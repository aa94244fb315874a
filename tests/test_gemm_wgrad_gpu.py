"""The weight-gradient GEMM on warp-level 3xTF32 MMAs (csrc/gemm_wgrad_kernel.cu): both operands stored [K][rows] and read as
they lie, per-row operand transforms applied on fragment load, split-K slice partials in the workspace layout the fold reads.

* against float64 at the tower's shape (288 x 288 over 16384 samples, 43 K slices, both transforms), the heads' shape (27 x 288),
  a ragged K and sizes that are not tile multiples, with the accumulation bound of tests/test_gemm_gpu.py;
* two launches give the same bits;
* hrl_gemm_fused routes the tower's and the heads' weight gradients to it, and the convolution weight gradient (conv_mode 2)
  and unaligned operands to the wgmma kernel (traced with torch.profiler).
"""
import ctypes as C

import pytest
import torch

from tower_ref import traced_gemms

pytestmark = pytest.mark.gpu


def _grid(shape, g, bits=10, span=4):
    """Values k / 2^bits with |k| < span * 2^bits: the operand transforms below are exact in fp32 (and in float64), so the
    reference sees exactly the operands the kernel splits into hi / lo halves."""
    return (torch.randint(-span * 2 ** bits + 1, span * 2 ** bits, shape, generator=g).double() / 2 ** bits).float()


def _pow2(n, g):
    return torch.pow(2.0, torch.randint(-1, 2, (n,), generator=g).float()) * (torch.randint(0, 2, (n,), generator=g).float() * 2 - 1)


def make_case(M, N, K, a_kind, b_kind, seed, lda=None, ldb=None):
    """A (K x lda) with a_kind 0 plain / 1 x*p + r / 2 x*p + y*q + r, B (K x ldb) with b_kind 0 plain / 1 relu(x*p + r)."""
    g = torch.Generator().manual_seed(seed)
    lda, ldb = lda or M, ldb or N
    case = dict(M=M, N=N, K=K, a=_grid((K, lda), g).cuda(), b=_grid((K, ldb), g).cuda(), a2=None, ac=None, bc=None)
    # small offsets r keep A_op zero-mean like the randn operands of tests/test_gemm_gpu.py (a per-row mean would make the fp32
    # accumulator's truncation coherent over K and exceed that bound on the wgmma kernel as well)
    r = lambda n: _grid((n,), g, span=1).cuda() / 16
    if a_kind == 2:
        case['a2'] = _grid((K, lda), g).cuda()
        case['ac'] = (_pow2(M, g).cuda(), _pow2(M, g).cuda(), r(M))
    elif a_kind == 1:
        case['ac'] = (_pow2(M, g).cuda(), r(M))
    if b_kind == 1:
        case['bc'] = (_pow2(N, g).cuda(), r(N))
    return case


def operands64(c):
    M, N = c['M'], c['N']
    A = c['a'][:, :M].double()
    if c['ac'] is not None:
        A = A * c['ac'][0].double() + c['ac'][-1].double()
        if c['a2'] is not None:
            A = A + c['a2'][:, :M].double() * c['ac'][1].double()
    B = c['b'][:, :N].double()
    if c['bc'] is not None:
        B = torch.relu(B * c['bc'][0].double() + c['bc'][1].double())
    return A, B


def launch(c, splits, out=None, ws=None):
    """hrl_gemm_fused on the case: C = A_op^T B_op (out, summed over the slices), or only the slice partials (ws, out None)."""
    from handyrl_b200._capi import HrlGemmArgs, check, lib
    from handyrl_b200.ops import _ptr, _stream_ptr
    args = HrlGemmArgs()
    for o, t, t2, consts, relu in ((args.a, c['a'], c['a2'], c['ac'], False), (args.b, c['b'], None, c['bc'], True)):
        o.ptr, o.ptr2, o.ld, o.kmajor, o.feature_is_row = _ptr(t), _ptr(t2), t.stride(0), 0, 1
        if consts is not None:
            o.p, o.r = _ptr(consts[0]), _ptr(consts[-1])
            o.q = _ptr(consts[1]) if len(consts) == 3 else None
            o.relu = int(relu)
    args.C, args.ldc = _ptr(out), (out.stride(0) if out is not None else c['N'])
    args.M, args.N, args.K, args.splits = c['M'], c['N'], c['K'], splits
    args.workspace = _ptr(ws)
    check(lib().hrl_gemm_fused(C.byref(args), _stream_ptr()))


def slices(K, splits):
    """[(k_begin, k_end)] of the K slices hrl_gemm_fused forms (whole 32-sample chunks, no empty slice)."""
    chunks = -(-K // 32)
    per = -(-chunks // max(1, min(splits, chunks)))
    return [(32 * s * per, min(K, 32 * (s + 1) * per)) for s in range(-(-chunks // per))]


def assert_bound(got, want, scale, k_slice, what):
    # the accumulation bound of tests/test_gemm_gpu.py: ~0.5 sqrt(K_slice) ulp of sum |a||b|
    err = ((got.double() - want).abs() / (scale + 1e-30)).max().item()
    assert err < 1.2e-7 * (0.8 * k_slice ** 0.5 + 4), (what, err, k_slice)


def test_tower_shape_slice_partials_match_float64():
    """288 x 288 over 16384 samples in 43 slices (tower.py's split of the cfg2 weight gradient), BatchNorm backward of two
    sources as A, relu(BatchNorm-apply) as B: every slice partial against float64."""
    from handyrl_b200._capi import lib
    c = make_case(288, 288, 16384, 2, 1, seed=1)
    splits = lib().hrl_gemm_effective_splits(16384, 44)
    assert splits == 43
    ws = torch.full((splits, 288, 288), float('nan'), device='cuda')
    launch(c, splits, ws=ws)
    torch.cuda.synchronize()
    A, B = operands64(c)
    sl = slices(16384, splits)
    assert len(sl) == splits
    for s, (k0, k1) in enumerate(sl):
        want, scale = A[k0:k1].t() @ B[k0:k1], A[k0:k1].abs().t() @ B[k0:k1].abs()
        assert_bound(ws[s], want, scale, k1 - k0, 'slice %d' % s)


@pytest.mark.parametrize('M,N,K,a_kind,b_kind,splits,lda,ldb', [
    (27, 288, 16384, 0, 1, 128, 28, None),      # the heads' weight gradient: dHpre (ld 28) x relu(bn(Y))
    (288, 288, 1013, 2, 1, 5, None, None),      # ragged K: the last chunk is partial
    (288, 288, 5000, 2, 0, 1, None, None),      # the first tower layer: plain activation operand, one slice
    (100, 300, 777, 1, 1, 3, None, None),       # M, N not tile multiples, N over two column tiles
    (50, 37, 300, 1, 0, 1, 52, 40),             # ragged everywhere; N % 4 != 0 (scalar stores), padded rows
])
def test_summed_product_matches_float64(M, N, K, a_kind, b_kind, splits, lda, ldb):
    from handyrl_b200._capi import lib
    c = make_case(M, N, K, a_kind, b_kind, seed=M * 7 + N * 3 + K, lda=lda, ldb=ldb)
    out = torch.full((M, N), float('nan'), device='cuda')
    ws = torch.empty(lib().hrl_gemm_workspace_floats(M, N, K, splits), device='cuda') if splits > 1 else None
    launch(c, splits, out=out, ws=ws)
    torch.cuda.synchronize()
    A, B = operands64(c)
    k_slice = max(k1 - k0 for k0, k1 in slices(K, splits))
    assert_bound(out, A.t() @ B, A.abs().t() @ B.abs(), k_slice, 'C')


def test_two_launches_are_bit_identical():
    c = make_case(288, 288, 16384, 2, 1, seed=3)
    outs = []
    for _ in range(2):
        ws = torch.empty((43, 288, 288), device='cuda')
        launch(c, 43, ws=ws)
        outs.append(ws)
    torch.cuda.synchronize()
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32))


def test_same_bits_as_the_wgmma_kernel():
    """The tower's product with operands whose rows are 289 floats (not 16-byte multiples) runs on the wgmma kernel: the same
    slices, the same hi / lo halves and the same product order give the same slice partials, bit for bit."""
    c = make_case(288, 288, 16384, 2, 1, seed=4)
    ws = torch.empty((43, 288, 288), device='cuda')
    launch(c, 43, ws=ws)
    odd = dict(c)
    for k in ('a', 'a2', 'b'):
        t = torch.zeros((16384, 289), device='cuda')
        t[:, :288] = c[k]
        odd[k] = t
    assert traced_gemms(lambda: launch(odd, 43, ws=torch.empty_like(ws)), runs=2, repeat=2) == {('gemm_tf32x3_kernel', 'false,false,false,144')}
    ws_wgmma = torch.empty_like(ws)
    launch(odd, 43, ws=ws_wgmma)
    torch.cuda.synchronize()
    assert torch.equal(ws.view(torch.int32), ws_wgmma.view(torch.int32))


def test_tower_weight_gradients_take_the_wgrad_kernel():
    """The fused tower (tictactoe net): the tower layers' weight gradients (A = BatchNorm backward of two sources; B =
    relu(bn(Y)), or the stem's plain output for the first layer) and the heads' (plain dHpre with 16-byte rows) run on the
    mma.sync kernel; the stem's, over observations whose rows are 27 floats, stays on the wgmma kernel."""
    from handyrl_b200 import nets, tower
    torch.manual_seed(0)
    net = nets.BoardNet(planes=3, board=(3, 3), width=32, depth=3, actions=9).cuda().train()
    M = 512
    eng = tower.FusedBoardNet(net, M, torch.device('cuda'))
    for p in net.parameters():
        p.grad = torch.zeros_like(p)
    x = (torch.rand(M, 3, 3, 3, device='cuda') < 0.4).float()
    out = eng.forward(x)
    dout = {k: torch.randn_like(v) for k, v in out.items()}

    seen = traced_gemms(lambda: eng.backward(dout['policy'], dout['value']), runs=2, repeat=2)
    wgrad = {args for k, args in seen if k == 'gemm_wgrad_kernel'}
    assert wgrad == {'2,1', '2,0', '0,1'}, seen
    assert ('gemm_tf32x3_kernel', 'false,false,false,16') in seen, seen       # the stem: x2d rows of 27 floats


def test_convolution_weight_gradient_and_unaligned_operands_keep_the_wgmma_kernel():
    from handyrl_b200 import ops
    g = torch.Generator(device='cuda').manual_seed(11)
    x = torch.randn(64, 16, 5, 5, device='cuda', generator=g).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    w = (0.2 * torch.randn(8, 16, 3, 3, device='cuda', generator=g)).requires_grad_(True)
    assert ops.conv_implicit_supported(x, w)
    ops.conv_weights_changed()
    dy = torch.randn(64, 8, 5, 5, device='cuda', generator=g).contiguous(memory_format=torch.channels_last)

    def conv():
        ops.conv_implicit(x, w).backward(dy)

    seen = traced_gemms(conv, runs=2, repeat=2)
    assert seen and all(k == 'gemm_tf32x3_kernel' for k, _ in seen), seen
    assert any(args.startswith('false,false,false,') for _, args in seen), seen    # the weight gradient (conv_mode 2)

    a = torch.randn(4000, 27, device='cuda', generator=g)                    # rows of 27 floats: not 16-byte aligned
    b = torch.randn(4000, 288, device='cuda', generator=g)
    seen = traced_gemms(lambda: ops.gemm_tf32x3(a, b, a_kmajor=False, b_kmajor=False, splits=4), runs=2, repeat=2)
    assert seen == {('gemm_tf32x3_kernel', 'false,false,false,144')}, seen
    b_off = torch.randn(4000 * 288 + 1, device='cuda', generator=g)[1:].view(4000, 288)      # base pointer off by 4 bytes
    a2 = torch.randn(4000, 288, device='cuda', generator=g)
    seen = traced_gemms(lambda: ops.gemm_tf32x3(a2, b_off, a_kmajor=False, b_kmajor=False, splits=4), runs=2, repeat=2)
    assert seen == {('gemm_tf32x3_kernel', 'false,false,false,144')}, seen
