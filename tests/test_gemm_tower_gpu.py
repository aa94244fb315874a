"""The tower's forward / input-gradient GEMM on wgmma with A from registers (csrc/gemm_tower_kernel.cu): a K-major A (plain,
relu(x*p + r), or x*p + y*q + r of two sources, per reduction index) times a packed hrl_board_pack image of 257..288 rows.

* against float64 over a 3x3 board: 32 -> 32 channels both ways (288 x 288), 30 <- 32 (N = 270), 32 <- 12 (K = 108, a tail
  chunk) and the heads' adjoint image (K = 27, rows of 28 floats), at M = 16384, 1000 and 130, every operand kind;
* the epilogues (relu, stats, mask_stats) on the product's C and column partials;
* the same bits as the wgmma kernel, forced by storing A in rows that are not 16-byte multiples;
* two launches give the same bits;
* hrl_gemm_fused routes the fused tower's forward and input-gradient products to it and keeps the stem and the heads'
  forward on the wgmma kernel (traced with torch.profiler).
"""
import ctypes as C

import pytest
import torch

from tower_ref import traced_gemms

pytestmark = pytest.mark.gpu

H = W = 3
SHAPES = {                   # (Cout, Cin, image): the forward image is N = Cout * 9 over K = Cin * 9, the adjoint the reverse
    '32x32_fwd': (32, 32, 'fwd'),
    '32x32_bwd': (32, 32, 'bwd'),
    '30x32_fwd': (30, 32, 'fwd'),
    '32x12_fwd': (32, 12, 'fwd'),
    'heads_bwd': (3, 32, 'bwd'),
}


def _grid(shape, g, bits=10, span=4):
    """Values k / 2^bits: the operand transforms below are exact in fp32, so float64 sees the operands the kernel splits."""
    return (torch.randint(-span * 2 ** bits + 1, span * 2 ** bits, shape, generator=g).double() / 2 ** bits).float()


def _pow2(n, g):
    return torch.pow(2.0, torch.randint(-1, 2, (n,), generator=g).float()) * (torch.randint(0, 2, (n,), generator=g).float() * 2 - 1)


def make_case(shape, M, kind, seed):
    from handyrl_b200._capi import check, lib
    from handyrl_b200.ops import _ptr, _stream_ptr
    Cout, Cin, which = SHAPES[shape]
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) / 8).cuda()
    rows_f, rows_b = Cout * H * W, Cin * H * W
    fwd = torch.zeros(lib().hrl_board_pack_floats(rows_f, rows_b), device='cuda')
    bwd = torch.zeros(lib().hrl_board_pack_floats(rows_b, rows_f), device='cuda')
    check(lib().hrl_board_pack(_ptr(w), Cout, Cin, 3, 3, H, W, _ptr(fwd), rows_f, 0, _ptr(bwd), rows_b, 0, _stream_ptr()))
    # dense matrix of the convolution in float64: y_flat = x_flat @ F, F (Cin*9 x Cout*9)
    eye = torch.eye(rows_b, dtype=torch.float64, device='cuda').view(rows_b, Cin, H, W)
    F = torch.nn.functional.conv2d(eye, w.double(), padding=1).reshape(rows_b, rows_f)
    if which == 'fwd':
        image, N, K, dense = fwd, rows_f, rows_b, F
    else:
        image, N, K, dense = bwd, rows_b, rows_f, F.t()
    ld = (K + 3) // 4 * 4                       # the heads' dHpre: 27 floats in rows of 28
    a = torch.zeros(M, ld, device='cuda')
    a[:, :K] = _grid((M, K), g).cuda()
    case = dict(M=M, N=N, K=K, a=a, a2=None, consts=None, relu=False, image=image, dense=dense)
    r = lambda n: _grid((n,), g, span=1).cuda() / 16
    if kind == 1:
        case.update(consts=(_pow2(K, g).cuda(), r(K)), relu=True)
    elif kind == 2:
        a2 = torch.zeros(M, ld, device='cuda')
        a2[:, :K] = _grid((M, K), g).cuda()
        case.update(a2=a2, consts=(_pow2(K, g).cuda(), _pow2(K, g).cuda(), r(K)))
    return case


def a_op64(c):
    K = c['K']
    A = c['a'][:, :K].double()
    if c['consts'] is not None:
        p, r = c['consts'][0].double(), c['consts'][-1].double()
        A = A * p + r
        if c['a2'] is not None:
            A = A + c['a2'][:, :K].double() * c['consts'][1].double()
        if c['relu']:
            A = torch.relu(A)
    return A


EPILOGUES = ('store', 'relu', 'stats', 'mask_stats')


def make_ep(c, seed):
    g = torch.Generator().manual_seed(seed)
    N = c['N']
    return dict(y=_grid((c['M'], N), g).cuda(), scale=_pow2(N, g).cuda(), shift=_grid((N,), g, span=1).cuda(),
                mean=_grid((N,), g, span=1).cuda(), rstd=_pow2(N, g).cuda())


def launch(c, epilogue='store', ep=None, a=None, a2=None):
    """hrl_gemm_fused on the case -> (C, col_partials or None).  a / a2: the same operand values stored elsewhere."""
    from handyrl_b200._capi import GEMM_EPILOGUES, HrlGemmArgs, check, lib
    from handyrl_b200.ops import _ptr, _stream_ptr
    a = c['a'] if a is None else a
    a2 = c['a2'] if a2 is None else a2
    M, N = c['M'], c['N']
    out = torch.full((M, N), float('nan'), device='cuda')
    cp = torch.full((-(-M // 128), 2, N), float('nan'), device='cuda') if epilogue in ('stats', 'mask_stats') else None
    args = HrlGemmArgs()
    args.a.ptr, args.a.ptr2, args.a.ld, args.a.kmajor = _ptr(a), _ptr(a2), a.stride(0), 1
    if c['consts'] is not None:
        args.a.p, args.a.r = _ptr(c['consts'][0]), _ptr(c['consts'][-1])
        args.a.q = _ptr(c['consts'][1]) if len(c['consts']) == 3 else None
        args.a.relu = int(c['relu'])
    args.b.ptr, args.b.kmajor, args.b.packed = _ptr(c['image']), 1, 1
    args.C, args.ldc, args.M, args.N, args.K, args.splits = _ptr(out), N, M, N, c['K'], 1
    args.epilogue = GEMM_EPILOGUES[epilogue]
    args.col_partials = _ptr(cp)
    if ep is not None:
        args.ep_mean = _ptr(ep['mean'])
        if epilogue == 'mask_stats':
            args.ep_y, args.ep_ldy = _ptr(ep['y']), ep['y'].stride(0)
            args.ep_scale, args.ep_shift, args.ep_rstd = _ptr(ep['scale']), _ptr(ep['shift']), _ptr(ep['rstd'])
    check(lib().hrl_gemm_fused(C.byref(args), _stream_ptr()))
    return out, cp


def odd_rows(t, K):
    """t's values in rows that are not a multiple of 4 floats (the wgmma kernel takes them, this kernel does not)."""
    if t is None:
        return None
    ld = K + 1 if (K + 1) % 4 else K + 2
    o = torch.zeros(t.shape[0], ld, device='cuda')
    o[:, :K] = t[:, :K]
    return o


@pytest.mark.parametrize('M', [16384, 1000, 130])
@pytest.mark.parametrize('kind', [0, 1, 2])
@pytest.mark.parametrize('shape', list(SHAPES))
def test_product_matches_float64(shape, kind, M):
    c = make_case(shape, M, kind, seed=M + 7 * kind + len(shape))
    out, _ = launch(c)
    torch.cuda.synchronize()
    A = a_op64(c)
    want, scale = A @ c['dense'], A.abs() @ c['dense'].abs()
    err = ((out.double() - want).abs() / (scale + 1e-30)).max().item()
    # the tensor core truncates each addition into the fp32 accumulator: with a ReLU'd (non-negative) operand the errors
    # do not cancel, so the bound is one ulp of sum |a||b| per reduction element (the wgmma kernel gives the same bits,
    # test_same_bits_as_the_wgmma_kernel)
    assert err < 2.0 ** -23 * (c['K'] + 8), err


@pytest.mark.parametrize('kind', [0, 1, 2])
@pytest.mark.parametrize('M', [1000, 130])
def test_epilogues_match_float64(M, kind):
    c = make_case('32x32_bwd', M, kind, seed=5 + kind)
    ep = make_ep(c, seed=9)
    base, _ = launch(c)
    relu, _ = launch(c, 'relu')
    stats, cp_s = launch(c, 'stats', ep)
    masked, cp_m = launch(c, 'mask_stats', ep)
    torch.cuda.synchronize()
    assert torch.equal(relu, torch.relu(base)) and torch.equal(stats, base)
    y = ep['y'].double()
    keep = (y * ep['scale'].double() + ep['shift'].double()) > 0
    assert torch.equal(masked, torch.where(keep, base, torch.zeros_like(base)))
    xhat = (y - ep['mean'].double()) * ep['rstd'].double()
    d = base.double() - ep['mean'].double()
    m = masked.double()
    for t in range(-(-M // 128)):
        rows = slice(128 * t, min(M, 128 * (t + 1)))
        for got, want, mag in ((cp_s[t, 0], d[rows].sum(0), d[rows].abs().sum(0)), (cp_s[t, 1], (d[rows] ** 2).sum(0), (d[rows] ** 2).sum(0)),
                               (cp_m[t, 0], m[rows].sum(0), m[rows].abs().sum(0)),
                               (cp_m[t, 1], (m[rows] * xhat[rows]).sum(0), (m[rows] * xhat[rows]).abs().sum(0))):
            assert ((got.double() - want).abs() <= 1e-6 * mag + 1e-30).all()


@pytest.mark.parametrize('M', [16384, 1000, 130])
@pytest.mark.parametrize('kind', [0, 1, 2])
@pytest.mark.parametrize('shape', list(SHAPES))
def test_same_bits_as_the_wgmma_kernel(shape, kind, M):
    """The same A values in rows of K+1 (or K+2) floats run on the wgmma kernel: the same transformed values, hi / lo halves,
    chunks, k8 steps and product order into the same accumulators, and the same epilogue, give the same C and column
    partials, bit for bit, for every epilogue."""
    c = make_case(shape, M, kind, seed=3 * M + kind)
    ep = make_ep(c, seed=11)
    a, a2 = odd_rows(c['a'], c['K']), odd_rows(c['a2'], c['K'])
    for epilogue in EPILOGUES:
        if epilogue in ('stats', 'mask_stats') and c['N'] % 4:
            continue
        got, cp = launch(c, epilogue, ep)
        want, cp_w = launch(c, epilogue, ep, a=a, a2=a2)
        torch.cuda.synchronize()
        assert torch.equal(got.view(torch.int32), want.view(torch.int32)), epilogue
        if cp is not None:
            assert torch.equal(cp.view(torch.int32), cp_w.view(torch.int32)), epilogue


@pytest.mark.parametrize('kind', [0, 1, 2])
def test_dispatch_of_direct_calls(kind):
    """16-byte rows take this kernel, the same operand in rows of K + 1 floats the wgmma kernel (one trace per kind: the
    tests above rely on the rule, not on a trace of every case)."""
    c = make_case('32x12_fwd', 1000, kind, seed=kind)
    assert traced_gemms(lambda: launch(c)) == {('gemm_tower_kernel', str(kind))}
    a, a2 = odd_rows(c['a'], c['K']), odd_rows(c['a2'], c['K'])
    assert {k for k, _ in traced_gemms(lambda: launch(c, a=a, a2=a2))} == {'gemm_tf32x3_kernel'}


def test_two_launches_are_bit_identical():
    c = make_case('32x32_bwd', 16384, 2, seed=1)
    ep = make_ep(c, seed=2)
    (c1, p1), (c2, p2) = launch(c, 'mask_stats', ep), launch(c, 'mask_stats', ep)
    torch.cuda.synchronize()
    assert torch.equal(c1.view(torch.int32), c2.view(torch.int32)) and torch.equal(p1.view(torch.int32), p2.view(torch.int32))


def test_fused_tower_dispatch():
    """One FusedBoardNet forward and backward: the tower layers' forward products (plain A0 for the first, relu(bn(Y)) for the
    others), their input gradients (BatchNorm backward of two sources) and the heads-to-tower input gradient (plain dHpre,
    K = 27 in rows of 28) take gemm_tower_kernel; the stem (27-float observation rows) and the heads' forward (N = 27) keep
    the wgmma kernel, the weight gradients the mma.sync kernel."""
    from handyrl_b200 import nets, tower
    torch.manual_seed(0)
    net = nets.BoardNet(planes=3, board=(3, 3), width=32, depth=3, actions=9).cuda().train()
    M = 512
    eng = tower.FusedBoardNet(net, M, torch.device('cuda'))
    for p in net.parameters():
        p.grad = torch.zeros_like(p)
    x = (torch.rand(M, 3, 3, 3, device='cuda') < 0.4).float()

    def step():
        out = eng.forward(x)
        eng.backward(torch.ones_like(out['policy']), torch.ones_like(out['value']))

    seen = traced_gemms(step)
    assert {args for k, args in seen if k == 'gemm_tower_kernel'} == {'0', '1', '2'}, seen
    assert {'true,true,true,144', 'true,true,true,16'} <= {args for k, args in seen if k == 'gemm_tf32x3_kernel'}, seen
    assert {args for k, args in seen if k == 'gemm_wgrad_kernel'} == {'2,1', '2,0', '0,1'}, seen
