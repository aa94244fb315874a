"""The bf16 mode of the net's tensor-core products (HrlGemmArgs.bf16, train_args['tensor_cores'] = 'bf16') on the GPU.

Every bound is derived from the arithmetic.  The product of two bf16 values is exact in fp32, so a bf16 product is the fp32
accumulation of exact terms: against float64 products of the operands rounded to bf16 (torch rounds to nearest even, as the
kernels do) its error is that of fp32 accumulation alone, the accumulation of the 3xTF32 form: the bound
test_gemm_gpu.py holds that kernel to, 1.2e-7 (0.8 sqrt(k) + 4) of sum|a||b| over a K slice of k terms.  Where an operand
transform runs first, its fp32 result decides the bf16 rounding: an element whose fp32 value sits at a rounding boundary may
round either way, at most one bf16 ulp of the element times |b|.
"""
import os
import pickle

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN
from tower_ref import U16, U32, _close, _conv, _conv_in, _conv_w, _transform_ref, _wgrad_bound, accum_bound, r16

pytestmark = pytest.mark.gpu

# the shapes of test_gemm_gpu.py: M, N, K, a_kmajor, b_kmajor, bias, splits
CASES = [
    (1000, 288, 288, True, True, False, 1),
    (16384, 288, 288, True, True, True, 1),
    (777, 288, 288, True, False, False, 1),
    (288, 288, 5000, False, False, False, 1),
    (288, 288, 16384, False, False, False, 37),
    (300, 288, 27, True, True, True, 1),
    (515, 27, 288, True, True, True, 1),
    (130, 600, 96, True, True, False, 1),
    (64, 16, 8, True, True, False, 1),
    (129, 272, 40, False, True, False, 2),
]


@pytest.mark.parametrize('M,N,K,a_k,b_k,with_bias,splits', CASES)
def test_gemm_bf16_matches_float64_on_rounded_operands(M, N, K, a_k, b_k, with_bias, splits):
    from handyrl_b200 import ops
    g = torch.Generator().manual_seed(M * 7 + N * 3 + K)
    a = torch.randn((M, K) if a_k else (K, M), generator=g).cuda()
    b = torch.randn((N, K) if b_k else (K, N), generator=g).cuda()
    bias = torch.randn(N, generator=g).cuda() if with_bias else None
    got = ops.gemm_bf16(a, b, bias, a_kmajor=a_k, b_kmajor=b_k, splits=splits).double()
    A = r16(a) if a_k else r16(a).t()
    B = r16(b) if b_k else r16(b).t()
    want, scale = A @ B.t(), A.abs() @ B.abs().t()
    if with_bias:
        want, scale = want + bias.double(), scale + bias.double().abs()
    bound = accum_bound(K, splits) * scale + 1e-30
    assert ((got - want).abs() <= bound).all(), ((got - want).abs() / bound).max().item()
    # the operands really were rounded: against the unrounded operands the error leaves the accumulation bound
    A0 = a.double() if a_k else a.double().t()
    B0 = b.double() if b_k else b.double().t()
    exact = A0 @ B0.t() + (bias.double() if with_bias else 0)
    assert ((got - exact).abs() > bound).any()


def test_gemm_bf16_is_repeatable():
    from handyrl_b200 import ops
    g = torch.Generator().manual_seed(3)
    a = torch.randn(9000, 288, generator=g).cuda()           # the weight-gradient form: both operands transposed, split over K
    b = torch.randn(9000, 272, generator=g).cuda()
    one = ops.gemm_bf16(a, b, a_kmajor=False, b_kmajor=False, splits=23)
    two = ops.gemm_bf16(a, b, a_kmajor=False, b_kmajor=False, splits=23)
    assert torch.equal(one, two)


def _product(a, image, M, N, K, bf16):
    import ctypes as C
    from handyrl_b200._capi import HrlGemmArgs, check, lib
    from handyrl_b200.ops import _ptr, _stream_ptr
    out = torch.empty(M, N, device='cuda')
    args = HrlGemmArgs()
    args.a.ptr, args.a.ld, args.a.kmajor = _ptr(a), a.stride(0), 1
    args.b.ptr, args.b.kmajor, args.b.packed = _ptr(image), 1, 1
    args.C, args.ldc, args.M, args.N, args.K, args.splits, args.bf16 = _ptr(out), N, M, N, K, 1, int(bf16)
    check(lib().hrl_gemm_fused(C.byref(args), _stream_ptr()))
    return out


@pytest.mark.parametrize('Cout,Cin,H,W,ksz,M', [(32, 32, 3, 3, 3, 1000), (32, 3, 3, 3, 3, 515), (2, 32, 3, 3, 1, 300), (8, 5, 4, 4, 3, 129)])
def test_packed_bf16_board_images_forward_and_input_gradient(Cout, Cin, H, W, ksz, M):
    """hrl_board_pack_many with HrlPackJob.bf16: a quarter of the hrl_board_pack_floats image, both directions."""
    import ctypes as C
    from handyrl_b200._capi import HrlPackJob, check, lib
    from handyrl_b200.ops import _ptr, _stream_ptr
    g = torch.Generator(device='cuda').manual_seed(Cout * 100 + Cin)
    w = torch.randn(Cout, Cin, ksz, ksz, device='cuda', generator=g)
    x = torch.randn(M, Cin, H, W, device='cuda', generator=g)
    dy = torch.randn(M, Cout, H, W, device='cuda', generator=g)
    row0 = 7 if Cout * H * W + 7 <= 288 else 0
    rows_f, rows_b = Cout * H * W + row0, Cin * H * W
    fwd = torch.zeros(lib().hrl_board_pack_floats(rows_f, rows_b) // 4, device='cuda')
    bwd = torch.zeros(lib().hrl_board_pack_floats(rows_b, rows_f) // 4, device='cuda')
    j = (HrlPackJob * 1)()
    j[0].w, j[0].Cout, j[0].Cin, j[0].kh, j[0].kw, j[0].H, j[0].W = _ptr(w), Cout, Cin, ksz, ksz, H, W
    j[0].image_fwd, j[0].fwd_rows, j[0].fwd_row0 = _ptr(fwd), rows_f, row0
    j[0].image_bwd, j[0].bwd_rows, j[0].bwd_k0 = _ptr(bwd), rows_b, row0
    j[0].bf16 = 1
    check(lib().hrl_board_pack_many(C.byref(j), 1, _stream_ptr()))
    xr, wr, dyr = r16(x), r16(w), r16(dy)
    y = _product(x.reshape(M, -1), fwd, M, rows_f, rows_b, True).double()
    assert (y[:, :row0] == 0).all()
    ref = F.conv2d(xr, wr, padding=ksz // 2).reshape(M, -1)
    scale = F.conv2d(xr.abs(), wr.abs(), padding=ksz // 2).reshape(M, -1)
    assert ((y[:, row0:] - ref).abs() <= accum_bound(rows_b) * scale).all()
    dyp = torch.cat([torch.randn(M, row0, device='cuda', generator=g), dy.reshape(M, -1)], 1).contiguous()
    dx = _product(dyp, bwd, M, rows_b, rows_f, True).double()
    ref = torch.nn.grad.conv2d_input(x.shape, wr, dyr, padding=ksz // 2).reshape(M, -1)
    scale = torch.nn.grad.conv2d_input(x.shape, wr.abs(), dyr.abs(), padding=ksz // 2).reshape(M, -1)
    assert ((dx - ref).abs() <= accum_bound(rows_f) * scale).all()


@pytest.mark.parametrize('Cout,Cin,taps', [(64, 64, 9), (32, 17 * 4, 9), (128, 32, 1)])
def test_conv_pack_bf16_images(Cout, Cin, taps):
    """hrl_conv_pack_bf16: forward and adjoint images of the implicit convolution, every weight rounded to nearest even,
    in a quarter of hrl_conv_pack_floats."""
    from handyrl_b200._capi import check, lib
    from handyrl_b200.ops import _ptr, _stream_ptr
    k = int(round(taps ** 0.5))
    w = torch.randn(Cout, Cin, k, k, device='cuda')
    n_f, n_a = lib().hrl_conv_pack_floats(Cout, Cin, taps), lib().hrl_conv_pack_floats(Cin, Cout, taps)
    fwd, adj = torch.zeros(n_f // 4, device='cuda'), torch.zeros(n_a // 4, device='cuda')
    check(lib().hrl_conv_pack_bf16(_ptr(w), Cout, Cin, k, k, _ptr(fwd), _ptr(adj), _stream_ptr()))
    torch.cuda.synchronize()

    def unpack(img, rows, ch):
        # [chunk][n_pad rows][32 bf16, 16-byte slot j at j ^ ((row >> 1) & 3)] -> (rows, taps * ch_pad)
        n_pad = lib().hrl_gemm_padded_rows(rows)
        ch_pad = -(-ch // 32) * 32
        e = img.view(torch.bfloat16).view(-1, n_pad, 4, 8)[:, :rows]
        r = torch.arange(rows, device='cuda')
        slot = torch.arange(4, device='cuda')[None, :] ^ ((r[:, None] >> 1) & 3)       # logical slot -> stored slot
        e = torch.gather(e, 2, slot[None, :, :, None].expand(e.shape[0], rows, 4, 8))
        return e.reshape(-1, rows, 32).permute(1, 0, 2).reshape(rows, taps, ch_pad)[:, :, :ch]
    wb = w.bfloat16()
    assert torch.equal(unpack(fwd, Cout, Cin), wb.reshape(Cout, Cin, taps).permute(0, 2, 1))
    assert torch.equal(unpack(adj, Cin, Cout), wb.reshape(Cout, Cin, taps).flip(2).permute(1, 2, 0))


@pytest.mark.parametrize('epilogue', ['stats', 'mask_stats'])
def test_fused_transforms_and_epilogues_bf16(epilogue):
    """BatchNorm-apply + ReLU of the A operand (per reduction index) with the STATS epilogue; the two-source BatchNorm backward
    dY = dZ*p + Y*q + r with per-row constants on transposed operands (the weight-gradient form, feature_is_row) and MASK_STATS."""
    import ctypes as C
    from handyrl_b200._capi import GEMM_EPILOGUES, HrlGemmArgs, check, lib
    from handyrl_b200.ops import _ptr, _stream_ptr
    from handyrl_b200.tower import _operand
    g = torch.Generator(device='cuda').manual_seed(11)
    rnd = lambda *s: torch.randn(*s, device='cuda', generator=g)
    M, N, K = 700, 96, 160
    cp = torch.empty(((M + 127) // 128, 2, N), device='cuda')
    out = torch.empty(M, N, device='cuda')
    args = HrlGemmArgs()
    args.M, args.N, args.K, args.splits, args.bf16 = M, N, K, 1, 1
    args.C, args.ldc, args.col_partials, args.epilogue = _ptr(out), N, _ptr(cp), GEMM_EPILOGUES[epilogue]
    if epilogue == 'stats':
        x, b = rnd(M, K), rnd(N, K)
        p, r = rnd(K), rnd(K)
        _operand(args.a, x, consts=(p, r), relu=True)
        _operand(args.b, b)
        ta, edge = _transform_ref(x, p[None], r[None], relu=True)
        B, eb = r16(b), torch.zeros_like(b, dtype=torch.float64)
        pivot = rnd(N)                                       # the shift of the statistics sums
        args.ep_mean = _ptr(pivot)
    else:
        dz, yy, b = rnd(K, M), rnd(K, M), rnd(K, N)          # A stored (K, M): per-row constants = per column of the memory
        p, q, r = rnd(M), rnd(M), rnd(M)
        _operand(args.a, dz, t2=yy, consts=(p, q, r), kmajor=False, by_row=True)
        _operand(args.b, b, kmajor=False)
        ta, edge = _transform_ref(dz, p[None], r[None], y=yy, q=q[None])
        ta, edge, B, eb = ta.t(), edge.t(), r16(b).t(), torch.zeros(N, K, dtype=torch.float64, device='cuda')
        ys, sc, sh = rnd(M, N), rnd(N), rnd(N)
        mu, rs = rnd(N), rnd(N).abs() + 0.5
        args.ep_y, args.ep_ldy, args.ep_scale, args.ep_shift = _ptr(ys), N, _ptr(sc), _ptr(sh)
        args.ep_mean, args.ep_rstd = _ptr(mu), _ptr(rs)
    check(lib().hrl_gemm_fused(C.byref(args), _stream_ptr()))
    torch.cuda.synchronize()
    acc = ta @ B.t()
    bound = accum_bound(K) * (ta.abs() @ B.abs().t()) + edge @ B.abs().t() + (ta.abs() @ eb.t())
    # column sums: fp32 additions over a row tile (M of them at most), per-tile partials summed here in float64
    s1, s2 = cp[:, 0].double().sum(0), cp[:, 1].double().sum(0)
    if epilogue == 'stats':
        assert ((out.double() - acc).abs() <= bound).all()
        d = (out - pivot).double()                           # d = C - pivot, one fp32 rounding (within 2^-24 |d|)
        assert ((s1 - d.sum(0)).abs() <= (M + 1) * U32 * d.abs().sum(0) + 1e-30).all()
        assert ((s2 - (d * d).sum(0)).abs() <= (M + 3) * U32 * (d * d).sum(0) + 1e-30).all()
    else:
        live = (ys.double() * sc.double() + sh.double()).float() > 0          # the epilogue's mask, fmaf in fp32
        want = torch.where(live, acc, torch.zeros_like(acc))
        assert ((out.double() - want).abs() <= torch.where(live, bound, torch.zeros_like(bound))).all()
        xh = ((ys - mu) * rs).double()                       # (y - mean) * rstd, the kernel's two fp32 operations
        assert ((s1 - out.double().sum(0)).abs() <= M * U32 * out.double().abs().sum(0) + 1e-30).all()
        assert ((s2 - (out.double() * xh).sum(0)).abs() <= (M + 1) * U32 * (out.double() * xh).abs().sum(0) + 1e-30).all()


@pytest.mark.parametrize('wrap', [False, True])
def test_conv_implicit_bf16_against_float64(wrap):
    from handyrl_b200 import ops
    g = torch.Generator(device='cuda').manual_seed(5 + wrap)
    N, Cin, Cout, H, W = 64, 32, 64, 7, 11
    x = torch.randn(N, Cin, H, W, device='cuda', generator=g)
    w = (torch.randn(Cout, Cin, 3, 3, device='cuda', generator=g) * 0.1).requires_grad_(True)
    b = torch.randn(Cout, device='cuda', generator=g).requires_grad_(True)
    dy = torch.randn(N, Cout, H, W, device='cuda', generator=g)
    xg = x.clone().requires_grad_(True)
    y = ops.conv_implicit(xg, w, b, wrap=wrap, bf16=True)
    y.backward(dy)
    xr, wr, dyr = r16(x).requires_grad_(True), r16(w.detach()).requires_grad_(True), r16(dy)
    mode = 'circular' if wrap else 'zeros'

    def conv(a, k, bias=None):
        if wrap:
            return F.conv2d(F.pad(a, (1, 1, 1, 1), mode='circular'), k, bias)
        return F.conv2d(a, k, bias, padding=1)
    ref = conv(xr, wr, b.detach().double())
    ref.backward(dyr)
    with torch.no_grad():
        sy = conv(xr.abs(), wr.abs(), b.detach().double().abs())
    assert ((y.double() - ref).abs() <= accum_bound(9 * Cin) * sy).all(), mode
    assert ((y.double() - conv(x.double(), w.detach().double(), b.detach().double())).abs() > accum_bound(9 * Cin) * sy).any()
    xa = xr.detach().abs().requires_grad_(True)
    conv(xa, wr.detach().abs()).backward(dyr.abs())
    assert ((xg.grad.double() - xr.grad).abs() <= accum_bound(9 * Cout) * xa.grad).all()
    wa = wr.detach().abs().requires_grad_(True)
    conv(xr.detach().abs(), wa).backward(dyr.abs())
    pixels = N * H * W
    assert ((w.grad.double() - wr.grad).abs() <= accum_bound(pixels) * wa.grad + 1e-30).all()
    db_bound = dy.double().abs().sum((0, 2, 3)) * (pixels * U32 + U16)      # fp32 sums of dy, or of dy rounded to bf16
    assert ((b.grad.double() - dy.double().sum((0, 2, 3))).abs() <= db_bound).all()


def test_deferred_segmented_weight_gradient_bf16():
    """The recurrent cells' deferred weight gradient in bf16 mode: one segmented product over the (dy, x) pairs of a shared
    weight, its ones row giving the bias gradient."""
    from handyrl_b200 import ops
    g = torch.Generator(device='cuda').manual_seed(9)
    N, C, H, W, steps = 32, 32, 6, 6, 5
    w = (torch.randn(C, C, 3, 3, device='cuda', generator=g) * 0.2).requires_grad_(True)
    b = torch.randn(C, device='cuda', generator=g).requires_grad_(True)
    xs = [torch.randn(N, C, H, W, device='cuda', generator=g) for _ in range(steps)]
    dys = [torch.randn(N, C, H, W, device='cuda', generator=g) for _ in range(steps)]
    with ops.deferred_weight_gradients():
        outs = [ops.conv_implicit(x, w, b, bf16=True) for x in xs]
        torch.autograd.backward(outs, dys)
    wr = r16(w.detach())
    dw = torch.zeros_like(wr)
    dwa = torch.zeros_like(wr)
    for x, dy in zip(xs, dys):
        dw += torch.nn.grad.conv2d_weight(r16(x), w.shape, r16(dy), padding=1)
        dwa += torch.nn.grad.conv2d_weight(r16(x).abs(), w.shape, r16(dy).abs(), padding=1)
    pixels = N * H * W
    # each pair's K slices, then a fixed-order sum of every slice of every pair
    assert ((w.grad.double() - dw).abs() <= (accum_bound(pixels) + steps * 132 * U32) * dwa).all()
    db = sum(dy.double().sum((0, 2, 3)) for dy in dys)
    dba = sum(dy.double().abs().sum((0, 2, 3)) for dy in dys)
    assert ((b.grad.double() - db).abs() <= dba * (steps * pixels * U32 + U16)).all()


# ---- the learner in bf16 mode -------------------------------------------------------------------------------------
with open(os.path.join(GOLDEN, 'step_cases.pkl'), 'rb') as f:
    STEP_CASES = pickle.load(f)
with open(os.path.join(GOLDEN, 'net_step_cases.pkl'), 'rb') as f:
    NET_CASES = pickle.load(f)


def _check_weights(c, final, steps, depth, sample=None, noise=None):
    for (k, v), (kr, vr) in zip(final.items(), c['state3'].items()):
        if noise is not None and noise(c, k):
            continue
        got = sample(kr, v.numpy()) if sample is not None else v.numpy()
        if 'running_' in k:
            # BatchNorm buffers follow the batch statistics, not Adam: each step moves them by momentum (0.1) times a batch
            # statistic whose activations carry the forward chain's rounding, depth x 2^-8 relative
            np.testing.assert_allclose(got, vr, rtol=0, atol=steps * 0.1 * depth * U16 * (np.abs(vr).max() + 1), err_msg=k)
        elif v.dtype.is_floating_point:
            # Adam moves a weight by at most ~lr a step whatever its gradient: 2 lr per step bounds any difference
            np.testing.assert_allclose(got, vr, rtol=0, atol=2 * c['lr'] * steps + 5e-5, err_msg='%s/%s' % (k, kr))
        else:
            assert int(v) == int(vr)


def _check_losses(got, ref, depth, s):
    # each product's operands are rounded once (2 x 2^-9 of sum|a||b| per product), `depth` products in the forward chain;
    # later steps add the weights' lr-sized differences, bounded as the step-0 error again per step
    scale = max(abs(v) for v in ref.values())
    for k, v in ref.items():
        assert abs(got[k] - v) <= (1 + s) * depth * U16 * scale + 1e-4, (s, k, got[k], v)


@pytest.mark.parametrize('name', sorted(STEP_CASES))
def test_learner_step_bf16_tictactoe_fused_tower(name):
    from handyrl_b200.nets import tictactoe_net, load_state_by_order
    from handyrl_b200.synthetic import synthetic_batch
    from handyrl_b200.train import LearnerStep
    c = STEP_CASES[name]
    B, T, P, A = c['dims']
    args = dict(c['args'], tensor_cores='bf16')
    net = load_state_by_order(tictactoe_net(), c['state0'])
    mk = lambda s: synthetic_batch(B, T, P, A, turn_based=args['turn_based_training'], observation=args['observation'], seed=40 + s)
    stepper = LearnerStep(net, args, mk(0), lr=c['lr'])
    assert stepper.tensor_cores == 'bf16' and stepper.engine is not None and stepper.engine.bf16
    depth = len(net.tower) + 3                    # stem, tower, squeeze heads, output layer
    for s, ref in enumerate(c['steps']):
        stepper.step(stepper.new_packed().fill(mk(s)))
        _check_losses(stepper.read_losses(), ref['losses'], depth, s)
    _check_weights(c, stepper.cpu_state_dict(), len(c['steps']), depth)


@pytest.mark.parametrize('name', sorted(NET_CASES))
def test_learner_step_bf16_geister_and_geese(name):
    from conftest import golden_sample, net_case_setup, noise_driven
    from handyrl_b200 import fastnet
    from handyrl_b200.train import LearnerStep
    c = NET_CASES[name]
    net, batches = net_case_setup(c)
    args = dict(c['args'], tensor_cores='bf16')
    stepper = LearnerStep(net, args, batches[0], lr=c['lr'])
    convs = [m for m in net.modules() if isinstance(m, fastnet.BoardConv2d)]
    assert convs and all(m.tensor_cores == 'bf16' for m in convs)
    depth = len(convs) + 2
    for s, (batch, ref) in enumerate(zip(batches, c['steps'])):
        stepper.step(stepper.new_packed().fill(batch))
        got = stepper.read_losses()
        _check_losses(got, ref['losses'], depth, s)
        assert got['dcnt'] == ref['dcnt']
    _check_weights(c, stepper.cpu_state_dict(), len(c['steps']), depth, golden_sample, noise_driven)


def test_bf16_graph_and_eager_steps_are_bit_identical():
    from handyrl_b200.nets import tictactoe_net, load_state_by_order
    from handyrl_b200.synthetic import synthetic_batch
    from handyrl_b200.train import LearnerStep
    c = STEP_CASES[sorted(STEP_CASES)[0]]
    B, T, P, A = c['dims']
    mk = lambda s: synthetic_batch(B, T, P, A, turn_based=c['args']['turn_based_training'], observation=c['args']['observation'],
                                   seed=40 + s)
    runs = {}
    for mode, graph in (('bf16', True), ('bf16', False), (True, True)):
        net = load_state_by_order(tictactoe_net(), c['state0'])
        st = LearnerStep(net, dict(c['args'], tensor_cores=mode), mk(0), lr=c['lr'], use_graph=graph)
        for s in range(3):
            st.step(st.new_packed().fill(mk(s)))
        runs[(mode, graph)] = (st.cpu_state_dict(), st.read_losses(), st.launches_per_step)
    (wg, lg, ng), (we, le, _), (_, _, n_default) = runs[('bf16', True)], runs[('bf16', False)], runs[(True, True)]
    assert lg == le
    for k in wg:
        assert torch.equal(wg[k], we[k]), k
    assert ng == n_default and ng > 0


# ---- the dense small-board convolution and the fused tower, product by product ----------------------------------------
@pytest.mark.parametrize('N', [100, 2048])
def test_board_conv_bf16_against_float64(N):
    """ops.board_conv in bf16 mode (the dense small-board convolution of fastnet, TicTacToe-sized boards): forward, input
    gradient, and the weight gradient as one product (N = 100) or as split-K slice partials folded by hrl_board_fold."""
    from handyrl_b200 import ops
    g = torch.Generator(device='cuda').manual_seed(N)
    Cin, Cout, H, W = 32, 32, 3, 3
    x = torch.randn(N, Cin, H, W, device='cuda', generator=g).requires_grad_(True)
    w = (torch.randn(Cout, Cin, 3, 3, device='cuda', generator=g) * 0.1).requires_grad_(True)
    dy = torch.randn(N, Cout, H, W, device='cuda', generator=g)
    y = ops.board_conv(x, w, bf16=True)
    y.backward(dy)
    torch.cuda.synchronize()
    xr, wr, dyr = r16(x.detach()), r16(w.detach()), r16(dy)
    D = Cin * H * W
    _close(y, _conv(xr, wr), accum_bound(D) * _conv(xr.abs(), wr.abs()), 'y')
    _close(x.grad, _conv_in(x.shape, wr, dyr), accum_bound(D) * _conv_in(x.shape, wr.abs(), dyr.abs()), 'dx')
    splits = ops.k_splits(Cout * H * W, Cin * H * W, N)
    assert (splits > 1) == (N > 1000)
    _close(w.grad, _conv_w(xr, w.shape, dyr), _wgrad_bound(N, splits, H * W) * _conv_w(xr.abs(), w.shape, dyr.abs()), 'dw')
    # rounding happened: against the unrounded operands the forward leaves its bound
    assert ((y.double() - _conv(x.detach().double(), w.detach().double())).abs() > accum_bound(D) * _conv(xr.abs(), wr.abs())).any()


TOWER_CASES = {
    'tictactoe': (dict(planes=3, board=(3, 3), width=32, depth=3, actions=9), 2048),
    'return_head': (dict(planes=2, board=(3, 3), width=16, depth=2, actions=7, return_head=True), 515),
}


@pytest.mark.parametrize('name', sorted(TOWER_CASES))
def test_fused_tower_bf16_against_float64_on_rounded_operands(name):
    """tower.FusedBoardNet(bf16=True), forward and backward, product by product against float64 F.conv2d / BatchNorm on the
    operands rounded to bf16 after their fp32 transform.  Each float64 product takes its inputs from the engine's own fp32
    buffers (the previous layer's output, the BatchNorm constants of the finalise kernels): an end-to-end float64 run would
    round some operand elements on the other side of a bf16 boundary than the engine, by amounts no bound derived per product
    covers.  Checked: every product's output (stem, tower layers, squeeze heads, the ReLU-masked input gradients through the
    adjoint images, the weight gradients with their per-row transforms on both operands), the heads, every parameter's .grad,
    the batch statistics and the running buffers."""
    from handyrl_b200 import nets, tower
    kw, M = TOWER_CASES[name]
    torch.manual_seed(17)
    net = nets.BoardNet(**kw).cuda().train()
    for blk in net.tower:                # non-trivial affine parameters and running statistics
        blk[1].weight.data.uniform_(0.5, 1.5)
        blk[1].bias.data.normal_(0, 0.3)
        blk[1].running_mean.normal_(0, 0.1)
        blk[1].running_var.uniform_(0.5, 2.0)
    run0 = [(blk[1].running_mean.double().clone(), blk[1].running_var.double().clone()) for blk in net.tower]
    H, W = kw['board']
    cells, planes = H * W, kw['planes']
    x = (torch.rand(M, planes, H, W, device='cuda') < 0.4).float()
    eng = tower.FusedBoardNet(net, M, torch.device('cuda'), bf16=True)
    for p in net.parameters():
        p.grad = torch.full_like(p, 7.0)           # backward must overwrite, not accumulate
    out = eng.forward(x)
    g = torch.Generator().manual_seed(5)
    dout = {k: torch.randn(v.shape, generator=g).cuda().double() for k, v in out.items()}
    eng.backward(dout['policy'].float(), dout['value'].float(), dout['return'].float() if 'return' in dout else None)
    torch.cuda.synchronize()
    L, C_, NH = eng.depth, eng.width, eng.NH
    n = M * cells
    img = lambda t, ch: t.double().reshape(M, ch, H, W)
    W16 = lambda w: r16(w.detach())
    Wabs = lambda w: r16(w.detach()).abs()

    def act(l):
        """the operand the engine builds from layer l's output: relu(fmaf(Y_l, scale, shift)) rounded to bf16 (l = -1: A0)"""
        if l < 0:
            return r16(eng.A0), torch.zeros(M, eng.D, dtype=torch.float64, device='cuda')
        st = eng.bn[l]
        return _transform_ref(eng.Y[l], st['scale'][None], st['shift'][None], relu=True)

    def mask(l):
        if l < 0:
            return eng.A0.double() > 0
        st = eng.bn[l]
        return (eng.Y[l].double() * st['scale'].double() + st['shift'].double()).float() > 0

    # ---- forward
    w0, b0 = net.stem.weight, net.stem.bias.detach().double()
    xr = r16(x)
    _close(eng.A0.view(M, C_, H, W), F.relu(_conv(xr, W16(w0), b0)), accum_bound(planes * cells) * _conv(xr, Wabs(w0), b0.abs()), 'A0')
    for l, blk in enumerate(net.tower):
        a, e = act(l - 1)
        wl = blk[0].weight
        bound = accum_bound(eng.D) * _conv(img(a, C_).abs(), Wabs(wl)) + _conv(img(e, C_), Wabs(wl))
        _close(eng.Y[l].view(M, C_, H, W), _conv(img(a, C_), W16(wl)), bound, 'Y%d' % l)
        # batch statistics (fp32 column sums over a row tile, summed in double) and the running buffers
        y = eng.Y[l].double().view(M, C_, cells)
        mean, var, ey2 = y.mean((0, 2)), y.var((0, 2), unbiased=False), (y * y).mean((0, 2))
        e_mean, e_var = 128 * U32 * y.abs().mean((0, 2)), 4 * 128 * U32 * ey2
        st, bn = eng.bn[l], blk[1]
        _close(st['mean'].view(C_, cells)[:, 0], mean, e_mean + 1e-30, 'mean%d' % l)
        rstd = (var + bn.eps).rsqrt()
        _close(st['rstd'].view(C_, cells)[:, 0], rstd, rstd * (e_var / (var + bn.eps) + 4 * U32), 'rstd%d' % l)
        m_, (rm0, rv0) = bn.momentum, run0[l]
        _close(bn.running_mean, (1 - m_) * rm0 + m_ * mean, m_ * e_mean + 4 * U32 * (rm0.abs() + mean.abs()), 'running_mean%d' % l)
        _close(bn.running_var, (1 - m_) * rv0 + m_ * var * n / (n - 1), m_ * e_var * n / (n - 1) + 4 * U32 * (rv0 + var), 'running_var%d' % l)
    sq = [net.p_squeeze, net.v_squeeze] + ([net.r_squeeze] if eng.rmaps else [])
    wsq = torch.cat([s.weight for s in sq])
    bsq = torch.cat([s.bias for s in sq]).detach().double()
    a_top, e_top = act(L - 1)
    hpre_ref = _conv(img(a_top, C_), W16(wsq), bsq).reshape(M, NH)
    bound = accum_bound(eng.D) * _conv(img(a_top, C_).abs(), Wabs(wsq), bsq.abs()) + _conv(img(e_top, C_), Wabs(wsq))
    _close(eng.Hpre[:, :NH], hpre_ref, bound.reshape(M, NH), 'Hpre')
    # heads (fp32 kernels): LeakyReLU, then the Linear layers (tanh on the value)
    pre = eng.Hpre[:, :NH].double()
    pc, vc = eng.pmaps * cells, eng.vmaps * cells
    parts = {'policy': (slice(0, pc), net.p_out), 'value': (slice(pc, pc + vc), net.v_out)}
    if eng.rmaps:
        parts['return'] = (slice(pc + vc, NH), net.r_out)
    for k, (cols, lin) in parts.items():
        h = F.leaky_relu(pre[:, cols], eng.slope)
        wl = lin.weight.detach().double()
        z, za = h @ wl.t(), h.abs() @ wl.abs().t()
        want = torch.tanh(z) if k == 'value' else z
        _close(out[k], want, (h.shape[1] + 2) * U32 * za + (4 * U32 if k == 'value' else 0), k)

    # ---- backward: heads
    dpre = torch.zeros_like(pre)
    for k, (cols, lin) in parts.items():
        wl = lin.weight.detach().double()
        dz = dout[k] * (1 - eng.value.double() ** 2) if k == 'value' else dout[k]
        slope = torch.where(pre[:, cols] > 0, 1.0, eng.slope)
        dpre[:, cols] = slope * (dz @ wl)
        h = F.leaky_relu(pre[:, cols], eng.slope)
        dza = dz.abs() + (4 * U32 * dout[k].abs() if k == 'value' else 0)
        _close(eng.dHpre[:, cols], dpre[:, cols], (wl.shape[0] + 2) * U32 * slope * (dza @ wl.abs()) + 4 * U32 * (dout[k].abs() @ wl.abs()) * (k == 'value'), 'dpre_' + k)
        _close(lin.weight.grad, dz.t() @ h, (M + 2) * U32 * (dza.t() @ h.abs()), k + '_out.grad')
    dh = r16(eng.dHpre[:, :NH])
    dhi, dhai = img(dh, NH // cells), img(dh.abs(), NH // cells)
    # squeeze convolutions: bias gradients (column sums of dpre), weight gradient over the samples (per-row BatchNorm-apply +
    # ReLU of the B operand), then the input gradient through the adjoint image with the last ReLU mask
    row = 0
    s_heads = eng.splits['heads']
    dw_ref = _conv_w(img(a_top, C_), wsq.shape, dhi)
    dw_bound = _wgrad_bound(M, s_heads, cells) * _conv_w(img(a_top, C_).abs(), wsq.shape, dhai) + _conv_w(img(e_top, C_), wsq.shape, dhai)
    for s in sq:
        o = s.out_channels
        _close(s.weight.grad, dw_ref[row:row + o], dw_bound[row:row + o], 'squeeze.weight.grad')
        seg = eng.dHpre[:, row * cells:(row + o) * cells].double().view(M, o, cells)
        _close(s.bias.grad, seg.sum((0, 2)), (n + 1) * U32 * seg.abs().sum((0, 2)), 'squeeze.bias.grad')
        row += o
    dz_ref = _conv_in((M, C_, H, W), W16(wsq), dhi).reshape(M, -1) * mask(L - 1)
    _close(eng.dZ[L - 1], dz_ref, accum_bound(NH) * _conv_in((M, C_, H, W), Wabs(wsq), dhai).reshape(M, -1), 'dZ%d' % (L - 1))

    # ---- backward: tower layers
    for l in range(L - 1, -1, -1):
        blk, st = net.tower[l], eng.bn[l]
        bn, wl = blk[1], blk[0].weight
        dz = eng.dZ[l].double().view(M, C_, cells)
        xh = ((eng.Y[l] - st['mean']) * st['rstd']).double().view(M, C_, cells)          # the epilogue's fp32 xhat
        _close(bn.bias.grad, dz.sum((0, 2)), (n + 1) * U32 * dz.abs().sum((0, 2)), 'bn%d.bias.grad' % l)
        _close(bn.weight.grad, (dz * xh).sum((0, 2)), (n + 2) * U32 * (dz * xh).abs().sum((0, 2)), 'bn%d.weight.grad' % l)
        # dY_l = dZ_l * p + Y_l * q + r, formed while staged; the layer's input operand as in the forward
        dy, e_dy = _transform_ref(eng.dZ[l], st['p'][None], st['r'][None], y=eng.Y[l], q=st['q'][None])
        a, e = act(l - 1)
        dyi, dyai, ei = img(dy, C_), img(dy.abs(), C_), img(e_dy, C_)
        ai, aai, eai = img(a, C_), img(a.abs(), C_), img(e, C_)
        shape = wl.shape
        bound = (_wgrad_bound(M, eng.splits['tower'], cells) * _conv_w(aai, shape, dyai) + _conv_w(eai, shape, dyai) +
                 _conv_w(aai, shape, ei) + _conv_w(eai, shape, ei))
        _close(wl.grad, _conv_w(ai, shape, dyi), bound, 'tower%d.weight.grad' % l)
        target = eng.dZ[l - 1] if l > 0 else eng.dZ0
        want = _conv_in((M, C_, H, W), W16(wl), dyi).reshape(M, -1) * mask(l - 1)
        bound = accum_bound(eng.D) * _conv_in((M, C_, H, W), Wabs(wl), dyai) + _conv_in((M, C_, H, W), Wabs(wl), ei)
        _close(target, want, bound.reshape(M, -1), 'dZ%d' % (l - 1))
    # ---- backward: stem
    dz0 = eng.dZ0.double().view(M, C_, cells)
    _close(net.stem.bias.grad, dz0.sum((0, 2)), (n + 1) * U32 * dz0.abs().sum((0, 2)), 'stem.bias.grad')
    d0 = r16(eng.dZ0)
    bound = _wgrad_bound(M, eng.splits['stem'], cells) * _conv_w(xr, w0.shape, img(d0.abs(), C_))
    _close(w0.grad, _conv_w(xr, w0.shape, img(d0, C_)), bound, 'stem.weight.grad')
    for p in net.parameters():
        assert not (p.grad == 7.0).all()
