"""The implicit convolution products (ops.conv_implicit: hrl_gemm_fused conv_mode 1 / 2 on the neighbour table, the packed images
of hrl_conv_pack / hrl_conv_pack_bf16, hrl_conv_wgrad_reduce, and the deferred segmented weight gradient with hrl_conv_wgrad_reduce2)
element by element against float64, in 3xTF32 and bf16, on the shapes they admit: every MMA width of the packed and the
weight-gradient instantiations, every odd kernel of at most 9 taps on boards of 1 to 256 cells with both paddings, several M and
N tiles and many K slices of the weight gradient, and both branches of the deferred flush.

The float64 reference (tower_ref.conv_ref*) is built from the index arithmetic of the convolution, not from hrl_conv_geometry.
Every element is held to a bound of its own arithmetic, relative to its own sum |a||b| (tower_ref.product_bound for a product
of K terms in its K slices: accum_bound, floored at the worst case of one 32-element chunk); bf16 products are compared on
operands rounded to bf16 (tower_ref.operand_ref):
* forward: product_bound(taps * Cin padded to 32) of |x| * |w|, and one rounding of the bias addition;
* input gradient: the same with the adjoint kernel, K = taps * (Cout padded to 32);
* weight gradient: product_bound(pixels, s) for the s K slices the call launched, plus (s + 1) U32 for hrl_conv_wgrad_reduce's
  fp32 sum of the slices; the deferred form sums n * per slices (n pairs) and rounds once more when it adds into a .grad;
* bias gradient: fp32 sums of dy, (pixels + 1) U32 of sum |dy|, or the ones row of the deferred product.
"""
import pytest
import torch

from tower_ref import (U32, _close, conv_ref, conv_ref_input, conv_ref_weight, conv_src, operand_ref,
                       product_bound, traced_gemms)

pytestmark = pytest.mark.gpu


def _pad32(c):
    return -(-c // 32) * 32


def _inputs(seed, N, Cin, Cout, H, W, kh, kw, bias, channels_last):
    g = torch.Generator(device='cuda').manual_seed(seed)
    x = torch.randn(N, Cin, H, W, device='cuda', generator=g)
    w = torch.randn(Cout, Cin, kh, kw, device='cuda', generator=g) * 0.2
    b = torch.randn(Cout, device='cuda', generator=g) if bias else None
    dy = torch.randn(N, Cout, H, W, device='cuda', generator=g)
    if channels_last:
        x, dy = x.contiguous(memory_format=torch.channels_last), dy.contiguous(memory_format=torch.channels_last)
    return x, w, b, dy


def _record(monkeypatch, fn, calls):
    """record the arguments of every call of the library function `fn` (and make it)"""
    from handyrl_b200 import _capi
    lib = _capi.lib()
    real = getattr(lib, fn)
    monkeypatch.setattr(lib, fn, lambda *a: (calls.append(a), real(*a))[1])


def check_conv(N, Cin, Cout, H, W, kh, kw, wrap, bias, bf16, channels_last, monkeypatch, seed=0):
    """one forward and backward of ops.conv_implicit, every output against float64; returns the weight gradient's K slices"""
    from handyrl_b200 import ops
    x, w, b, dy = _inputs(seed or N * 1000 + Cin * 10 + Cout, N, Cin, Cout, H, W, kh, kw, bias, channels_last)
    assert ops.conv_implicit_supported(x, w)
    xs, ws = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    bs = b.clone().requires_grad_(True) if bias else None
    ops.conv_weights_changed()
    calls = []
    with monkeypatch.context() as m:
        _record(m, 'hrl_conv_wgrad_reduce', calls)
        y = ops.conv_implicit(xs, ws, bs, wrap, bf16=bf16)
        y.backward(dy)
    (reduce,) = calls
    s = reduce[1]
    pixels, taps = N * H * W, kh * kw
    src = conv_src(H, W, kh, kw, wrap)
    (xr, ex), (wr, ew), (dyr, edy) = operand_ref(x, bf16), operand_ref(w, bf16), operand_ref(dy, bf16)
    xa, wa, dya = xr.abs(), wr.abs(), dyr.abs()
    bd = b.double() if bias else None

    assert y.shape == (N, Cout, H, W)
    mag = conv_ref(xa, wa, src)
    bound = product_bound(taps * _pad32(Cin)) * mag + conv_ref(ex, wa, src) + conv_ref(xa, ew, src)
    if bias:
        bound = bound + U32 * (mag + bd.abs()[None, :, None, None])
    _close(y, conv_ref(xr, wr, src, bd), bound, 'output')

    bound = (product_bound(taps * _pad32(Cout)) * conv_ref_input(dya, wa, src) + conv_ref_input(edy, wa, src)
             + conv_ref_input(dya, ew, src))
    _close(xs.grad, conv_ref_input(dyr, wr, src), bound, 'input gradient')

    bound = ((product_bound(pixels, s) + (s + 1) * U32) * conv_ref_weight(dya, xa, src, kh, kw)
             + conv_ref_weight(edy, xa, src, kh, kw) + conv_ref_weight(dya, ex, src, kh, kw))
    _close(ws.grad, conv_ref_weight(dyr, xr, src, kh, kw), bound, 'weight gradient')
    if bias:
        dyd = dy.double()
        _close(bs.grad, dyd.sum((0, 2, 3)), (pixels + 1) * U32 * dyd.abs().sum((0, 2, 3)), 'bias gradient')
    return s


# ---- every MMA width --------------------------------------------------------------------------------------------------
# Cout, Cin, kh, kw.  The forward's width is padded_rows(Cout) / 2, the input gradient's padded_rows(Cin) / 2 and the weight
# gradient's padded_rows(min(taps * Cin, 288)) / 2.  The first twenty rows give the forward one Cout per width and the input
# gradient the same spread over Cin, mostly with padded rows (Cout, Cin = 12 mod 16) and with Cin % 32 in {4, 28, 0}; the last
# nine give the weight gradient the widths those leave out.
WIDTH_CASES = [
    (4, 288, 1, 1), (12, 284, 3, 3), (28, 256, 1, 3), (44, 252, 3, 1), (60, 236, 5, 1), (76, 220, 1, 1), (92, 204, 1, 5),
    (108, 188, 7, 1), (124, 172, 1, 1), (140, 156, 1, 9), (156, 140, 1, 1), (172, 124, 3, 3), (188, 108, 1, 3),
    (204, 92, 3, 1), (220, 76, 5, 1), (236, 60, 1, 1), (252, 44, 1, 5), (256, 28, 7, 1), (284, 12, 1, 1), (288, 4, 1, 9),
    (8, 4, 1, 7), (16, 8, 3, 3), (24, 12, 7, 1), (32, 12, 9, 1), (40, 24, 1, 5), (48, 52, 1, 3), (20, 36, 5, 1),
    (36, 76, 3, 1), (68, 28, 3, 3),
]


def _width(n):
    from handyrl_b200._capi import lib
    return lib().hrl_gemm_padded_rows(min(n, 288)) // 2


def test_width_sweep_launches_every_mma_width():
    """the 17 widths of the dispatch (8 ... 128 in steps of 8, and 144), for the packed products and the weight gradient"""
    every = {_width(n) for n in range(1, 289)}
    assert every == set(range(8, 129, 8)) | {144}
    assert {_width(co) for co, _, _, _ in WIDTH_CASES[:20]} == every                     # forward
    assert {_width(ci) for _, ci, _, _ in WIDTH_CASES[:20]} == every                     # input gradient
    assert {_width(kh * kw * ci) for _, ci, kh, kw in WIDTH_CASES} == every              # weight gradient
    assert {ci % 32 for _, ci, _, _ in WIDTH_CASES[:20]} >= {4, 28, 0}


@pytest.mark.parametrize('bf16', [False, True])
@pytest.mark.parametrize('Cout,Cin,kh,kw', WIDTH_CASES)
def test_every_width_matches_float64(Cout, Cin, kh, kw, bf16, monkeypatch):
    i = WIDTH_CASES.index((Cout, Cin, kh, kw))
    check_conv(3, Cin, Cout, 7, 11, kh, kw, wrap=i % 2 == 0, bias=i % 3 != 0, bf16=bf16, channels_last=i % 2 == 1,
               monkeypatch=monkeypatch)


@pytest.mark.parametrize('bf16', [False, True])
@pytest.mark.parametrize('Cout,Cin,kh,kw', [(4, 288, 1, 1), (188, 108, 1, 3), (16, 8, 3, 3)])
def test_conv_products_run_the_expected_instantiations(Cout, Cin, kh, kw, bf16):
    """forward and input gradient on the packed <k-major, k-major, packed, NW> instantiation, the weight gradient on the
    <plain, plain, plain, NW> one, at the widths the shape asks for; never the tower or the weight-gradient kernel"""
    from handyrl_b200 import ops
    x, w, b, dy = _inputs(7, 3, Cin, Cout, 7, 11, kh, kw, True, True)
    xs, ws = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    ops.conv_weights_changed()

    def step():
        ops.conv_implicit(xs, ws, b, True, bf16=bf16).backward(dy)
    seen = traced_gemms(step, runs=2, repeat=2)
    kernel = 'gemm_bf16_kernel' if bf16 else 'gemm_tf32x3_kernel'
    assert seen == {(kernel, 'true,true,true,%d' % _width(Cout)), (kernel, 'true,true,true,%d' % _width(Cin)),
                    (kernel, 'false,false,false,%d' % _width(kh * kw * Cin))}, seen


# ---- every odd kernel of at most 9 taps, on boards of 1 to 256 cells ---------------------------------------------------------
KERNELS = [(1, 1), (1, 3), (3, 1), (3, 3), (1, 5), (5, 1), (1, 7), (7, 1), (1, 9), (9, 1)]
BOARDS = {        # H, W, boards in the batch: M = N * H * W is not a multiple of 128 below 256 cells (row tiles straddle boards)
    '1x1': (1, 1, 37),
    '3x3': (3, 3, 15),            # a 1x9 / 9x1 kernel is wider / taller than the board: wrapped taps alias the same cell
    '6x6': (6, 6, 5),
    '7x11': (7, 11, 3),
    '1x256': (1, 256, 2),         # 256-cell boards: full neighbour tables (up to 2304 entries)
    '16x16': (16, 16, 2),
    '2x128': (2, 128, 2),
}


@pytest.mark.parametrize('bf16', [False, True])
@pytest.mark.parametrize('wrap', [False, True])
@pytest.mark.parametrize('kh,kw', KERNELS)
@pytest.mark.parametrize('board', list(BOARDS))
def test_every_kernel_and_board_matches_float64(board, kh, kw, wrap, bf16, monkeypatch):
    H, W, N = BOARDS[board]
    i = KERNELS.index((kh, kw))
    Cin, Cout = (36, 20) if i % 2 else (20, 36)
    check_conv(N, Cin, Cout, H, W, kh, kw, wrap, bias=True, bf16=bf16, channels_last=i % 2 == 0, monkeypatch=monkeypatch)


# ---- weight-gradient tiling ---------------------------------------------------------------------------------------------------
WGRAD_CASES = {   # N, Cin, Cout, H, W, kh, kw, wrap
    'one_slice': (2, 16, 24, 6, 6, 3, 3, False),         # 72 pixels: one K slice, written straight into the result
    'split_k': (512, 32, 32, 7, 11, 3, 3, True),         # 39,424 pixels in 132 K slices
    'cout132': (5, 32, 132, 6, 6, 3, 3, False),          # two M tiles
    'cout288': (9, 16, 288, 7, 11, 3, 3, True),          # three M tiles
    'cin288': (40, 288, 20, 6, 6, 3, 3, False),          # N = 9 * 288 = 2592: nine N tiles
}


@pytest.mark.parametrize('bf16', [False, True])
@pytest.mark.parametrize('name', list(WGRAD_CASES))
def test_weight_gradient_tiling_matches_float64(name, bf16, monkeypatch):
    N, Cin, Cout, H, W, kh, kw, wrap = WGRAD_CASES[name]
    s = check_conv(N, Cin, Cout, H, W, kh, kw, wrap, bias=True, bf16=bf16, channels_last=not bf16, monkeypatch=monkeypatch)
    assert (s == 1) == (name == 'one_slice'), s
    if name == 'split_k':
        assert s > 100


# the shapes the suite has always checked (Geister's ConvLSTM gates, the Geese torus block, padded chunks, a board smaller than
# a chunk, one-row and one-column kernels at the widest operand tile), now element by element
REFERENCE_CASES = [
    # N, Cin, Cout, H, W, kh, kw, wrap, bias
    (37, 64, 128, 6, 6, 3, 3, False, True),
    (21, 32, 32, 7, 11, 3, 3, True, True),
    (9, 36, 20, 6, 6, 3, 3, False, False),
    (130, 8, 12, 3, 3, 3, 3, False, True),
    (5, 16, 288, 5, 4, 1, 3, True, False),
    (3, 288, 8, 4, 4, 3, 1, False, True),
]


@pytest.mark.parametrize('N,Cin,Cout,H,W,kh,kw,wrap,bias', REFERENCE_CASES)
@pytest.mark.parametrize('channels_last', [True, False])
def test_conv_implicit_matches_float64(N, Cin, Cout, H, W, kh, kw, wrap, bias, channels_last, monkeypatch):
    check_conv(N, Cin, Cout, H, W, kh, kw, wrap, bias, False, channels_last, monkeypatch)


# ---- deferred weight gradients -----------------------------------------------------------------------------------------------
DEFER_CASES = {   # boards per pair, H, W, pairs, bf16, whether the bias gradient is the product's ones row
    # Geese's torus block (Cin = 32, 3x3: 288 columns): the ones row would open a second N tile and halve the K slices, so
    # the bias gradient is a sum of each pair's dy
    'cfg4': (60, 7, 11, 2, False, False),
    'ones_alone': (1, 7, 11, 3, False, True),           # 77 pixels, one slice: the ones row alone in its second N tile
    'many_pairs': (2, 7, 11, 70, False, False),         # two segmented products (64 + 6 pairs), column sums of 70 pairs
    'bf16': (1, 7, 11, 5, True, True),
    'bf16_cfg4': (60, 7, 11, 2, True, False),
}


@pytest.mark.parametrize('prefilled', [False, True])
@pytest.mark.parametrize('name', list(DEFER_CASES))
def test_deferred_weight_gradient_matches_float64(name, prefilled, monkeypatch):
    """one weight (Cin = Cout = 32, 3x3, with bias) applied to several inputs; inside deferred_weight_gradients() its gradient is
    ONE segmented product per 64 pairs and one hrl_conv_wgrad_reduce2 each, which adds into .grad: the ones row's column into
    bias.grad, or (when that column would cost K slices) torch sums of each pair's dy"""
    from handyrl_b200 import ops
    N, H, W, pairs, bf16, ones = DEFER_CASES[name]
    C, taps = 32, 9
    g = torch.Generator(device='cuda').manual_seed(31 + pairs)
    w = torch.nn.Parameter(torch.randn(C, C, 3, 3, device='cuda', generator=g) * 0.2)
    b = torch.nn.Parameter(torch.randn(C, device='cuda', generator=g))
    xs = [torch.randn(N, C, H, W, device='cuda', generator=g) for _ in range(pairs)]
    dys = [torch.randn(N, C, H, W, device='cuda', generator=g) for _ in range(pairs)]
    g0 = (torch.randn(C, C, 3, 3, device='cuda', generator=g), torch.randn(C, device='cuda', generator=g))
    w.grad, b.grad = (g0[0].clone(), g0[1].clone()) if prefilled else (None, None)
    ops.conv_weights_changed()
    outs = [ops.conv_implicit(x, w, b, True, bf16=bf16) for x in xs]
    calls = []
    before = ops.LAUNCHES['n']
    with monkeypatch.context() as m:
        _record(m, 'hrl_conv_wgrad_reduce2', calls)
        with ops.deferred_weight_gradients():
            torch.autograd.backward(outs, dys)
    chunks = -(-pairs // 64)
    assert ops.LAUNCHES['n'] - before == 2 * chunks          # one segmented product and one reduction per 64 pairs, nothing else
    assert len(calls) == chunks
    assert all(c[2] == taps * C + ones and (c[4] is not None) == ones for c in calls), calls
    slices = sum(c[1] for c in calls)
    per = max(c[1] // min(64, pairs - 64 * i) for i, c in enumerate(calls))
    pixels = N * H * W
    if name in ('cfg4', 'bf16_cfg4'):
        assert per > 1

    src = conv_src(H, W, 3, 3, True)
    want, mag, edge = 0, 0, 0
    for x, dy in zip(xs, dys):
        (xr, ex), (dyr, edy) = operand_ref(x, bf16), operand_ref(dy, bf16)
        want = want + conv_ref_weight(dyr, xr, src, 3, 3)
        mag = mag + conv_ref_weight(dyr.abs(), xr.abs(), src, 3, 3)
        edge = edge + conv_ref_weight(edy, xr.abs(), src, 3, 3) + conv_ref_weight(dyr.abs(), ex, src, 3, 3)
    g0w, g0b = (g0[0].double(), g0[1].double()) if prefilled else (0, 0)
    _close(w.grad, want + g0w, (product_bound(pixels, per) + (slices + chunks + 2) * U32) * mag + edge + U32 * abs(want + g0w),
           'weight gradient')
    # the ones row multiplies dy as the product reads it (rounded to bf16 in bf16 mode); the column sums read fp32 dy
    dys_b = [operand_ref(dy, bf16 and ones) for dy in dys]
    db = sum(d.sum((0, 2, 3)) for d, _ in dys_b)
    dba = sum(d.abs().sum((0, 2, 3)) for d, _ in dys_b)
    dbe = sum(e.sum((0, 2, 3)) for _, e in dys_b)
    k_terms = product_bound(pixels, per) + (slices + chunks + 2) * U32 if ones else (pixels + pairs + 2) * U32
    _close(b.grad, db + g0b, k_terms * dba + dbe + U32 * abs(db + g0b), 'bias gradient')


def test_deferred_pair_of_another_pixel_count_takes_the_immediate_product(monkeypatch):
    """pairs of one segmented product cover the same pixels: an application to a batch of another size gets its own product"""
    from handyrl_b200 import ops
    g = torch.Generator(device='cuda').manual_seed(41)
    C, H, W = 32, 6, 6
    w = torch.nn.Parameter(torch.randn(C, C, 3, 3, device='cuda', generator=g) * 0.2)
    b = torch.nn.Parameter(torch.randn(C, device='cuda', generator=g))
    xs = [torch.randn(N, C, H, W, device='cuda', generator=g) for N in (4, 4, 3)]
    dys = [torch.randn(x.shape, device='cuda', generator=g) for x in xs]
    ops.conv_weights_changed()
    outs = [ops.conv_implicit(x, w, b, False) for x in xs]
    deferred, immediate = [], []
    before = ops.LAUNCHES['n']
    with monkeypatch.context() as m:
        _record(m, 'hrl_conv_wgrad_reduce2', deferred)
        _record(m, 'hrl_conv_wgrad_reduce', immediate)
        with ops.deferred_weight_gradients():
            torch.autograd.backward(outs[:2], dys[:2])
            outs[2].backward(dys[2])
    assert ops.LAUNCHES['n'] - before == 4 and len(deferred) == 1 and len(immediate) == 1
    # hrl_conv_wgrad_reduce goes through hrl_conv_wgrad_reduce2 inside the library, not through the binding: one call each
    slices = deferred[0][1] + immediate[0][1]
    src = conv_src(H, W, 3, 3, False)
    want = sum(conv_ref_weight(dy.double(), x.double(), src, 3, 3) for x, dy in zip(xs, dys))
    mag = sum(conv_ref_weight(dy.double().abs(), x.double().abs(), src, 3, 3) for x, dy in zip(xs, dys))
    _close(w.grad, want, (product_bound(144, 1) + (slices + 4) * U32) * mag, 'weight gradient')
    db = sum(dy.double().sum((0, 2, 3)) for dy in dys)
    dba = sum(dy.double().abs().sum((0, 2, 3)) for dy in dys)
    _close(b.grad, db, (product_bound(144, 1) + (slices + 4 + 144) * U32) * dba, 'bias gradient')


@pytest.mark.parametrize('bf16', [False, True])
def test_deferred_weight_applied_to_two_geometries_matches_float64(bf16, monkeypatch):
    """one weight applied to boards of two shapes with equal pixel counts (6 boards of 6x6, 4 of 9x6), and on one board shape
    with both paddings: every pair is reduced over its own neighbour table, one deferred product per geometry"""
    from handyrl_b200 import ops
    g = torch.Generator(device='cuda').manual_seed(43)
    C = 32
    w = torch.nn.Parameter(torch.randn(C, C, 3, 3, device='cuda', generator=g) * 0.2)
    b = torch.nn.Parameter(torch.randn(C, device='cuda', generator=g))
    apps = [((6, 6, 6), False), ((4, 9, 6), False), ((6, 6, 6), True), ((6, 6, 6), False)]      # (N, H, W), wrap
    xs = [torch.randn(N, C, H, W, device='cuda', generator=g) for (N, H, W), _ in apps]
    dys = [torch.randn(x.shape, device='cuda', generator=g) for x in xs]
    ops.conv_weights_changed()
    outs = [ops.conv_implicit(x, w, b, wrap, bf16=bf16) for x, (_, wrap) in zip(xs, apps)]
    calls = []
    with monkeypatch.context() as m:
        _record(m, 'hrl_conv_wgrad_reduce2', calls)
        with ops.deferred_weight_gradients():
            torch.autograd.backward(outs, dys)
    slices = sum(c[1] for c in calls)
    want, mag, edge, db, dba = 0, 0, 0, 0, 0
    for x, dy, ((N, H, W), wrap) in zip(xs, dys, apps):
        src = conv_src(H, W, 3, 3, wrap)
        (xr, ex), (dyr, edy) = operand_ref(x, bf16), operand_ref(dy, bf16)
        want = want + conv_ref_weight(dyr, xr, src, 3, 3)
        mag = mag + conv_ref_weight(dyr.abs(), xr.abs(), src, 3, 3)
        edge = edge + conv_ref_weight(edy, xr.abs(), src, 3, 3) + conv_ref_weight(dyr.abs(), ex, src, 3, 3)
        db, dba = db + dyr.sum((0, 2, 3)), dba + dyr.abs().sum((0, 2, 3)) + edy.sum((0, 2, 3))
    _close(w.grad, want, (product_bound(216, 1) + (slices + 6) * U32) * mag + edge, 'weight gradient')
    _close(b.grad, db, (product_bound(216, 1) + (slices + 6) * U32) * dba, 'bias gradient')
    assert len(calls) == 3                                  # 6x6 zero padding (two pairs), 9x6, 6x6 wrapped
