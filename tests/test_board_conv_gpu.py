"""The dense small-board convolution (fastnet.BoardConv2d -> ops.board_conv: hrl_board_expand, the forward and input-gradient
products of hrl_gemm_fused, the split-K weight-gradient product left as slice partials, hrl_board_fold) element by element
against float64, in 3xTF32 and bf16, on the shapes BoardConv2d._eligible admits: boards of 1 to 16 cells, square and not,
kernels larger than the board, one to 57 N tiles, both weight-gradient kernels with one K slice and many, 1 to 16,384 samples,
and dense matrices up to the 2^20-element limit.

Every element is held to a bound of its own arithmetic, relative to its own sum |a||b| (the convolution of the absolute values):
* a product of K terms in s K slices of whole 32-element chunks: 1.2e-7 (0.8 sqrt(k_slice) + 4) of sum|a||b| for the largest
  slice (test_gemm_gpu.py), never below 40 U32: a slice of one chunk is 12 truncating wgmma accumulations (3xTF32), the worst
  case of which the sqrt form leaves out at small K;
* forward: the product over K = Cin*HW, then one rounding of the bias addition;
* input gradient: the product over K = Cout*HW;
* weight gradient: the product over the N samples in its s slices, then hrl_board_fold's fp32 sums over the slices and over
  the output cells, (s + HW + 1) U32;
* bias gradient: torch's fp32 sum of N*HW terms of dy;
* bf16: the same bounds on operands rounded to bf16 first (a bf16 product is exact in fp32, only the accumulation rounds).
Each bound is shown to discriminate: a reference with the kernel flipped in both spatial axes, and one that drops the last
32-element chunk of the forward product, both leave it by far.
"""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -23          # fp32 accumulation, truncating: relative error of one addition

# Cout, Cin, kh, kw, H, W, N, mode, weight-gradient K slices.  Forward: ceil(Cout*HW / 288) N tiles of the generic wgmma kernel,
# input gradient: ceil(Cin*HW / 288) N tiles with the dense matrix read as stored (not K-major).  Weight gradient: Cout*HW rows
# by Cin*HW columns reduced over N, on gemm_wgrad (mma.sync) when both are multiples of 4 in 3xTF32, else on the generic kernel
# with both operands transposed; one K slice -> hrl_board_fold's single-part branch, more -> its slice-run branch.
CASES = [
    (32, 32, 3, 3, 3, 3, 16384, 'tf32x3', 43),    # TicTacToe: 288 columns (MMA width 144), gemm_wgrad, 43 slices
    (32, 32, 3, 3, 3, 3, 2048, 'bf16', 32),       # TicTacToe in bf16: the generic kernel's transposed weight gradient
    (1, 3, 3, 3, 3, 3, 127, 'tf32x3', 1),         # Cout*HW = 9: MMA width 8, K = 27 inside one chunk; generic weight gradient
    (30, 10, 1, 1, 1, 1, 129, 'tf32x3', 2),       # 1x1 board: 9 fold groups of 2 channels over 10, generic, 2 slices
    (9, 5, 1, 1, 1, 1, 1, 'bf16', 1),             # 1x1 board, one sample: one row of the row tile
    (8, 6, 5, 5, 2, 2, 128, 'tf32x3', 2),         # 5x5 kernel on a 2x2 board: only its middle 3x3 taps reach a cell
    (16, 8, 5, 5, 3, 3, 129, 'bf16', 2),          # 5x5 on 3x3, one sample past a row tile
    (17, 11, 3, 3, 4, 4, 3000, 'tf32x3', 32),     # 4x4: Cout*HW = 272, a ragged single tile (MMA width 136), gemm_wgrad
    (64, 3, 1, 3, 1, 16, 2000, 'tf32x3', 16),     # 1x16 with a 1x3 kernel: Cout*HW = 1024, four N tiles, the last 160 wide
    (18, 7, 3, 1, 16, 1, 1, 'tf32x3', 1),         # 16x1 with a 3x1 kernel, one sample: Cout*HW = 288, gemm_wgrad, one slice
    (5, 9, 3, 5, 2, 8, 127, 'tf32x3', 1),         # 2x8 with a 3x5 kernel: taller than the board, gemm_wgrad, one slice
    (9, 11, 3, 5, 3, 5, 4096, 'tf32x3', 64),      # 3x5 with a 3x5 kernel: 135 x 165, two M tiles, generic kernel split-K
    # the fold's shared memory once held every input channel's columns: these three exceeded it
    (16, 256, 3, 3, 4, 4, 129, 'tf32x3', 2),      # exactly 2^20 dense elements; input gradient over 15 N tiles
    (16, 200, 3, 3, 4, 4, 2000, 'tf32x3', 5),     # 819,200 elements, 12 N tiles
    (2, 1024, 1, 1, 4, 4, 300, 'tf32x3', 2),      # a 1x1 head: K = 16,384 forward, 57 N tiles in the input gradient
    (2, 1024, 1, 1, 4, 4, 128, 'bf16', 2),        # the same head in bf16
]


def _id(case):
    Cout, Cin, kh, kw, H, W, N, mode, _ = case
    return '%d-%d-k%dx%d-b%dx%d-n%d-%s' % (Cout, Cin, kh, kw, H, W, N, mode)


def _wgrad_kernel(Cout, Cin, H, W, mode):
    return 'gemm_wgrad' if (Cout * H * W) % 4 == 0 and (Cin * H * W) % 4 == 0 and mode == 'tf32x3' else 'generic'


def _k_slice(K, splits):
    """the largest K slice of a product of K terms in `splits` slices of whole 32-element chunks"""
    from handyrl_b200._capi import lib
    chunks = -(-K // 32)
    return min(K, 32 * -(-chunks // lib().hrl_gemm_effective_splits(K, splits)))


def product_bound(K, splits=1):
    """the error of a tensor-core product of K terms in `splits` K slices, relative to its sum |a||b|"""
    return max(1.2e-7 * (0.8 * _k_slice(K, splits) ** 0.5 + 4), 40 * U32)


def _r16(t):
    return t.bfloat16().double()


def _conv64(x, w, dy, b=None):
    """float64 output, input gradient and weight gradient of the stride-1 "same" convolution (F.conv2d and its autograd)"""
    x, w = x.double().requires_grad_(True), w.double().requires_grad_(True)
    y = F.conv2d(x, w, None if b is None else b.double(), padding=(w.shape[2] // 2, w.shape[3] // 2))
    dx, dw = torch.autograd.grad(y, (x, w), dy.double())
    return y.detach(), dx, dw


def _close(got, want, bound, what):
    err = (got.double() - want).abs()
    assert (err <= bound).all(), (what, (err - bound).max().item(), (err / (bound + 1e-300)).max().item())


def _discriminates(alt, want, bound, what):
    """a wrong reference leaves the bound by far: by more than 10x at a tenth of the elements or more"""
    far = ((alt - want).abs() > 10 * bound).double().mean().item()
    assert far >= 0.1, (what, far)


def _inputs(case):
    Cout, Cin, kh, kw, H, W, N, _, _ = case
    g = torch.Generator().manual_seed(CASES.index(case) * 7919 + N)
    x = torch.randn(N, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, kh, kw, generator=g) * (2.0 / (Cin * kh * kw)) ** 0.5
    b = torch.randn(Cout, generator=g)
    dy = torch.randn(N, Cout, H, W, generator=g)
    return x.cuda(), w.cuda(), b.cuda(), dy.cuda()


def _module(w, b, mode):
    from handyrl_b200 import fastnet
    Cout, Cin, kh, kw = w.shape
    conv = nn.Conv2d(Cin, Cout, (kh, kw), padding=(kh // 2, kw // 2)).cuda()
    with torch.no_grad():
        conv.weight.copy_(w)
        conv.bias.copy_(b)
    assert fastnet.optimize_small_boards(nn.Sequential(conv), tensor_cores='bf16' if mode == 'bf16' else True) == 1
    return conv


def test_case_table_covers_the_admitted_shapes():
    """the routes the table is there for, from the shapes alone"""
    from handyrl_b200 import fastnet
    hw = lambda c: c[4] * c[5]
    assert {(c[4], c[5]) for c in CASES} >= {(1, 1), (2, 2), (3, 3), (4, 4), (1, 16), (16, 1), (2, 8), (3, 5)}
    assert {(c[2], c[3], c[4], c[5]) for c in CASES} >= {(5, 5, 2, 2), (5, 5, 3, 3)}
    assert {(c[2], c[3]) for c in CASES} >= {(1, 1), (3, 3), (5, 5), (1, 3), (3, 1), (3, 5)}
    assert {c[0] * hw(c) for c in CASES} >= {9, 272, 288, 1024}
    assert max(c[1] * hw(c) for c in CASES) == 16384
    assert {_wgrad_kernel(c[0], c[1], c[4], c[5], c[7]) for c in CASES} == {'gemm_wgrad', 'generic'}
    assert any(_wgrad_kernel(c[0], c[1], c[4], c[5], c[7]) == 'generic' and c[8] > 1 and c[7] == 'tf32x3' for c in CASES)
    assert {c[8] > 1 for c in CASES} == {False, True}
    assert {c[6] for c in CASES} >= {1, 127, 128, 129}
    assert all(c[6] <= 4096 or c[:6] == (32, 32, 3, 3, 3, 3) for c in CASES)
    assert max(c[0] * c[1] * hw(c) ** 2 for c in CASES) == fastnet.DENSE_MAX_ELEMS
    assert all(hw(c) <= fastnet.DENSE_MAX_CELLS and c[0] * c[1] * hw(c) ** 2 <= fastnet.DENSE_MAX_ELEMS for c in CASES)


@pytest.mark.parametrize('case', CASES, ids=_id)
def test_board_conv_matches_float64(case, monkeypatch):
    from handyrl_b200 import _capi, fastnet, ops
    Cout, Cin, kh, kw, H, W, N, mode, want_splits = case
    HW, bf16 = H * W, mode == 'bf16'
    x, w, b, dy = _inputs(case)
    conv = _module(w, b, mode)
    splits = ops.k_splits(Cout * HW, Cin * HW, N)
    assert splits == want_splits, splits

    folds = []
    lib = _capi.lib()
    real = lib.hrl_board_fold
    monkeypatch.setattr(lib, 'hrl_board_fold', lambda *a: (folds.append(a[1]), real(*a))[1])
    xs = x.clone().requires_grad_(True)
    before = fastnet.BoardConv2d.dense_calls
    y = conv(xs)
    assert fastnet.BoardConv2d.dense_calls == before + 1
    params = (xs, conv.weight, conv.bias)
    grads = torch.autograd.grad(y, params, dy, retain_graph=True)
    again = torch.autograd.grad(y, params, dy)
    assert folds == [splits, splits]
    # the slices and the fold are summed in a fixed order
    for g0, g1, what in zip(grads, again, ('input', 'weight', 'bias')):
        assert torch.equal(g0, g1), what
    if case[:7] == (32, 32, 3, 3, 3, 3, 16384):
        with torch.no_grad():
            assert torch.equal(conv(x), y)
    dx, dw, db = grads

    (xr, wr, dyr) = (_r16(x), _r16(w), _r16(dy)) if bf16 else (x.double(), w.double(), dy.double())
    bd = b.double()
    want_y, want_dx, want_dw = _conv64(xr, wr, dyr, bd)
    mag_y, mag_dx, mag_dw = _conv64(xr.abs(), wr.abs(), dyr.abs())

    assert y.shape == (N, Cout, H, W)
    bound_y = product_bound(Cin * HW) * mag_y + U32 * (mag_y + bd.abs()[None, :, None, None])
    _close(y, want_y, bound_y, 'output')
    bound_dx = product_bound(Cout * HW) * mag_dx
    _close(dx, want_dx, bound_dx, 'input gradient')
    bound_dw = (product_bound(N, splits) + (splits + HW + 1) * U32) * mag_dw
    _close(dw, want_dw, bound_dw, 'weight gradient')
    dyd = dy.double()
    _close(db, dyd.sum((0, 2, 3)), (N * HW + 1) * U32 * dyd.abs().sum((0, 2, 3)), 'bias gradient')

    if kh * kw > 1:
        flip_y, flip_dx, _ = _conv64(xr, wr.flip(2, 3), dyr, bd)
        _discriminates(flip_y, want_y, bound_y, 'output, flipped kernel')
        _discriminates(flip_dx, want_dx, bound_dx, 'input gradient, flipped kernel')
        _discriminates(want_dw.flip(2, 3), want_dw, bound_dw, 'weight gradient, flipped')
    K = Cin * HW
    short = xr.reshape(N, K).clone()
    short[:, (K - 1) // 32 * 32:] = 0
    drop_y = F.conv2d(short.view(N, Cin, H, W), wr, bd, padding=(kh // 2, kw // 2))
    _discriminates(drop_y, want_y, bound_y, 'output without its last K chunk')


def test_one_element_over_the_dense_limit_takes_another_path():
    """Conv2d(256, 16, 3) on 4x4 boards has exactly 2^20 dense elements (a case above); one input channel more does not take the
    dense path, and still computes the convolution"""
    from handyrl_b200 import fastnet
    g = torch.Generator().manual_seed(5)
    x = torch.randn(64, 257, 4, 4, generator=g).cuda()
    w = torch.randn(16, 257, 3, 3, generator=g).cuda() * 0.05
    b = torch.randn(16, generator=g).cuda()
    dy = torch.randn(64, 16, 4, 4, generator=g).cuda()
    conv = _module(w, b, 'tf32x3')
    assert not conv._eligible(x)
    xs = x.clone().requires_grad_(True)
    before = fastnet.BoardConv2d.dense_calls
    y = conv(xs)
    assert fastnet.BoardConv2d.dense_calls == before
    y.backward(dy)
    want_y, want_dx, want_dw = _conv64(x, w, dy, b)
    mag_y, mag_dx, mag_dw = _conv64(x.abs(), w.abs(), dy.abs())
    # whichever path runs may use TF32 (cuDNN's default: 2^-10 per operand) or a transform algorithm: held to 2^-7
    _close(y, want_y, 2.0 ** -7 * (mag_y + b.double().abs()[None, :, None, None]), 'output')
    _close(xs.grad, want_dx, 2.0 ** -7 * mag_dx, 'input gradient')
    _close(conv.weight.grad, want_dw, 2.0 ** -7 * mag_dw, 'weight gradient')
