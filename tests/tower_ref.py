"""Float64 references and error bounds shared by the tensor-core product tests (test_bf16_gpu.py, test_tower_products_gpu.py,
test_gemm_tower_gpu.py, test_conv_products_gpu.py): the board convolutions and their gradients (zero or wrap-around padding,
any odd kernel, by explicit index arithmetic), the operand transforms as the kernels compute them in fp32, the accumulation
bounds of the products and of the weight-gradient fold, and a trace of the GEMM kernels a call launches."""
import re
import time

import torch
import torch.nn.functional as F

U32 = 2.0 ** -23          # fp32 accumulation, truncating: relative error of one addition
U16 = 2.0 ** -8           # bf16 round to nearest: relative error of one rounding <= 2^-9 (8 stored mantissa bits)


def r16(t):
    """t rounded to bf16 (nearest even), as float64"""
    return t.bfloat16().double()


def accum_bound(K, splits=1):
    """fp32 accumulation error of K exact terms in `splits` K slices, relative to sum|a||b| (test_gemm_gpu.py)"""
    from handyrl_b200._capi import lib
    k_slice = -(-K // lib().hrl_gemm_effective_splits(K, splits))
    return 1.2e-7 * (0.8 * k_slice ** 0.5 + 4)


def product_bound(K, splits=1):
    """accum_bound, but never below U32 (32 + 8): a K slice of one 32-element chunk is 12 truncating wgmma accumulations (3xTF32)
    whose worst case accum_bound's sqrt(K) form leaves out at small K (test_tower_products_gpu.tf32x3_bound of one chunk)"""
    return max(accum_bound(K, splits), 40 * U32)


def _conv(a, w, b=None):
    return F.conv2d(a, w, b, padding=w.shape[-1] // 2)


def _conv_in(shape, w, dy):
    return torch.nn.grad.conv2d_input(shape, w, dy, padding=w.shape[-1] // 2)


def _conv_w(a, shape, dy):
    return torch.nn.grad.conv2d_weight(a, shape, dy, padding=shape[-1] // 2)


def _close(got, want, bound, what):
    err = (got.double() - want).abs()
    assert (err <= bound).all(), (what, (err - bound).max().item(), (err / (bound + 1e-300)).max().item())


def _wgrad_bound(K, splits, cells, product=accum_bound):
    """a weight gradient of the dense products: K samples in `splits` slices (each within product(K, splits) of its sum|a||b|),
    then hrl_board_fold's fp32 sums over the slices and over the output cells"""
    return product(K, splits) + (splits + cells + 1) * U32


def _transform_ref(x, p, r, y=None, q=None, relu=False, bf16=True):
    """the kernel's operand transform fmaf(x, p, fmaf(y, q, r)) in float32 (each fmaf exact in float64, rounded once), then
    bf16 rounding; also the elements whose float32 value sits at a bf16 rounding boundary (one float32 ulp decides them).
    bf16=False: the float32 operand itself (what the 3xTF32 products split exactly into hi and lo), with no such elements."""
    inner = r.double() if y is None else (y.double() * q.double() + r.double()).float().double()
    t = (x.double() * p.double() + inner).float()
    if relu:
        t = t.clamp_min(0)
    if not bf16:
        return t.double(), torch.zeros_like(t, dtype=torch.float64)
    up, dn = torch.nextafter(t, torch.full_like(t, float('inf'))), torch.nextafter(t, torch.full_like(t, -float('inf')))
    edge = up.bfloat16() != dn.bfloat16()
    ulp = (t.abs().bfloat16().float() * 2.0 ** -7).double()          # at most one bf16 ulp of the element
    return r16(t), torch.where(edge, ulp, torch.zeros_like(ulp))


def operand_ref(t, bf16):
    """an untransformed operand as the products see it: (value, boundary term) of _transform_ref with p = 1, r = 0"""
    one = torch.ones((), dtype=torch.float32, device=t.device)
    return _transform_ref(t, one, torch.zeros_like(one), bf16=bf16)


_CONV_SRC = {}


def conv_src(H, W, kh, kw, wrap):
    """src[cell, tap] (CPU, int64): the input cell tap (a, b) of output cell (y, x) reads, (y + a - kh//2, x + b - kw//2) taken
    modulo H and W (wrap) or H*W -- an extra zero cell -- off the board.  Index arithmetic only: valid for kernels larger than
    the board, whose wrapped taps read the same cell more than once."""
    key = (H, W, kh, kw, bool(wrap))
    if key not in _CONV_SRC:
        src = torch.empty(H * W, kh * kw, dtype=torch.long)
        for y in range(H):
            for x in range(W):
                for a in range(kh):
                    for b in range(kw):
                        yy, xx = y + a - kh // 2, x + b - kw // 2
                        if wrap:
                            yy, xx = yy % H, xx % W
                        src[y * W + x, a * kw + b] = yy * W + xx if 0 <= yy < H and 0 <= xx < W else H * W
        _CONV_SRC[key] = src
    return _CONV_SRC[key]


def _conv_cols(x, src):
    """x (N, C, H, W) -> (N, C, cells, taps): the input each tap of each output cell reads"""
    N, Cin, H, W = x.shape
    xp = torch.cat([x.reshape(N, Cin, H * W), x.new_zeros(N, Cin, 1)], 2)
    return xp[:, :, src.to(x.device)]


def conv_ref(x, w, src, b=None):
    """y[n, o, cell] = sum over (i, tap) of w[o, i, tap] x[n, i, src[cell, tap]] (+ b[o])"""
    N, _, H, W = x.shape
    y = torch.einsum('nipt,oit->nop', _conv_cols(x, src), w.reshape(w.shape[0], w.shape[1], -1))
    if b is not None:
        y = y + b[None, :, None]
    return y.reshape(N, -1, H, W)


def conv_ref_input(dy, w, src):
    """the input gradient of conv_ref: dy[n, o, cell] w[o, i, tap] scattered onto x[n, i, src[cell, tap]]"""
    N, Cout, H, W = dy.shape
    Cin = w.shape[1]
    g = torch.einsum('nop,oit->nipt', dy.reshape(N, Cout, H * W), w.reshape(Cout, Cin, -1))
    dx = dy.new_zeros(N, Cin, H * W + 1)
    dx.index_add_(2, src.to(dy.device).reshape(-1), g.reshape(N, Cin, -1))
    return dx[:, :, :H * W].reshape(N, Cin, H, W)


def conv_ref_weight(dy, x, src, kh, kw):
    """the weight gradient of conv_ref: sum over (n, cell) of dy[n, o, cell] x[n, i, src[cell, tap]]"""
    N, Cout = dy.shape[:2]
    dw = torch.einsum('nop,nipt->oit', dy.reshape(N, Cout, -1), _conv_cols(x, src))
    return dw.reshape(Cout, x.shape[1], kh, kw)


_GEMM_RE = re.compile(r'(gemm_tower_kernel|gemm_wgrad_kernel|gemm_tf32x3_kernel|gemm_bf16_kernel)<([^>]*)>')


def traced_gemms(fn, attempts=3, runs=1, repeat=1):
    """The GEMM kernels fn() launches, as {(kernel, template arguments)} from a torch.profiler (CUPTI) trace (taken again when
    the tracer dropped every GEMM record).  The tracer can miss launches in its first moments (a fused tower's whole forward pass
    at a small batch) and the record of a kernel that ends as the window closes, so fn() runs after a settled start and the
    window stays open a little after it.  Within a long test session it can also drop the record of a kernel launched once in
    a trace; for an fn() that launches the same kernels every time, repeat > 1 calls it that many times in each trace and
    runs > 1 returns the union of that many traces: a kernel seen in any of them was launched."""
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    union = set()
    for _ in range(runs):
        seen = set()
        for _ in range(attempts):
            with torch.profiler.profile(activities=acts) as prof:
                torch.zeros(1, device='cuda').add_(1)
                torch.cuda.synchronize()
                time.sleep(0.05)
                for _ in range(repeat):
                    fn()
                torch.cuda.synchronize()
                time.sleep(0.002)
            names = set()
            for e in prof.events():
                names.add(e.name)
                names.update(k.name for k in getattr(e, 'kernels', []))
            seen = {(m.group(1), m.group(2).replace(' ', '')) for m in map(_GEMM_RE.search, names) if m}
            if seen:
                break
        union |= seen
    return union
