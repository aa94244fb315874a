"""Float64 references and error bounds shared by the fused tower's tests (test_bf16_gpu.py, test_tower_products_gpu.py,
test_gemm_tower_gpu.py): the board convolutions and their gradients, the operand transforms as the kernels compute them in
fp32, the accumulation bounds of the products and of the weight-gradient fold, and a trace of the GEMM kernels a call
launches."""
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


_GEMM_RE = re.compile(r'(gemm_tower_kernel|gemm_wgrad_kernel|gemm_tf32x3_kernel)<([^>]*)>')


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
