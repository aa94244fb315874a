"""Time ops.gemm_tf32x3 (3xTF32 hrl_gemm_fused) at the shapes of the TicTacToe tower (CUDA events, back to back, L2-warm) vs cuBLAS fp32."""
import ctypes, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from handyrl_b200 import ops
from handyrl_b200._capi import lib

torch.backends.cuda.matmul.allow_tf32 = False
M = int(sys.argv[1]) if len(sys.argv) > 1 else 16384
x = torch.randn(M, 288, device='cuda'); w = torch.randn(288, 288, device='cuda') * 0.1; dy = torch.randn(M, 288, device='cuda')

def timeit(fn, reps=30):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e3

dbg = getattr(lib(), 'hrl_gemm_set_debug', None)
for mode in (0, 1, 2):
    if dbg is None and mode: break
    if dbg is not None: dbg(mode)
    print('debug', mode, 'fwd %.1f us' % timeit(lambda: ops.gemm_tf32x3(x, w)),
          'dgrad %.1f us' % timeit(lambda: ops.gemm_tf32x3(dy, w, b_kmajor=False)),
          'wgrad(48 splits) %.1f us' % timeit(lambda: ops.gemm_tf32x3(dy, x, a_kmajor=False, b_kmajor=False, splits=48)))
if dbg is not None: dbg(0)
print('cublas fp32: fwd %.1f us' % timeit(lambda: x @ w.t()), 'dgrad %.1f us' % timeit(lambda: dy @ w), 'wgrad %.1f us' % timeit(lambda: dy.t() @ x))
