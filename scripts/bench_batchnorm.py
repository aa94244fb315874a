"""Time hrl_bn_train_fwd / _bwd (csrc/bn_kernel.cu) of this build against another build of the library, alternating them.

    python scripts/bench_batchnorm.py --baseline-lib PATH/libhrl_b200.so [--reps 50] [--rounds 5]

Shapes: the BatchNorm activations of the Geister net (configs[2]: 256 x 20 x 2 positions of a 6x6 board, 32 maps, NCHW and
channels-last) and of the Hungry Geese tower (configs[3]: 256 x 32 x 4 positions of a 7x11 board, 32 maps, channels-last).
Each round times `reps` forward + backward calls of one library with CUDA events, then the other; the lines report the median
over rounds per library and the card's name and power limit, which the times belong to.  Both libraries are loaded by
path with their own ctypes bindings, so the baseline may be any build that exports the same two functions.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = [('cfg3 geister', (10240, 32, 6, 6), False), ('cfg3 geister', (10240, 32, 6, 6), True),
          ('cfg4 geese', (32768, 32, 7, 11), True)]


def load(path):
    h = C.CDLL(path)
    h.hrl_bn_workspace_floats.restype = C.c_size_t
    h.hrl_bn_workspace_floats.argtypes = [C.c_int64, C.c_int32, C.c_int32, C.c_int32]
    h.hrl_bn_train_fwd.restype = C.c_int
    h.hrl_bn_train_fwd.argtypes = [C.c_void_p] * 8 + [C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_float, C.c_void_p, C.c_void_p]
    h.hrl_bn_train_bwd.restype = C.c_int
    h.hrl_bn_train_bwd.argtypes = [C.c_void_p] * 8 + [C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    return h


def card():
    import torch
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        out = torch.cuda.get_device_name() + ', power limit unknown'
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--baseline-lib', required=True)
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--rounds', type=int, default=5)
    opt = ap.parse_args()
    import torch
    from handyrl_b200 import _capi
    assert torch.cuda.is_available(), 'bench_batchnorm needs a GPU'
    libs = {'this build': load(_capi.LIB_PATH), 'baseline': load(os.path.abspath(opt.baseline_lib))}
    gpu = card()
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    for name, shape, cl in SHAPES:
        N, Cn, H, W = shape
        g = torch.Generator(device='cuda').manual_seed(0)
        fmt = torch.channels_last if cl else torch.contiguous_format
        x = torch.randn(shape, device='cuda', generator=g).contiguous(memory_format=fmt)
        dy = torch.randn(shape, device='cuda', generator=g).contiguous(memory_format=fmt)
        y, dx = torch.empty_like(x), torch.empty_like(x)
        gamma, beta = torch.ones(Cn, device='cuda'), torch.zeros(Cn, device='cuda')
        mean, rstd, rm, rv, dg, db = (torch.zeros(Cn, device='cuda') for _ in range(6))
        ws = torch.empty(max(h.hrl_bn_workspace_floats(N, Cn, H * W, int(cl)) for h in libs.values()), device='cuda')
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

        def run(h):
            assert h.hrl_bn_train_fwd(p(x), p(gamma), p(beta), p(y), p(mean), p(rstd), p(rm), p(rv), N, Cn, H * W, int(cl), 1e-5, 0.1,
                                      p(ws), stream) == 0
            assert h.hrl_bn_train_bwd(p(x), p(dy), p(gamma), p(mean), p(rstd), p(dx), p(dg), p(db), N, Cn, H * W, int(cl), p(ws),
                                      stream) == 0

        times = {k: [] for k in libs}
        for h in libs.values():          # warm-up: module load of each library
            for _ in range(5):
                run(h)
        torch.cuda.synchronize()
        for _ in range(opt.rounds):
            for k, h in libs.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(opt.reps):
                    run(h)
                e1.record()
                e1.synchronize()
                times[k].append(e0.elapsed_time(e1) * 1e3 / opt.reps)
        moved = 8 * x.numel() * 4           # forward reads x twice and writes y; backward reads x and dy twice and writes dx
        for k, t in times.items():
            us = statistics.median(t)
            print(json.dumps({'shape': name, 'nchw' if not cl else 'channels_last': list(shape), 'lib': k, 'us_fwd_bwd': round(us, 1),
                              'spread_us': [round(min(t), 1), round(max(t), 1)], 'GB_per_s_min_traffic': round(moved / us * 1e-3, 1),
                              'gpu': gpu}), flush=True)


if __name__ == '__main__':
    main()
