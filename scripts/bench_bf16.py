"""Speed of the bf16 mode of the net's tensor-core products (train_args['tensor_cores'] = 'bf16') against the default 3xTF32 on
one GPU, both forms alternated in one process:
  * the three products of a cfg2 tower layer alone (16384 x 288 x 288: forward and input gradient on packed weight images, the
    weight gradient on transposed operands split over K slices), 20 launches per CUDA graph, best of `--rounds`; FLOP/s of
    2 M N K against each form's ceiling (3xTF32: a third of the dense TF32 rate; bf16: the dense BF16 rate, H100 SXM data sheet);
  * the cfg2 LearnerStep (TicTacToe, fused tower) and the cfg4 LearnerStep (Hungry Geese, module path), CUDA graphs on resident
    batches, CUDA events around blocks of steps, best block of `--rounds`, and the library launches per step of each mode.

    python scripts/bench_bf16.py [--steps 300] [--steps-cfg4 60] [--rounds 3] [--out results/bench_bf16.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from bench_diagnostics import time_block  # noqa: E402

CEILING_TFLOPS = {'tf32x3': 494.7 / 3, 'bf16': 989.4}      # dense, H100 SXM data sheet (700 W)


def gpu_name_and_power():
    """name, power limit and max SM clock of the card, read with the measurement"""
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()
    except Exception:
        return torch.cuda.get_device_name()


def tower_products(rounds):
    """the forward / input-gradient / weight-gradient products of one cfg2 tower layer, 3xTF32 and bf16"""
    from handyrl_b200._capi import HrlGemmArgs, HrlPackJob, check, lib
    from handyrl_b200.ops import _ptr, k_splits
    M, D, C_, H = 16384, 288, 32, 3
    g = torch.Generator(device='cuda').manual_seed(1)
    w = torch.randn(C_, C_, 3, 3, device='cuda', generator=g) * 0.1
    x = torch.randn(M, D, device='cuda', generator=g)
    dy = torch.randn(M, D, device='cuda', generator=g)
    out = torch.empty(M, D, device='cuda')
    splits = k_splits(D, D, M)
    ws = torch.empty(splits * D * D, device='cuda')
    stream = torch.cuda.Stream()
    images, calls = {}, {}
    for form in ('tf32x3', 'bf16'):
        bf = form == 'bf16'
        n = lib().hrl_board_pack_floats(D, D) // (4 if bf else 1)
        fwd, bwd = torch.zeros(n, device='cuda'), torch.zeros(n, device='cuda')
        j = (HrlPackJob * 1)()
        j[0].w, j[0].Cout, j[0].Cin, j[0].kh, j[0].kw, j[0].H, j[0].W = _ptr(w), C_, C_, 3, 3, H, H
        j[0].image_fwd, j[0].fwd_rows, j[0].image_bwd, j[0].bwd_rows, j[0].bf16 = _ptr(fwd), D, _ptr(bwd), D, int(bf)
        check(lib().hrl_board_pack_many(C.byref(j), 1, torch.cuda.current_stream().cuda_stream))
        images[form] = (fwd, bwd)

        def args(kind, bf=bf, fwd=fwd, bwd=bwd):
            a = HrlGemmArgs()
            a.bf16 = int(bf)
            if kind == 'wgrad':          # dW = dY^T X over the samples: both operands transposed, split over K
                a.a.ptr, a.a.ld, a.a.kmajor = _ptr(dy), D, 0
                a.b.ptr, a.b.ld, a.b.kmajor = _ptr(x), D, 0
                a.C, a.ldc, a.M, a.N, a.K, a.splits, a.workspace = None, D, D, D, M, splits, _ptr(ws)
            else:
                a.a.ptr, a.a.ld, a.a.kmajor = _ptr(x if kind == 'fwd' else dy), D, 1
                a.b.ptr, a.b.kmajor, a.b.packed = _ptr(fwd if kind == 'fwd' else bwd), 1, 1
                a.C, a.ldc, a.M, a.N, a.K, a.splits = _ptr(out), D, M, D, D, 1
            return a
        for kind in ('fwd', 'dgrad', 'wgrad'):
            calls[(form, kind)] = args(kind)
    torch.cuda.synchronize()
    graphs = {}
    for key, a in calls.items():
        with torch.cuda.stream(stream):
            check(lib().hrl_gemm_fused(C.byref(a), stream.cuda_stream))
        stream.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=stream):
            for _ in range(20):
                check(lib().hrl_gemm_fused(C.byref(a), stream.cuda_stream))
        graphs[key] = gr
        time_block(stream, lambda i, gr=gr: gr.replay(), 5)
    best = {k: float('inf') for k in graphs}
    for r in range(rounds):
        for form in (('tf32x3', 'bf16') if r % 2 == 0 else ('bf16', 'tf32x3')):
            for kind in ('fwd', 'dgrad', 'wgrad'):
                gr = graphs[(form, kind)]
                best[(form, kind)] = min(best[(form, kind)], time_block(stream, lambda i, gr=gr: gr.replay(), 10) / 20 * 1e3)
    res = {}
    flop = 2.0 * M * D * D
    for (form, kind), us in best.items():
        tflops = flop / (us * 1e-6) / 1e12
        res['%s_%s' % (kind, form)] = {'us': us, 'tflops': tflops, 'pct_of_ceiling': 100.0 * tflops / CEILING_TFLOPS[form]}
    res['splits_wgrad'] = splits
    return res


def step_times(name, steps, rounds, warmup, ring_size):
    import bench
    from handyrl_b200.train import LearnerStep, PackedBatch
    w = bench.WORKLOADS[name]
    args = bench.train_args(w)
    example = bench.make_batch(w, 10_000)
    steppers = {on: LearnerStep(bench.make_net(w), dict(args, tensor_cores='bf16' if on else True), example, lr=3e-8 * w['B'] * w['T'],
                                use_graph=True)
                for on in (False, True)}
    ring = torch.stack([PackedBatch(steppers[False].layout).fill(bench.make_batch(w, 20_000 + i)).buffer.cuda() for i in range(ring_size)])
    torch.cuda.synchronize()
    res = {False: [], True: []}
    for on, st in steppers.items():
        time_block(st.stream, lambda i: st.step_resident(ring[i % len(ring)]), warmup)
    for r in range(rounds):
        for on in ((False, True) if r % 2 == 0 else (True, False)):
            st = steppers[on]
            res[on].append(time_block(st.stream, lambda i: st.step_resident(ring[i % len(ring)]), steps))
    info = {'launches_per_step': {('bf16' if k else 'tf32x3'): s.launches_per_step for k, s in steppers.items()},
            'fused_tower': steppers[True].engine is not None}
    for s in steppers.values():
        s.close()
    off, on = min(res[False]), min(res[True])
    return {'tf32x3_ms_per_step': res[False], 'bf16_ms_per_step': res[True], 'best_tf32x3': off, 'best_bf16': on,
            'speedup': off / on, **info}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=300)
    ap.add_argument('--steps-cfg4', type=int, default=60)
    ap.add_argument('--warmup', type=int, default=30)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--configs', default='cfg2,cfg4')
    ap.add_argument('--out', default=None)
    opt = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_bf16 needs a GPU'
    import __graft_entry__
    __graft_entry__.build()
    out = {'gpu': gpu_name_and_power(), 'tower_products': tower_products(opt.rounds)}
    for name in [n for n in opt.configs.split(',') if n]:
        steps = opt.steps if name == 'cfg2' else opt.steps_cfg4
        out[name + '_step'] = dict(step_times(name, steps, opt.rounds, opt.warmup, 16 if name == 'cfg2' else 8), steps_per_block=steps)
    line = json.dumps(out)
    print(line)
    if opt.out:
        os.makedirs(os.path.dirname(os.path.abspath(opt.out)), exist_ok=True)
        with open(opt.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
