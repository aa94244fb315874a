"""Cost of policy distillation (train_args['distill']) on one GPU.
  * the kernel alone (hrl_distill_fwd_bwd) at the cfg2, cfg3 and cfg5-shard loss shapes: one CUDA graph of `--launches`
    launches per block, blocks timed with CUDA events, the best block kept; µs per launch and algorithmic GB/s (student and
    teacher logits, the action mask and the gradient's read and write: 20 bytes per action of each policy row) against the
    3.35 TB/s of the H100 SXM data sheet;
  * the cfg2 (fused tower) and cfg4 (module path) LearnerStep with the key off and on (a teacher of the same architecture and
    other weights, c0 = 1, no annealing): ms per step and launches per step, the two forms alternated over `--rounds` blocks.
The card's name, power limit and maximum SM clock are read in the same run.  Prints one JSON line.

    python scripts/bench_distill.py [--launches 200] [--steps 100] [--steps-cfg4 30] [--rounds 3] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from bench_diagnostics import time_block  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
KERNEL_SHAPES = {       # B, T, P, A, turn_based, observation, burn_in
    'cfg2': (512, 32, 2, 9, True, False, 0),
    'cfg3': (256, 20, 2, 214, True, True, 4),
    'cfg5shard': (512, 64, 2, 512, True, False, 0),
}


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip() or q.stderr.strip()


def kernel(name, launches, rounds):
    from handyrl_b200 import ops
    from handyrl_b200.synthetic import synthetic_batch, synthetic_outputs
    B, T, P, A, tb, obs, bi = KERNEL_SHAPES[name]
    batch = {k: v.cuda() for k, v in synthetic_batch(B, T, P, A, turn_based=tb, observation=obs, burn_in=bi, seed=0,
                                                      with_obs=False).items()}
    outs = {k: v.cuda() for k, v in synthetic_outputs(batch, seed=1).items()}
    teacher = outs['policy'] + 0.5 * torch.randn_like(outs['policy'])
    args = {'gamma': 0.8, 'lambda': 0.7, 'entropy_regularization': 0.1, 'entropy_regularization_decay': 0.1,
            'policy_target': 'UPGO', 'value_target': 'VTRACE', 'turn_based_training': tb, 'observation': obs, 'burn_in_steps': bi}
    buf = ops.loss_fwd_bwd(outs, batch, args)
    step = torch.zeros(1, dtype=torch.int64, device='cuda')
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            ops.distill_fwd_bwd(outs['policy'], teacher, batch, args, buf, step, 1.0)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(launches):
                ops.distill_fwd_bwd(outs['policy'], teacher, batch, args, buf, step, 1.0)
    times = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(s):          # replay() launches on the current stream: the events bracket it there
            e0.record()
            g.replay()
            e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1) * 1e3 / launches)
    rows = B * T * (1 if (tb and not obs) else P)
    nbytes = 20 * A * rows
    best = min(times)
    return {'B': B, 'T': T, 'P': P, 'A': A, 'rows': rows, 'us': times, 'best_us': best, 'algorithmic_bytes': nbytes,
            'GB_per_s': nbytes / (best * 1e-6) / 1e9, 'share_of_hbm': nbytes / (best * 1e-6) / HBM_BYTES_PER_S}


def step(name, steps, rounds, warmup=10):
    import bench
    from handyrl_b200.train import LearnerStep, PackedBatch
    w = dict(bench.WORKLOADS[name])
    args = bench.train_args(w)
    example = bench.make_batch(w, 10_000)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, 'teacher.pth')
        g = torch.Generator().manual_seed(123)
        torch.save({k: v + 0.05 * torch.randn(v.shape, generator=g) if v.is_floating_point() else v
                    for k, v in bench.make_net(w).state_dict().items()}, path)
        steppers = {'off': LearnerStep(bench.make_net(w), args, example, lr=3e-8 * w['B'] * w['T']),
                    'on': LearnerStep(bench.make_net(w), dict(args, distill={'teacher': path}), example, lr=3e-8 * w['B'] * w['T'])}
    batch = PackedBatch(steppers['off'].layout).fill(example).buffer.cuda()
    for st in steppers.values():
        time_block(st.stream, lambda i, st=st: st.step_resident(batch), warmup)
    res = {k: [] for k in steppers}
    for r in range(rounds):
        for k in (('off', 'on') if r % 2 == 0 else ('on', 'off')):
            st = steppers[k]
            res[k].append(time_block(st.stream, lambda i, st=st: st.step_resident(batch), steps))
    out = {'B': w['B'], 'T': w['T'], 'fused_tower': steppers['off'].engine is not None}
    for k, st in steppers.items():
        out[k] = {'ms_per_step': res[k], 'best_ms': min(res[k]), 'launches_per_step': st.launches_per_step}
        if k == 'on':
            out[k]['launches_per_teacher'] = st.launches_per_teacher
        st.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--launches', type=int, default=200)
    ap.add_argument('--steps', type=int, default=100)
    ap.add_argument('--steps-cfg4', type=int, default=30)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_distill.py measures on the GPU; there is none')
    res = {'card': card(), 'kernel': {n: kernel(n, a.launches, a.rounds) for n in KERNEL_SHAPES},
           'step': {'cfg2': step('cfg2', a.steps, a.rounds), 'cfg4': step('cfg4', a.steps_cfg4, a.rounds)}}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
