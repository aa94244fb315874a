"""Cost of the guard against non-finite steps (train_args['skip_nonfinite']) on one GPU, with the key off and on, alternated in one
process: the cfg2 LearnerStep (TicTacToe, fused tower) and the cfg4 LearnerStep (Hungry Geese, module path), both as CUDA graphs
on resident batches of finite data, CUDA events around blocks of steps, best block of `--rounds`.  What the key adds per step is
one device-to-device copy of the BatchNorm buffers and the hrl_step_commit launch; the guarded optimiser launch replaces the
unguarded one.

    python scripts/bench_nonfinite_guard.py [--steps 300] [--steps-cfg4 60] [--rounds 3] [--out results/bench_nonfinite_guard.json]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from bench_diagnostics import gpu_name_and_power, summary, time_block  # noqa: E402


def step_times(name, steps, rounds, warmup, ring_size):
    import bench
    from handyrl_b200.train import LearnerStep, PackedBatch
    w = bench.WORKLOADS[name]
    args = bench.train_args(w)
    example = bench.make_batch(w, 10_000)
    steppers = {on: LearnerStep(bench.make_net(w), dict(args, skip_nonfinite=on), example, lr=3e-8 * w['B'] * w['T'], use_graph=True)
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
    st = steppers[True]
    st.stream.synchronize()
    info = {'launches_per_step': {str(k): s.launches_per_step for k, s in steppers.items()},
            'fused_tower': st.engine is not None,
            'saved_buffer_bytes': st.guard_saved.numel() if st.guard_saved is not None else 0,
            'skipped': float(st.skipped)}
    for s in steppers.values():
        s.close()
    return res, info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=300)
    ap.add_argument('--steps-cfg4', type=int, default=60)
    ap.add_argument('--warmup', type=int, default=30)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    opt = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_nonfinite_guard needs a GPU'
    out = {'gpu': gpu_name_and_power()}
    for name, steps, ring in (('cfg2', opt.steps, 16), ('cfg4', opt.steps_cfg4, 8)):
        res, info = step_times(name, steps, opt.rounds, opt.warmup, ring)
        out[name + '_step'] = dict(summary(res, 'ms_per_step'), steps_per_block=steps, **info)
    line = json.dumps(out)
    print(line)
    if opt.out:
        os.makedirs(os.path.dirname(os.path.abspath(opt.out)), exist_ok=True)
        with open(opt.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
