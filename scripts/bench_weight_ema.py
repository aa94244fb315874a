"""Cost of the moving average of the weights (train_args['weight_ema']) on one GPU, with averaging off and on, alternated in one process:
  * the cfg2 LearnerStep (TicTacToe, fused tower) and the cfg4 LearnerStep (Hungry Geese, module path), both as CUDA graphs on
    resident batches, CUDA events around blocks of steps, best block of `--rounds`;
  * the averaging kernel alone (hrl_weight_ema) on each net's fp32 state, 20 launches per CUDA graph.

    python scripts/bench_weight_ema.py [--steps 300] [--steps-cfg4 60] [--rounds 3] [--out results/bench_weight_ema.json]
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


def step_times(name, steps, rounds, warmup, ring_size, decay):
    import bench
    from handyrl_b200 import ops
    from handyrl_b200.train import LearnerStep, PackedBatch
    w = bench.WORKLOADS[name]
    args = bench.train_args(w)
    example = bench.make_batch(w, 10_000)
    steppers = {on: LearnerStep(bench.make_net(w), dict(args, weight_ema=decay if on else None), example, lr=3e-8 * w['B'] * w['T'],
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
    st = steppers[True]
    info = {'launches_per_step': {str(k): s.launches_per_step for k, s in steppers.items()},
            'fused_tower': st.engine is not None, 'state_fp32_words': st.avg.numel()}
    # the kernel alone on this net's state: 20 launches per graph
    stream = torch.cuda.Stream()
    avg, x, step = st.avg.clone(), st.state.bytes[:st.state.i_off].view(torch.float32), st.opt.step_count
    with torch.cuda.stream(stream):
        ops.weight_ema_update(avg, x, step, decay, False)
    stream.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        for _ in range(20):
            ops.weight_ema_update(avg, x, step, decay, False)
    time_block(stream, lambda i: graph.replay(), 10)
    kernel_us = min(time_block(stream, lambda i: graph.replay(), 50) / 20 * 1e3 for _ in range(rounds))
    info['kernel_us'] = kernel_us
    info['kernel_bytes'] = 3 * 4 * avg.numel()          # read the state and the average, write the average
    info['kernel_gb_per_s'] = info['kernel_bytes'] / (kernel_us * 1e-6) / 1e9
    for s in steppers.values():
        s.close()
    return res, info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=300)
    ap.add_argument('--steps-cfg4', type=int, default=60)
    ap.add_argument('--warmup', type=int, default=30)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--decay', type=float, default=0.999)
    ap.add_argument('--out', default=None)
    opt = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_weight_ema needs a GPU'
    out = {'gpu': gpu_name_and_power(), 'decay': opt.decay}
    for name, steps, ring in (('cfg2', opt.steps, 16), ('cfg4', opt.steps_cfg4, 8)):
        res, info = step_times(name, steps, opt.rounds, opt.warmup, ring, opt.decay)
        out[name + '_step'] = dict(summary(res, 'ms_per_step'), steps_per_block=steps, **info)
    line = json.dumps(out)
    print(line)
    if opt.out:
        os.makedirs(os.path.dirname(os.path.abspath(opt.out)), exist_ok=True)
        with open(opt.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
