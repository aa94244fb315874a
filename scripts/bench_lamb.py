"""Cost of LAMB (train_args['optimizer'] = 'lamb') against Adam on one GPU, alternated in one process:

 * the optimiser alone (hrl_grad_sumsq + hrl_clip_adam_step, against hrl_grad_sumsq + hrl_clip_lamb_step) on the bucket layouts
   of the TicTacToe, Geister and Geese nets, as CUDA graphs of 20 optimiser steps, CUDA events around blocks of replays;
 * the cfg2 LearnerStep (TicTacToe, fused tower) and the cfg4 LearnerStep (Hungry Geese, module path) as CUDA graphs on
   resident batches, key off and on.

Best block of `--rounds` for each.

    python scripts/bench_lamb.py [--replays 200] [--steps 300] [--steps-cfg4 60] [--rounds 3] [--out results/bench_lamb.json]
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

GRAPH_STEPS = 20


def optimiser_times(name, replays, rounds):
    from handyrl_b200 import nets, ops
    net = {'tictactoe': nets.tictactoe_net, 'geister': nets.geister_net, 'geese': nets.geese_net}[name]()
    numels = [p.numel() for p in net.parameters()]
    g = torch.Generator().manual_seed(1)
    graphs, res, info = {}, {False: [], True: []}, {}
    stream = torch.cuda.Stream()
    for lamb in (False, True):
        params = [torch.nn.Parameter(torch.zeros(k, device='cuda')) for k in numels]
        opt = ops.FlatLamb(params, lr=1e-4) if lamb else ops.FlatAdam(params, lr=1e-4)
        with torch.no_grad():
            opt.flat_param[:opt.n].copy_(0.1 * torch.randn(opt.n, generator=g))
            opt.flat_grad[:opt.n].copy_(1e-3 * torch.randn(opt.n, generator=g))
        before = ops.LAUNCHES['n']
        stream.wait_stream(torch.cuda.current_stream())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            for _ in range(GRAPH_STEPS):
                opt.step()
        info['launches_per_step_' + ('lamb' if lamb else 'adam')] = (ops.LAUNCHES['n'] - before) // GRAPH_STEPS
        graphs[lamb] = (graph, opt)
        if lamb:
            info['chunks'] = int(opt.plan.shape[0])
    info['words'] = sum(numels)
    info['tensors'] = len(numels)
    for lamb, (graph, _) in graphs.items():
        time_block(stream, lambda i: graph.replay(), 10)
    for r in range(rounds):
        for lamb in ((False, True) if r % 2 == 0 else (True, False)):
            graph = graphs[lamb][0]
            res[lamb].append(1e3 * time_block(stream, lambda i: graph.replay(), replays) / GRAPH_STEPS)
    return res, info


def step_times(name, steps, rounds, warmup, ring_size):
    import bench
    from handyrl_b200.train import LearnerStep, PackedBatch
    w = bench.WORKLOADS[name]
    args = bench.train_args(w)
    example = bench.make_batch(w, 10_000)
    steppers = {on: LearnerStep(bench.make_net(w), dict(args, optimizer='lamb' if on else None), example, lr=3e-8 * w['B'] * w['T'],
                                use_graph=True) for on in (False, True)}
    ring = torch.stack([PackedBatch(steppers[False].layout).fill(bench.make_batch(w, 20_000 + i)).buffer.cuda() for i in range(ring_size)])
    torch.cuda.synchronize()
    res = {False: [], True: []}
    for on, st in steppers.items():
        time_block(st.stream, lambda i: st.step_resident(ring[i % len(ring)]), warmup)
    for r in range(rounds):
        for on in ((False, True) if r % 2 == 0 else (True, False)):
            st = steppers[on]
            res[on].append(time_block(st.stream, lambda i: st.step_resident(ring[i % len(ring)]), steps))
    info = {'launches_per_step': {str(k): s.launches_per_step for k, s in steppers.items()},
            'fused_tower': steppers[True].engine is not None}
    for s in steppers.values():
        s.close()
    return res, info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--replays', type=int, default=200)
    ap.add_argument('--steps', type=int, default=300)
    ap.add_argument('--steps-cfg4', type=int, default=60)
    ap.add_argument('--warmup', type=int, default=30)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    opt = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_lamb needs a GPU'
    out = {'gpu': gpu_name_and_power()}
    for name in ('tictactoe', 'geister', 'geese'):
        res, info = optimiser_times(name, opt.replays, opt.rounds)
        out[name + '_optimiser'] = dict(summary(res, 'us_per_step'), graph_steps=GRAPH_STEPS, replays_per_block=opt.replays, **info)
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
