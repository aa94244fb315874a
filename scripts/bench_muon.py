"""Cost of Muon (train_args['optimizer'] = 'muon') against Adam and LAMB on one GPU, alternated in one process:

 * the optimiser alone (hrl_grad_sumsq + hrl_clip_adam_step / hrl_clip_lamb_step / hrl_clip_muon_step) on the bucket layouts
   of the cfg2, cfg3 and cfg4 nets (TicTacToe, Geister, Geese), as CUDA graphs of 20 optimiser steps, CUDA events around
   blocks of replays;
 * the cfg2 LearnerStep (TicTacToe, fused tower) and the cfg4 LearnerStep (Hungry Geese, module path) as CUDA graphs on
   resident batches, key off and on, three blocks each.

Best block of `--rounds` for each.  The card's name and power limit are read in the same run.

    python scripts/bench_muon.py [--replays 200] [--steps 300] [--steps-cfg4 60] [--rounds 3] [--out results/bench_muon.json]
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
OPTIMISERS = ('adam', 'lamb', 'muon')


def optimiser_times(name, replays, rounds):
    from handyrl_b200 import nets, ops
    net = {'tictactoe': nets.tictactoe_net, 'geister': nets.geister_net, 'geese': nets.geese_net}[name]()
    shapes = [tuple(p.shape) for p in net.parameters()]
    g = torch.Generator().manual_seed(1)
    graphs, res, info = {}, {k: [] for k in OPTIMISERS}, {}
    stream = torch.cuda.Stream()
    for kind in OPTIMISERS:
        params = [torch.nn.Parameter(torch.zeros(s, device='cuda')) for s in shapes]
        opt = {'adam': ops.FlatAdam, 'lamb': ops.FlatLamb, 'muon': ops.FlatMuon}[kind](params, lr=1e-4)
        with torch.no_grad():
            opt.flat_param[:opt.n].copy_(0.1 * torch.randn(opt.n, generator=g))
            opt.flat_grad[:opt.n].copy_(1e-3 * torch.randn(opt.n, generator=g))
        opt.step()                                     # eager first: module load, shared-memory attribute
        before = ops.LAUNCHES['n']
        stream.wait_stream(torch.cuda.current_stream())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            for _ in range(GRAPH_STEPS):
                opt.step()
        info['launches_per_step_' + kind] = (ops.LAUNCHES['n'] - before) // GRAPH_STEPS
        graphs[kind] = (graph, opt)
        if kind == 'muon':
            info['muon_matrices'] = int(opt.mats.shape[0])
            info['adam_spans'] = int(opt.spans.shape[0])
    info['words'] = sum(p.numel() for p in net.parameters())
    for kind, (graph, _) in graphs.items():
        time_block(stream, lambda i: graph.replay(), 10)
    for r in range(rounds):
        for kind in (OPTIMISERS if r % 2 == 0 else tuple(reversed(OPTIMISERS))):
            graph = graphs[kind][0]
            res[kind].append(1e3 * time_block(stream, lambda i: graph.replay(), replays) / GRAPH_STEPS)
    return {'us_per_step_' + k: v for k, v in res.items()} | {'best_' + k: min(v) for k, v in res.items()} | info


def step_times(name, steps, rounds, warmup, ring_size):
    import bench
    from handyrl_b200.train import LearnerStep, PackedBatch
    w = bench.WORKLOADS[name]
    args = bench.train_args(w)
    example = bench.make_batch(w, 10_000)
    steppers = {on: LearnerStep(bench.make_net(w), dict(args, optimizer='muon' if on else None), example, lr=3e-8 * w['B'] * w['T'],
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
    assert torch.cuda.is_available(), 'bench_muon needs a GPU'
    out = {'gpu': gpu_name_and_power()}
    for cfg, name in (('cfg2', 'tictactoe'), ('cfg3', 'geister'), ('cfg4', 'geese')):
        out[cfg + '_optimiser'] = dict(optimiser_times(name, opt.replays, opt.rounds), net=name, graph_steps=GRAPH_STEPS,
                                       replays_per_block=opt.replays)
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
