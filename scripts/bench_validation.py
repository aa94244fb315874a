"""Cost of the held-out validation loss (train_args['validation_rate']) on one GPU, in one process:
  (a) the forward-only loss kernel (hrl_loss_fwd) against the fused forward+backward one (hrl_loss_fwd_bwd) at the cfg2, cfg3 and
      cfg5-shard shapes: 20 launches per CUDA graph, blocks of the two alternated, best block each way;
  (b) the cfg2 LearnerStep (TicTacToe, fused tower) and the cfg4 LearnerStep (Hungry Geese, module path) with the key off and at
      r = 0.05: ms per training step (the two learners' blocks alternated), ms per validation pass, launches per step and per
      pass, and the per-step cost with one pass every round(1 / r) steps.

    python scripts/bench_validation.py [--steps 300] [--steps-cfg4 60] [--rounds 3] [--out results/bench_validation.json]
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

SHAPES = {
    'cfg2': dict(B=512, T=32, P=2, A=9, turn_based=True, observation=False, reward_kind='zero', burn_in=0, ret=False,
                 policy_target='UPGO', value_target='VTRACE'),
    'cfg3': dict(B=256, T=20, P=2, A=214, turn_based=True, observation=True, reward_kind='step', burn_in=4, ret=True,
                 policy_target='TD', value_target='TD'),
    'cfg5shard': dict(B=512, T=64, P=2, A=512, turn_based=True, observation=False, reward_kind='zero', burn_in=0, ret=False,
                      policy_target='UPGO', value_target='VTRACE'),
}


def loss_times(name, iters, rounds):
    from handyrl_b200 import ops
    from handyrl_b200.synthetic import synthetic_batch, synthetic_outputs
    c = SHAPES[name]
    args = {'turn_based_training': c['turn_based'], 'observation': c['observation'], 'gamma': 0.8, 'lambda': 0.7,
            'burn_in_steps': c['burn_in'], 'entropy_regularization': 0.1, 'entropy_regularization_decay': 0.1,
            'policy_target': c['policy_target'], 'value_target': c['value_target']}
    batch = synthetic_batch(c['B'], c['T'], c['P'], c['A'], turn_based=c['turn_based'], observation=c['observation'],
                            reward_kind=c['reward_kind'], burn_in=c['burn_in'], seed=0, with_obs=False)
    outs = synthetic_outputs(batch, has_value=True, has_return=c['ret'], seed=1)
    db, do = {k: v.cuda() for k, v in batch.items()}, {k: v.cuda() for k, v in outs.items()}
    full = ops.loss_fwd_bwd(do, db, args)
    fwd_buf = ops.LossBuffers(c['B'], c['T'], full.dims[2], full.dims[3], c['A'], True, c['ret'], 'cuda', grads=False)
    fwd = ops.loss_fwd(do, db, args, buffers=fwd_buf)
    torch.cuda.synchronize()
    assert torch.equal(fwd, full.losses)
    calls = {'fwd_bwd': lambda: ops.loss_fwd_bwd(do, db, args, buffers=full), 'fwd': lambda: ops.loss_fwd(do, db, args, buffers=fwd_buf)}
    stream = torch.cuda.Stream()
    graphs = {}
    for k, call in calls.items():
        with torch.cuda.stream(stream):
            for _ in range(3):
                call()
        stream.synchronize()
        graphs[k] = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graphs[k], stream=stream):
            for _ in range(20):
                call()
    res = {'fwd_bwd': [], 'fwd': []}
    for k in res:
        time_block(stream, lambda i: graphs[k].replay(), 10)
    for r in range(rounds):
        for k in (('fwd_bwd', 'fwd') if r % 2 == 0 else ('fwd', 'fwd_bwd')):
            res[k].append(time_block(stream, lambda i: graphs[k].replay(), max(1, iters // 20)) / 20 * 1e3)
    P, Pa, A = full.dims[2], full.dims[3], c['A']
    best = {k: min(v) for k, v in res.items()}
    return {'fwd_bwd_us': res['fwd_bwd'], 'fwd_us': res['fwd'], 'best_fwd_bwd_us': best['fwd_bwd'], 'best_fwd_us': best['fwd'],
            'saving_pct': 100.0 * (best['fwd_bwd'] - best['fwd']) / best['fwd_bwd'],
            'policy_bytes_per_cell': {'fwd_bwd': 12 * Pa * A, 'fwd': 8 * Pa * A}, 'P': P, 'Pa': Pa, 'calls_per_block': iters}


def learner_times(name, steps, rounds, warmup, ring_size, rate):
    import bench
    from handyrl_b200.train import LearnerStep, PackedBatch
    w = bench.WORKLOADS[name]
    args = bench.train_args(w)
    example = bench.make_batch(w, 10_000)
    steppers = {on: LearnerStep(bench.make_net(w), dict(args, validation_rate=rate if on else None), example,
                                lr=3e-8 * w['B'] * w['T'], use_graph=True)
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
    time_block(st.stream, lambda i: st.validate_in_place(), warmup)
    val_ms = min(time_block(st.stream, lambda i: st.validate_in_place(), steps) for _ in range(rounds))
    every = max(1, int(round(1.0 / rate)))
    info = {'validation_ms_per_pass': val_ms, 'validation_every_steps': every,
            'launches_per_step': {str(k): s.launches_per_step for k, s in steppers.items()},
            'launches_per_validation': st.launches_per_validation, 'fused_tower': st.engine is not None}
    info['ms_per_step_with_validation'] = min(res[True]) + val_ms / every
    info['validation_overhead_pct'] = 100.0 * (info['ms_per_step_with_validation'] - min(res[False])) / min(res[False])
    for s in steppers.values():
        s.close()
    return res, info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=300)
    ap.add_argument('--steps-cfg4', type=int, default=60)
    ap.add_argument('--warmup', type=int, default=30)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--loss-iters', type=int, default=500)
    ap.add_argument('--rate', type=float, default=0.05)
    ap.add_argument('--out', default=None)
    opt = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_validation needs a GPU'
    out = {'gpu': gpu_name_and_power(), 'validation_rate': opt.rate}
    for name in ('cfg2', 'cfg3', 'cfg5shard'):
        out['loss_kernel_' + name] = loss_times(name, opt.loss_iters, opt.rounds)
    for name, steps, ring in (('cfg2', opt.steps, 16), ('cfg4', opt.steps_cfg4, 8)):
        res, info = learner_times(name, steps, opt.rounds, opt.warmup, ring, opt.rate)
        out[name + '_learner'] = dict(summary(res, 'ms_per_step'), steps_per_block=steps, **info)
    line = json.dumps(out)
    print(line)
    if opt.out:
        os.makedirs(os.path.dirname(os.path.abspath(opt.out)), exist_ok=True)
        with open(opt.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
