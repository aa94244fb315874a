"""Cost of the learner diagnostics on one GPU, with the diagnostics off and on, alternated in one process:
  * the cfg2 LearnerStep (CUDA graph, resident batches), CUDA events around blocks of steps;
  * the fused loss kernel alone (hrl_loss_fwd_bwd vs hrl_loss_fwd_bwd_diag) at the cfg3 and cfg5-shard shapes.

    python scripts/bench_diagnostics.py [--steps 300] [--rounds 3] [--out results/bench_diagnostics.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_name_and_power():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()
    except Exception:
        return torch.cuda.get_device_name()


def time_block(stream, fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(stream):
        e0.record()
        for i in range(n):
            fn(i)
        e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def step_times(steps, rounds, warmup):
    import bench
    from handyrl_b200.train import LearnerStep, PackedBatch
    w = bench.WORKLOADS['cfg2']
    args = bench.train_args(w)
    example = bench.make_batch(w, 10_000)
    steppers = {on: LearnerStep(bench.make_net(w), dict(args, diagnostics=on), example, lr=3e-8 * w['B'] * w['T'], use_graph=True)
                for on in (False, True)}
    nbytes = steppers[False].layout.nbytes
    ring = torch.stack([PackedBatch(steppers[False].layout).fill(bench.make_batch(w, 20_000 + i)).buffer.cuda() for i in range(16)])
    torch.cuda.synchronize()
    assert ring.shape[1] == nbytes
    res = {False: [], True: []}
    for on, st in steppers.items():
        time_block(st.stream, lambda i: st.step_resident(ring[i % len(ring)]), warmup)
    for r in range(rounds):
        for on in ((False, True) if r % 2 == 0 else (True, False)):
            st = steppers[on]
            res[on].append(time_block(st.stream, lambda i: st.step_resident(ring[i % len(ring)]), steps))
    launches = {on: st.launches_per_step for on, st in steppers.items()}
    for st in steppers.values():
        st.close()
    return res, launches


def loss_times(name, iters, rounds):
    from handyrl_b200 import ops
    from handyrl_b200.synthetic import synthetic_batch, synthetic_outputs
    shapes = {'cfg3': dict(B=256, T=20, P=2, A=214, turn_based=True, observation=True, reward_kind='step', burn_in=4, ret=True,
                           policy_target='TD', value_target='TD'),
              'cfg5shard': dict(B=512, T=64, P=2, A=512, turn_based=True, observation=False, reward_kind='zero', burn_in=0, ret=False,
                                policy_target='UPGO', value_target='VTRACE')}
    c = shapes[name]
    args = {'turn_based_training': c['turn_based'], 'observation': c['observation'], 'gamma': 0.8, 'lambda': 0.7,
            'burn_in_steps': c['burn_in'], 'entropy_regularization': 0.1, 'entropy_regularization_decay': 0.1,
            'policy_target': c['policy_target'], 'value_target': c['value_target']}
    batch = synthetic_batch(c['B'], c['T'], c['P'], c['A'], turn_based=c['turn_based'], observation=c['observation'],
                            reward_kind=c['reward_kind'], burn_in=c['burn_in'], seed=0, with_obs=False)
    outs = synthetic_outputs(batch, has_value=True, has_return=c['ret'], seed=1)
    db, do = {k: v.cuda() for k, v in batch.items()}, {k: v.cuda() for k, v in outs.items()}
    bufs = {on: ops.loss_fwd_bwd(do, db, args, diagnostics=on) for on in (False, True)}
    torch.cuda.synchronize()
    assert torch.equal(bufs[False].losses, bufs[True].losses) and torch.equal(bufs[False].dpolicy, bufs[True].dpolicy)
    # 20 back-to-back launches per CUDA graph: the timing is the kernel's, not the Python call's
    stream = torch.cuda.Stream()
    graphs = {}
    for on in (False, True):
        with torch.cuda.stream(stream):
            for _ in range(3):
                ops.loss_fwd_bwd(do, db, args, buffers=bufs[on], diagnostics=on)
        stream.synchronize()
        graphs[on] = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graphs[on], stream=stream):
            for _ in range(20):
                ops.loss_fwd_bwd(do, db, args, buffers=bufs[on], diagnostics=on)
    res = {False: [], True: []}
    for on in (False, True):
        time_block(stream, lambda i: graphs[on].replay(), 10)
    for r in range(rounds):
        for on in ((False, True) if r % 2 == 0 else (True, False)):
            res[on].append(time_block(stream, lambda i: graphs[on].replay(), max(1, iters // 20)) / 20 * 1e3)
    return res


def summary(res, unit):
    off, on = min(res[False]), min(res[True])
    return {'off_' + unit: res[False], 'on_' + unit: res[True], 'best_off': off, 'best_on': on, 'overhead_pct': 100.0 * (on - off) / off}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=300)
    ap.add_argument('--warmup', type=int, default=50)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--loss-iters', type=int, default=500)
    ap.add_argument('--out', default=None)
    opt = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_diagnostics needs a GPU'
    out = {'gpu': gpu_name_and_power()}
    res, launches = step_times(opt.steps, opt.rounds, opt.warmup)
    out['cfg2_step'] = dict(summary(res, 'ms_per_step'), steps_per_block=opt.steps, launches_per_step={str(k): v for k, v in launches.items()})
    for name in ('cfg3', 'cfg5shard'):
        out['loss_kernel_' + name] = dict(summary(loss_times(name, opt.loss_iters, opt.rounds), 'us_per_call'), calls_per_block=opt.loss_iters)
    line = json.dumps(out)
    print(line)
    if opt.out:
        os.makedirs(os.path.dirname(os.path.abspath(opt.out)), exist_ok=True)
        with open(opt.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
