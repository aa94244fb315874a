"""Cost of prioritised replay (train_args['prioritized_replay']) on one GPU, in one process:
  (a) the fused loss kernel with a NULL window-weight pointer against a set one, at the cfg2, cfg3 and cfg5-shard shapes;
  (b) the device sampler hrl_replay_sample alone at 1k, 10k and 100k stored episodes, B = 512;
  (c) the priority update hrl_replay_priority_update alone at the cfg2 and cfg4 step shapes;
  (d) GpuBatcher.fill + LearnerStep.step_in_place per step, key off (host sampler, descriptor copy) and on (device sampler,
      importance weights, priority update), on cfg2 (TicTacToe, fused tower) and cfg4 (Hungry Geese, module path) with
      episodes resident in the device ring.
CUDA events around blocks of calls, the key off and on alternated block by block, best block each way.  (a)-(c) are captured
in CUDA graphs; (d) replays the step graph, with the fill enqueued by the host as in training.

    python scripts/bench_prioritized_replay.py [--rounds 3] [--out results/bench_prioritized_replay.json]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from bench_diagnostics import gpu_name_and_power, summary, time_block  # noqa: E402

SPEC = {'alpha': 0.6, 'beta': 0.4, 'epsilon': 0.01}


def graph_of(fn, n):
    """A CUDA graph of n calls of fn (after one eager warm-up call)."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        for _ in range(n):
            fn()
    return g, s


def alternate(calls, n, rounds):
    """calls {False: fn, True: fn}: graphs of n calls each, replayed in alternated blocks; us per call."""
    graphs = {k: graph_of(fn, n) for k, fn in calls.items()}
    res = {False: [], True: []}
    for k in graphs:
        graphs[k][0].replay()
    torch.cuda.synchronize()
    for r in range(rounds):
        for k in ((False, True) if r % 2 == 0 else (True, False)):
            g, s = graphs[k]
            res[k].append(1e3 * time_block(s, lambda i: g.replay(), 5) / n)
    return res


def loss_times(name, n, rounds):
    import bench
    from handyrl_b200 import ops
    from handyrl_b200.synthetic import synthetic_batch, synthetic_outputs
    w = bench.WORKLOADS[name]
    args = bench.train_args(w)
    has_return = name == 'cfg3'
    if has_return:
        host = {k: v for k, v in bench.make_batch(w, 3).items() if k != 'observation'}
    else:
        host = synthetic_batch(w['B'], w['T'], w['P'], w['A'], turn_based=w['turn_based'], observation=w['observation'],
                               reward_kind=w['reward_kind'], seed=3, with_obs=False)
    batch = {k: v.cuda() for k, v in host.items()}
    outs = {k: v.cuda() for k, v in synthetic_outputs(host, has_value=True, has_return=has_return, seed=1).items()}
    weight = torch.from_numpy(np.random.default_rng(0).uniform(0.5, 2.0, w['B']).astype(np.float32)).cuda()
    bufs = {on: None for on in (False, True)}

    def call(on):
        bufs[on] = ops.loss_fwd_bwd(outs, batch, args, buffers=bufs[on], window_weight=weight if on else None)
    call(False), call(True)
    return alternate({on: (lambda on=on: call(on)) for on in (False, True)}, n, rounds)


def fake_episodes(n, steps, Ps, A, obs_shape, seed):
    from handyrl_b200.batch import FlatEpisode
    g = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        fe = FlatEpisode()
        fe.steps, fe.players = steps, list(range(Ps))
        fe.obs = (g.random((steps, Ps) + obs_shape) < 0.3).astype(np.float32)
        fe.prob = g.uniform(0.1, 1.0, (steps, Ps)).astype(np.float32)
        fe.action = g.integers(0, A, (steps, Ps)).astype(np.int32)
        fe.amask = np.zeros((steps, Ps, A), np.float32)
        fe.value = g.uniform(-1, 1, (steps, Ps, 1)).astype(np.float32)
        fe.reward = np.zeros((steps, Ps), np.float32)
        fe.ret = np.zeros((steps, Ps), np.float32)
        fe.flags = np.full((steps, Ps), 3, np.uint8)
        fe.turn = (np.arange(steps) % Ps).astype(np.int32)
        fe.outcome = g.choice([-1.0, 1.0], Ps).astype(np.float32)
        out.append(fe)
    return out


def sampler_times(episodes, B, n, rounds):
    """The sampler alone ('on'; 'off' is the same graph again, for the spread between blocks)."""
    from handyrl_b200 import ops, priority
    from handyrl_b200.replay import DeviceReplay
    steps = 12
    rp = DeviceReplay(episodes * steps + 64, episodes, mirror=True)
    for lo in range(0, episodes, 4096):
        rp.add_flat_many(fake_episodes(min(4096, episodes - lo), steps, 2, 4, (2,), lo))
    args = {'burn_in_steps': 0, 'forward_steps': 8, 'turn_based_training': True, 'maximum_episodes': episodes}
    st = priority.PriorityState(SPEC, episodes + 1, B, torch.device('cuda'))
    win = torch.empty((B, 32), dtype=torch.uint8, device='cuda')
    head, count = rp.snapshot(episodes)
    st.prio.uniform_(0.05, 3.0)
    st.prio_serial.copy_(rp.dir_dev[:, 3])
    torch.cuda.synchronize()
    fn = lambda: ops.replay_sample(st, rp, head, count, args, win, 1, 0, False)
    return alternate({False: fn, True: fn}, n, rounds)


def update_times(name, n, rounds):
    import bench
    from handyrl_b200 import ops, priority
    w = bench.WORKLOADS[name]
    B, T, P = w['B'], w['T'], (w['P'] if w['turn_based'] else 1)
    st = priority.PriorityState(SPEC, 100_001, B, torch.device('cuda'))
    g = torch.Generator(device='cuda').manual_seed(0)
    adv = torch.randn((B, T, P, 1), device='cuda', generator=g)
    tm = (torch.rand((B, T, P, 1), device='cuda', generator=g) < 0.5).float()
    st.win_slot.copy_(torch.randint(0, 100_000, (B,), device='cuda', generator=g, dtype=torch.int32))
    st.prio_serial.copy_(torch.arange(100_001, device='cuda'))
    st.win_serial.copy_(st.win_slot.long())
    fn = lambda: ops.priority_update(st, adv, tm, 0)
    return alternate({False: fn, True: fn}, n, rounds)


def fill_step_times(name, steps, rounds, warmup):
    import bench
    from handyrl_b200.train import EpisodeDeque, GpuBatcher, LearnerStep
    w = bench.WORKLOADS[name]
    obs_shape = w['obs_shape']
    eps = fake_episodes(4000, 40, w['P'], w['A'], obs_shape, 1)
    res, info = {False: [], True: []}, {}
    setups = {}
    for on in (False, True):
        args = dict(bench.train_args(w), maximum_episodes=5000, replay_capacity_steps=4000 * 40 + 64,
                    prioritized_replay=SPEC if on else None)
        gb = GpuBatcher(args, EpisodeDeque(), torch.device('cuda'), seed=5)
        gb.replay.add_flat_many(eps)
        win = gb.replay.sample_windows(w['B'], args, np.random.default_rng(1))
        example = {k: v.cpu() for k, v in gb.replay.gather(win, args).items() if not k.startswith('_')}
        example['observation'] = example['observation'].reshape(*example['observation'].shape[:3], *obs_shape)
        torch.cuda.synchronize()
        st = LearnerStep(bench.make_net(w), args, example, lr=3e-8 * w['B'] * w['T'], use_graph=True)
        st.warm_up()
        setups[on] = (gb, st)
        info['launches_per_step_' + ('on' if on else 'off')] = st.launches_per_step
    fill_step = lambda on: (lambda i: (setups[on][0].fill(setups[on][1]), setups[on][1].step_in_place()))
    for on in (False, True):
        time_block(setups[on][1].stream, fill_step(on), warmup)
    for r in range(rounds):
        for on in ((False, True) if r % 2 == 0 else (True, False)):
            res[on].append(time_block(setups[on][1].stream, fill_step(on), steps))
    st = setups[True][1]
    st.stream.synchronize()
    p = st.prio_state.prio.cpu().numpy()
    info['prio_moved'] = bool(np.any(p[:4000] != 1.0))
    info['max_prio'] = float(st.prio_state.max_prio)
    for gb, s in setups.values():
        s.close()
    return res, info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--calls', type=int, default=200)
    ap.add_argument('--steps', type=int, default=300)
    ap.add_argument('--steps-cfg4', type=int, default=60)
    ap.add_argument('--warmup', type=int, default=30)
    ap.add_argument('--out', default=None)
    opt = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_prioritized_replay needs a GPU'
    out = {'gpu': gpu_name_and_power()}
    for name in ('cfg2', 'cfg3', 'cfg5shard'):
        out['loss_kernel_' + name] = dict(summary(loss_times(name, opt.calls, opt.rounds), 'us_per_call'), note='off: NULL weights, on: set')
        print(name, json.dumps(out['loss_kernel_' + name]), flush=True)
    for n in (1000, 10_000, 100_000):
        r = sampler_times(n, 512, opt.calls, opt.rounds)
        out['sampler_%d_episodes' % n] = {'us_per_call': r[True] + r[False], 'best_us': min(r[True] + r[False]), 'B': 512}
        print(n, json.dumps(out['sampler_%d_episodes' % n]), flush=True)
    for name in ('cfg2', 'cfg4'):
        r = update_times(name, opt.calls, opt.rounds)
        out['update_' + name] = {'us_per_call': r[True] + r[False], 'best_us': min(r[True] + r[False])}
    for name, steps in (('cfg2', opt.steps), ('cfg4', opt.steps_cfg4)):
        res, info = fill_step_times(name, steps, opt.rounds, opt.warmup)
        out[name + '_fill_step'] = dict(summary(res, 'ms_per_step'), steps_per_block=steps, **info)
        print(name, json.dumps(out[name + '_fill_step']), flush=True)
    line = json.dumps(out)
    print(line)
    if opt.out:
        os.makedirs(os.path.dirname(os.path.abspath(opt.out)), exist_ok=True)
        with open(opt.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
