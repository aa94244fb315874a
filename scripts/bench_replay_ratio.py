"""The replay ratio limit (train_args['replay_ratio']) on one GPU: the drop-in Trainer on cfg2 (TicTacToe net, fused tower,
B=512, forward_steps=32) fed by a producer thread that appends episodes at a fixed rate, with epoch hand-offs (update()) at a
fixed period, as the Learner does.  Runs, in one process:
  * key off and a limit too large ever to bind (--free), alternated --rounds times each: steps/s of each run and their spread;
  * two binding limits (--binding): steps/s, and per epoch the achieved ratio (trained samples over stored steps) and the
    fraction of the epoch the trainer thread waited for credit.

    python scripts/bench_replay_ratio.py [--seconds 8] [--rounds 3] [--episodes-per-s 1000] [--binding 32 256]
                                         [--out results/bench_replay_ratio.json]
"""
import argparse
import json
import os
import statistics
import sys
import threading
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from bench_diagnostics import gpu_name_and_power  # noqa: E402


def producer(tr, episodes, per_s, stop, maximum):
    """Append episodes to tr.episodes at `per_s` episodes per second, in slices every 10 ms, on a fixed schedule."""
    t0, sent = time.perf_counter(), 0
    while not stop.is_set():
        due = int((time.perf_counter() - t0) * per_s)
        if due > sent:
            tr.episodes.extend(episodes[(sent + i) % len(episodes)] for i in range(due - sent))
            sent = due
            while len(tr.episodes) > maximum:
                tr.episodes.popleft()
        time.sleep(0.01)


def run(ratio, opt, backlog, fresh):
    import bench
    from handyrl_b200.train import Trainer
    w = bench.WORKLOADS['cfg2']
    args = dict(bench.train_args(w), minimum_episodes=len(backlog), maximum_episodes=20000, gpu_replay=True, num_gpus=1,
                forward_steps=w['T'])
    if ratio:
        args['replay_ratio'] = ratio
    tr = Trainer(args, bench.make_net(w))
    tr.episodes.extend(backlog)
    th = threading.Thread(target=tr.run, daemon=True)
    th.start()
    tr.update()                                    # the first epoch builds and captures the step
    stop = threading.Event()
    prod = threading.Thread(target=producer, args=(tr, fresh, opt.episodes_per_s, stop, args['maximum_episodes']), daemon=True)
    prod.start()
    while tr.steps < opt.warm_steps:
        time.sleep(0.005)
    tr.update()                                    # the timed region starts with an epoch
    tr.stepper.stream.synchronize()
    s0, t0 = tr.steps, time.perf_counter()
    stored0 = tr.replay_ratio_stats()['stored'] if ratio else None
    epochs = []
    while time.perf_counter() - t0 < opt.seconds:
        time.sleep(opt.epoch_s)
        tr.update()
        if ratio:
            ep = tr.replay_ratio_stats()['epoch']
            epochs.append({'ratio': ep['ratio'], 'waited': ep['waited'], 'wall_s': ep['wall'], 'steps': ep['trained'] // (w['B'] * w['T'])})
    tr.stepper.stream.synchronize()
    dt, n = time.perf_counter() - t0, tr.steps - s0
    out = {'replay_ratio': ratio, 'steps_per_s': n / dt, 'samples_per_s': n * w['B'] * w['T'] / dt, 'steps': n, 'seconds': dt}
    if ratio:
        stats = tr.replay_ratio_stats()
        out['stored_steps_per_s'] = (stats['stored'] - stored0) / dt
        out['epochs'] = epochs
    stop.set()
    prod.join(timeout=5)
    tr.stop()
    th.join(timeout=30)
    return out


def spread(xs):
    med = statistics.median(xs)
    return {'median': med, 'min': min(xs), 'max': max(xs), 'spread_pct': 100.0 * (max(xs) - min(xs)) / med}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--seconds', type=float, default=8.0, help='timed region of each run')
    ap.add_argument('--epoch-s', type=float, default=1.0, help='period of the update() hand-offs')
    ap.add_argument('--rounds', type=int, default=3, help='alternated key-off / non-binding runs, each')
    ap.add_argument('--warm-steps', type=int, default=50)
    ap.add_argument('--episodes-per-s', type=float, default=1000.0, help='producer rate (6 reference workers: about 900)')
    ap.add_argument('--free', type=float, default=1e9, help='a limit too large to bind')
    ap.add_argument('--binding', type=float, nargs='*', default=[32.0, 256.0])
    ap.add_argument('--out', default=None)
    opt = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_replay_ratio needs a GPU'
    from handyrl_b200.synthetic import tictactoe_episodes
    backlog, fresh = tictactoe_episodes(4000, seed=7), tictactoe_episodes(4000, seed=8)
    res = {'gpu': gpu_name_and_power(), 'workload': 'cfg2 Trainer, TicTacToe net, B=512 forward_steps=32',
           'producer_episodes_per_s': opt.episodes_per_s, 'mean_episode_steps': sum(e['steps'] for e in fresh) / len(fresh),
           'timing': 'host wall clock over the timed region, step stream synchronised at both ends'}
    runs = {'off': [], 'free': []}
    for r in range(opt.rounds):
        for arm in (('off', 'free') if r % 2 == 0 else ('free', 'off')):
            runs[arm].append(run(opt.free if arm == 'free' else None, opt, backlog, fresh))
            print(arm, json.dumps(runs[arm][-1]), flush=True)
    res['off'] = dict(spread([x['steps_per_s'] for x in runs['off']]), runs=runs['off'])
    res['free'] = dict(spread([x['steps_per_s'] for x in runs['free']]), runs=runs['free'], replay_ratio=opt.free)
    res['free_vs_off_pct'] = 100.0 * (res['free']['median'] - res['off']['median']) / res['off']['median']
    res['binding'] = []
    for ratio in opt.binding:
        out = run(ratio, opt, backlog, fresh)
        print('binding', json.dumps(out), flush=True)
        res['binding'].append(out)
    line = json.dumps(res)
    print(line)
    if opt.out:
        os.makedirs(os.path.dirname(os.path.abspath(opt.out)), exist_ok=True)
        with open(opt.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
