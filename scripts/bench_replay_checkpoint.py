"""Cost of train_args['save_replay'] on one GPU, in one command:

  1. step time of the cfg2 Trainer (TicTacToe net, fused tower, B=512, forward_steps=32) with the key off and on, alternated in blocks (the key adds nothing to the step, so the two
     must agree within the spread of the blocks);
  2. at 1k / 10k / 100k resident episodes: the time GpuBatcher.snapshot() takes (what the trainer thread spends at an epoch
     boundary), the time update() spends handing the file to the writer, the write time and file size, and the time from
     the file to a GpuBatcher whose restored backlog is resident (load + feed).

The episodes of leg 2 repeat a pool of 2000 distinct ones; pickle stores a repeated payload once, so write time, file size
and load time beyond 2000 episodes are lower bounds.

Prints one JSON line, with the card's name and power limit read in the same run.

    python scripts/bench_replay_checkpoint.py [--blocks 3] [--epochs 6] [--sizes 1000,10000,100000]
"""
import argparse
import json
import os
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

import torch  # noqa: E402

from bench_diagnostics import gpu_name_and_power  # noqa: E402


def trainer_args(**extra):
    import bench
    w = bench.WORKLOADS['cfg2']
    return dict(bench.train_args(w), minimum_episodes=100, maximum_episodes=20000, gpu_replay=True, num_gpus=1,
                forward_steps=w['T'], **extra)


def step_time(on, episodes, epochs, epoch_seconds):
    """Mean wall time per step of `epochs` epochs of a Trainer (device work included: each update() waits for its epoch)."""
    import bench
    from handyrl_b200.train import Trainer
    tr = Trainer(trainer_args(**({'save_replay': True} if on else {})), bench.make_net(bench.WORKLOADS['cfg2']))
    tr.episodes.extend(episodes)
    th = threading.Thread(target=tr.run, daemon=True)
    th.start()
    try:
        _, s0 = tr.update()                       # capture and warm-up are in the first epoch
        while tr.gpu_batcher.fed < len(episodes):
            time.sleep(0.01)
        _, s0 = tr.update()
        t0 = time.perf_counter()
        for _ in range(epochs):
            time.sleep(epoch_seconds)
            _, s1 = tr.update()
        dt = time.perf_counter() - t0
    finally:
        tr.stop()
        th.join(timeout=30)
    return 1e6 * dt / (s1 - s0), s1 - s0


def sizes_leg(n, episodes_pool, directory):
    from handyrl_b200.train import EpisodeDeque, GpuBatcher, ReplayCheckpoints, load_replay_file, replay_file
    args = dict(trainer_args(save_replay=True, prioritized_replay=True), maximum_episodes=n)
    eps = [dict(episodes_pool[i % len(episodes_pool)]) for i in range(n)]          # n distinct episode objects
    dq = EpisodeDeque()
    dq.extend(eps)
    gb = GpuBatcher(args, dq, torch.device('cuda'))
    gb.run()
    while not gb.ready():
        time.sleep(0.01)
    torch.cuda.synchronize()
    ts = []
    for _ in range(5):
        t0 = time.perf_counter()
        snap = gb.snapshot()
        ts.append(time.perf_counter() - t0)
    ring = n + 1
    state = {'slot_serial': torch.arange(ring), 'priority': torch.rand(ring) + 0.01, 'max_prio': 1.5}
    files = ReplayCheckpoints(directory, keep=1)
    t0 = time.perf_counter()
    obj = replay_file(snap, state, None, 0, 1)
    files.submit(1, obj)
    submit = time.perf_counter() - t0
    t0 = time.perf_counter()
    files.close()
    write = time.perf_counter() - t0
    path = files.path(1)
    size = os.path.getsize(path)
    resident = len(snap['episodes'])
    gb.stop()
    del gb, dq, snap, obj
    torch.cuda.empty_cache()
    t0 = time.perf_counter()
    d = load_replay_file(path)
    load = time.perf_counter() - t0
    dq = EpisodeDeque()
    dq.extend(d['episodes'])
    gb = GpuBatcher(args, dq, torch.device('cuda'), restore=d)
    gb.run()
    while not gb.ready():
        time.sleep(0.005)
    torch.cuda.synchronize()
    restore = time.perf_counter() - t0
    gb.restore_sampler(d['sampler'])
    gb.stop()
    os.remove(path)
    return {'episodes': resident, 'snapshot_ms': 1e3 * sorted(ts)[len(ts) // 2], 'snapshot_ms_max': 1e3 * max(ts),
            'submit_ms': 1e3 * submit, 'write_s': write, 'file_mb': size / 1e6, 'load_s': load, 'file_to_ready_s': restore}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--blocks', type=int, default=3)
    ap.add_argument('--epochs', type=int, default=6)
    ap.add_argument('--epoch-seconds', type=float, default=1.0)
    ap.add_argument('--sizes', default='1000,10000,100000')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_replay_checkpoint.py needs a CUDA device')
    from handyrl_b200.synthetic import tictactoe_episodes
    result = {'gpu': gpu_name_and_power(), 'workload': 'cfg2 Trainer, TicTacToe net, B=512 forward_steps=32'}
    pool = tictactoe_episodes(2000, seed=4)
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)                             # the Trainer writes models/ relative to the working directory
        blocks = {'off': [], 'on': []}
        for _ in range(a.blocks):
            for name, on in (('off', False), ('on', True)):
                us, steps = step_time(on, pool, a.epochs, a.epoch_seconds)
                blocks[name].append(round(us, 2))
        result['step_us'] = blocks
        result['sizes'] = [sizes_leg(int(n), pool, os.path.join(tmp, 'sizes')) for n in a.sizes.split(',') if n]
    print(json.dumps(result))


if __name__ == '__main__':
    main()
