"""Cost of board-symmetry augmentation (train_args['symmetry']) on one GPU, in one process:
  (a) the replay gather/pad kernel alone, hrl_gather_pad against hrl_gather_pad_sym with a random transform per window, at
      four shapes: cfg2 (TicTacToe 3x3, dihedral), cfg3 (Geister: mirror over its 6x6 planes, actions fixed), a 19x19 board
      with 362 actions (dihedral, pass fixed) and cfg5's 64x64 observation with 512 actions (dihedral on the board, actions
      fixed).  Episodes resident in the device ring, distinct outputs in rotation that together exceed L2, blocks of the two
      kernels alternated, best block each way; CUDA events.  Bandwidth = batch bytes written / time, against 3.35 TB/s.
  (b) bench.py's e2e_trainer leg (the drop-in Trainer on cfg2) with the key off and on.

    python scripts/bench_symmetry.py [--reps 20] [--rounds 3] [--trainer-steps 2000] [--out results/bench_symmetry.json]
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

from bench_diagnostics import gpu_name_and_power  # noqa: E402

HBM_TBS = 3.35          # H100 SXM HBM3 peak
L2_BYTES = 50e6

# name: (B, T, burn_in, P, observation (Pa = P), A, {leaf: per-step shape}, board group, board, actions move with the board)
SHAPES = {
    'cfg2_tictactoe_dihedral': (512, 32, 0, 2, False, 9, {'board': (3, 3, 3)}, 'dihedral', (3, 3), True),
    'cfg3_geister_mirror': (256, 20, 4, 2, True, 214, {'scalar': (18,), 'board': (7, 6, 6)}, 'mirror', (6, 6), False),
    'go19_dihedral': (256, 32, 0, 2, False, 362, {'board': (4, 19, 19)}, 'dihedral', (19, 19), True),
    'cfg5shard_64x64_dihedral': (512, 64, 0, 2, False, 512, {'board': (1, 64, 64)}, 'dihedral', (64, 64), False),
}


def make_replay(B, T, burn_in, P, A, leaves, g):
    from handyrl_b200.batch import FlatEpisode
    from handyrl_b200.replay import DeviceReplay
    steps = 3 * T
    obs_elems = sum(int(np.prod(s)) for s in leaves.values())
    n_eps = max(8, min(64, int(1.5e9 / (steps * P * (obs_elems + A) * 4))))
    rp = DeviceReplay(capacity_steps=n_eps * steps + 1, max_episodes=n_eps + 1)
    fes = []
    for _ in range(n_eps):
        fe = FlatEpisode()
        fe.steps, fe.players = steps, list(range(P))
        fe.obs = {k: (g.random((steps, P) + s) < 0.3).astype(np.float32) for k, s in leaves.items()}
        fe.prob = g.random((steps, P), dtype=np.float32)
        fe.action = g.integers(0, A, (steps, P)).astype(np.int32)
        fe.amask = np.where(g.random((steps, P, A)) < 0.7, 0, 1e32).astype(np.float32)
        fe.value = g.random((steps, P, 1), dtype=np.float32)
        fe.reward = np.zeros((steps, P), np.float32)
        fe.ret = np.zeros((steps, P), np.float32)
        fe.flags = np.full((steps, P), 3, np.uint8)
        fe.turn = (np.arange(steps) % P).astype(np.int32)
        fe.outcome = np.zeros(P, np.float32)
        fes.append(fe)
    rp.add_flat_many(fes)
    return rp


def tables_for(rp, group, board, actions_move):
    from handyrl_b200 import symmetry
    if actions_move:
        obs_src, act_dst = symmetry.board_tables(group, board, rp.leaf_shapes, rp.A)
    else:                         # custom tables: the board turns, the actions stay (timing only)
        obs_src = symmetry.board_tables(group, board, rp.leaf_shapes, max(rp.A, board[0] * board[1]))[0]
        act_dst = np.tile(np.arange(rp.A), (len(obs_src), 1))
    return symmetry.SymmetryTables(obs_src, act_dst, rp.OE, rp.A)


def gather_times(name, reps, rounds):
    from handyrl_b200 import symmetry
    B, T, burn_in, P, observation, A, leaves, group, board, actions_move = SHAPES[name]
    g = np.random.default_rng(0)
    rp = make_replay(B, T, burn_in, P, A, leaves, g)
    tables = tables_for(rp, group, board, actions_move)
    args = {'turn_based_training': True, 'observation': observation, 'burn_in_steps': burn_in, 'forward_steps': T - burn_in,
            'maximum_episodes': 1 << 20}
    probe = rp.empty_batch(B, args)
    batch_bytes = sum(t.numel() * t.element_size() for t in probe.values())
    n_out = max(2, min(16, int(2 * L2_BYTES / batch_bytes) + 1))
    outs = [probe] + [rp.empty_batch(B, args) for _ in range(n_out - 1)]
    wins = [rp.sample_windows(B, args, g) for _ in range(n_out)]
    wdev = [torch.from_numpy(x.view(np.uint8).reshape(B, -1)).cuda() for x in wins]
    ks = [torch.from_numpy(symmetry.draw(g, B, tables.K)).cuda() for _ in range(n_out)]
    tables.device(rp.device)
    live = float(np.mean([(x['end'] - x['start']).sum() / (B * T) for x in wins]))
    calls = {'plain': lambda i: rp.gather(wdev[i], args, out=outs[i]),
             'sym': lambda i: rp.gather(wdev[i], args, out=outs[i], sym=ks[i], tables=tables)}
    for fn in calls.values():
        for i in range(n_out):
            fn(i)
    torch.cuda.synchronize()
    res = {'plain': [], 'sym': []}
    for r in range(rounds):
        for k in (('plain', 'sym') if r % 2 == 0 else ('sym', 'plain')):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                for i in range(n_out):
                    calls[k](i)
            e1.record()
            e1.synchronize()
            res[k].append(e0.elapsed_time(e1) / (reps * n_out) * 1e3)
    best = {k: min(v) for k, v in res.items()}
    out = {'B': B, 'T': T, 'Pa': P if observation else 1, 'OE': rp.OE, 'A': A, 'K': tables.K, 'batch_MB': batch_bytes / 1e6,
           'live_fraction': live, 'outputs_in_rotation': n_out, 'plain_us': res['plain'], 'sym_us': res['sym']}
    for k in ('plain', 'sym'):
        out['best_%s_us' % k] = best[k]
        out['%s_write_TBs' % k] = batch_bytes / (best[k] * 1e-6) / 1e12
        out['%s_write_frac_of_hbm' % k] = out['%s_write_TBs' % k] / HBM_TBS
    out['sym_over_plain'] = best['sym'] / best['plain']
    return out


def trainer_rates(steps):
    """bench.py's e2e_trainer leg on cfg2, key off then on (the key added to the args that leg builds)."""
    import bench
    base = bench.train_args
    res = {}
    for on in (False, True):
        bench.train_args = (lambda w: dict(base(w), symmetry={'group': 'dihedral', 'board': [3, 3]})) if on else base
        try:
            r = bench.trainer_leg(bench.WORKLOADS['cfg2'], steps=steps)
        finally:
            bench.train_args = base
        res['on' if on else 'off'] = {k: r[k] for k in ('value', 'unit', 'ms_per_step', 'steps')}
    res['on_over_off'] = res['on']['value'] / res['off']['value']
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--trainer-steps', type=int, default=2000)
    ap.add_argument('--no-trainer', action='store_true')
    ap.add_argument('--out', default=None)
    opt = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_symmetry needs a GPU'
    out = {'gpu': gpu_name_and_power()}
    for name in SHAPES:
        out['gather_' + name] = gather_times(name, opt.reps, opt.rounds)
        torch.cuda.empty_cache()
        print(name, json.dumps({k: v for k, v in out['gather_' + name].items() if not isinstance(v, list)}), flush=True)
    if not opt.no_trainer:
        out['e2e_trainer_cfg2'] = trainer_rates(opt.trainer_steps)
    line = json.dumps(out)
    print(line)
    if opt.out:
        os.makedirs(os.path.dirname(os.path.abspath(opt.out)), exist_ok=True)
        with open(opt.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
