"""Host side of replay batching: decode an episode ONCE into flat arrays, then slice/pad windows.

Mirrors the reference's make_batch (handyrl/train.py:33-124) and Batcher.select_episode
(train.py:291-315) in behaviour, but not in structure: the reference re-decompresses and
re-walks nested per-player dicts for every sampled window; here an episode is decoded once
into a `FlatEpisode` (the same row layout the device replay store and the gather/pad kernel
use, include/hrl_b200.h HrlGatherArgs) and a batch is a gather over those rows.

Known, documented deviation: `selected_prob` is always float32 (the reference silently
produces float64 when a player's entry is None, SURVEY.md hard part 4).
"""
import bz2
import pickle
import random

import numpy as np
import torch


def tree_map(fn, *trees):
    """Apply fn leaf-wise over nested dict/list/tuple structures of equal shape."""
    t0 = trees[0]
    if isinstance(t0, dict):
        return type(t0)((k, tree_map(fn, *[t[k] for t in trees])) for k in t0)
    if isinstance(t0, (list, tuple)):
        return type(t0)(tree_map(fn, *[t[i] for t in trees]) for i in range(len(t0)))
    return fn(*trees)


def tree_leaves(tree):
    if isinstance(tree, dict):
        return [l for v in tree.values() for l in tree_leaves(v)]
    if isinstance(tree, (list, tuple)):
        return [l for v in tree for l in tree_leaves(v)]
    return [tree]


class FlatEpisode:
    """One episode as step-major arrays; row s = episode step s, column = player slot."""
    __slots__ = ('steps', 'players', 'obs', 'prob', 'action', 'amask', 'value', 'reward', 'ret', 'flags',
                 'turn', 'outcome')


def decode_moments(blocks):
    out = []
    for blk in blocks:
        out.extend(pickle.loads(bz2.decompress(blk)))
    return out


def flatten_moments(moments, outcome, players=None):
    """Nested per-player moment dicts (generation.py:32-33, 72) -> FlatEpisode.

    Absent entries take the reference's defaults (train.py:70-82): zero observation, prob 1,
    action 0, action_mask 1e32, value 0, reward 0, return 0.
    """
    fe = FlatEpisode()
    S = len(moments)
    if players is None:
        players = list(moments[0]['observation'].keys())
    Ps = len(players)
    fe.steps, fe.players = S, players

    obs_tmpl = amask_tmpl = None
    for m in moments:
        tp = m['turn'][0]
        if obs_tmpl is None and m['observation'][tp] is not None:
            obs_tmpl = tree_map(lambda o: np.zeros_like(np.asarray(o)), m['observation'][tp])
        if amask_tmpl is None and m['action_mask'][tp] is not None:
            amask_tmpl = np.zeros_like(np.asarray(m['action_mask'][tp]))
        if obs_tmpl is not None and amask_tmpl is not None:
            break
    A = amask_tmpl.shape[-1]

    fe.obs = tree_map(lambda z: np.zeros((S, Ps) + z.shape, dtype=z.dtype), obs_tmpl)
    obs_leaves = tree_leaves(fe.obs)
    fe.prob = np.ones((S, Ps), np.float32)
    fe.action = np.zeros((S, Ps), np.int32)
    fe.amask = np.full((S, Ps, A), 1e32, np.float32)
    vdim = 1
    for m in moments:
        v = next((x for x in m['value'].values() if x is not None), None)
        if v is not None:
            vdim = int(np.asarray(v).size)
            break
    fe.value = np.zeros((S, Ps, vdim), np.float32)
    fe.reward = np.zeros((S, Ps), np.float32)
    fe.ret = np.zeros((S, Ps), np.float32)
    fe.flags = np.zeros((S, Ps), np.uint8)
    fe.turn = np.zeros(S, np.int32)
    slot = {p: i for i, p in enumerate(players)}
    for s, m in enumerate(moments):
        fe.turn[s] = slot[m['turn'][0]]
        for p, i in slot.items():
            o = m['observation'][p]
            if o is not None:
                for dst, src in zip(obs_leaves, tree_leaves(o)):
                    dst[s, i] = src
                fe.flags[s, i] |= 2
            sp = m['selected_prob'][p]
            if sp is not None:
                fe.prob[s, i] = sp
                fe.flags[s, i] |= 1
            if m['action'][p] is not None:
                fe.action[s, i] = m['action'][p]
            if m['action_mask'][p] is not None:
                fe.amask[s, i] = m['action_mask'][p]
            if m['value'][p] is not None:
                fe.value[s, i] = np.asarray(m['value'][p], np.float32).reshape(-1)
            if m['reward'][p] is not None:
                fe.reward[s, i] = m['reward'][p]
            if m['return'][p] is not None:
                fe.ret[s, i] = m['return'][p]
    fe.outcome = np.array([outcome[p] for p in players], np.float32)
    return fe


def reduce_values(fe, value_bins):
    """A FlatEpisode whose stored values are a categorical value head's K logits (train_args['value_bins'], parsed by
    value_bins.config) with each present value reduced to its expectation: fe.value becomes (S, Ps, 1), what the replay
    stores.  A value is present where the player observed (flags bit 1); absent ones stay 0.  Episodes with scalar values,
    and every episode when the value head is not categorical, are returned as they are."""
    spec = (value_bins or {}).get('value')
    if spec is None or fe.value.shape[-1] == 1:
        return fe
    if fe.value.shape[-1] != spec['bins']:
        raise ValueError("train_args['value_bins']['value'] has %d bins, but an episode stores %d values per moment"
                         % (spec['bins'], fe.value.shape[-1]))
    from .value_bins import reduce_values as reduce
    fe.value = reduce(fe.value, (fe.flags & 2) != 0, spec)
    return fe


def window_rows(T, burn_in, start, end, train_start):
    """Where a window [start, end) lands in the T batch steps (train.py:92-95): returns
    (t0, n) = first batch step holding real data and how many."""
    n = end - start
    pad_before = burn_in - (train_start - start) if n < T else 0
    return pad_before, n


def gather_windows(windows, args, rng=random):
    """Collate windows into the reference's batch dict (numpy arrays).

    windows: list of (FlatEpisode, local_start, local_end, start, train_start, total) where
    local_* index rows of the FlatEpisode and start/train_start/total are episode step numbers.
    """
    T = args['burn_in_steps'] + args['forward_steps']
    burn_in = args['burn_in_steps']
    B = len(windows)
    fe0 = windows[0][0]
    Ps = len(fe0.players)
    alternating = args['turn_based_training'] and not args['observation']
    solo = not args['turn_based_training']
    P = 1 if solo else Ps
    Pa = 1 if alternating else P
    A = fe0.amask.shape[-1]
    vdim = fe0.value.shape[-1]

    obs = tree_map(lambda z: np.zeros((B, T, Pa) + z.shape[2:], z.dtype), fe0.obs)
    obs_leaves = tree_leaves(obs)
    prob = np.ones((B, T, Pa, 1), np.float32)
    act = np.zeros((B, T, Pa, 1), np.int64)
    amask = np.full((B, T, Pa, A), 1e32, np.float32)
    value = np.zeros((B, T, P, vdim), np.float32)
    reward = np.zeros((B, T, P, 1), np.float32)
    ret = np.zeros((B, T, P, 1), np.float32)
    outcome = np.zeros((B, 1, P, 1), np.float32)
    emask = np.zeros((B, T, 1, 1), np.float32)
    tmask = np.zeros((B, T, P, 1), np.float32)
    omask = np.zeros((B, T, P, 1), np.float32)
    progress = np.ones((B, T, 1), np.float32)

    for b, (fe, l0, l1, start, train_start, total) in enumerate(windows):
        t0, n = window_rows(T, burn_in, start, start + (l1 - l0), train_start)
        rows = slice(l0, l1)
        dst = slice(t0, t0 + n)
        if solo:   # train.py:57-58: one random player per sampled window
            vp = [rng.choice(range(Ps))]
        else:
            vp = list(range(Ps))
        if alternating:
            pp = fe.turn[rows]                              # (n,) the turn player's slot
            sel = (np.arange(l0, l1), pp)
            for d, s in zip(obs_leaves, tree_leaves(fe.obs)):
                d[b, dst, 0] = s[sel]
            prob[b, dst, 0, 0] = fe.prob[sel]
            act[b, dst, 0, 0] = fe.action[sel]
            amask[b, dst, 0] = fe.amask[sel]
        else:
            for d, s in zip(obs_leaves, tree_leaves(fe.obs)):
                d[b, dst] = s[rows][:, vp]
            prob[b, dst, :, 0] = fe.prob[rows][:, vp]
            act[b, dst, :, 0] = fe.action[rows][:, vp]
            amask[b, dst] = fe.amask[rows][:, vp]
        value[b, dst] = fe.value[rows][:, vp]
        value[b, t0 + n:] = fe.outcome[vp].reshape(1, P, 1)                 # train.py:98
        reward[b, dst, :, 0] = fe.reward[rows][:, vp]
        ret[b, dst, :, 0] = fe.ret[rows][:, vp]
        fl = fe.flags[rows][:, vp]
        tmask[b, dst, :, 0] = (fl & 1) != 0
        omask[b, dst, :, 0] = (fl & 2) != 0
        emask[b, dst] = 1
        outcome[b, 0, :, 0] = fe.outcome[vp]
        progress[b, dst, 0] = np.arange(start, start + n, dtype=np.float32) / np.float32(total)   # train.py:89

    return {
        'observation': obs, 'selected_prob': prob, 'value': value, 'action': act, 'outcome': outcome,
        'reward': reward, 'return': ret, 'episode_mask': emask, 'turn_mask': tmask,
        'observation_mask': omask, 'action_mask': amask, 'progress': progress,
    }


def make_batch(episodes, args):
    """Drop-in for handyrl.train.make_batch: list of 'minimum episode' dicts
    (train.py:309-314) -> dict of torch tensors with the layouts of train.py:114-124."""
    windows = []
    for ep in episodes:
        fe = flatten_moments(decode_moments(ep['moment']), ep['outcome'])
        l0, l1 = ep['start'] - ep['base'], ep['end'] - ep['base']
        windows.append((fe, l0, l1, ep['start'], ep['train_start'], ep['total']))
    np_batch = gather_windows(windows, args)
    return tree_map(lambda a: torch.from_numpy(np.ascontiguousarray(a)), np_batch)


def sample_window(n_episodes, fetch, args, rng=random):
    """Recency-biased episode choice + window placement (train.py:291-308).

    `fetch(idx)` returns (steps, episode) for the idx-th oldest episode and may raise IndexError if the replay
    shrank concurrently (train.py:298-302 retries).  The episode object is fetched ONCE and handed back, so the
    window always fits the episode it was drawn for even when the deque shifts underneath.
    Returns (episode index, start, end, train_start, episode).
    """
    while True:
        count = min(n_episodes(), args['maximum_episodes'])
        idx = rng.randrange(count)
        accept = 1 - (count - 1 - idx) / count
        if rng.random() >= accept:
            continue
        try:
            steps, episode = fetch(idx)
        except IndexError:
            continue
        break
    candidates = 1 + max(0, steps - args['forward_steps'])
    train_start = rng.randrange(candidates)
    start = max(0, train_start - args['burn_in_steps'])
    end = min(train_start + args['forward_steps'], steps)
    return idx, start, end, train_start, episode
