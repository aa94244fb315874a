"""Prioritised replay (train_args['prioritized_replay']).

Every stored window is trained on many times, because the learner consumes windows faster than the workers produce
episodes.  With the key set, the GPU replay draws episodes in proportion to how wrong the learner still is on them and
corrects the bias with importance weights.  The priorities live on the device and the sampler is a kernel
(hrl_replay_sample, csrc/replay_priority_kernel.cu), so the learner still never waits on the host.

The law (INTEGRATION.md):
  priority of a window   q_b = sum(tm * |Adv|) / sum(tm) + epsilon over its trained cells (t >= burn_in), tm the turn mask and
                         Adv the loss pass's total advantage (tap_advantage); sum(tm) == 0 gives no priority
  priority of an episode p_i, one per slot of the replay directory: a step that trained windows of episode i sets p_i to the
                         largest of their q_b; an episode the sampler has not seen starts at max_prio, the largest priority ever
                         stored (initially 1); a step rejected by skip_nonfinite writes nothing
  draw                   episode i (0 = the oldest of the `count` considered) with probability proportional to (i+1) * p_i^alpha:
                         the reference's recency law times the priority, so alpha = 0 is the recency law itself
  importance weight      w_b = B * p_b^(-alpha*beta) / sum_b' p_b'^(-alpha*beta), the (P/Q)^-beta correction of the priority
                         factor, normalised to mean 1 over the batch; beta = 0 gives exactly 1

This module parses the key, owns the device buffers (PriorityState) and holds the host references of the kernels.
"""
import numbers

import numpy as np

DEFAULTS = {'alpha': 0.6, 'beta': 0.4, 'epsilon': 0.01}


def config(args):
    """train_args['prioritized_replay'] -> {'alpha', 'beta', 'epsilon'} (floats), or None when the feature is off (key absent,
    None or False).  True takes the defaults; a dict overrides any of them.  Raises ValueError for any other value, an unknown
    key, a value out of range (alpha >= 0, 0 <= beta <= 1, epsilon > 0), and for the key with gpu_replay: False."""
    value = args.get('prioritized_replay')
    if value is None or value is False:
        return None
    if value is True:
        spec = dict(DEFAULTS)
    elif isinstance(value, dict):
        unknown = sorted(set(value) - set(DEFAULTS), key=str)
        if unknown:
            raise ValueError("train_args['prioritized_replay']: unknown key(s) %s (known: alpha, beta, epsilon)" % unknown)
        spec = dict(DEFAULTS)
        for k, v in value.items():
            if isinstance(v, bool) or not isinstance(v, numbers.Real) or not np.isfinite(float(v)):
                raise ValueError("train_args['prioritized_replay']['%s'] must be a finite number; got %r" % (k, v))
            spec[k] = float(v)
    else:
        raise ValueError("train_args['prioritized_replay'] must be True, False, None or a dict of alpha, beta, epsilon; got %r"
                         % (value,))
    if not spec['alpha'] >= 0:
        raise ValueError("train_args['prioritized_replay']: alpha=%r must be >= 0" % spec['alpha'])
    if not 0 <= spec['beta'] <= 1:
        raise ValueError("train_args['prioritized_replay']: beta=%r must lie in [0, 1]" % spec['beta'])
    if not spec['epsilon'] > 0:
        raise ValueError("train_args['prioritized_replay']: epsilon=%r must be > 0" % spec['epsilon'])
    if not args.get('gpu_replay', True):
        raise ValueError("train_args['prioritized_replay'] needs the GPU replay (gpu_replay: True): the sampler is a kernel")
    return spec


def ring_slots(args):
    """Slots of the replay directory ring (DeviceReplay keeps maximum_episodes + 1)."""
    return int(args['maximum_episodes']) + 1


def sampler_key(seed):
    """Philox key of a batch sampler seeded with `seed` (its own stream: the host generators are left alone)."""
    return (int(seed) * 0x9E3779B97F4A7C15 + 3) % (1 << 64)


class PriorityState:
    """The device buffers of prioritised replay for one learner (one rank):
      prio [ring] float32, prio_serial [ring] int64 (-1: no episode yet), max_prio [1] float32 = 1,
      cdf [ring] float64 (the sampler's prefix sums),
      win_slot [B] int32, win_serial [B] int64 (-1: the window updates nothing), win_weight [B] float32 = 1.
    The learner step owns it because its captured graph bakes in the update kernel's pointers; the batcher fills the
    per-window buffers through the sampler."""

    def __init__(self, spec, ring, B, device):
        import torch
        self.alpha, self.beta, self.epsilon = spec['alpha'], spec['beta'], spec['epsilon']
        self.ring, self.B = int(ring), int(B)
        self.prio = torch.ones(self.ring, dtype=torch.float32, device=device)
        self.prio_serial = torch.full((self.ring,), -1, dtype=torch.int64, device=device)
        self.max_prio = torch.ones(1, dtype=torch.float32, device=device)
        self.cdf = torch.zeros(self.ring, dtype=torch.float64, device=device)
        self.win_slot = torch.zeros(self.B, dtype=torch.int32, device=device)
        self.win_serial = torch.full((self.B,), -1, dtype=torch.int64, device=device)
        self.win_weight = torch.ones(self.B, dtype=torch.float32, device=device)


# ---------------------------------------------------------------- host references of the kernels

def window_priorities(advantage, turn_mask, burn_in, epsilon):
    """q_b of each window (float64): advantage and turn_mask (B, T, P[, 1]).  NaN where the window gives no priority
    (sum(tm) == 0 over its trained cells)."""
    adv = np.asarray(advantage, np.float64).reshape(advantage.shape[0], advantage.shape[1], -1)[:, burn_in:]
    tm = np.asarray(turn_mask, np.float64).reshape(adv.shape[0], -1, adv.shape[2])[:, burn_in:]
    num = (tm * np.abs(adv)).sum(axis=(1, 2))
    den = tm.sum(axis=(1, 2))
    with np.errstate(invalid='ignore', divide='ignore'):
        return np.where(den != 0, num / np.where(den != 0, den, 1) + epsilon, np.nan)


def draw_probabilities(prio, alpha):
    """Probability of drawing each of count episodes (oldest first) with priorities prio: (i+1) * p_i^alpha, normalised."""
    p = np.asarray(prio, np.float64)
    w = np.arange(1, p.size + 1, dtype=np.float64) * p ** alpha
    return w / w.sum()


def importance_weights(prio_drawn, alpha, beta):
    """w_b = B * p_b^(-alpha*beta) / sum_b' p_b'^(-alpha*beta) for the priorities of the drawn windows."""
    x = np.asarray(prio_drawn, np.float64) ** (-alpha * beta)
    return x.size * x / x.sum()


def update(prio, prio_serial, max_prio, slots, serials, q, skip=False):
    """The priority update of one step on host arrays (returns new prio, new max_prio; prio_serial is read only): windows
    with serial < 0, with a serial that no longer matches their slot, or without priority (NaN q) write nothing; windows on
    one slot resolve to their largest q; max_prio rises to the largest q written; skip: nothing at all."""
    prio = np.array(prio, np.float32, copy=True)
    max_prio = float(max_prio)
    if skip:
        return prio, max_prio
    best = {}
    for s, ser, qb in zip(np.asarray(slots), np.asarray(serials), np.asarray(q, np.float64)):
        if ser < 0 or not np.isfinite(qb) or prio_serial[s] != ser:
            continue
        best[int(s)] = max(best.get(int(s), -np.inf), float(np.float32(qb)))
    for s, v in best.items():
        prio[s] = v
        max_prio = max(max_prio, v)
    return prio, np.float32(max_prio)


def refresh(prio, prio_serial, dir_serial, live_slots, max_prio):
    """The sampler's first step on host arrays: live slots whose directory serial differs from prio_serial start at max_prio.
    Returns new (prio, prio_serial)."""
    prio = np.array(prio, np.float32, copy=True)
    prio_serial = np.array(prio_serial, np.int64, copy=True)
    for s in live_slots:
        if prio_serial[s] != dir_serial[s]:
            prio[s] = max_prio
            prio_serial[s] = dir_serial[s]
    return prio, prio_serial


# ---------------------------------------------------------------- priorities in the replay checkpoints (train_args['save_replay'])

def image(slot_serial, priority, max_prio, resident_serials):
    """The priorities a replay checkpoint stores, keyed by serial: of the per-slot state (PriorityState.prio_serial and prio
    as host arrays), the slots whose serial belongs to a resident episode.  A slot that never held an episode (-1) or whose
    episode has left the ring is dropped; a resident episode the sampler has not seen yet has no entry."""
    slot_serial, priority = np.asarray(slot_serial, np.int64), np.asarray(priority, np.float32)
    resident = np.asarray(resident_serials, np.int64)
    keep = (slot_serial >= 0) & np.isin(slot_serial, resident[resident >= 0])
    order = np.argsort(slot_serial[keep], kind='stable')
    return {'serial': slot_serial[keep][order], 'priority': priority[keep][order], 'max_prio': float(max_prio)}


def restore_entries(saved, saved_serials, positions, slots, serials):
    """Where a checkpoint's priorities go in a restored ring.  saved: {'serial', 'priority'} (image()); saved_serials: the
    serial each position of the checkpoint's episode list had (-1: held out); positions: for each episode resident now, oldest
    first, its position in that list, or -1 for an episode that was not in it; slots, serials: the directory slot and the
    serial each has now.  Returns (slots, serials, priorities) of the episodes that get their saved priority; the others keep
    none and start at max_prio, as a new episode does.  A serial is unique in a ring and a position maps to one episode, so no
    slot appears twice; repeated positions or serials raise ValueError."""
    key = np.asarray(saved['serial'], np.int64)
    prio = np.asarray(saved['priority'], np.float32)
    saved_serials, positions = np.asarray(saved_serials, np.int64), np.asarray(positions, np.int64)
    slots, serials = np.asarray(slots, np.int64), np.asarray(serials, np.int64)
    if key.shape != prio.shape or positions.shape != slots.shape or slots.shape != serials.shape:
        raise ValueError('restore_entries: array lengths differ')
    if np.unique(key).size != key.size:
        raise ValueError('restore_entries: a serial appears twice in the saved priorities')
    known = positions >= 0
    if positions[known].size and (positions[known].max() >= saved_serials.size or
                                  np.unique(positions[known]).size != positions[known].size):
        raise ValueError('restore_entries: positions outside the saved list or repeated')
    old = np.full(positions.shape, -1, np.int64)
    old[known] = saved_serials[positions[known]]
    order = np.argsort(key, kind='stable')
    at = np.searchsorted(key[order], old)
    hit = (old >= 0) & (at < key.size)
    hit[hit] = key[order][at[hit]] == old[hit]
    return slots[hit], serials[hit], prio[order][at[hit]]
