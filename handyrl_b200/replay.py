"""GPU-resident replay: episodes are decoded ONCE on arrival into flat device arrays; a training batch is
B window descriptors + one gather/pad kernel (csrc/gather_kernel.cu, C ABI hrl_gather_pad).

Replaces, for the learner, the reference's per-sample bz2+pickle decode and Python collation
(make_batch, handyrl/train.py:33-124) and the batcher process pool that ships pickled batches through
pipes (train.py:270-289, connection.py:133-173).  Sampling semantics (recency-biased episode choice,
window placement, burn-in) are those of Batcher.select_episode (train.py:291-315), shared with the
host path through batch.sample_window.

Store layout = include/hrl_b200.h HrlGatherArgs: one row per episode step, columns per player slot.
Nested observations are stored as the concatenation of their flattened leaves.
"""
import collections
import ctypes as C
import hashlib
import random
import threading

import numpy as np
import torch

from . import _capi
from ._capi import HrlGatherArgs, HrlWindow, check, lib
from .batch import flatten_moments, decode_moments, sample_window, tree_leaves, tree_map

WINDOW_DTYPE = np.dtype([('first_step', '<i8'), ('start', '<i4'), ('end', '<i4'), ('train_start', '<i4'),
                         ('total', '<i4'), ('outcome_row', '<i4'), ('player', '<i4')])
assert WINDOW_DTYPE.itemsize == C.sizeof(HrlWindow)


def held_out(fe, rate):
    """True when the episode (a FlatEpisode) belongs to the held-out validation split of rate r: an 8-byte BLAKE2b digest of its
    step arrays (action, selected prob, turn) and outcome, read as a fraction in [0, 1), is below r.  The decision depends on the
    episode's content alone -- not on Python's salted hash(), the arrival order, the rank or the wire format it came in -- so every
    rank and every restart splits the replay the same way.  rate None or 0: never."""
    if not rate:
        return False
    h = hashlib.blake2b(digest_size=8)
    for a in (fe.action, fe.prob, fe.turn, fe.outcome):
        h.update(np.ascontiguousarray(a).tobytes())
    return int.from_bytes(h.digest(), 'little') < rate * 2.0 ** 64


class EpisodeHandle:
    """Where one stored episode lives: first row of the step ring, number of steps, row of the outcome table."""
    __slots__ = ('first_step', 'steps', 'outcome_row')

    def __init__(self, first_step, steps, outcome_row):
        self.first_step, self.steps, self.outcome_row = int(first_step), int(steps), int(outcome_row)

    def __eq__(self, other):
        return (self.first_step, self.steps, self.outcome_row) == (other.first_step, other.steps, other.outcome_row)

    def __repr__(self):
        return 'EpisodeHandle(first_step=%d, steps=%d, outcome_row=%d)' % (self.first_step, self.steps, self.outcome_row)


class DeviceReplay:
    """Ring of decoded episodes in HBM.

    capacity_steps bounds the stored steps, max_episodes the stored episodes (the reference trims its
    deque to `maximum_episodes`, train.py:474-483); when either is exceeded the oldest episodes go.
    The episode directory (first row / length / outcome row, oldest first) is a numpy ring so that B windows
    are drawn with array operations instead of a Python loop per window.

    track=True (train_args['save_replay']): `resident` holds, for every directory entry and in its order, the item the caller
    staged with that episode (stage(fes, items); the GPU batcher passes the episode as it arrived), appended and evicted with
    the directory under `lock`.  References only: nothing is copied and nothing is done per step.
    """

    def __init__(self, capacity_steps, max_episodes, device='cuda', mirror=False, track=False):
        self.device = torch.device(device)
        self.capacity = int(capacity_steps)
        self.max_episodes = int(max_episodes)
        self._dir = np.zeros((self.max_episodes + 1, 3), np.int64)      # (first_step, steps, outcome_row), a ring
        self._head = 0
        self._count = 0
        self.write = 0
        self.ready = False
        self.next_outcome_row = 0
        self.lock = threading.Lock()       # guards the directory (feeder thread appends, learner thread samples)
        self.resident = collections.deque() if track else None
        # every stored episode gets the next serial, so a directory slot that is reused is told apart from its old episode
        self._serial = np.full(self.max_episodes + 1, -1, np.int64)
        self.next_serial = 0
        # mirror=True (prioritised replay): a device copy of the directory, [slot] = (first_step, steps, outcome_row, serial),
        # which commit() updates on its stream for the slots it appends; the device sampler reads it
        self.dir_dev = (torch.full((self.max_episodes + 1, 4), -1, dtype=torch.int64, device=self.device) if mirror else None)

    # ------------------------------------------------------------------ directory
    def __len__(self):
        return self._count

    def _entry(self, i):
        return self._dir[(self._head + i) % self._dir.shape[0]]

    @property
    def handles(self):
        """Stored episodes, oldest first (a snapshot; the directory itself is the numpy ring)."""
        return [EpisodeHandle(*self._entry(i)) for i in range(self._count)]

    def _popleft(self):
        self._head = (self._head + 1) % self._dir.shape[0]
        self._count -= 1
        if self.resident is not None:
            self.resident.popleft()

    def _append(self, first_step, steps, row, item=None):
        slot = (self._head + self._count) % self._dir.shape[0]
        self._dir[slot] = (first_step, steps, row)
        self._serial[slot] = self.next_serial
        self.next_serial += 1
        self._count += 1
        if self.resident is not None:
            self.resident.append(item)
        return slot

    def positions(self):
        """(slots, serials) of the stored episodes, oldest first: the directory slot each sits in and the serial it was given
        (int64 arrays; take them under self.lock when a feeder runs)."""
        slots = (self._head + np.arange(self._count, dtype=np.int64)) % self._dir.shape[0]
        return slots, self._serial[slots].copy()

    def snapshot(self, max_count):
        """(head slot, count) of the directory now, count capped at max_count (the sampler's view; take it under self.lock)."""
        return self._head, min(self._count, int(max_count))

    def _allocate(self, fe):
        S, dev = self.capacity, self.device
        self.Ps = len(fe.players)
        self.A = fe.amask.shape[-1]
        self.obs_template = tree_map(lambda a: a[0, 0], fe.obs)                  # one observation, nested
        self.leaf_shapes = [tuple(l.shape[2:]) for l in tree_leaves(fe.obs)]
        self.leaf_sizes = [int(np.prod(s)) if len(s) else 1 for s in self.leaf_shapes]
        self.OE = int(sum(self.leaf_sizes))
        if fe.value.shape[-1] != 1:
            raise ValueError('DeviceReplay stores a scalar behaviour value per player; got %d values' % fe.value.shape[-1])
        f = dict(dtype=torch.float32, device=dev)
        self.st_obs = torch.zeros((S, self.Ps, self.OE), **f)
        self.st_prob = torch.ones((S, self.Ps), **f)
        self.st_action = torch.zeros((S, self.Ps), dtype=torch.int32, device=dev)
        self.st_amask = torch.zeros((S, self.Ps, self.A), **f)
        self.st_value = torch.zeros((S, self.Ps), **f)
        self.st_reward = torch.zeros((S, self.Ps), **f)
        self.st_return = torch.zeros((S, self.Ps), **f)
        self.st_flags = torch.zeros((S, self.Ps), dtype=torch.uint8, device=dev)
        self.st_turn = torch.zeros((S,), dtype=torch.int32, device=dev)
        self.n_outcome_rows = self.max_episodes + 64
        self.st_outcome = torch.zeros((self.n_outcome_rows, self.Ps), **f)
        self.ready = True

    @staticmethod
    def bytes_per_step(fe):
        """HBM bytes one stored step of this kind of episode takes (sizing the ring from free memory)."""
        Ps = len(fe.players)
        OE = sum(int(np.prod(l.shape[2:])) if l.ndim > 2 else 1 for l in tree_leaves(fe.obs))
        return Ps * (4 * OE + 4 * fe.amask.shape[-1] + 4 * 5 + 1) + 4

    def add(self, episode):
        """Decode one episode dict (the reference's wire format, generation.py:84-91, or the flat format of
        wire.py) and upload it."""
        from .wire import episode_to_flat
        return self.add_flat(episode_to_flat(episode))

    def add_flat(self, fe):
        return self.add_flat_many([fe])[0]

    def add_flat_many(self, fes):
        """Upload several decoded episodes (stage + commit)."""
        return self.commit(self.stage(fes)) if fes else []

    def stage(self, fes, items=None):
        """Host half of an upload: concatenate the episodes' step rows column by column into page-locked staging
        tensors.  Touches neither the ring nor the directory, so a feeder thread can do it without holding any lock
        the learner needs.  `items` (one per episode, with track=True): what commit() puts in `resident` for each."""
        if not self.ready:
            self._allocate(fes[0])
        pin = self.device.type == 'cuda'

        def host(parts, dtype):
            a = np.concatenate(parts) if len(parts) > 1 else parts[0]
            t = torch.from_numpy(np.ascontiguousarray(a, dtype=dtype))
            return t.pin_memory() if pin else t

        cols = {
            'obs': host([np.concatenate([l.reshape(fe.steps, self.Ps, -1).astype(np.float32, copy=False)
                                         for l in tree_leaves(fe.obs)], axis=2) for fe in fes], np.float32),
            'prob': host([fe.prob for fe in fes], np.float32), 'action': host([fe.action for fe in fes], np.int32),
            'amask': host([fe.amask for fe in fes], np.float32), 'value': host([fe.value[..., 0] for fe in fes], np.float32),
            'reward': host([fe.reward for fe in fes], np.float32), 'return': host([fe.ret for fe in fes], np.float32),
            'flags': host([fe.flags for fe in fes], np.uint8), 'turn': host([fe.turn for fe in fes], np.int32),
        }
        if items is not None and len(items) != len(fes):
            raise ValueError('stage: %d items for %d episodes' % (len(items), len(fes)))
        return {'steps': [int(fe.steps) for fe in fes], 'cols': cols, 'items': items,
                'outcome': host([np.stack([fe.outcome for fe in fes])], np.float32)}

    def commit(self, staged):
        """Device half of an upload: place the staged episodes in the ring (evicting what they overwrite and the
        oldest episodes beyond max_episodes) and enqueue the copies on the current stream.  Rows are placed back to
        back, so every run of episodes that does not cross the end of the ring is ONE copy per store column."""
        handles, segments = [], []        # segments: [dst_lo, src_lo, n]
        rows, appended = [], []
        with self.lock:
            src = 0
            items = staged.get('items') or [None] * len(staged['steps'])
            for n, item in zip(staged['steps'], items):
                if n > self.capacity:
                    raise ValueError('episode of %d steps exceeds the replay capacity of %d steps' % (n, self.capacity))
                if self.write + n > self.capacity:          # episodes are stored contiguously: wrap
                    # the previous lap's episodes beyond the write pointer are the oldest ones: drop them so
                    # that directory order == ring order again
                    while self._count and self._entry(0)[0] >= self.write:
                        self._popleft()
                    self.write = 0
                lo, hi = self.write, self.write + n
                # evict whatever the new rows overwrite, and the oldest episode beyond max_episodes
                while self._count and (self._count >= self.max_episodes or
                                       (self._entry(0)[0] < hi and self._entry(0)[0] + self._entry(0)[1] > lo)):
                    self._popleft()
                row = self.next_outcome_row
                self.next_outcome_row = (row + 1) % self.n_outcome_rows
                if segments and segments[-1][0] + segments[-1][2] == lo:
                    segments[-1][2] += n
                else:
                    segments.append([lo, src, n])
                rows.append(row)
                appended.append(self._append(lo, n, row, item))
                handles.append(EpisodeHandle(lo, n, row))
                self.write = hi
                src += n
            store = {'obs': self.st_obs, 'prob': self.st_prob, 'action': self.st_action, 'amask': self.st_amask,
                     'value': self.st_value, 'reward': self.st_reward, 'return': self.st_return, 'flags': self.st_flags,
                     'turn': self.st_turn}
            for dst_lo, src_lo, n in segments:
                for k, t in store.items():
                    t[dst_lo:dst_lo + n].copy_(staged['cols'][k][src_lo:src_lo + n], non_blocking=True)
            idx = torch.tensor(rows, dtype=torch.long)
            self.st_outcome.index_copy_(0, idx.to(self.device, non_blocking=True),
                                        staged['outcome'].to(self.device, non_blocking=True))
            if self.dir_dev is not None and appended:
                # a slot reused inside one upload is copied once, with its final episode
                slots = np.unique(np.asarray(appended, np.int64))
                ent = np.concatenate([self._dir[slots], self._serial[slots, None]], axis=1)
                self.dir_dev.index_copy_(0, torch.from_numpy(slots).to(self.device, non_blocking=True),
                                         torch.from_numpy(np.ascontiguousarray(ent)).to(self.device, non_blocking=True))
        return handles

    # ------------------------------------------------------------------ batches
    def batch_shapes(self, args):
        T = args['burn_in_steps'] + args['forward_steps']
        alternating = bool(args['turn_based_training'] and not args['observation'])
        P = 1 if not args['turn_based_training'] else self.Ps
        Pa = 1 if alternating else P
        return T, P, Pa, alternating

    def empty_batch(self, B, args):
        """Allocate the output tensors of one batch in the reference layout (train.py:114-124)."""
        T, P, Pa, _ = self.batch_shapes(args)
        f = dict(dtype=torch.float32, device=self.device)
        return {
            'observation': torch.empty((B, T, Pa, self.OE), **f),
            'selected_prob': torch.empty((B, T, Pa, 1), **f), 'value': torch.empty((B, T, P, 1), **f),
            'action': torch.empty((B, T, Pa, 1), dtype=torch.int64, device=self.device),
            'outcome': torch.empty((B, 1, P, 1), **f), 'reward': torch.empty((B, T, P, 1), **f),
            'return': torch.empty((B, T, P, 1), **f), 'episode_mask': torch.empty((B, T, 1, 1), **f),
            'turn_mask': torch.empty((B, T, P, 1), **f), 'observation_mask': torch.empty((B, T, P, 1), **f),
            'action_mask': torch.empty((B, T, Pa, self.A), **f), 'progress': torch.empty((B, T, 1), **f),
        }

    def sample_windows(self, B, args, rng=random):
        """B window descriptors drawn like Batcher.select_episode (train.py:291-315).

        rng = a numpy Generator: all B windows are drawn with array operations (the learner's path: the same
        recency-biased acceptance law and uniform window placement, B at a time).
        rng = the `random` module / a random.Random: the reference's own call sequence, window by window, so a seeded
        stream reproduces the reference's picks exactly (tests)."""
        solo = not args['turn_based_training']
        win = np.zeros(B, WINDOW_DTYPE)
        if isinstance(rng, np.random.Generator):
            with self.lock:
                count = min(self._count, args['maximum_episodes'])
                if count <= 0:
                    raise IndexError('the replay is empty')
                idx = np.empty(0, np.int64)
                while idx.size < B:           # accept idx with probability (idx+1)/count (train.py:294-297)
                    cand = rng.integers(0, count, size=2 * (B - idx.size) + 8)
                    idx = np.concatenate([idx, cand[rng.random(cand.size) < (cand + 1) / count]])
                ent = self._dir[(self._head + idx[:B]) % self._dir.shape[0]]
            steps = ent[:, 1]
            train_start = (rng.random(B) * (1 + np.maximum(0, steps - args['forward_steps']))).astype(np.int64)
            win['first_step'], win['total'], win['outcome_row'] = ent[:, 0], steps, ent[:, 2]
            win['train_start'] = train_start
            win['start'] = np.maximum(0, train_start - args['burn_in_steps'])
            win['end'] = np.minimum(train_start + args['forward_steps'], steps)
            if solo:
                win['player'] = rng.integers(0, self.Ps, size=B)
            return win
        with self.lock:
            for b in range(B):
                _, st, ed, tst, ent = sample_window(lambda: self._count, lambda i: (self._entry(i)[1], self._entry(i).copy()),
                                                    args, rng)
                win[b] = (ent[0], st, ed, tst, ent[1], ent[2], 0)
        if solo:
            for b in range(B):          # make_batch draws the solo player per window, in order (train.py:57-58)
                win[b]['player'] = rng.choice(range(self.Ps))
        return win

    def gather(self, windows, args, out=None, sym=None, tables=None):
        """Run the gather/pad kernel for an array of WINDOW_DTYPE descriptors; returns the batch dict
        (observation as the concatenated-leaf tensor; see split_observation).

        sym (with tables, a symmetry.SymmetryTables): the transform of each window, an int32 array of B values in [0, K)
        (checked here) or an int32 device tensor the caller has checked; the batch is then gathered through those
        transforms (hrl_gather_pad_sym).  sym=None: the plain gather (hrl_gather_pad)."""
        B = len(windows)
        T, P, Pa, alternating = self.batch_shapes(args)
        if out is None:
            out = self.empty_batch(B, args)
        if torch.is_tensor(windows):          # descriptors already staged on the device (pinned double buffering)
            wdev = windows
        else:
            wdev = torch.from_numpy(windows.view(np.uint8).reshape(B, -1)).to(self.device, non_blocking=True)
        g = HrlGatherArgs()
        g.B, g.T, g.P, g.Pa, g.A, g.Ps = B, T, P, Pa, self.A, self.Ps
        g.burn_in = args['burn_in_steps']
        g.obs_elems = self.OE
        g.turn_alternating = int(alternating)
        ptr = lambda t: C.c_void_p(t.data_ptr())
        g.windows = ptr(wdev)
        g.st_obs, g.st_prob, g.st_action, g.st_amask = ptr(self.st_obs), ptr(self.st_prob), ptr(self.st_action), ptr(self.st_amask)
        g.st_value, g.st_reward, g.st_return = ptr(self.st_value), ptr(self.st_reward), ptr(self.st_return)
        g.st_flags, g.st_turn, g.st_outcome = ptr(self.st_flags), ptr(self.st_turn), ptr(self.st_outcome)
        g.observation, g.selected_prob, g.value, g.action = (ptr(out['observation']), ptr(out['selected_prob']),
                                                             ptr(out['value']), ptr(out['action']))
        g.outcome, g.reward, g.ret = ptr(out['outcome']), ptr(out['reward']), ptr(out['return'])
        g.episode_mask, g.turn_mask, g.observation_mask = ptr(out['episode_mask']), ptr(out['turn_mask']), ptr(out['observation_mask'])
        g.action_mask, g.progress = ptr(out['action_mask']), ptr(out['progress'])
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        if sym is None:
            check(lib().hrl_gather_pad(C.byref(g), stream))
        else:
            if tables is None:
                raise ValueError('gather: sym needs the transform tables')
            if not torch.is_tensor(sym):
                sym = np.ascontiguousarray(sym, np.int32)
                if sym.shape != (B,):
                    raise ValueError('gather: sym must hold one transform per window (%d); got shape %s' % (B, sym.shape))
                tables.check_sym(sym)
                sym = torch.from_numpy(sym).to(self.device, non_blocking=True)
            elif sym.dtype != torch.int32 or sym.numel() != B or not sym.is_contiguous():
                raise ValueError('gather: sym must be a contiguous int32 tensor of %d transforms' % B)
            if tables.OE != self.OE or tables.A != self.A:
                raise ValueError('gather: the tables are for OE=%d, A=%d; the replay stores OE=%d, A=%d'
                                 % (tables.OE, tables.A, self.OE, self.A))
            t = tables.device(self.device)
            check(lib().hrl_gather_pad_sym(C.byref(g), ptr(sym), ptr(t['obs_src']), ptr(t['act_src']), ptr(t['act_dst']),
                                           tables.K, stream))
            out['_sym'] = sym       # keep the transform buffer alive until the kernel has run
        from . import ops
        ops._count()
        out['_windows'] = wdev      # keep the descriptor buffer alive until the kernel has run
        return out

    def split_observation(self, flat_obs):
        """(B,T,Pa,OE) concatenated leaves -> the env's nested observation structure."""
        pieces, off = [], 0
        for shape, size in zip(self.leaf_shapes, self.leaf_sizes):
            pieces.append(flat_obs[..., off:off + size].reshape(*flat_obs.shape[:3], *shape))
            off += size
        it = iter(pieces)
        return tree_map(lambda _: next(it), self.obs_template)
