"""Board-symmetry augmentation of replay batches (train_args['symmetry']).

If a board position is valid, so is its rotation or mirror image: the policy target moves with the board and the value does
not change.  With the key set, every window the GPU replay gathers for training goes through one transform k of a group,
drawn uniformly per window; the gather kernel applies it while it copies (hrl_gather_pad_sym, csrc/gather_kernel.cu), so
the augmentation moves no extra bytes.

A group is a set of K permutation tables over the stored layout:
  obs_src [K, OE]  element e of the transformed flat observation (the concatenated flattened leaves DeviceReplay stores)
                   is element obs_src[k][e] of the stored one;
  act_dst [K, A]   stored action a becomes act_dst[k][a];
  act_src [K, A]   its inverse: slot a of the transformed action mask is slot act_src[k][a] of the stored one.

Forms of the key:
  {'group': 'mirror' | 'flips' | 'dihedral', 'board': [H, W]}   built-in board groups (2, 4, 8 transforms; k = 0 is the
      identity).  Every observation leaf whose last two dimensions are (H, W) is transformed on them, all leading channels
      alike; other leaves pass unchanged.  Actions a < H*W are the cells (a // W, a % W) and move with the board; actions
      a >= H*W map to themselves.
  {'tables': 'package.module:function'}   function(leaf_shapes, A) -> (obs_src, act_dst), for envs whose actions are not
      board cells.
"""
import importlib
import numbers

import numpy as np

GROUPS = {'mirror': 2, 'flips': 4, 'dihedral': 8}
MAX_TRANSFORMS = 64          # HRL_SYM_MAX_TRANSFORMS of include/hrl_b200.h


def config(args):
    """train_args['symmetry'] -> the parsed spec ({'group': name, 'board': (H, W)} or {'tables': 'module:function'}), or None
    when augmentation is off (key absent, None or False).  Raises ValueError for anything the config alone shows malformed,
    and for the key together with gpu_replay: False (the augmentation happens in the GPU replay's gather)."""
    value = args.get('symmetry')
    if value is None or value is False:
        return None
    if not isinstance(value, dict):
        raise ValueError("train_args['symmetry'] must be {'group': 'mirror'|'flips'|'dihedral', 'board': [H, W]} or "
                         "{'tables': 'package.module:function'}; got %r" % (value,))
    keys = set(value)
    if keys == {'group', 'board'}:
        group, board = value['group'], value['board']
        if group not in GROUPS:
            raise ValueError("train_args['symmetry']: unknown group %r (one of %s)" % (group, ', '.join(sorted(GROUPS))))
        if (not isinstance(board, (list, tuple)) or len(board) != 2 or
                not all(isinstance(n, numbers.Integral) and not isinstance(n, bool) and n > 0 for n in board)):
            raise ValueError("train_args['symmetry']: 'board' must be two positive integers [H, W]; got %r" % (board,))
        H, W = int(board[0]), int(board[1])
        if group == 'dihedral' and H != W:
            raise ValueError("train_args['symmetry']: the 'dihedral' group needs a square board; got %dx%d" % (H, W))
        spec = {'group': group, 'board': (H, W)}
    elif keys == {'tables'}:
        resolve_tables(value['tables'])
        spec = {'tables': value['tables']}
    else:
        raise ValueError("train_args['symmetry'] takes either the keys 'group' and 'board' or the key 'tables'; got %s"
                         % sorted(keys))
    if not args.get('gpu_replay', True):
        raise ValueError("train_args['symmetry'] needs the GPU replay (gpu_replay: True): the gather kernel applies it")
    return spec


def resolve_tables(path):
    """'package.module:function' -> the function (ValueError when it cannot be imported)."""
    if not isinstance(path, str) or path.count(':') != 1 or not all(path.split(':')):
        raise ValueError("train_args['symmetry']['tables'] must be a 'package.module:function' string; got %r" % (path,))
    mod, name = path.split(':')
    try:
        fn = getattr(importlib.import_module(mod), name)
    except (ImportError, AttributeError) as e:
        raise ValueError("train_args['symmetry']: cannot load the table builder %r: %s" % (path, e))
    if not callable(fn):
        raise ValueError("train_args['symmetry']: %r is not callable" % (path,))
    return fn


def board_cell_src(group, H, W):
    """[K, H*W]: cell e of the transformed board is cell cell_src[k][e] of the stored one (k = 0 the identity).
    mirror: identity, left-right flip.  flips: identity, flip rows, flip columns, both.  dihedral: k % 4 quarter turns
    (counter-clockwise) after a left-right flip when k >= 4."""
    idx = np.arange(H * W).reshape(H, W)
    if group == 'mirror':
        grids = [idx, idx[:, ::-1]]
    elif group == 'flips':
        grids = [idx, idx[::-1, :], idx[:, ::-1], idx[::-1, ::-1]]
    elif group == 'dihedral':
        grids = [np.rot90(idx[:, ::-1] if k >= 4 else idx, k % 4) for k in range(8)]
    else:
        raise ValueError("train_args['symmetry']: unknown group %r" % (group,))
    return np.stack([g.reshape(-1) for g in grids]).astype(np.int64)


def board_tables(group, board, leaf_shapes, A):
    """Built-in tables of `group` on an (H, W) board for observation leaves of `leaf_shapes` and A actions."""
    H, W = board
    if group == 'dihedral' and H != W:
        raise ValueError("train_args['symmetry']: the 'dihedral' group needs a square board; got %dx%d" % (H, W))
    if A < H * W:
        raise ValueError("train_args['symmetry']: %d actions cannot hold the %dx%d board's %d cells" % (A, H, W, H * W))
    cells = board_cell_src(group, H, W)
    K = cells.shape[0]
    pieces, off, matched = [], 0, False
    for shape in leaf_shapes:
        size = int(np.prod(shape)) if len(shape) else 1
        if len(shape) >= 2 and tuple(shape[-2:]) == (H, W):
            lead = size // (H * W)
            base = off + np.arange(lead)[:, None] * (H * W)                     # [lead, 1]
            pieces.append((base[None] + cells[:, None, :]).reshape(K, size))
            matched = True
        else:
            pieces.append(np.broadcast_to(off + np.arange(size), (K, size)))
        off += size
    if not matched:
        raise ValueError("train_args['symmetry']: no observation leaf ends in the board shape %dx%d (leaves: %s)"
                         % (H, W, [tuple(s) for s in leaf_shapes]))
    obs_src = np.concatenate(pieces, axis=1) if pieces else np.zeros((K, 0), np.int64)
    act_dst = np.tile(np.arange(A), (K, 1))
    act_dst[:, :H * W] = np.argsort(cells, axis=1)           # stored cell c lands where cell_src points back at it
    return obs_src, act_dst


def inverse(perm):
    """Row-wise inverse of a [K, n] stack of permutations."""
    perm = np.asarray(perm)
    inv = np.empty_like(perm)
    np.put_along_axis(inv, perm, np.broadcast_to(np.arange(perm.shape[1]), perm.shape), axis=1)
    return inv


def _check_perms(name, a, K, n):
    if a.shape != (K, n):
        raise ValueError("train_args['symmetry']: %s has shape %s, expected %s" % (name, a.shape, (K, n)))
    if n and not np.array_equal(np.sort(a, axis=1), np.broadcast_to(np.arange(n), (K, n))):
        bad = [k for k in range(K) if not np.array_equal(np.sort(a[k]), np.arange(n))]
        raise ValueError("train_args['symmetry']: row(s) %s of %s are not permutations of [0, %d)" % (bad[:8], name, n))


class SymmetryTables:
    """The K transforms of one group for one kind of episode: obs_src [K, OE], act_dst and act_src [K, A] (int32, host),
    and their device copies, uploaded once (device())."""

    def __init__(self, obs_src, act_dst, OE, A):
        obs_src, act_dst = np.asarray(obs_src), np.asarray(act_dst)
        if obs_src.ndim != 2 or act_dst.ndim != 2:
            raise ValueError("train_args['symmetry']: the tables must be 2-D [K, OE] and [K, A]; got shapes %s and %s"
                             % (obs_src.shape, act_dst.shape))
        K = act_dst.shape[0]
        if not 1 <= K <= MAX_TRANSFORMS:
            raise ValueError("train_args['symmetry']: K=%d transforms, outside [1, %d]" % (K, MAX_TRANSFORMS))
        if not (np.issubdtype(obs_src.dtype, np.integer) and np.issubdtype(act_dst.dtype, np.integer)):
            raise ValueError("train_args['symmetry']: the tables must be integer arrays")
        _check_perms('obs_src', obs_src, K, OE)
        _check_perms('act_dst', act_dst, K, A)
        self.K, self.OE, self.A = K, OE, A
        self.obs_src = np.ascontiguousarray(obs_src, np.int32)
        self.act_dst = np.ascontiguousarray(act_dst, np.int32)
        self.act_src = np.ascontiguousarray(inverse(self.act_dst), np.int32)
        self._dev = {}

    def device(self, device):
        """{'obs_src', 'act_src', 'act_dst'} as int32 device tensors (uploaded on the first call per device)."""
        import torch
        key = str(device)
        if key not in self._dev:
            self._dev[key] = {k: torch.from_numpy(getattr(self, k)).to(device)
                              for k in ('obs_src', 'act_src', 'act_dst')}
        return self._dev[key]

    def check_sym(self, sym):
        """Raise ValueError unless every transform index of `sym` lies in [0, K) (the kernel trusts them)."""
        sym = np.asarray(sym)
        if sym.size and (sym.min() < 0 or sym.max() >= self.K):
            raise ValueError('symmetry: transform indices must lie in [0, %d); got [%d, %d]' % (self.K, sym.min(), sym.max()))


def build_tables(spec, leaf_shapes, A):
    """The SymmetryTables of a parsed spec (config()) for observation leaves of `leaf_shapes` (per-step shapes, the order
    DeviceReplay concatenates them in) and A actions.  ValueError when they do not fit."""
    leaf_shapes = [tuple(int(n) for n in s) for s in leaf_shapes]
    OE = sum(int(np.prod(s)) if len(s) else 1 for s in leaf_shapes)
    if 'group' in spec:
        obs_src, act_dst = board_tables(spec['group'], spec['board'], leaf_shapes, A)
    else:
        out = resolve_tables(spec['tables'])(leaf_shapes, A)
        if not isinstance(out, (tuple, list)) or len(out) != 2:
            raise ValueError("train_args['symmetry']: %s must return (obs_src, act_dst)" % spec['tables'])
        obs_src, act_dst = out
        if np.asarray(obs_src).shape[:1] != np.asarray(act_dst).shape[:1]:
            raise ValueError("train_args['symmetry']: obs_src and act_dst disagree on K: %s vs %s"
                             % (np.asarray(obs_src).shape, np.asarray(act_dst).shape))
    return SymmetryTables(obs_src, act_dst, OE, A)


def sampler_rng(seed):
    """The generator the transforms of a batch sampler seeded with `seed` are drawn from: its own stream, so the window
    descriptors drawn for a seed are the same with augmentation on and off."""
    return np.random.default_rng(seed + 2)


def draw(rng, B, K):
    """Transform index of each of B windows, uniform in [0, K) (int32)."""
    return rng.integers(0, K, size=B, dtype=np.int32)


def apply_tables(batch, k, tables):
    """Host reference of hrl_gather_pad_sym: transform an un-augmented gather output (the dict DeviceReplay.gather returns,
    flat observation (B, T, Pa, OE)) window by window with transform k[b].  Returns a new dict of numpy arrays; observation
    and action_mask are permuted, live actions (episode_mask 1) remapped, every other tensor copied as it is."""
    def host(t):
        return t.detach().cpu().numpy() if hasattr(t, 'detach') else np.asarray(t)

    k = np.asarray(k, np.int64)
    tables.check_sym(k)
    out = {key: host(v).copy() for key, v in batch.items() if not key.startswith('_')}
    obs = out['observation']
    for b in range(obs.shape[0]):
        obs[b] = obs[b][..., tables.obs_src[k[b]]]
        out['action_mask'][b] = out['action_mask'][b][..., tables.act_src[k[b]]]
        act = out['action'][b]                                   # (T, Pa, 1)
        live = (out['episode_mask'][b, :, 0, 0] > 0)[:, None, None] & (act >= 0) & (act < tables.A)
        act[...] = np.where(live, tables.act_dst[k[b]][np.clip(act, 0, tables.A - 1)], act)
    return out
