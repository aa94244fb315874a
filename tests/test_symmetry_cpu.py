"""Board-symmetry augmentation without a GPU: the built-in groups' tables, how the key is read and refused, custom tables, the
host reference transform, the binding, and the sampler's draws."""
import os
import re

import numpy as np
import pytest

from handyrl_b200 import symmetry

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TTT_LEAVES, TTT_A = [(3, 3, 3)], 9
GEISTER_LEAVES, GEISTER_A = [(18,), (7, 6, 6)], 214
BOARDS = {'mirror': [(3, 3), (6, 6), (4, 7)], 'flips': [(3, 3), (4, 7), (2, 5)], 'dihedral': [(3, 3), (6, 6), (19, 19)]}


def direction_tables(leaf_shapes, A):
    """Custom tables for the tests: a 4-direction action set on a 7x11 torus board whose flips exchange the
    directions (0 north, 1 south, 2 west, 3 east)."""
    spec = symmetry.board_tables('flips', (7, 11), leaf_shapes, 77)
    obs_src = spec[0]
    act_dst = np.array([[0, 1, 2, 3], [1, 0, 2, 3], [0, 1, 3, 2], [1, 0, 3, 2]])
    assert A == 4
    return obs_src, act_dst


def not_a_permutation(leaf_shapes, A):
    OE = sum(int(np.prod(s)) for s in leaf_shapes)
    return np.zeros((2, OE), np.int64), np.tile(np.arange(A), (2, 1))


def too_many(leaf_shapes, A):
    OE = sum(int(np.prod(s)) for s in leaf_shapes)
    return np.tile(np.arange(OE), (65, 1)), np.tile(np.arange(A), (65, 1))


def _is_perm(row):
    return np.array_equal(np.sort(row), np.arange(len(row)))


@pytest.mark.parametrize('group', sorted(BOARDS))
def test_builtin_tables_are_groups_of_permutations(group):
    for H, W in BOARDS[group]:
        leaves = [(2, H, W), (5,)]
        A = H * W + 1
        t = symmetry.build_tables({'group': group, 'board': (H, W)}, leaves, A)
        assert t.K == symmetry.GROUPS[group]
        assert t.obs_src.shape == (t.K, 2 * H * W + 5) and t.act_dst.shape == (t.K, A) and t.act_src.shape == (t.K, A)
        assert t.obs_src.dtype == np.int32 and t.act_dst.dtype == np.int32 and t.act_src.dtype == np.int32
        for k in range(t.K):
            assert _is_perm(t.obs_src[k]) and _is_perm(t.act_dst[k]) and _is_perm(t.act_src[k])
            assert np.array_equal(t.act_src[k][t.act_dst[k]], np.arange(A))
        assert np.array_equal(t.obs_src[0], np.arange(t.OE)) and np.array_equal(t.act_dst[0], np.arange(A))
        rows = {tuple(r) for r in t.obs_src}
        acts = {tuple(r) for r in t.act_dst}
        if H * W > 1:
            assert len(rows) == t.K and len(acts) == t.K        # K distinct transforms
        for i in range(t.K):
            for j in range(t.K):
                # applying j then i: new[e] = old[src_j[src_i[e]]]; stored action a goes to dst_i[dst_j[a]]
                assert tuple(t.obs_src[j][t.obs_src[i]]) in rows
                assert tuple(t.act_dst[i][t.act_dst[j]]) in acts


@pytest.mark.parametrize('group', sorted(BOARDS))
def test_observation_and_action_maps_agree_on_tictactoe(group):
    t = symmetry.build_tables({'group': group, 'board': (3, 3)}, TTT_LEAVES, TTT_A)
    for k in range(t.K):
        for c in range(9):
            for ch in range(3):
                board = np.zeros((3, 3, 3), np.float32)
                board[ch].flat[c] = 1.0
                new = board.reshape(-1)[t.obs_src[k]].reshape(3, 3, 3)
                assert new[ch].flat[t.act_dst[k][c]] == 1.0 and new.sum() == 1.0
    # the quarter turn and the mirror of the dihedral group are what their names say
    if group == 'dihedral':
        b = np.arange(9).reshape(3, 3)
        x = np.tile(b, (3, 1, 1)).reshape(-1)
        assert np.array_equal(x[t.obs_src[1]].reshape(3, 3, 3)[0], np.rot90(b))
        assert np.array_equal(x[t.obs_src[4]].reshape(3, 3, 3)[0], b[:, ::-1])


def test_non_board_leaves_and_extra_actions_are_fixed():
    t = symmetry.build_tables({'group': 'mirror', 'board': (6, 6)}, GEISTER_LEAVES, GEISTER_A)
    assert t.K == 2
    for k in range(t.K):
        assert np.array_equal(t.obs_src[k][:18], np.arange(18))              # Geister's scalar leaf
        assert np.array_equal(t.act_dst[k][36:], np.arange(36, GEISTER_A))
        assert not k or not np.array_equal(t.obs_src[k][18:], np.arange(18, 18 + 7 * 36))
    go = symmetry.build_tables({'group': 'dihedral', 'board': (19, 19)}, [(17, 19, 19)], 362)
    assert go.K == 8 and (go.act_dst[:, 361] == 361).all()                   # pass
    # one channel row, reshaped: every channel moves alike
    src = go.obs_src[3].reshape(17, 361)
    assert np.array_equal(src - src[:, :1], np.broadcast_to(src[0] - src[0, 0], src.shape))


def test_key_off_and_forms():
    assert symmetry.config({}) is None
    assert symmetry.config({'symmetry': None}) is None
    assert symmetry.config({'symmetry': False}) is None
    assert symmetry.config({'symmetry': {'group': 'dihedral', 'board': [3, 3]}}) == {'group': 'dihedral', 'board': (3, 3)}
    assert symmetry.config({'symmetry': {'group': 'flips', 'board': (4, 7)}, 'gpu_replay': True})['board'] == (4, 7)
    spec = symmetry.config({'symmetry': {'tables': 'test_symmetry_cpu:direction_tables'}})
    assert spec == {'tables': 'test_symmetry_cpu:direction_tables'}


@pytest.mark.parametrize('value', [
    True, 'dihedral', {'group': 'rotations', 'board': [3, 3]}, {'group': 'dihedral', 'board': [3, 4]},
    {'group': 'mirror'}, {'board': [3, 3]}, {'group': 'mirror', 'board': [3]}, {'group': 'mirror', 'board': [0, 3]},
    {'group': 'mirror', 'board': [3.0, 3]}, {'group': 'mirror', 'board': [3, 3], 'tables': 'a:b'},
    {'tables': 'no_such_module_anywhere:fn'}, {'tables': 'test_symmetry_cpu:no_such_function'}, {'tables': 'nocolon'},
    {'tables': 3}])
def test_malformed_configs_are_refused(value):
    with pytest.raises(ValueError):
        symmetry.config({'symmetry': value})


def test_shape_errors_are_refused_when_the_leaves_are_known():
    with pytest.raises(ValueError):      # no leaf ends in the board
        symmetry.build_tables({'group': 'mirror', 'board': (4, 4)}, TTT_LEAVES, 16)
    with pytest.raises(ValueError):      # fewer actions than cells
        symmetry.build_tables({'group': 'mirror', 'board': (6, 6)}, [(7, 6, 6)], 30)
    with pytest.raises(ValueError):      # a table row that is not a permutation
        symmetry.build_tables({'tables': 'test_symmetry_cpu:not_a_permutation'}, TTT_LEAVES, TTT_A)
    with pytest.raises(ValueError):      # K out of range
        symmetry.build_tables({'tables': 'test_symmetry_cpu:too_many'}, TTT_LEAVES, TTT_A)
    with pytest.raises(ValueError):      # wrong width
        symmetry.SymmetryTables(np.tile(np.arange(5), (2, 1)), np.tile(np.arange(9), (2, 1)), 27, 9)
    with pytest.raises(ValueError):      # K = 0
        symmetry.SymmetryTables(np.zeros((0, 27), np.int64), np.zeros((0, 9), np.int64), 27, 9)


def test_custom_tables_load_from_a_module_function():
    t = symmetry.build_tables({'tables': 'test_symmetry_cpu:direction_tables'}, [(3, 7, 11)], 4)
    assert t.K == 4 and t.OE == 3 * 77 and t.A == 4
    assert np.array_equal(t.act_dst[1], [1, 0, 2, 3]) and np.array_equal(t.act_src[3], [1, 0, 3, 2])


def test_trainer_and_learner_step_refuse_a_bad_key():
    """Both constructors check the key before touching a device, and the key needs the GPU replay."""
    import torch
    from handyrl_b200.train import LearnerStep, Trainer
    from handyrl_b200.nets import tictactoe_net
    args = {'batch_size': 4, 'forward_steps': 4, 'gpu_replay': True}
    for bad in ({'symmetry': {'group': 'dihedral', 'board': [3, 4]}}, {'symmetry': {'group': 'spin', 'board': [3, 3]}},
                {'symmetry': {'group': 'mirror', 'board': [3, 3]}, 'gpu_replay': False}):
        with pytest.raises(ValueError):
            Trainer(dict(args, **bad), tictactoe_net())
        with pytest.raises(ValueError):
            LearnerStep(torch.nn.Linear(2, 2), dict(args, **bad), None, lr=1e-3)


def test_apply_tables_transforms_live_windows_only():
    t = symmetry.build_tables({'group': 'dihedral', 'board': (3, 3)}, TTT_LEAVES, TTT_A)
    rng = np.random.default_rng(0)
    B, T, Pa = 5, 4, 2
    batch = {'observation': rng.standard_normal((B, T, Pa, 27)).astype(np.float32),
             'action_mask': rng.standard_normal((B, T, Pa, 9)).astype(np.float32),
             'action': rng.integers(0, 9, (B, T, Pa, 1)).astype(np.int64),
             'episode_mask': np.ones((B, T, 1, 1), np.float32), 'progress': rng.random((B, T, 1)).astype(np.float32)}
    batch['episode_mask'][1, 2:] = 0
    k = np.array([0, 1, 4, 7, 3], np.int32)
    out = symmetry.apply_tables(batch, k, t)
    assert np.array_equal(out['observation'][0], batch['observation'][0]) and np.array_equal(out['action'][0], batch['action'][0])
    for b in range(B):
        assert np.array_equal(out['observation'][b], batch['observation'][b][..., t.obs_src[k[b]]])
        assert np.array_equal(out['action_mask'][b], batch['action_mask'][b][..., t.act_src[k[b]]])
    assert np.array_equal(out['action'][1, 2:], batch['action'][1, 2:])                 # pad cells keep their action
    assert np.array_equal(out['action'][1, :2], t.act_dst[1][batch['action'][1, :2]])
    assert np.array_equal(out['progress'], batch['progress'])
    with pytest.raises(ValueError):
        symmetry.apply_tables(batch, np.array([0, 1, 2, 3, 8]), t)


def test_binding_mirrors_the_header():
    from handyrl_b200 import _capi
    header = open(os.path.join(ROOT, 'include', 'hrl_b200.h')).read()
    assert 'hrl_gather_pad_sym' in _capi.SYMBOLS
    assert re.search(r'#define HRL_SYM_MAX_TRANSFORMS 64\b', header) and symmetry.MAX_TRANSFORMS == 64
    assert re.search(r'int hrl_gather_pad_sym\(const HrlGatherArgs \*args,', header)
    assert _capi.HRL_ABI_VERSION == 3 and '#define HRL_ABI_VERSION 3' in header


def test_sampler_draws_the_same_windows_with_the_key_on():
    from handyrl_b200.replay import DeviceReplay
    from handyrl_b200.synthetic import tictactoe_episodes
    from handyrl_b200.train import sample_batch
    replay = DeviceReplay(4096, 64, device='cpu')
    for ep in tictactoe_episodes(20, seed=1):
        replay.add(ep)
    args = {'turn_based_training': True, 'observation': False, 'burn_in_steps': 0, 'forward_steps': 4, 'maximum_episodes': 64}
    seed = 123
    K = 8
    off = [sample_batch(replay, 64, args, np.random.default_rng(seed))[0] for _ in range(1)]
    rng, srng = np.random.default_rng(seed), symmetry.sampler_rng(seed)
    win, ks = sample_batch(replay, 64, args, rng, srng, K)
    assert np.array_equal(win, off[0])
    assert ks.dtype == np.int32 and ks.shape == (64,) and ks.min() >= 0 and ks.max() < K
    win2, ks2 = sample_batch(replay, 64, args, np.random.default_rng(seed), symmetry.sampler_rng(seed), K)
    assert np.array_equal(win2, win) and np.array_equal(ks2, ks)
    assert len(set(ks.tolist())) > 1
    # later batches too: the two streams never interleave
    a = [sample_batch(replay, 16, args, rng)[0] for _ in range(3)]
    rng_b = np.random.default_rng(seed)
    sample_batch(replay, 64, args, rng_b)
    b = [sample_batch(replay, 16, args, rng_b, symmetry.sampler_rng(seed + 1), K)[0] for _ in range(3)]
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
