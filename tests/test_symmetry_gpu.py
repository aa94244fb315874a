"""Board-symmetry augmentation on the GPU: hrl_gather_pad_sym against the plain gather and the host reference transform, the
transforms' distribution, a learner step fed an augmented gather, and the Trainer with the key on."""
import copy
import os
import pickle
import random
import threading

import numpy as np
import pytest
import torch

from conftest import GOLDEN

pytestmark = pytest.mark.gpu

with open(os.path.join(GOLDEN, 'batch_cases.pkl'), 'rb') as f:
    BATCH_CASES = pickle.load(f)

# the group each golden setup is augmented with: TicTacToe boards turn and mirror; Geister mirrors its 6x6 planes (its
# 18-wide scalar leaf and its actions >= 36 stay fixed)
SPECS = {'tictactoe': {'group': 'dihedral', 'board': (3, 3)}, 'tictactoe_obs': {'group': 'dihedral', 'board': (3, 3)},
         'parallel_ttt': {'group': 'flips', 'board': (3, 3)}, 'geister_burnin': {'group': 'mirror', 'board': (6, 6)}}


def windows_for(case, replay, handles):
    """The golden batch's window descriptors (as tests/test_replay_gpu.py draws them)."""
    from handyrl_b200.replay import WINDOW_DTYPE
    eps = case['episodes']
    win = np.zeros(len(case['selected']), WINDOW_DTYPE)
    solo = not case['args']['turn_based_training']
    random.seed(9)
    for b, sel in enumerate(case['selected']):
        cs = case['args']['compress_steps']
        idx = next(i for i, ep in enumerate(eps)
                   if ep['steps'] == sel['total'] and ep['moment'][sel['base'] // cs:sel['base'] // cs + len(sel['moment'])] == sel['moment'])
        h = handles[idx]
        player = random.choice(range(replay.Ps)) if solo else 0
        win[b] = (h.first_step, sel['start'], sel['end'], sel['train_start'], sel['total'], h.outcome_row, player)
    return win


def _golden(name):
    from handyrl_b200.replay import DeviceReplay
    from handyrl_b200 import symmetry
    case = BATCH_CASES[name]
    replay = DeviceReplay(capacity_steps=4096, max_episodes=64)
    handles = [replay.add(ep) for ep in case['episodes']]
    tables = symmetry.build_tables(SPECS[name], replay.leaf_shapes, replay.A)
    return case, replay, windows_for(case, replay, handles), tables


def _host(batch):
    return {k: v.cpu().numpy() for k, v in batch.items() if not k.startswith('_')}


def _assert_batches_equal(got, want, what):
    assert sorted(got) == sorted(want)
    for k in want:
        assert got[k].shape == want[k].shape and got[k].dtype == want[k].dtype, (what, k)
        assert np.array_equal(got[k].view(np.uint8), want[k].view(np.uint8)), (what, k)       # bit for bit


def _poisoned(replay, B, args):
    """Output buffers full of NaN / -1: every byte the kernel leaves unwritten would show."""
    out = replay.empty_batch(B, args)
    for v in out.values():
        v.fill_(-1 if not v.is_floating_point() else float('nan'))
    return out


@pytest.mark.parametrize('name', sorted(BATCH_CASES))
def test_identity_transform_equals_the_plain_gather(name):
    case, replay, win, tables = _golden(name)
    B = len(win)
    plain = _host(replay.gather(win, case['args'], out=_poisoned(replay, B, case['args'])))
    sym = replay.gather(win, case['args'], out=_poisoned(replay, B, case['args']), sym=np.zeros(B, np.int32), tables=tables)
    torch.cuda.synchronize()
    _assert_batches_equal(_host(sym), plain, name)


@pytest.mark.parametrize('name', sorted(BATCH_CASES))
def test_random_transforms_equal_the_host_reference(name):
    from handyrl_b200 import symmetry
    case, replay, win, tables = _golden(name)
    B = len(win)
    plain = replay.gather(win, case['args'])
    torch.cuda.synchronize()
    rng = np.random.default_rng(17)
    for trial in range(6):
        k = rng.integers(0, tables.K, size=B).astype(np.int32)
        k[trial % B] = tables.K - 1
        got = replay.gather(win, case['args'], out=_poisoned(replay, B, case['args']), sym=k, tables=tables)
        torch.cuda.synchronize()
        _assert_batches_equal(_host(got), symmetry.apply_tables(plain, k, tables), (name, trial))


def _fake_episode(steps, Ps, A, obs_shape, rng):
    from handyrl_b200.batch import FlatEpisode
    fe = FlatEpisode()
    fe.steps, fe.players = steps, list(range(Ps))
    fe.obs = rng.standard_normal((steps, Ps) + obs_shape).astype(np.float32)
    fe.prob = rng.random((steps, Ps), dtype=np.float32)
    fe.action = rng.integers(0, A, (steps, Ps)).astype(np.int32)
    fe.amask = np.where(rng.random((steps, Ps, A)) < 0.3, 1e32, 0).astype(np.float32)
    fe.value = rng.random((steps, Ps, 1), dtype=np.float32)
    fe.reward = rng.standard_normal((steps, Ps)).astype(np.float32)
    fe.ret = rng.standard_normal((steps, Ps)).astype(np.float32)
    fe.flags = np.full((steps, Ps), 3, np.uint8)
    fe.turn = (np.arange(steps) % Ps).astype(np.int32)
    fe.outcome = np.array([1, -1][:Ps], np.float32)
    return fe


def half_identity_tables(leaf_shapes, A):
    """Custom tables whose transforms 1 and 3 are the identity and 2 the mirror of an 8x8 board (tests the identity
    row path at k != 0)."""
    from handyrl_b200 import symmetry
    obs_src, act_dst = symmetry.board_tables('mirror', (8, 8), leaf_shapes, A)
    return obs_src[[1, 0, 1, 0]], act_dst[[1, 0, 1, 0]]


@pytest.mark.parametrize('spec', [{'group': 'dihedral', 'board': (8, 8)}, {'tables': 'test_symmetry_gpu:half_identity_tables'}],
                         ids=['dihedral', 'custom'])
@pytest.mark.parametrize('alternating', [True, False])
def test_vectorised_rows_equal_the_host_reference(spec, alternating):
    """Rows whose width is a multiple of 4 (16-byte copies): an 8x8 board of 4 planes, 68 actions."""
    from handyrl_b200 import symmetry
    from handyrl_b200.replay import DeviceReplay
    rng = np.random.default_rng(3)
    replay = DeviceReplay(capacity_steps=8192, max_episodes=128)
    for _ in range(40):
        replay.add_flat(_fake_episode(int(rng.integers(4, 40)), 2, 68, (4, 8, 8), rng))
    tables = symmetry.build_tables(spec, replay.leaf_shapes, replay.A)
    assert replay.OE % 4 == 0 and replay.A % 4 == 0
    args = {'turn_based_training': True, 'observation': not alternating, 'burn_in_steps': 2, 'forward_steps': 16,
            'maximum_episodes': 128}
    B = 96
    win = replay.sample_windows(B, args, np.random.default_rng(5))
    plain = replay.gather(win, args)
    k = rng.integers(0, tables.K, size=B).astype(np.int32)
    got = replay.gather(win, args, out=_poisoned(replay, B, args), sym=k, tables=tables)
    torch.cuda.synchronize()
    _assert_batches_equal(_host(got), symmetry.apply_tables(plain, k, tables), 'vectorised')
    em = plain['episode_mask'].cpu().numpy()
    assert (em == 0).any() and (em == 1).any()           # pad cells before and after the windows


def test_bad_transform_indices_are_refused_on_the_host():
    from handyrl_b200 import _capi
    case, replay, win, tables = _golden('tictactoe')
    B = len(win)
    for bad in (np.full(B, tables.K, np.int32), np.full(B, -1, np.int32), np.zeros(B + 1, np.int32)):
        with pytest.raises(ValueError):
            replay.gather(win, case['args'], sym=bad, tables=tables)
    with pytest.raises(_capi.HrlError):   # the C entry point checks its pointers and K before it launches anything
        _capi.check(_capi.lib().hrl_gather_pad_sym(None, None, None, None, None, 1, None))


def test_each_transform_is_drawn_uniformly():
    """The transforms GpuBatcher draws (train.sample_batch) over 65536 windows: every k within 5 sigma of N / K."""
    from handyrl_b200 import symmetry
    from handyrl_b200.replay import DeviceReplay
    from handyrl_b200.synthetic import tictactoe_episodes
    from handyrl_b200.train import sample_batch
    replay = DeviceReplay(4096, 64)
    for ep in tictactoe_episodes(20, seed=2):
        replay.add(ep)
    args = dict(BATCH_CASES['tictactoe']['args'], maximum_episodes=64)
    tables = symmetry.build_tables({'group': 'dihedral', 'board': (3, 3)}, replay.leaf_shapes, replay.A)
    N, K = 65536, tables.K
    win, k = sample_batch(replay, N, args, np.random.default_rng(4), symmetry.sampler_rng(4), K)
    counts = np.bincount(k, minlength=K)
    p = 1.0 / K
    assert counts.sum() == N and len(counts) == K
    assert np.all(np.abs(counts - N * p) <= 5 * np.sqrt(N * p * (1 - p))), counts
    out = replay.gather(win, args, sym=k, tables=tables)     # and the kernel takes a batch of that size
    torch.cuda.synchronize()
    assert out['action'].shape[0] == N


# ---------------------------------------------------------------------------------------------------------------- learner
def _trainer_args(**extra):
    case = BATCH_CASES['tictactoe']
    return dict(case['args'], batch_size=8, minimum_episodes=4, num_batchers=1, **{'lambda': 0.7},
                entropy_regularization=0.1, entropy_regularization_decay=0.1, policy_target='UPGO', value_target='VTRACE',
                gpu_replay=True, num_gpus=1, **extra)


def _wait(cond, n=1000):
    for _ in range(n):
        if cond():
            return True
        threading.Event().wait(0.01)
    return cond()


def _to_step_batch(flat, replay):
    """A gather output (numpy, flat observation) -> the host batch a LearnerStep packs (the env's observation shape)."""
    b = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in flat.items()}
    b['observation'] = b['observation'].reshape(*b['observation'].shape[:3], *replay.leaf_shapes[0])
    return b


@pytest.mark.parametrize('use_graph', [False, True], ids=['eager', 'graph'])
def test_learner_step_on_an_augmented_gather_equals_the_host_transformed_batch(use_graph):
    from handyrl_b200 import symmetry
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.synthetic import tictactoe_episodes
    from handyrl_b200.train import EpisodeDeque, GpuBatcher, LearnerStep
    from test_validation_gpu import _cpu_losses
    args = _trainer_args(symmetry={'group': 'dihedral', 'board': [3, 3]}, seed=5)
    torch.manual_seed(0)
    make = lambda: copy.deepcopy(net0)
    net0 = tictactoe_net()
    q = EpisodeDeque()
    q.extend(tictactoe_episodes(40, seed=13))
    gb = GpuBatcher(args, q, torch.device('cuda', 0), seed=77)
    gb.run()
    assert _wait(lambda: gb.fed >= 40)
    gb.stop()
    torch.cuda.synchronize()
    replay, B = gb.replay, args['batch_size']
    # the draws GpuBatcher.fill will make, reproduced from its seed
    win, k = replay.sample_windows(B, args, np.random.default_rng(77)), symmetry.draw(symmetry.sampler_rng(77), B, 8)
    assert len(set(k.tolist())) > 1
    host = _to_step_batch(symmetry.apply_tables(replay.gather(win, args), k, gb.sym_tables), replay)
    torch.cuda.synchronize()
    results = []
    for path in ('gather', 'host'):
        st = LearnerStep(make(), args, host, lr=1e-3, use_graph=use_graph, cudnn_benchmark=False)
        assert st.engine is not None                     # the fused tower
        st.warm_up()
        if path == 'gather':
            gb.fill(st)
            st.step_in_place()
        else:
            st.step(st.new_packed().fill(host))
        st.stream.synchronize()
        results.append((st.read_losses(), st.cpu_state_dict()))
        st.close()
    (la, wa), (lb, wb) = results
    assert la == lb, (la, lb)
    for key in wa:
        assert torch.equal(wa[key], wb[key]), key
    want, dcnt = _cpu_losses(make, net0.state_dict(), host, args)
    assert la['dcnt'] == dcnt > 0
    for key, v in want.items():
        assert abs(la[key] - v) <= 2e-4 * abs(v) + 1e-4, (key, la[key], v)   # test_step_gpu.py's tolerance


# ---------------------------------------------------------------------------------------------------------------- trainer
def _line_kinds(text):
    return [l.split(' = ')[0] if ' = ' in l else l for l in text.splitlines()]


def _run_trainer(extra, episodes, spy, capsys):
    """Two epochs of a Trainer once every episode is stored and the held-out ring holds one; returns it (stopped) and the
    lines those epochs printed."""
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.train import Trainer
    torch.manual_seed(0)
    tr = Trainer(_trainer_args(validation_rate=0.7, seed=3, **extra), tictactoe_net())
    tr.episodes.extend(episodes)
    th = threading.Thread(target=tr.run, daemon=True)
    th.start()
    try:
        tr.update()
        assert _wait(lambda: tr.gpu_batcher.fed >= len(episodes) and tr.gpu_batcher.validation_ready())
        tr.update()
        spy.clear()
        capsys.readouterr()
        out = [tr.update()[1] for _ in range(2)]
        lines = capsys.readouterr().out
        assert out[1] > out[0]
    finally:
        tr.stop()
        th.join(timeout=10)
    return tr, lines


def test_trainer_with_the_key_prints_the_same_lines_and_validates_on_real_data(tmp_path, monkeypatch, capsys):
    from handyrl_b200.replay import DeviceReplay
    from handyrl_b200.synthetic import tictactoe_episodes
    monkeypatch.chdir(tmp_path)
    calls = []
    real_gather = DeviceReplay.gather

    def spy(self, windows, args, out=None, sym=None, tables=None):
        calls.append((self, sym is not None))
        return real_gather(self, windows, args, out=out, sym=sym, tables=tables)

    monkeypatch.setattr(DeviceReplay, 'gather', spy)
    episodes = tictactoe_episodes(60, seed=21)
    kinds = {}
    for on in (False, True):
        extra = {'symmetry': {'group': 'dihedral', 'board': [3, 3]}} if on else {}
        tr, lines = _run_trainer(extra, episodes, calls, capsys)
        kinds[on] = _line_kinds(lines)
        gb = tr.gpu_batcher
        train_calls = [s for r, s in calls if r is gb.replay]
        val_calls = [s for r, s in calls if r is gb.val_replay]
        assert train_calls and val_calls
        assert all(s == on for s in train_calls) and not any(val_calls)
    assert kinds[True] == kinds[False], kinds
    assert 'validation' in kinds[True] and 'loss' in kinds[True]
    # a held-out batch is the plain gather of its descriptors
    st = tr.stepper
    state = copy.deepcopy(gb.val_rng.bit_generator.state)
    gb.fill_validation(st)
    st.stream.synchronize()
    rng = np.random.default_rng()
    rng.bit_generator.state = state
    win = gb.val_replay.sample_windows(st.dims[0], tr.args, rng)
    want = _host(real_gather(gb.val_replay, win, tr.args))
    torch.cuda.synchronize()
    got = {k: v.cpu().numpy() for k, v in st.dev.items()}
    got['observation'] = got['observation'].reshape(want['observation'].shape)
    for key in got:
        assert np.array_equal(got[key], want[key]), key
