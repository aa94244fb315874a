"""Prioritised replay on the GPU: the window weight of the fused loss (bit-identical at 1, exact scaling otherwise), the device
sampler (distribution, weights, determinism, live windows, new episodes), the priority update, the learner step and the
Trainer with the key on."""
import os
import pickle
import re

import numpy as np
import pytest
import torch
from scipy import stats

from conftest import GOLDEN, case_args, load_cases
from test_diagnostics_gpu import VARIANTS, assert_same_outputs, split, to_dev
from test_nonfinite_guard_gpu import _poisoned, _setup, deterministic_cudnn  # noqa: F401  (a fixture)

pytestmark = pytest.mark.gpu

LOSS_CASES = load_cases('loss_cases.npz')
SPEC = {'alpha': 0.6, 'beta': 0.4, 'epsilon': 0.01}


def _loss(outs, batch, args, tuning=None, weight=None, diagnostics=False):
    from handyrl_b200 import ops
    res = ops.loss_fwd_bwd(outs, batch, args, tuning=tuning, window_weight=weight, diagnostics=diagnostics)
    torch.cuda.synchronize()
    return res


# ---------------------------------------------------------------------------------------------------------------- K1 weights
@pytest.mark.parametrize('recurrence', ['serial', 'scan'])
@pytest.mark.parametrize('variant', VARIANTS)
@pytest.mark.parametrize('name', sorted(LOSS_CASES))
def test_null_and_unit_weights_are_bit_identical(name, variant, recurrence):
    case = LOSS_CASES[name]
    batch, outs = split(case)
    args = case_args(case['meta'])
    db, do = to_dev(batch), to_dev(outs)
    tuning = {'variant': variant, 'recurrence': recurrence}
    B = do['policy'].shape[0]
    ones = torch.ones(B, device='cuda')
    assert_same_outputs(_loss(do, db, args, tuning), _loss(do, db, args, tuning, weight=ones))
    plain, unit = _loss(do, db, args, tuning, diagnostics=True), _loss(do, db, args, tuning, weight=ones, diagnostics=True)
    assert_same_outputs(plain, unit)
    assert torch.equal(plain.diagnostics, unit.diagnostics)


@pytest.mark.parametrize('cluster', [1, 2, 4, 8])
def test_bulk_cluster_and_bf16_logits_with_weights(cluster):
    from handyrl_b200.synthetic import synthetic_batch, synthetic_outputs
    from test_diagnostics_gpu import ARGS
    batch = synthetic_batch(64, 32, 2, 512, seed=3, with_obs=False)
    outs = synthetic_outputs(batch, seed=4)
    db, do = {k: v.cuda() for k, v in batch.items()}, {k: v.cuda() for k, v in outs.items()}
    tuning = {'variant': 'bulk', 'cluster': cluster}
    ones = torch.ones(64, device='cuda')
    w = torch.from_numpy(np.random.default_rng(cluster).uniform(0.5, 2.0, 64).astype(np.float32)).cuda()
    for policy in (do['policy'], do['policy'].to(torch.bfloat16)):
        o = dict(do, policy=policy)
        plain = _loss(o, db, ARGS, tuning)
        assert_same_outputs(plain, _loss(o, db, ARGS, tuning, weight=ones))
        if policy.dtype == torch.float32:
            _assert_scaled(plain, _loss(o, db, ARGS, tuning, weight=w), w.cpu().numpy())


def _assert_scaled(plain, weighted, w):
    """Every gradient row of window b is w[b] times the unweighted row (1e-6 relative); dcnt is unweighted."""
    for k in ('dpolicy', 'dvalue', 'dreturn'):
        a, g = getattr(plain, k), getattr(weighted, k)
        if a is None:
            assert g is None
            continue
        a, g = a.float().cpu().numpy(), g.float().cpu().numpy()
        want = a * w.reshape((-1,) + (1,) * (a.ndim - 1)).astype(np.float64)
        np.testing.assert_allclose(g, want, rtol=1e-6, atol=1e-6 * max(np.abs(want).max(), 1e-30), err_msg=k)
    assert float(weighted.losses[5]) == float(plain.losses[5])


_PER_WINDOW = {}


@pytest.mark.parametrize('variant', VARIANTS)
@pytest.mark.parametrize('name', sorted(LOSS_CASES))
def test_random_weights_scale_rows_and_sums(name, variant):
    """Loss sums = sum_b w_b L_b of per-window float64 oracle runs (1e-5 relative); rows scale by w_b; dcnt and the
    diagnostics sums are the unweighted ones."""
    from oracle import oracle
    case = LOSS_CASES[name]
    batch, outs = split(case)
    args = case_args(case['meta'])
    B = outs['policy'].shape[0]
    if name not in _PER_WINDOW:
        _PER_WINDOW[name] = np.stack([oracle.loss({k: v[b:b + 1] for k, v in batch.items()},
                                                  {k: v[b:b + 1] for k, v in outs.items()}, args, dtype=np.float64)['losses']
                                      for b in range(B)])
    per = _PER_WINDOW[name]
    w = np.random.default_rng(B).uniform(0.5, 2.0, B).astype(np.float32)
    db, do = to_dev(batch), to_dev(outs)
    wd = torch.from_numpy(w).cuda()
    tuning = {'variant': variant}
    plain, weighted = _loss(do, db, args, tuning, diagnostics=True), _loss(do, db, args, tuning, weight=wd, diagnostics=True)
    _assert_scaled(plain, weighted, w)
    assert torch.equal(plain.diagnostics, weighted.diagnostics)
    got = weighted.losses.cpu().numpy().astype(np.float64)
    want = (w.astype(np.float64)[:, None] * per).sum(axis=0)
    for i in range(5):
        assert abs(got[i] - want[i]) <= 1e-5 * abs(want[i]) + 1e-5, (name, variant, i, got[i], want[i])
    assert got[5] == per[:, 5].sum()


# ---------------------------------------------------------------------------------------------------------------- sampler
def _replay(lengths, max_episodes, Ps=2, A=9, seed=0):
    from handyrl_b200.replay import DeviceReplay
    from test_symmetry_gpu import _fake_episode
    rng = np.random.default_rng(seed)
    replay = DeviceReplay(capacity_steps=int(sum(lengths)) + 64, max_episodes=max_episodes, mirror=True)
    for n in lengths:
        replay.add_flat(_fake_episode(int(n), Ps, A, (3, 3), rng))
    torch.cuda.synchronize()
    return replay


def _state(spec, replay, B):
    from handyrl_b200 import priority
    return priority.PriorityState(spec, replay.max_episodes + 1, B, torch.device('cuda'))


def _sample(st, replay, args, counter, seed=11, solo=False):
    """One sampler launch; returns (descriptors as WINDOW_DTYPE, slots, serials, weights) on the host."""
    from handyrl_b200 import ops
    from handyrl_b200.replay import WINDOW_DTYPE
    with replay.lock:
        head, count = replay.snapshot(args['maximum_episodes'])
    win = torch.empty((st.B, WINDOW_DTYPE.itemsize), dtype=torch.uint8, device='cuda')
    ops.replay_sample(st, replay, head, count, args, win, seed, counter, solo)
    torch.cuda.synchronize()
    return (win.cpu().numpy().view(WINDOW_DTYPE).reshape(-1), st.win_slot.cpu().numpy(), st.win_serial.cpu().numpy(),
            st.win_weight.cpu().numpy())


def _live(replay, max_count):
    head, count = replay.snapshot(max_count)
    return (head + np.arange(count)) % (replay.max_episodes + 1)


ARGS = {'burn_in_steps': 2, 'forward_steps': 8, 'turn_based_training': True, 'maximum_episodes': 64}


@pytest.mark.parametrize('alpha', [0.0, 0.6, 1.0])
def test_sampler_frequencies_follow_the_law(alpha):
    from handyrl_b200 import priority
    replay = _replay([20] * 40, 64)
    B = 65536
    st = _state(dict(SPEC, alpha=alpha), replay, B)
    _sample(st, replay, ARGS, 0)                                 # first sight: every episode at max_prio
    slots = _live(replay, 64)
    assert np.all(st.prio.cpu().numpy()[slots] == 1.0)
    prio = np.random.default_rng(1).uniform(0.05, 4.0, slots.size).astype(np.float32)
    st.prio[torch.from_numpy(slots).cuda()] = torch.from_numpy(prio).cuda()
    counts, starts = np.zeros(slots.size), np.zeros(13)
    pos = {int(s): i for i, s in enumerate(slots)}
    for c in range(1, 17):                                       # 16 x 65536 > 10^6 draws
        win, slot, _, weight = _sample(st, replay, ARGS, c)
        idx = np.array([pos[int(s)] for s in slot])
        counts += np.bincount(idx, minlength=slots.size)
        starts += np.bincount(win['train_start'], minlength=13)
        np.testing.assert_allclose(weight, priority.importance_weights(prio[idx], alpha, SPEC['beta']), rtol=1e-6)
    expected = priority.draw_probabilities(prio, alpha) * counts.sum()
    assert stats.chisquare(counts, expected).pvalue > 1e-4, (counts[:8], expected[:8])
    assert starts.size == 13                                     # train_start uniform on [0, 1 + 20 - 8)
    assert stats.chisquare(starts).pvalue > 1e-4, starts


def test_beta_zero_gives_unit_weights():
    replay = _replay([12] * 10, 16)
    st = _state(dict(SPEC, beta=0.0), replay, 512)
    st.prio.uniform_(0.1, 5.0)
    st.prio_serial.copy_(replay.dir_dev[:, 3])
    _, _, _, w = _sample(st, replay, dict(ARGS, maximum_episodes=16), 3)
    assert np.all(w == 1.0)


@pytest.mark.parametrize('solo', [False, True])
def test_same_key_same_windows_inside_live_episodes(solo):
    lengths = np.random.default_rng(2).integers(3, 40, 50)
    replay = _replay(lengths, 32, Ps=2)                          # 50 episodes into 32: the oldest are evicted
    args = dict(ARGS, maximum_episodes=32, turn_based_training=not solo)
    st = _state(SPEC, replay, 2048)
    a = _sample(st, replay, args, 5, seed=9, solo=solo)
    st.prio.mul_(torch.rand_like(st.prio) + 0.5)                 # (the drawn windows depend on the priorities...)
    st.prio_serial.copy_(replay.dir_dev[:, 3])
    prio = st.prio.clone()
    b = _sample(st, replay, args, 5, seed=9, solo=solo)
    st.prio.copy_(prio)
    c = _sample(st, replay, args, 5, seed=9, solo=solo)          # (...and on nothing else: same key, counter, priorities)
    d = _sample(st, replay, args, 6, seed=9, solo=solo)
    for x, y in zip(b, c):
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8))
    assert not np.array_equal(c[0].view(np.uint8), d[0].view(np.uint8))
    live = set(int(s) for s in _live(replay, 32))
    win, slot, serial, _ = a
    for b_ in range(len(win)):
        s = int(slot[b_])
        assert s in live
        first, steps, row = replay._dir[s]
        w = win[b_]
        assert (w['first_step'], w['total'], w['outcome_row']) == (first, steps, row) and serial[b_] == replay._serial[s]
        ts = int(w['train_start'])
        assert 0 <= ts <= max(0, steps - args['forward_steps'])
        assert w['start'] == max(0, ts - args['burn_in_steps']) and w['end'] == min(ts + args['forward_steps'], steps)
        assert (0 <= w['player'] < 2) if solo else w['player'] == 0
    if solo:
        assert len(set(win['player'].tolist())) == 2


def test_new_episodes_start_at_max_prio():
    replay = _replay([10] * 10, 12)
    args = dict(ARGS, maximum_episodes=12)
    st = _state(SPEC, replay, 256)
    _sample(st, replay, args, 0)
    old = _live(replay, 12)
    st.prio.fill_(0.5)
    st.max_prio.fill_(3.5)
    from test_symmetry_gpu import _fake_episode
    rng = np.random.default_rng(7)
    for _ in range(4):
        replay.add_flat(_fake_episode(10, 2, 9, (3, 3), rng))   # 14 episodes into 12: two evicted, four new
    torch.cuda.synchronize()
    _sample(st, replay, args, 1)
    live = _live(replay, 12)
    prio, pser = st.prio.cpu().numpy(), st.prio_serial.cpu().numpy()
    assert np.array_equal(pser[live], replay._serial[live])
    new = [s for s in live if replay._serial[s] >= 10]
    assert len(new) == 4
    assert np.all(prio[new] == 3.5)
    assert np.all(prio[[s for s in live if s not in new]] == 0.5) and set(old) - set(live)


def test_sampler_refuses_bad_arguments():
    from handyrl_b200 import _capi
    with pytest.raises(_capi.HrlError):
        _capi.check(_capi.lib().hrl_replay_sample(None, None))
    with pytest.raises(_capi.HrlError):
        _capi.check(_capi.lib().hrl_replay_priority_update(4, 4, 2, 0, None, None, 0.01, None, None, None, None, None, None, None))


# ---------------------------------------------------------------------------------------------------------------- update
def test_update_matches_the_host_reference():
    from handyrl_b200 import ops, priority
    B, T, P, burn, ring = 96, 12, 2, 3, 40
    rng = np.random.default_rng(4)
    st = priority.PriorityState(SPEC, ring, B, torch.device('cuda'))
    pser = np.arange(ring, dtype=np.int64) + 100
    st.prio_serial.copy_(torch.from_numpy(pser))
    adv = (3 * rng.standard_normal((B, T, P, 1))).astype(np.float32)
    tm = (rng.random((B, T, P, 1)) < 0.5).astype(np.float32)
    tm[5, burn:] = 0                                             # no trained turn: no priority
    slots = rng.integers(0, ring, B).astype(np.int32)
    slots[:8] = 7                                                # duplicates
    serials = pser[slots]
    serials[10] = 999                                            # stale
    serials[11] = -1                                             # no serial
    st.win_slot.copy_(torch.from_numpy(slots))
    st.win_serial.copy_(torch.from_numpy(serials))
    dadv, dtm = torch.from_numpy(adv).cuda(), torch.from_numpy(tm).cuda()
    skip = torch.ones(1, dtype=torch.int32, device='cuda')
    ops.priority_update(st, dadv, dtm, burn, skip=skip)          # a rejected step writes nothing
    torch.cuda.synchronize()
    assert torch.all(st.prio == 1.0) and float(st.max_prio) == 1.0
    skip.zero_()
    ops.priority_update(st, dadv, dtm, burn, skip=skip)
    torch.cuda.synchronize()
    q = priority.window_priorities(adv, tm, burn, SPEC['epsilon'])
    want, mx = priority.update(np.ones(ring, np.float32), pser, 1.0, slots, serials, q)
    got = st.prio.cpu().numpy()
    np.testing.assert_allclose(got, want, rtol=1e-6)
    assert got[7] == pytest.approx(np.nanmax(q[:8]), rel=1e-6)
    if slots[10] not in slots[np.arange(B) != 10]:
        assert got[slots[10]] == 1.0
    assert float(st.max_prio) == pytest.approx(float(mx), rel=1e-6) and float(st.max_prio) > 1.0
    before = st.prio.clone()
    ops.priority_update(st, dadv, dtm, burn)                     # no guard: the same result again
    torch.cuda.synchronize()
    assert torch.equal(st.prio, before)


# ---------------------------------------------------------------------------------------------------------------- learner
def _learner(kind, on, use_graph=True, **extra):
    from handyrl_b200.train import LearnerStep
    make, args, good, lr = _setup(kind)
    a = dict(args, maximum_episodes=100, prioritized_replay=True if on else None, **extra)
    st = LearnerStep(make(), a, good[0], lr=lr, use_graph=use_graph, cudnn_benchmark=False)
    return st, a, good


@pytest.mark.parametrize('use_graph', [True, False], ids=['graph', 'eager'])
@pytest.mark.parametrize('kind', ['tictactoe', 'geese'])
def test_unit_weights_train_exactly_as_without_the_key(kind, use_graph, deterministic_cudnn):
    out = {}
    for on in (False, True):
        st, _, good = _learner(kind, on, use_graph)
        assert (st.engine is not None) == (kind == 'tictactoe')
        for b in good + good:
            st.step(st.new_packed().fill(b))
        st.stream.synchronize()
        out[on] = (st.state.bytes.cpu(), st.opt.exp_avg.cpu(), st.opt.exp_avg_sq.cpu(), st.accum.cpu(), st.launches_per_step)
        if on:      # serials of -1: the warm-up, capture and these steps move no priority
            ps = st.prio_state
            assert torch.all(ps.prio == 1.0) and float(ps.max_prio) == 1.0 and torch.all(ps.win_weight == 1.0)
        st.close()
    for x, y in zip(out[False][:4], out[True][:4]):
        assert torch.equal(x, y)
    assert out[True][4] == out[False][4] + 1


def test_a_step_stores_priorities_and_a_rejected_step_does_not():
    from handyrl_b200 import priority
    st, args, good = _learner('tictactoe', True, skip_nonfinite=True)
    ps = st.prio_state
    B = st.dims[0]
    st.warm_up()
    slots = np.arange(B, dtype=np.int32) % 50
    ps.prio_serial[:50] = torch.arange(50, device='cuda')
    ps.win_slot.copy_(torch.from_numpy(slots))
    ps.win_serial.copy_(torch.from_numpy(slots.astype(np.int64)))
    st.step(st.new_packed().fill(_poisoned(good[1], args)))
    st.stream.synchronize()
    assert float(st.skipped) == 1.0
    assert torch.all(ps.prio == 1.0) and float(ps.max_prio) == 1.0
    st.step(st.new_packed().fill(good[0]))
    st.stream.synchronize()
    q = priority.window_priorities(st.loss_buf.advantage.cpu().numpy(), st.dev['turn_mask'].cpu().numpy(),
                                   args.get('burn_in_steps', 0), SPEC['epsilon'])
    want, mx = priority.update(np.ones(ps.ring, np.float32), ps.prio_serial.cpu().numpy(), 1.0, slots, slots, q)
    np.testing.assert_allclose(ps.prio.cpu().numpy(), want, rtol=1e-6)
    assert float(ps.max_prio) == pytest.approx(float(mx), rel=1e-6)
    assert not torch.all(ps.prio == 1.0)
    st.close()


def test_the_key_is_checked_when_the_step_is_built():
    from handyrl_b200.train import LearnerStep
    make, args, good, lr = _setup('tictactoe')
    for bad in ({'alpha': -1}, {'beta': 2}, 'on'):
        with pytest.raises(ValueError):
            LearnerStep(make(), dict(args, maximum_episodes=100, prioritized_replay=bad), good[0], lr=lr)
    with pytest.raises(ValueError):
        LearnerStep(make(), dict(args, maximum_episodes=100, prioritized_replay=True, gpu_replay=False), good[0], lr=lr)


# ---------------------------------------------------------------------------------------------------------------- trainer
@pytest.mark.parametrize('extra', [{}, {'symmetry': {'group': 'dihedral', 'board': [3, 3]}, 'skip_nonfinite': True}],
                         ids=['plain', 'symmetry+guard'])
def test_trainer_with_the_key(extra, tmp_path, monkeypatch, capsys):
    from handyrl_b200 import ops
    from handyrl_b200.replay import DeviceReplay
    from handyrl_b200.synthetic import tictactoe_episodes
    from test_symmetry_gpu import _line_kinds, _run_trainer
    monkeypatch.chdir(tmp_path)
    calls, samples = [], []
    real_gather, real_sample = DeviceReplay.gather, ops.replay_sample

    def spy(self, windows, args, out=None, sym=None, tables=None):
        calls.append((self, torch.is_tensor(windows)))
        return real_gather(self, windows, args, out=out, sym=sym, tables=tables)

    def spy_sample(state, replay, *a, **k):
        samples.append(replay)
        return real_sample(state, replay, *a, **k)

    monkeypatch.setattr(DeviceReplay, 'gather', spy)
    monkeypatch.setattr(ops, 'replay_sample', spy_sample)
    episodes = tictactoe_episodes(60, seed=21)
    kinds = {}
    for on in (False, True):
        e = dict(extra, prioritized_replay=True if on else None)
        samples.clear()
        tr, lines = _run_trainer(e, episodes, calls, capsys)
        kinds[on] = _line_kinds(lines)
        gb = tr.gpu_batcher
        assert (gb.replay.dir_dev is not None) == on
        if on:
            assert samples and all(r is gb.replay for r in samples)        # validation keeps the host sampler
            assert any(r is gb.val_replay for r, _ in calls)
            ps = tr.stepper.prio_state
            live = _live(gb.replay, tr.args['maximum_episodes'])
            p = ps.prio.cpu().numpy()[live]
            assert np.all(np.isfinite(p)) and np.any(p != 1.0) and float(ps.max_prio) >= 1.0
        else:
            assert not samples
        losses = [l for l in lines.splitlines() if l.startswith('loss = ')]
        assert losses and all(np.isfinite(float(v)) for l in losses for v in re.findall(r':(-?[0-9.]+(?:e-?[0-9]+)?|nan|-?inf)', l))
    assert kinds[True] == kinds[False], kinds


# ---------------------------------------------------------------------------------------------------------------- multi-GPU
NGPU = torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(NGPU < 2, reason='needs at least 2 GPUs')
def test_two_ranks_stay_identical_with_the_key():
    """Each rank draws its shard from its own priorities and Philox stream; the all-reduced step keeps the weights equal."""
    import threading
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.train import Trainer
    with open(os.path.join(GOLDEN, 'batch_cases.pkl'), 'rb') as f:
        case = pickle.load(f)['tictactoe']
    args = dict(case['args'], batch_size=8, minimum_episodes=4, num_batchers=1, **{'lambda': 0.7}, seed=3,
                entropy_regularization=0.1, entropy_regularization_decay=0.1, policy_target='UPGO', value_target='VTRACE',
                gpu_replay=True, num_gpus=2, multi_gpu_probe=True, multi_gpu_chunk=4, prioritized_replay=True)
    tr = Trainer(args, tictactoe_net())
    assert tr.world == 2
    tr.episodes.extend(case['episodes'])
    th = threading.Thread(target=tr.run, daemon=True)
    th.start()
    try:
        for _ in range(3):
            model, steps = tr.update()
            (helper_sum, _), = tr.fleet.collect_reports()
            mine = torch.cat([p.detach().reshape(-1) for p in model.parameters()]).double()
            pad = torch.zeros(tr.stepper.state.n_pad - mine.numel(), dtype=torch.float64)
            assert abs(float(torch.cat([mine, pad]).sum()) - helper_sum) <= 1e-9 * max(1.0, abs(helper_sum))
    finally:
        tr.stop()
        th.join(timeout=30)
