"""Held-out validation loss on the GPU: hrl_loss_fwd against hrl_loss_fwd_bwd bit for bit, the learner's validation pass against
the eager CPU port, its graph against eager launches, no trace of it on training, the averaged pass, the epoch hand-off, the
Trainer's held-out split and printed lines, and sharded learners."""
import os
import pickle
import threading

import numpy as np
import pytest
import torch

from conftest import GOLDEN, case_args, load_cases

pytestmark = pytest.mark.gpu

LOSS_CASES = load_cases('loss_cases.npz')
VARIANTS = ['rows-direct', 'rows-staged', 'bulk', 'element', 'group']
ARGS = {'turn_based_training': True, 'observation': False, 'gamma': 0.8, 'lambda': 0.7, 'burn_in_steps': 0,
        'entropy_regularization': 0.1, 'entropy_regularization_decay': 0.1, 'policy_target': 'UPGO', 'value_target': 'VTRACE'}
SENTINEL = 12345.0


def to_dev(d):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in d.items()}


def split(case):
    batch = {k[3:]: v for k, v in case.items() if k.startswith('in.')}
    outs = {k[4:]: v for k, v in case.items() if k.startswith('out.')}
    return batch, outs


def fwd_against_fwd_bwd(outs, batch, args, tuning=None):
    """Sums of loss_fwd (NULL gradient pointers, then gradient buffers filled with a sentinel) equal loss_fwd_bwd's bit for bit,
    and the sentinel buffers are untouched."""
    from handyrl_b200 import ops
    full = ops.loss_fwd_bwd(outs, batch, args, tuning=tuning)
    fwd = ops.loss_fwd(outs, batch, args, tuning=tuning)
    B, T, Pa, A = outs['policy'].shape
    P = batch['turn_mask'].shape[2]
    guarded = ops.LossBuffers(B, T, P, Pa, A, 'value' in outs, 'return' in outs, outs['policy'].device,
                              policy_dtype=outs['policy'].dtype)
    grads = [g for g in (guarded.dpolicy, guarded.dvalue, guarded.dreturn) if g is not None]
    for g in grads:
        g.fill_(SENTINEL)
    again = ops.loss_fwd(outs, batch, args, buffers=guarded, tuning=tuning)
    torch.cuda.synchronize()
    assert torch.equal(fwd, full.losses), (fwd.tolist(), full.losses.tolist())
    assert torch.equal(again, full.losses)
    for g in grads:
        assert bool((g == SENTINEL).all())
    return full


@pytest.mark.parametrize('recurrence', ['serial', 'scan'])
@pytest.mark.parametrize('variant', VARIANTS)
@pytest.mark.parametrize('name', sorted(LOSS_CASES))
def test_golden_cases_every_variant_and_recurrence(name, variant, recurrence):
    case = LOSS_CASES[name]
    batch, outs = split(case)
    fwd_against_fwd_bwd(to_dev(outs), to_dev(batch), case_args(case['meta']), tuning={'variant': variant, 'recurrence': recurrence})


FULL = [  # the full-size shapes of test_loss_gpu.py
    dict(id='cfg2', B=512, T=32, P=2, A=9, turn_based=True, observation=False, has_return=False,
         policy_target='UPGO', value_target='VTRACE', reward_kind='zero', burn_in=0),
    dict(id='cfg2_sim', B=512, T=32, P=2, A=9, turn_based=False, observation=False, has_return=False,
         policy_target='UPGO', value_target='VTRACE', reward_kind='zero', burn_in=0),
    dict(id='cfg3_geister', B=256, T=20, P=2, A=214, turn_based=True, observation=True, has_return=True,
         policy_target='TD', value_target='TD', reward_kind='step', burn_in=4),
    dict(id='cfg4_geese', B=256, T=32, P=4, A=4, turn_based=False, observation=False, has_return=False,
         policy_target='VTRACE', value_target='VTRACE', reward_kind='zero', burn_in=0),
    dict(id='cfg5_shard', B=512, T=64, P=2, A=512, turn_based=True, observation=False, has_return=False,
         policy_target='UPGO', value_target='VTRACE', reward_kind='zero', burn_in=0),
]


@pytest.mark.parametrize('cfg', FULL, ids=[c['id'] for c in FULL])
def test_full_size_shapes(cfg):
    from handyrl_b200.synthetic import synthetic_batch, synthetic_outputs
    cfg = dict(cfg)
    args = {'turn_based_training': cfg['turn_based'], 'observation': cfg['observation'], 'gamma': 0.8, 'lambda': 0.7,
            'burn_in_steps': cfg['burn_in'], 'entropy_regularization': 0.1, 'entropy_regularization_decay': 0.1,
            'policy_target': cfg['policy_target'], 'value_target': cfg['value_target']}
    batch = synthetic_batch(cfg['B'], cfg['T'], cfg['P'], cfg['A'], turn_based=cfg['turn_based'], observation=cfg['observation'],
                            reward_kind=cfg['reward_kind'], burn_in=cfg['burn_in'], seed=0, with_obs=False)
    outs = synthetic_outputs(batch, has_value=True, has_return=cfg['has_return'], seed=1)
    db, do = {k: v.cuda() for k, v in batch.items()}, {k: v.cuda() for k, v in outs.items()}
    for recurrence in ('serial', 'scan'):
        fwd_against_fwd_bwd(do, db, args, tuning={'recurrence': recurrence})


@pytest.mark.parametrize('cluster', [1, 2, 4])
def test_wide_rows_bulk_clusters_and_bf16_logits(cluster):
    from handyrl_b200.synthetic import synthetic_batch, synthetic_outputs
    batch = synthetic_batch(64, 32, 2, 512, seed=3, with_obs=False)
    outs = synthetic_outputs(batch, seed=4)
    db, do = {k: v.cuda() for k, v in batch.items()}, {k: v.cuda() for k, v in outs.items()}
    tuning = {'variant': 'bulk', 'cluster': cluster}
    fwd_against_fwd_bwd(do, db, ARGS, tuning=tuning)
    fwd_against_fwd_bwd(dict(do, policy=do['policy'].to(torch.bfloat16)), db, ARGS, tuning=tuning)


# ---------------------------------------------------------------------------------------------------------------- learner
with open(os.path.join(GOLDEN, 'step_cases.pkl'), 'rb') as f:
    STEP_CASES = pickle.load(f)
with open(os.path.join(GOLDEN, 'net_step_cases.pkl'), 'rb') as f:
    NET_CASES = pickle.load(f)
NSTEPS = 3
KINDS = ['tictactoe', 'geese', 'geister']


def _setup(kind):
    """(net factory, args, [batches], lr): the fused-tower TicTacToe net, the module-path Geese net, the recurrent Geister net."""
    if kind == 'tictactoe':
        from handyrl_b200.nets import tictactoe_net, load_state_by_order
        from handyrl_b200.synthetic import synthetic_batch
        c = STEP_CASES[sorted(STEP_CASES)[0]]
        B, T, P, A = c['dims']
        args = c['args']
        batches = [synthetic_batch(B, T, P, A, turn_based=args['turn_based_training'], observation=args['observation'], seed=40 + s)
                   for s in range(NSTEPS + 1)]
        return (lambda: load_state_by_order(tictactoe_net(), c['state0'])), args, batches, c['lr']
    from conftest import net_case_setup
    name = [n for n in sorted(NET_CASES) if NET_CASES[n]['net'] == kind][0]
    c = NET_CASES[name]
    _, batches = net_case_setup(c)
    batches = (batches * (NSTEPS + 1))[:NSTEPS + 1]
    return (lambda: net_case_setup(c)[0]), c['args'], batches, c['lr']


@pytest.fixture
def deterministic_cudnn():
    # the Geese stem (17 input channels) stays on cuDNN: pin deterministic algorithms so that runs compare bit for bit
    old = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.deterministic = old


def _load(st, batch):
    """Write a host batch into st.dev on the step stream (what GpuBatcher.fill_validation does with a held-out batch)."""
    packed = st.new_packed().fill(batch)
    with torch.cuda.stream(st.stream):
        st.dev_buffer.copy_(packed.buffer, non_blocking=True)
    st.stream.synchronize()


def _stepper(kind, use_graph=True, validation=True, **extra):
    from handyrl_b200.train import LearnerStep
    make, args, batches, lr = _setup(kind)
    st = LearnerStep(make(), dict(args, **extra), batches[0], lr=lr, use_graph=use_graph, cudnn_benchmark=False,
                     validation=validation)
    return st, make, args, batches


def _cpu_losses(make, state, batch, args):
    """The eager CPU port of the reference's training-mode loss: oracle.torch_learner on the net's forward with `state`."""
    from oracle.torch_learner import loss_from_raw, recurrent_raw_outputs, _walk
    net = make()
    net.load_state_dict({k: state[k] for k in net.state_dict()})
    net.train()
    batch = {k: v for k, v in batch.items()}
    B, T, Pa = batch['action'].shape[:3]
    with torch.no_grad():
        if hasattr(net, 'init_hidden'):
            raw = recurrent_raw_outputs(net, net.init_hidden([B, batch['turn_mask'].shape[2]]), batch, args)
        else:
            outs = net(_walk(lambda o: o.flatten(0, 2), batch['observation']), None)
            raw = {k: v.unflatten(0, (B, T, Pa)) for k, v in outs.items() if v is not None and k != 'hidden'}
        losses, dcnt = loss_from_raw(raw, batch, args)
    return {k: float(v) for k, v in losses.items()}, float(dcnt)


@pytest.mark.parametrize('kind', KINDS)
def test_validation_pass_equals_the_eager_cpu_port_and_graph_equals_eager(kind, deterministic_cudnn):
    sums = {}
    for use_graph in (True, False):
        st, make, args, batches = _stepper(kind, use_graph=use_graph)
        assert (st.engine is not None) == (kind == 'tictactoe') and (st.hidden0 is not None) == (kind == 'geister')
        st.step(st.new_packed().fill(batches[0]))
        _load(st, batches[1])
        st.validate_in_place()
        sums[use_graph] = st.pop_validation()['validation']
        state = st.cpu_state_dict()
        assert st.launches_per_validation > 0
        st.close()
    assert sums[True] == sums[False], (sums[True], sums[False])
    want, dcnt = _cpu_losses(make, state, batches[1], args)
    got = sums[True]
    assert got['dcnt'] == dcnt
    scale = max(abs(v) for v in want.values())
    for k, v in want.items():
        # test_step_gpu.py's tolerances for these nets' loss sums at the reference's weights
        tol = 2e-4 * abs(v) + 1e-4 if kind == 'tictactoe' else 1e-4 * scale + 1e-4
        assert abs(got[k] - v) <= tol, (kind, k, got[k], v)


def _train(kind, validate, use_graph=True):
    st, make, args, batches = _stepper(kind, use_graph=use_graph, validation=validate, weight_ema=0.9)
    for b in batches[:NSTEPS]:
        st.step(st.new_packed().fill(b))
        if validate:
            with torch.cuda.stream(st.stream):
                st.dev_buffer.copy_(st.new_packed().fill(batches[NSTEPS]).buffer)
            st.validate_in_place()
            st.validate_in_place(averaged=True)
    st.stream.synchronize()
    out = {'live': st.cpu_state_dict(), 'avg': st.ema_state_dict(), 'm': st.opt.exp_avg.cpu(), 'v': st.opt.exp_avg_sq.cpu(),
           'step': int(st.opt.step_count.item()), 'accum': st.accum.cpu(), 'last': st.last_losses.cpu(),
           'launches': st.launches_per_step}
    if validate:
        out['val'] = st.pop_validation()
    st.close()
    return out


@pytest.mark.parametrize('kind', KINDS)
def test_validation_leaves_no_trace_on_training(kind, deterministic_cudnn):
    from handyrl_b200.train import LearnerStep
    off, on = _train(kind, False), _train(kind, True)
    for part in ('live', 'avg'):
        for k in off[part]:
            assert torch.equal(off[part][k], on[part][k]), (part, k)
    assert any(k.endswith('running_var') for k in off['live']) or kind == 'tictactoe'
    for k in ('m', 'v', 'accum', 'last'):
        assert torch.equal(off[k], on[k]), k
    assert off['step'] == on['step'] == NSTEPS
    assert on['val']['validation']['dcnt'] > 0 and on['val']['validation_ema']['dcnt'] > 0
    # launches of the step with the key on or off
    make, args, batches, lr = _setup(kind)
    plain = LearnerStep(make(), args, batches[0], lr=lr, cudnn_benchmark=False)
    plain.warm_up()
    keyed = LearnerStep(make(), dict(args, validation_rate=0.05), batches[0], lr=lr, cudnn_benchmark=False)
    keyed.warm_up()
    assert plain.validation is False and keyed.validation is True
    assert plain.launches_per_step == keyed.launches_per_step
    plain.close()
    keyed.close()


@pytest.mark.parametrize('kind', ['tictactoe', 'geese'])
def test_averaged_pass_equals_a_live_pass_on_the_average(kind, deterministic_cudnn):
    from handyrl_b200.train import LearnerStep
    st, make, args, batches = _stepper(kind, weight_ema=0.7)
    for b in batches[:NSTEPS]:
        st.step(st.new_packed().fill(b))
    _load(st, batches[NSTEPS])
    st.validate_in_place(averaged=True)
    got = st.pop_validation()
    avg = st.ema_state_dict()
    st.close()
    assert got['validation']['dcnt'] == 0                    # only the averaged form ran
    net = make()
    net.load_state_dict({k: avg[k] for k in net.state_dict()})
    seeded = LearnerStep(net, args, batches[0], lr=1e-3, cudnn_benchmark=False, validation=True)
    seeded.warm_up()                 # the capture writes its own batch into self.dev
    _load(seeded, batches[NSTEPS])
    seeded.validate_in_place()
    want = seeded.pop_validation()['validation']
    seeded.close()
    assert got['validation_ema'] == want, (got['validation_ema'], want)


def test_hand_off_never_synchronises_the_step_stream_and_equals_pop_validation(deterministic_cudnn):
    from handyrl_b200.nets import tictactoe_net
    st, make, args, batches = _stepper('tictactoe', weight_ema=0.9)

    def passes():
        for b in batches[:2]:
            _load(st, b)
            st.validate_in_place()
            st.validate_in_place(averaged=True)

    for b in batches[:NSTEPS]:
        st.step(st.new_packed().fill(b))
    passes()
    st.stream.synchronize()
    stream_cls = type(st.stream)
    calls = []
    real = stream_cls.synchronize
    stream_cls.synchronize = lambda self: (calls.append(self), real(self))[1]
    try:
        pending = st.end_epoch(NSTEPS, NSTEPS, 3e-8, tictactoe_net(), ['p', 'v', 'ent', 'total'])
        pending.resolve()
    finally:
        stream_cls.synchronize = real
    assert not any(s is st.stream for s in calls)
    assert st.pop_validation()['validation']['dcnt'] == 0        # end_epoch moved the sums out
    passes()                                                      # the same passes on the same weights
    want = st.pop_validation()
    st.close()
    assert pending.validation == want and want['validation']['dcnt'] > 0


# ---------------------------------------------------------------------------------------------------------------- trainer
def _trainer_args(**extra):
    with open(os.path.join(GOLDEN, 'batch_cases.pkl'), 'rb') as f:
        case = pickle.load(f)['tictactoe']
    args = dict(case['args'], batch_size=8, minimum_episodes=4, num_batchers=1, **{'lambda': 0.7},
                entropy_regularization=0.1, entropy_regularization_decay=0.1, policy_target='UPGO', value_target='VTRACE',
                gpu_replay=True, num_gpus=1, **extra)
    return args


def _split(episodes, rate):
    from handyrl_b200.replay import held_out
    from handyrl_b200.wire import episode_to_flat
    train = [ep for ep in episodes if not held_out(episode_to_flat(ep), rate)]
    val = [ep for ep in episodes if held_out(episode_to_flat(ep), rate)]
    return train, val


def test_trainer_holds_episodes_out_and_prints_the_lines(tmp_path, monkeypatch, capsys):
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.replay import DeviceReplay, held_out
    from handyrl_b200.synthetic import tictactoe_episodes
    from handyrl_b200.train import Trainer
    monkeypatch.chdir(tmp_path)
    rate = 0.7                                   # round(1 / r) == 1: a validation pass after every step
    train_eps, val_eps = _split(tictactoe_episodes(60, seed=21), rate)
    assert len(train_eps) >= 4 and len(val_eps) >= 4
    staged = []
    real_stage = DeviceReplay.stage

    def spy(self, fes):
        staged.append((self, list(fes)))
        return real_stage(self, fes)

    monkeypatch.setattr(DeviceReplay, 'stage', spy)
    tr = Trainer(_trainer_args(validation_rate=rate, weight_ema=0.9), tictactoe_net())
    tr.episodes.extend(train_eps[:4])
    th = threading.Thread(target=tr.run, daemon=True)
    th.start()
    try:
        tr.update()
        before = capsys.readouterr().out
        tr.episodes.extend(val_eps + train_eps[4:])
        for _ in range(500):
            if tr.gpu_batcher.validation_ready():
                break
            threading.Event().wait(0.01)
        assert tr.gpu_batcher.validation_ready()
        for _ in range(500):
            if tr.gpu_batcher.fed >= len(train_eps) + len(val_eps):
                break
            threading.Event().wait(0.01)
        tr.update()                 # the epoch in which the held-out ring filled
        capsys.readouterr()
        tr.update()
        tr.update()
        after = capsys.readouterr().out
    finally:
        tr.stop()
        th.join(timeout=10)
    assert 'loss = ' in before and 'validation' not in before
    lines = after.splitlines()
    for name in ('validation = ', 'validation_ema = '):
        assert sum(l.startswith(name) for l in lines) == 2, after
    for i, l in enumerate(lines):
        if l.startswith('loss = '):
            assert lines[i + 1].startswith('validation = ') and lines[i + 2].startswith('validation_ema = '), after
    train_ring, val_ring = tr.gpu_batcher.replay, tr.gpu_batcher.val_replay
    to_train = [fe for r, fes in staged if r is train_ring for fe in fes]
    to_val = [fe for r, fes in staged if r is val_ring for fe in fes]
    assert len(to_train) == len(train_eps) and len(to_val) == len(val_eps)
    assert not any(held_out(fe, rate) for fe in to_train)
    assert all(held_out(fe, rate) for fe in to_val)
    want = sorted(fe.action.tobytes() + fe.prob.tobytes() for fe in to_val)
    from handyrl_b200.wire import episode_to_flat
    assert want == sorted(episode_to_flat(ep).action.tobytes() + episode_to_flat(ep).prob.tobytes() for ep in val_eps)


def test_helper_ranks_train_on_the_same_episodes_and_keep_no_held_out_ring(monkeypatch):
    """A helper rank's feeder (keep_validation=False) commits exactly rank 0's training episodes and stores nothing else."""
    from handyrl_b200.replay import DeviceReplay
    from handyrl_b200.synthetic import tictactoe_episodes
    from handyrl_b200.train import EpisodeDeque, GpuBatcher
    args = _trainer_args(validation_rate=0.3)
    staged = []
    real_stage = DeviceReplay.stage
    monkeypatch.setattr(DeviceReplay, 'stage', lambda self, fes: (staged.append((self, list(fes))), real_stage(self, fes))[1])
    episodes = tictactoe_episodes(80, seed=5)
    batchers = {}
    for keep in (True, False):
        q = EpisodeDeque()
        q.extend(episodes)
        gb = GpuBatcher(args, q, torch.device('cuda', 0), keep_validation=keep)
        gb.run()
        for _ in range(500):
            if gb.fed >= len(episodes):
                break
            threading.Event().wait(0.01)
        gb.stop()
        batchers[keep] = gb
    torch.cuda.synchronize()
    assert batchers[False].val_replay is None and batchers[True].validation_ready()

    def contents(ring):
        return sorted(fe.action.tobytes() + fe.prob.tobytes() for r, fes in staged if r is ring for fe in fes)

    assert contents(batchers[True].replay) == contents(batchers[False].replay)
    assert len(contents(batchers[True].replay)) + len(contents(batchers[True].val_replay)) == len(episodes)


NGPU = torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(NGPU < 2, reason='needs at least 2 GPUs')
def test_sharded_trainer_validates_on_rank0_and_ranks_stay_identical():
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.synthetic import tictactoe_episodes
    from handyrl_b200.train import Trainer
    args = _trainer_args(validation_rate=0.5, seed=3, multi_gpu_probe=True, multi_gpu_chunk=4)
    args['num_gpus'] = 2
    tr = Trainer(args, tictactoe_net())
    assert tr.world == 2
    tr.episodes.extend(tictactoe_episodes(40, seed=9))
    th = threading.Thread(target=tr.run, daemon=True)
    th.start()
    try:
        for _ in range(3):
            model, steps = tr.update()
            (helper_sum, helper_lr), = tr.fleet.collect_reports()
            mine = torch.cat([p.detach().reshape(-1) for p in model.parameters()]).double()
            pad = torch.zeros(tr.stepper.state.n_pad - mine.numel(), dtype=torch.float64)
            assert abs(float(torch.cat([mine, pad]).sum()) - helper_sum) <= 1e-9 * max(1.0, abs(helper_sum))
            assert helper_lr == float(tr.stepper.opt.lr.item())
    finally:
        tr.stop()
        th.join(timeout=30)
    assert tr.stepper.validation
