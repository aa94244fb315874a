"""Optimiser state with each checkpoint, on the GPU: a learner resumed from the handed-over state continues bit for bit,
the key changes nothing about training, the hand-off never synchronises the step stream, the Trainer's files and restart,
and helper ranks of a sharded learner."""
import os
import pickle
import threading

import numpy as np
import pytest
import torch

from conftest import GOLDEN

pytestmark = pytest.mark.gpu

with open(os.path.join(GOLDEN, 'step_cases.pkl'), 'rb') as f:
    STEP_CASES = pickle.load(f)
with open(os.path.join(GOLDEN, 'net_step_cases.pkl'), 'rb') as f:
    NET_CASES = pickle.load(f)
K, M = 4, 3            # steps before and after the epoch boundary
HEADS = ['p', 'v', 'ent', 'total']


def _setup(kind):
    """(net factory, args, [K + M batches], lr) of a fused-tower TicTacToe case or a module-path Geese case."""
    if kind == 'tictactoe':
        from handyrl_b200.nets import tictactoe_net, load_state_by_order
        from handyrl_b200.synthetic import synthetic_batch
        c = STEP_CASES[sorted(STEP_CASES)[0]]
        B, T, P, A = c['dims']
        args = c['args']
        batches = [synthetic_batch(B, T, P, A, turn_based=args['turn_based_training'], observation=args['observation'], seed=40 + s)
                   for s in range(K + M)]
        return (lambda: load_state_by_order(tictactoe_net(), c['state0'])), args, batches, c['lr']
    from conftest import net_case_setup
    name = [n for n in sorted(NET_CASES) if NET_CASES[n]['net'] == 'geese'][0]
    c = NET_CASES[name]
    _, batches = net_case_setup(c)
    batches = (batches * (K + M))[:K + M]
    return (lambda: net_case_setup(c)[0]), c['args'], batches, c['lr']


def _template(kind):
    from handyrl_b200 import nets
    return nets.tictactoe_net() if kind == 'tictactoe' else nets.geese_net()


@pytest.fixture
def deterministic_cudnn():
    # the Geese stem (17 input channels) stays on cuDNN: pin deterministic algorithms so that runs compare bit for bit
    old = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.deterministic = old


def _stepper(net, args, batches, lr, use_graph, **kw):
    from handyrl_b200.train import LearnerStep
    return LearnerStep(net, args, batches[0], lr=lr, use_graph=use_graph, cudnn_benchmark=False, **kw)


def _steps(st, batches):
    for b in batches:
        st.step(st.new_packed().fill(b))


def _result(st):
    st.stream.synchronize()
    out = {'live': st.cpu_state_dict(), 'm': st.opt.exp_avg.cpu(), 'v': st.opt.exp_avg_sq.cpu(),
           'step': int(st.opt.step_count.item()), 'lr': st.opt.lr.cpu(), 'ema': st.ema.cpu(), 'sums': st.accum.cpu(),
           'launches': st.launches_per_step}
    st.close()
    return out


def _differences(a, b):
    bad = [k for k in a['live'] if not torch.equal(a['live'][k], b['live'][k])]
    bad += [k for k in ('m', 'v', 'lr') if not torch.equal(a[k].view(torch.int32), b[k].view(torch.int32))]
    bad += ['step'] if a['step'] != b['step'] else []
    return bad


def _arm_a(kind, use_graph):
    """One learner: K steps, the epoch boundary, M more steps."""
    make, args, batches, lr = _setup(kind)
    st = _stepper(make(), dict(args, save_optimizer=True), batches, lr, use_graph)
    _steps(st, batches[:K])
    st.end_epoch(K, K, 3e-8, _template(kind), HEADS).resolve()
    _steps(st, batches[K:])
    return _result(st)


def _arm_b(kind, use_graph, load=True):
    """K steps and the epoch boundary on one learner, then a second learner, built like a restarted Learner's (a fresh net
    holding the handed-over weights), resumed from the handed-over optimiser state, runs the same M batches."""
    make, args, batches, lr = _setup(kind)
    st = _stepper(make(), dict(args, save_optimizer=True), batches, lr, use_graph)
    _steps(st, batches[:K])
    pending = st.end_epoch(K, K, 3e-8, _template(kind), HEADS)
    model, _ = pending.resolve()
    state = pending.optim_state
    assert state is not None and state['schedule']['steps'] == K
    st.close()
    net = make()
    net.load_state_dict(model.state_dict(), strict=True)
    st2 = _stepper(net, dict(args, save_optimizer=True), batches, lr, use_graph)
    if load:
        st2.load_optimizer_state(state)
    _steps(st2, batches[K:])
    return _result(st2)


@pytest.mark.parametrize('kind,use_graph', [('tictactoe', True), ('geese', True), ('tictactoe', False)],
                         ids=['tictactoe-graph', 'geese-graph', 'tictactoe-eager'])
def test_a_resumed_learner_continues_bit_for_bit(kind, use_graph, deterministic_cudnn):
    a = _arm_a(kind, use_graph)
    b = _arm_b(kind, use_graph)
    assert a['step'] == b['step'] == K + M
    assert _differences(a, b) == []
    assert any(k.endswith('running_var') for k in a['live'])         # BatchNorm buffers are part of the comparison
    if use_graph and kind == 'tictactoe':
        # without the load the second learner starts its moments, step count and learning rate afresh: it must differ
        cold = _arm_b(kind, use_graph, load=False)
        bad = _differences(a, cold)
        assert 'm' in bad and 'v' in bad and 'step' in bad and 'lr' in bad
        assert any(k in a['live'] for k in bad)


@pytest.mark.parametrize('kind', ['tictactoe', 'geese'])
def test_the_key_leaves_training_alone(kind, deterministic_cudnn):
    res = {}
    for on in (False, True):
        make, args, batches, lr = _setup(kind)
        st = _stepper(make(), dict(args, save_optimizer=on), batches, lr, True)
        assert (st.optim_snap is not None) == on
        _steps(st, batches[:K])
        pending = st.end_epoch(K, K, 3e-8, _template(kind), HEADS)
        _, sums = pending.resolve()
        assert (pending.optim_state is not None) == on
        _steps(st, batches[K:])
        res[on] = dict(_result(st), epoch_sums=sums)
    assert _differences(res[False], res[True]) == []
    assert torch.equal(res[False]['sums'], res[True]['sums'])
    assert res[False]['epoch_sums'] == res[True]['epoch_sums']
    assert res[False]['launches'] == res[True]['launches']


def _assert_same_dict(got, want):
    assert list(got) == list(want)
    assert got['param_names'] == want['param_names'] and got['schedule'] == want['schedule']
    assert got['max_norm'] == want['max_norm']
    assert got['optimizer']['param_groups'] == want['optimizer']['param_groups']
    assert sorted(got['optimizer']['state']) == sorted(want['optimizer']['state'])
    for i, s in want['optimizer']['state'].items():
        for k, t in s.items():
            assert torch.equal(got['optimizer']['state'][i][k], t), (i, k)


def test_the_hand_off_never_synchronises_the_step_stream_and_equals_a_blocking_read(deterministic_cudnn):
    make, args, batches, lr = _setup('tictactoe')
    st = _stepper(make(), dict(args, save_optimizer=True), batches, lr, True)
    _steps(st, batches[:K])
    st.stream.synchronize()
    stream_cls = type(st.stream)
    calls = []
    real = stream_cls.synchronize
    stream_cls.synchronize = lambda self: (calls.append(self), real(self))[1]
    try:
        pending = st.end_epoch(K, 123, 3e-8, _template('tictactoe'), HEADS)
        pending.resolve()
    finally:
        stream_cls.synchronize = real
    assert not any(s is st.stream for s in calls)
    want = st.optimizer_state_dict()                  # blocking read at the same point
    _assert_same_dict(pending.optim_state, want)
    assert want['schedule']['steps'] == 123 and float(want['optimizer']['state'][0]['step']) == K
    assert want['schedule']['lr'] == float(st.opt.lr.item()) == want['optimizer']['param_groups'][0]['lr']
    assert want['schedule']['data_cnt_ema'] == float(st.ema.item())
    # what a load reads back is what was handed over; a dict that does not fit changes nothing
    from handyrl_b200.train import OptimizerStateFormat
    m, v, step, lr_, ema, steps = OptimizerStateFormat(st.model.named_parameters()).unpack(want)
    assert torch.equal(m, st.opt.exp_avg.cpu()) and torch.equal(v, st.opt.exp_avg_sq.cpu())
    assert not m[st.opt.n:].any()
    st2 = _stepper(make(), dict(args, save_optimizer=True), batches, lr, True)
    before = st2.optimizer_state_dict()
    bad = dict(want, max_norm=1.0)
    with pytest.raises(ValueError):
        st2.load_optimizer_state(bad)
    bad = dict(want, param_names=want['param_names'][:-1] + ['extra.weight'])
    with pytest.raises(KeyError):
        st2.load_optimizer_state(bad)
    _assert_same_dict(st2.optimizer_state_dict(), before)
    st2.load_optimizer_state(want)
    _assert_same_dict(st2.optimizer_state_dict(), want)
    st2.warm_up()                                     # the capture's warm-up steps leave the loaded state in place
    _assert_same_dict(st2.optimizer_state_dict(), want)
    with pytest.raises(RuntimeError):
        st2.load_optimizer_state(want)
    st2.close()
    st.close()


# ---------------------------------------------------------------------------------------------------------------- trainer
def _trainer_args(**extra):
    with open(os.path.join(GOLDEN, 'batch_cases.pkl'), 'rb') as f:
        case = pickle.load(f)['tictactoe']
    args = dict(case['args'], batch_size=8, minimum_episodes=4, num_batchers=1, **{'lambda': 0.7},
                entropy_regularization=0.1, entropy_regularization_decay=0.1, policy_target='UPGO', value_target='VTRACE',
                gpu_replay=True, num_gpus=1)
    args.update(extra)
    return args, case['episodes']


def _two_epochs(args, episodes, check_sync=False):
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.train import Trainer
    tr = Trainer(args, tictactoe_net())
    tr.episodes.extend(episodes)
    th = threading.Thread(target=tr.run, daemon=True)
    th.start()
    calls = []
    try:
        tr.update()
        stream_cls = type(tr.stepper.stream)
        real = stream_cls.synchronize
        if check_sync:
            stream_cls.synchronize = lambda self: (calls.append(self), real(self))[1]
        try:
            tr.update()
        finally:
            stream_cls.synchronize = real
    finally:
        tr.stop()
        th.join(timeout=10)
    assert not any(s is tr.stepper.stream for s in calls)
    return tr


def test_trainer_writes_the_files_and_a_restart_resumes_them(tmp_path, monkeypatch, capsys):
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.train import Trainer
    monkeypatch.chdir(tmp_path)
    args, episodes = _trainer_args(save_optimizer=True)
    tr = _two_epochs(args, episodes, check_sync=True)
    assert sorted(os.listdir('models')) == ['1.optim.pth', '2.optim.pth', 'latest.optim.pth']
    saved = torch.load('models/2.optim.pth')
    _assert_same_dict(torch.load('models/latest.optim.pth'), saved)
    opt = torch.optim.Adam(tictactoe_net().parameters(), lr=3e-8, weight_decay=1e-5)
    opt.load_state_dict(saved['optimizer'])
    assert saved['schedule']['steps'] > 0 and float(saved['optimizer']['state'][0]['step']) == saved['schedule']['steps']

    # restarted at epoch 2: the stepper holds exactly the file's state after _start_stepper (warm-up included)
    tr = Trainer(dict(args, restart_epoch=2), tictactoe_net())
    tr.episodes.extend(episodes)
    try:
        tr._start_stepper()
        st = tr.stepper
        sched = saved['schedule']
        assert (tr.steps, tr.data_cnt_ema, tr.lr) == (sched['steps'], sched['data_cnt_ema'], sched['lr'])
        _assert_same_dict(st.optimizer_state_dict(), saved)
        assert int(st.opt.step_count.item()) == sched['steps']
        assert float(st.opt.lr.item()) == sched['lr'] and float(st.ema.item()) == sched['data_cnt_ema']
    finally:
        tr.stop()

    # restarted at an epoch without a file: one line, a fresh optimiser
    capsys.readouterr()
    tr = Trainer(dict(args, restart_epoch=5), tictactoe_net())
    tr.episodes.extend(episodes)
    try:
        tr._start_stepper()
        assert int(tr.stepper.opt.step_count.item()) == 0 and tr.steps == 0
        assert not tr.stepper.opt.exp_avg.any()
    finally:
        tr.stop()
    out = [line for line in capsys.readouterr().out.splitlines() if 'optimiser' in line]
    assert out == ['handyrl_b200: no %s, the optimiser state starts fresh' % os.path.join('models', '5.optim.pth')]


def test_trainer_pairs_the_averages_and_writes_nothing_without_the_key(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    args, episodes = _trainer_args(save_optimizer=True, weight_ema=0.9)
    tr = _two_epochs(args, episodes)
    assert tr.ema_files is tr.optim_files
    assert sorted(os.listdir('models')) == ['1.ema.pth', '1.optim.pth', '2.ema.pth', '2.optim.pth',
                                            'latest.ema.pth', 'latest.optim.pth']
    launches_on = tr.stepper.launches_per_step
    (tmp_path / 'off').mkdir()
    monkeypatch.chdir(tmp_path / 'off')
    args_off, _ = _trainer_args(weight_ema=0.9)
    tr = _two_epochs(args_off, episodes)
    assert sorted(os.listdir('models')) == ['1.ema.pth', '2.ema.pth', 'latest.ema.pth']
    assert tr.stepper.launches_per_step == launches_on
    (tmp_path / 'none').mkdir()
    monkeypatch.chdir(tmp_path / 'none')
    args_none, _ = _trainer_args()
    tr = _two_epochs(args_none, episodes)
    assert os.listdir('.') == []
    assert tr.optim_files is None and tr.stepper.optim_snap is None


# ---------------------------------------------------------------------------------------------------------------- multi-GPU
NGPU = torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(NGPU < 2, reason='needs at least 2 GPUs')
def test_helper_ranks_start_from_the_loaded_state(tmp_path, monkeypatch):
    """A one-GPU run writes its state; the run restarted on two GPUs loads it on both ranks: after an epoch the helper's
    weights (checksum) and device learning rate equal rank 0's, which they would not if it had started afresh."""
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.train import Trainer
    monkeypatch.chdir(tmp_path)
    args, episodes = _trainer_args(save_optimizer=True, seed=3)
    _two_epochs(args, episodes)
    saved = torch.load('models/2.optim.pth')
    tr = Trainer(dict(args, restart_epoch=2, num_gpus=2, multi_gpu_probe=True, multi_gpu_chunk=4), tictactoe_net())
    assert tr.world == 2
    tr.episodes.extend(episodes)
    th = threading.Thread(target=tr.run, daemon=True)
    th.start()
    try:
        model, steps = tr.update()
        assert steps > saved['schedule']['steps']
        (helper_sum, helper_lr), = tr.fleet.collect_reports()
        mine = torch.cat([p.detach().reshape(-1) for p in model.parameters()]).double()
        pad = torch.zeros(tr.stepper.state.n_pad - mine.numel(), dtype=torch.float64)
        assert abs(float(torch.cat([mine, pad]).sum()) - helper_sum) <= 1e-9 * max(1.0, abs(helper_sum))
        assert helper_lr == float(tr.stepper.opt.lr.item())
        assert sorted(os.listdir('models')) == ['1.optim.pth', '2.optim.pth', '3.optim.pth', 'latest.optim.pth']
        assert float(torch.load('models/3.optim.pth')['optimizer']['state'][0]['step']) > saved['schedule']['steps']
    finally:
        tr.stop()
        th.join(timeout=30)
    assert np.isfinite(helper_sum)
