"""Optimiser state with each checkpoint, without a GPU: the flat <-> per-parameter conversion, the dict against a real
torch.optim.Adam state_dict, what `step` means for bias correction (torch.optim.Adam against the oracle of the learner's
clip + Adam step), the checks a load makes before it touches anything, and the numbering of the .optim.pth files."""
import copy
import os
import queue
import types

import numpy as np
import pytest
import torch

from handyrl_b200.train import PendingModel

ARGS = {'batch_size': 4, 'forward_steps': 2, 'num_batchers': 1, 'minimum_episodes': 1, 'maximum_episodes': 10}
NETS = ['tictactoe_net', 'geese_net']


def _format(net):
    from handyrl_b200.train import OptimizerStateFormat
    return OptimizerStateFormat(net.named_parameters())


def _flat_state(fmt, seed):
    """Random moments over the n parameter words, zero padding up to n_pad (as FlatAdam keeps them)."""
    g = torch.Generator().manual_seed(seed)
    m, v = torch.zeros(fmt.n_pad), torch.zeros(fmt.n_pad)
    m[:fmt.n] = torch.randn(fmt.n, generator=g) * 1e-3
    v[:fmt.n] = torch.rand(fmt.n, generator=g) * 1e-5
    return m, v


def _net(name):
    from handyrl_b200 import nets
    torch.manual_seed(3)
    return getattr(nets, name)()


@pytest.mark.parametrize('name', NETS)
def test_flat_and_per_parameter_forms_round_trip_bit_for_bit(name, tmp_path):
    net = _net(name)
    fmt = _format(net)
    assert fmt.n == sum(p.numel() for p in net.parameters()) and fmt.n_pad % 4 == 0
    m, v = _flat_state(fmt, 1)
    lr, ema = float(np.float32(2.7e-6)), float(np.float32(123.456))
    d = fmt.to_dict(m, v, 4321, lr, ema, 987)
    assert d['param_names'] == [k for k, _ in net.named_parameters()]
    for i, p in enumerate(net.parameters()):
        assert d['optimizer']['state'][i]['exp_avg'].shape == p.shape
    torch.save(d, tmp_path / 'x.optim.pth')
    for src in (d, torch.load(tmp_path / 'x.optim.pth')):             # torch.load's default weights_only=True reads it
        m2, v2, step, lr2, ema2, steps = fmt.unpack(src)
        assert torch.equal(m2.view(torch.int32), m.view(torch.int32))      # bit for bit, padding (zero) included
        assert torch.equal(v2.view(torch.int32), v.view(torch.int32))
        assert (step, lr2, ema2, steps) == (4321, lr, ema, 987)
    assert d['schedule'] == {'steps': 987, 'data_cnt_ema': ema, 'lr': lr}
    assert d['max_norm'] == 4.0
    # padding is not part of the format: whatever the source held there, a load yields zeros
    m[fmt.n:] = 7.0
    assert not fmt.unpack(fmt.to_dict(m, v, 1, lr, ema, 0))[0][fmt.n:].any()


@pytest.mark.parametrize('name', NETS)
def test_the_dict_loads_into_torch_adam_on_a_fresh_net(name):
    net = _net(name)
    fmt = _format(net)
    m, v = _flat_state(fmt, 2)
    d = fmt.to_dict(m, v, 17, 1e-4, 50.0, 17)
    fresh = _net(name)
    opt = torch.optim.Adam(fresh.parameters(), lr=3e-8, weight_decay=1e-5)
    opt.load_state_dict(d['optimizer'])
    assert opt.param_groups[0]['lr'] == 1e-4
    for i, p in enumerate(fresh.parameters()):
        st = opt.state[p]
        assert float(st['step']) == 17
        off = fmt.offsets[i]
        assert torch.equal(st['exp_avg'].reshape(-1), m[off:off + p.numel()])
        assert torch.equal(st['exp_avg_sq'].reshape(-1), v[off:off + p.numel()])


def test_keys_match_a_real_adam_state_dict_after_one_step():
    net = _net('tictactoe_net')
    opt = torch.optim.Adam(net.parameters(), lr=1e-3, weight_decay=1e-5)
    sum(o.float().sum() for o in net(torch.randn(2, 3, 3, 3), None).values() if o is not None).backward()
    opt.step()
    real = opt.state_dict()
    fmt = _format(net)
    d = fmt.to_dict(*_flat_state(fmt, 3), 1, 1e-3, 8.0, 1)['optimizer']
    assert list(d) == list(real)
    assert len(d['param_groups']) == len(real['param_groups']) == 1
    assert d['param_groups'][0] == real['param_groups'][0]
    assert sorted(d['state']) == sorted(real['state'])
    for i, s in real['state'].items():
        assert list(d['state'][i]) == list(s)
        for k, t in s.items():
            assert d['state'][i][k].dtype == t.dtype and d['state'][i][k].shape == t.shape, (i, k)
    assert torch.equal(d['state'][0]['step'], real['state'][0]['step'])


@pytest.mark.parametrize('saved_step', [0, 3, 500])
def test_a_torch_adam_step_from_the_saved_state_matches_the_learners_step(saved_step):
    """From the same saved state and gradient: torch.optim.Adam with the gradient clipped to norm 4 on the CPU, and the oracle
    of the learner's clip + Adam kernel on the flat state.  The oracle reads the step count the file holds as the number of
    steps already taken (bias correction at t = step + 1), as torch does."""
    from oracle import oracle
    net = _net('tictactoe_net')
    fmt = _format(net)
    m, v = _flat_state(fmt, 4)
    lr = float(np.float32(1e-3))
    d = fmt.to_dict(m, v, saved_step, lr, 16.0, saved_step)
    g = torch.Generator().manual_seed(5)
    grads = [torch.randn(p.shape, generator=g) for p in net.parameters()]      # norm ~ 170: clipped to 4
    flat_p = torch.zeros(fmt.n_pad)
    flat_g = torch.zeros(fmt.n_pad)
    for p, gr, off in zip(net.parameters(), grads, fmt.offsets):
        flat_p[off:off + p.numel()] = p.detach().reshape(-1)
        flat_g[off:off + p.numel()] = gr.reshape(-1)

    ref = copy.deepcopy(net)
    opt = torch.optim.Adam(ref.parameters(), lr=3e-8, weight_decay=1e-5)
    opt.load_state_dict(d['optimizer'])
    for p, gr in zip(ref.parameters(), grads):
        p.grad = gr.clone()
    torch.nn.utils.clip_grad_norm_(ref.parameters(), d['max_norm'])
    opt.step()

    p_o, m_o, v_o = flat_p.numpy().copy(), m.numpy().copy(), v.numpy().copy()
    oracle.clip_adam(p_o, flat_g.numpy().copy(), m_o, v_o, lr, saved_step, max_norm=d['max_norm'])
    got = torch.cat([p.detach().reshape(-1) for p in ref.parameters()]).numpy()
    assert np.abs(got - p_o[:fmt.n]).max() <= 1e-6
    after = opt.state_dict()['state']
    assert float(after[0]['step']) == saved_step + 1
    for name, arr in (('exp_avg', m_o), ('exp_avg_sq', v_o)):
        mine = torch.cat([after[i][name].reshape(-1) for i in range(len(fmt.names))]).numpy()
        assert np.abs(mine - arr[:fmt.n]).max() <= 1e-6 * max(1.0, np.abs(arr).max()), name


def _target(fmt):
    """What load_optimizer_state writes to, on the CPU: the flat moments, the step counter, lr and the data-count average."""
    opt = types.SimpleNamespace(exp_avg=torch.full((fmt.n_pad,), 0.25), exp_avg_sq=torch.full((fmt.n_pad,), 0.5),
                                step_count=torch.full((1,), 9, dtype=torch.int64), lr=torch.full((1,), 1e-3),
                                betas=fmt.betas, eps=fmt.eps)
    return types.SimpleNamespace(opt=opt, ema=torch.full((1,), 64.0), optim_format=fmt, schedule_steps=9, _captured=False)


def _snapshot(t):
    return [x.clone() for x in (t.opt.exp_avg, t.opt.exp_avg_sq, t.opt.step_count, t.opt.lr, t.ema)] + [t.schedule_steps]


def _same(a, b):
    return all(torch.equal(x, y) for x, y in zip(a[:-1], b[:-1])) and a[-1] == b[-1]


def _mismatches(d):
    """(description, exception type, broken copy of d) for every way a dict may not fit the learner."""
    out = []

    def case(what, exc, edit):
        bad = copy.deepcopy(d)
        edit(bad)
        out.append((what, exc, bad))

    names = d['param_names']
    case('a name missing', KeyError, lambda b: b['param_names'].__setitem__(0, 'nope.weight'))
    case('a name extra', KeyError, lambda b: b['param_names'].append('extra.weight'))
    case('no state for a parameter', KeyError, lambda b: b['optimizer']['state'].pop(len(names) - 1))
    case('no schedule', KeyError, lambda b: b.pop('schedule'))
    case('a shape', ValueError, lambda b: b['optimizer']['state'][1].__setitem__('exp_avg', torch.zeros(3)))
    case('a shape', ValueError,
         lambda b: b['optimizer']['state'][2].__setitem__('exp_avg_sq', b['optimizer']['state'][2]['exp_avg_sq'].reshape(1, -1)))
    case('betas', ValueError, lambda b: b['optimizer']['param_groups'][0].__setitem__('betas', (0.8, 0.999)))
    case('eps', ValueError, lambda b: b['optimizer']['param_groups'][0].__setitem__('eps', 1e-6))
    case('weight_decay', ValueError, lambda b: b['optimizer']['param_groups'][0].__setitem__('weight_decay', 0.0))
    case('max_norm', ValueError, lambda b: b.__setitem__('max_norm', 1.0))
    case('step counts differ', ValueError, lambda b: b['optimizer']['state'][3].__setitem__('step', torch.tensor(2.0)))
    return out


@pytest.mark.parametrize('name', NETS)
def test_every_mismatch_raises_and_leaves_the_target_unchanged(name):
    from handyrl_b200.train import LearnerStep
    net = _net(name)
    fmt = _format(net)
    m, v = _flat_state(fmt, 6)
    d = fmt.to_dict(m, v, 12, 2e-4, 40.0, 12)
    cases = _mismatches(d)
    assert len(cases) == 11
    t = _target(fmt)
    before = _snapshot(t)
    for what, exc, bad in cases:
        with pytest.raises(exc):
            LearnerStep.load_optimizer_state(t, bad)
        assert _same(_snapshot(t), before), what
    # the intact dict loads; after a step or warm_up a load is refused
    LearnerStep.load_optimizer_state(t, d)
    assert torch.equal(t.opt.exp_avg, m) and torch.equal(t.opt.exp_avg_sq, v)
    assert int(t.opt.step_count) == 12 and float(t.opt.lr) == float(np.float32(2e-4)) and float(t.ema) == 40.0
    assert t.schedule_steps == 12
    t._captured = True
    with pytest.raises(RuntimeError):
        LearnerStep.load_optimizer_state(t, fmt.to_dict(v, m, 1, 1e-3, 8.0, 1))
    assert torch.equal(t.opt.exp_avg, m)


def test_a_learner_with_other_settings_refuses_the_dict():
    from handyrl_b200.train import OptimizerStateFormat
    net = _net('tictactoe_net')
    d = _format(net).to_dict(*_flat_state(_format(net), 7), 1, 1e-3, 8.0, 1)
    for kw in ({'betas': (0.9, 0.99)}, {'eps': 1e-7}, {'weight_decay': 1e-4}, {'max_norm': 2.0}):
        with pytest.raises(ValueError):
            OptimizerStateFormat(net.named_parameters(), **kw).unpack(d)


# ---------------------------------------------------------------------------------------------------------------- files
class _Epoch(PendingModel):
    """Stands in for the PendingModel of one epoch: what resolve() hands back, with its averaged and optimiser states."""

    def __init__(self, dcnt, tag):        # (no device copy to wait for)
        self.dcnt, self.tag, self.batch_cnt = dcnt, tag, 1
        self.ema_state = {'w': torch.full((2,), float(tag))}
        self.optim_state = {'schedule': {'steps': tag}}

    def resolve(self):
        return 'model%d' % self.tag, {'dcnt': self.dcnt}


def _trainer_with_epochs(epochs, **extra):
    from handyrl_b200.train import Trainer
    tr = Trainer(dict(ARGS, **extra), torch.nn.Identity())
    tr.update_queue = queue.Queue()
    for i, e in enumerate(epochs):
        tr.update_queue.put((e, 10 * (i + 1)))
    return tr


@pytest.mark.parametrize('with_average', [False, True], ids=['optim', 'optim+ema'])
def test_files_share_the_numbering_across_skipped_epochs(with_average, tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    extra = {'save_optimizer': True}
    if with_average:
        extra['weight_ema'] = 0.9
    # epochs 2, 4 and 5 have no sample with a turn in them: update() skips them, and they get no number
    tr = _trainer_with_epochs([_Epoch(5, 1), _Epoch(0, 2), _Epoch(3, 3), _Epoch(0, 4), _Epoch(0, 5), _Epoch(7, 6)], **extra)
    assert (tr.ema_files is tr.optim_files) == with_average
    assert [tr.update() for _ in range(3)] == [('model1', 10), ('model3', 30), ('model6', 60)]
    want = ['1.optim.pth', '2.optim.pth', '3.optim.pth', 'latest.optim.pth']
    if with_average:
        want += ['1.ema.pth', '2.ema.pth', '3.ema.pth', 'latest.ema.pth']
    assert sorted(os.listdir('models')) == sorted(want)
    for epoch, tag in ((1, 1), (2, 3), (3, 6), ('latest', 6)):
        assert torch.load(os.path.join('models', '%s.optim.pth' % epoch))['schedule']['steps'] == tag
        if with_average:            # <e>.ema.pth and <e>.optim.pth come from the same epoch
            assert torch.equal(torch.load(os.path.join('models', '%s.ema.pth' % epoch))['w'], torch.full((2,), float(tag)))


def test_a_restarted_run_continues_the_numbering_and_finds_its_file(tmp_path, monkeypatch):
    from handyrl_b200.train import AveragedCheckpoints
    monkeypatch.chdir(tmp_path)
    assert AveragedCheckpoints(7).seed_path('optim') is None
    os.makedirs('models')
    torch.save({'w': torch.zeros(2)}, os.path.join('models', '7.ema.pth'))
    assert AveragedCheckpoints(7).seed_path('optim') is None               # an average alone is not an optimiser state
    torch.save({'schedule': {'steps': 70}}, os.path.join('models', '7.optim.pth'))
    assert AveragedCheckpoints(7).seed_path('optim') == os.path.join('models', '7.optim.pth')
    assert AveragedCheckpoints(7, suffix='optim').seed_path() == os.path.join('models', '7.optim.pth')
    assert AveragedCheckpoints(0).seed_path('optim') is None                # restart_epoch 0 never resumes
    tr = _trainer_with_epochs([_Epoch(0, 1), _Epoch(2, 2), _Epoch(2, 3)], save_optimizer=True, weight_ema=0.99, restart_epoch=7)
    tr.update()
    tr.update()
    assert sorted(os.listdir('models')) == ['7.ema.pth', '7.optim.pth', '8.ema.pth', '8.optim.pth', '9.ema.pth', '9.optim.pth',
                                            'latest.ema.pth', 'latest.optim.pth']
    assert torch.load(os.path.join('models', '8.optim.pth'))['schedule']['steps'] == 2


def test_without_the_key_nothing_is_written(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    for extra in ({}, {'save_optimizer': False}):
        tr = _trainer_with_epochs([_Epoch(3, 1)], **extra)
        assert tr.optim_files is None and tr.checkpoint_files is None
        assert tr.update() == ('model1', 10)
        assert not os.path.exists('models')
