"""The LAMB optimiser without a GPU: the train_args key, the chunk plan of hrl_lamb_plan on the reference nets' parameter
shapes, the optimiser file format, and the float64 restatement (tests/lamb_ref.py) on a hand-worked case."""
import math

import numpy as np
import pytest
import torch

from lamb_ref import lamb_step

BAD = ['sgd', 'Lamb', 'LAMB', 'adamw', '', 0, 1, True, ['lamb'], {'name': 'adam'}, {}, {'lr_scale': 2.0},
       {'name': 'lamb', 'lr': 1.0}, {'name': 'lamb', 'lr_scale': 0.0}, {'name': 'lamb', 'lr_scale': -1.0},
       {'name': 'lamb', 'lr_scale': float('nan')}, {'name': 'lamb', 'lr_scale': float('inf')},
       {'name': 'lamb', 'lr_scale': True}, {'name': 'lamb', 'lr_scale': '2'}, {'name': 'lamb', 'lr_scale': None}]


# ---------------------------------------------------------------- the key


def test_absent_none_and_adam_mean_adam():
    from handyrl_b200.train import optimizer_config
    for value in (None, 'adam'):
        assert optimizer_config(value) == {'name': 'adam'}


def test_both_lamb_forms_are_accepted():
    from handyrl_b200.train import optimizer_config
    assert optimizer_config('lamb') == {'name': 'lamb', 'lr_scale': 1.0}
    assert optimizer_config({'name': 'lamb'}) == {'name': 'lamb', 'lr_scale': 1.0}
    assert optimizer_config({'name': 'lamb', 'lr_scale': 30}) == {'name': 'lamb', 'lr_scale': 30.0}
    assert optimizer_config({'name': 'lamb', 'lr_scale': 2.5e-3}) == {'name': 'lamb', 'lr_scale': 2.5e-3}


@pytest.mark.parametrize('value', BAD, ids=[repr(v) for v in BAD])
def test_bad_values_raise_at_build(value):
    """optimizer_config, LearnerStep and Trainer all refuse the value before they touch a device or the net."""
    from handyrl_b200.train import LearnerStep, Trainer, optimizer_config
    with pytest.raises(ValueError):
        optimizer_config(value)
    with pytest.raises(ValueError):
        LearnerStep(None, {'optimizer': value}, None, lr=1e-3)
    with pytest.raises(ValueError):
        LearnerStep(None, {}, None, lr=1e-3, optimizer=value)
    with pytest.raises(ValueError):
        Trainer({'optimizer': value}, None)


# ---------------------------------------------------------------- the chunk plan


def _nets():
    from handyrl_b200 import nets
    torch.manual_seed(0)
    return {'tictactoe': nets.tictactoe_net(), 'geister': nets.geister_net(), 'geese': nets.geese_net()}


@pytest.mark.parametrize('name', ['tictactoe', 'geister', 'geese'])
def test_plan_covers_every_word_of_every_tensor_once(name):
    from handyrl_b200.ops import lamb_plan
    numels = [p.numel() for p in _nets()[name].parameters()]
    offsets = np.cumsum([0] + numels)
    n = int(offsets[-1])
    plan = lamb_plan(numels).numpy()
    assert plan.ndim == 2 and plan.shape[1] == 5
    seen = np.zeros(n + 3, np.int64)           # + the padding words up to a multiple of 4: never in a chunk
    first_of = {}
    for c, (start, length, tensor, first, count) in enumerate(plan):
        assert 0 < length <= 1024
        assert offsets[tensor] <= start and start + length <= offsets[tensor + 1], 'chunk %d crosses tensor %d' % (c, tensor)
        first_of.setdefault(tensor, c)
        assert first == first_of[tensor] and count == math.ceil(numels[tensor] / 1024)
        assert (plan[first:first + count, 2] == tensor).all()
        seen[start:start + length] += 1
    assert (seen[:n] == 1).all() and (seen[n:] == 0).all()
    assert sorted(first_of) == list(range(len(numels)))
    assert list(plan[:, 0]) == sorted(plan[:, 0])                    # chunks in bucket order
    assert len(plan) == sum(math.ceil(k / 1024) for k in numels)


def test_plan_refuses_empty_tensors():
    from handyrl_b200 import _capi
    from handyrl_b200.ops import lamb_plan
    with pytest.raises(_capi.HrlError):
        lamb_plan([3, 0, 5])
    with pytest.raises(_capi.HrlError):
        lamb_plan([])


# ---------------------------------------------------------------- the file format


def _format(optimizer=None):
    from handyrl_b200.train import OptimizerStateFormat
    net = _nets()['tictactoe']
    kw = {} if optimizer is None else {'optimizer': optimizer}
    return OptimizerStateFormat(net.named_parameters(), **kw)


def _dict(fmt):
    m = torch.arange(fmt.n_pad, dtype=torch.float32)
    return fmt.to_dict(m, m + 1, 7, 1e-3, 512.0, 7)


def test_lamb_dict_carries_the_algorithm_and_adam_dict_keeps_todays_keys():
    from handyrl_b200.train import optimizer_config
    adam = _dict(_format())
    assert sorted(adam) == ['max_norm', 'optimizer', 'param_names', 'schedule']
    assert sorted(_dict(_format(optimizer_config('adam')))) == sorted(adam)
    lamb = _dict(_format(optimizer_config({'name': 'lamb', 'lr_scale': 20.0})))
    assert lamb['algorithm'] == 'lamb' and lamb['lr_scale'] == 20.0
    assert sorted(lamb) == sorted(list(adam) + ['algorithm', 'lr_scale'])
    for i, s in adam['optimizer']['state'].items():                  # the moments and the step mean the same thing
        for k in s:
            assert torch.equal(s[k], lamb['optimizer']['state'][i][k])
    assert lamb['optimizer']['param_groups'] == adam['optimizer']['param_groups']


def test_cross_loading_raises_and_lr_scale_is_not_compared():
    from handyrl_b200.train import optimizer_config
    adam_fmt = _format()
    lamb_fmt = _format(optimizer_config('lamb'))
    adam, lamb = _dict(adam_fmt), _dict(_format(optimizer_config({'name': 'lamb', 'lr_scale': 3.0})))
    with pytest.raises(ValueError, match='lamb'):
        adam_fmt.unpack(lamb)
    with pytest.raises(ValueError, match='adam'):
        lamb_fmt.unpack(adam)
    m, v, step, lr, ema, steps = lamb_fmt.unpack(lamb)                 # lr_scale 3.0 into a learner of 1.0
    assert torch.equal(m[:lamb_fmt.n], torch.arange(lamb_fmt.n, dtype=torch.float32)) and step == 7


# ---------------------------------------------------------------- the float64 restatement


def test_restatement_on_a_hand_worked_two_tensor_case():
    """t = 1 from zero moments, so u = g' / (|g'| + eps) elementwise.  Tensor 0 is all zero (r = 1); tensor 1 has no gradient
    and no decay (u = 0, r = 1, w unchanged); tensor 2 has |w| = 5 and u = +-1 / (1 + 1e-8), so r |u| = 5 / sqrt(2)."""
    lr, eps = 1e-2, 1e-8
    ws = [np.zeros(2), np.array([2.0]), np.array([3.0, 4.0])]
    gs = [np.array([3.0, 4.0]), np.array([0.0]), np.array([1.0, -1.0])]
    zeros = [np.zeros_like(w) for w in ws]
    w, m, v, r, norm = lamb_step(ws, gs, zeros, zeros, 1, lr, weight_decay=0.0, eps=eps)
    assert norm == pytest.approx(math.sqrt(27.0), rel=1e-15)
    c = 4.0 / (math.sqrt(27.0) + 1e-6)                                # clip active: |g| = 5.196 > 4
    assert r[0] == 1.0 and r[1] == 1.0
    assert r[2] == pytest.approx(5.0 * (1 + eps / c) / math.sqrt(2.0), rel=1e-12)
    np.testing.assert_allclose(w[0], [-lr * 3 * c / (3 * c + eps), -lr * 4 * c / (4 * c + eps)], rtol=1e-14)
    np.testing.assert_allclose(w[0], [-lr, -lr], rtol=1e-8)
    assert w[1][0] == 2.0
    np.testing.assert_allclose(w[2], [3.0 - lr * 5 / math.sqrt(2.0), 4.0 + lr * 5 / math.sqrt(2.0)], rtol=1e-14)
    np.testing.assert_allclose(m[2], [0.1 * c, -0.1 * c], rtol=1e-14)
    np.testing.assert_allclose(v[2], [1e-3 * c * c, 1e-3 * c * c], rtol=1e-12)
    assert m[1][0] == 0.0 and v[1][0] == 0.0
    # lr_scale multiplies the step and nothing else
    w2, _, _, r2, _ = lamb_step(ws, gs, zeros, zeros, 1, lr, lr_scale=3.0, weight_decay=0.0, eps=eps)
    assert r2 == r
    np.testing.assert_allclose(w2[2] - ws[2], 3.0 * (w[2] - ws[2]), rtol=1e-12)


def test_restatement_adds_the_decay_to_the_update_not_the_gradient():
    """With a zero gradient and zero moments u = wd * w, so r = 1 / wd and the tensor shrinks by lr * |w| / |w| * w."""
    lr, wd = 1e-2, 1e-5
    w0 = np.array([0.6, -0.8])
    w, m, v, r, _ = lamb_step([w0], [np.zeros(2)], [np.zeros(2)], [np.zeros(2)], 3, lr, weight_decay=wd)
    assert (m[0] == 0).all() and (v[0] == 0).all()
    assert r[0] == pytest.approx(1.0 / wd, rel=1e-12)
    np.testing.assert_allclose(w[0], w0 * (1 - lr), rtol=1e-12)
