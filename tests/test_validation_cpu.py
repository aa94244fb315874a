"""Held-out validation loss without a GPU: the content-based membership rule, the key's checks, the printed lines, and the C ABI
mirror of the forward-only loss kernel."""
import math
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADS = ['p', 'v', 'ent', 'total']


def _episodes(n, seed=0):
    from handyrl_b200.synthetic import tictactoe_episodes
    return tictactoe_episodes(n, seed=seed)


def _decisions(episodes, rate):
    from handyrl_b200.replay import held_out
    from handyrl_b200.wire import episode_to_flat
    return [held_out(episode_to_flat(ep), rate) for ep in episodes]


def test_membership_is_deterministic_across_interpreters():
    eps = _episodes(200, seed=3)
    here = _decisions(eps, 0.3)
    assert here == _decisions(eps, 0.3)
    # a fresh interpreter (another hash() salt) decides the same
    code = ('import sys; sys.path[:0] = [%r, %r]\n'
            'from test_validation_cpu import _episodes, _decisions\n'
            'print("".join("1" if d else "0" for d in _decisions(_episodes(200, seed=3), 0.3)))' % (ROOT, os.path.join(ROOT, 'tests')))
    env = dict(os.environ, PYTHONHASHSEED='12345')
    out = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, check=True, env=env, cwd=ROOT)
    assert out.stdout.strip() == ''.join('1' if d else '0' for d in here)
    assert 0 < sum(here) < len(here)


def test_membership_is_the_same_for_both_wire_formats():
    from handyrl_b200.wire import pack_episode
    eps = _episodes(100, seed=5)
    ref = _decisions(eps, 0.5)
    assert _decisions([pack_episode(ep) for ep in eps], 0.5) == ref
    assert _decisions([pack_episode(ep, drop_moments=True) for ep in eps], 0.5) == ref


def test_membership_is_monotone_in_the_rate_and_off_at_zero():
    eps = _episodes(100, seed=7)
    small, large = _decisions(eps, 0.1), _decisions(eps, 0.4)
    assert all(b for a, b in zip(small, large) if a)          # held out at r: held out at any r' > r
    assert not any(_decisions(eps, 0)) and not any(_decisions(eps, None))


@pytest.mark.parametrize('rate', [0.05, 0.3])
def test_held_out_fraction_is_within_a_binomial_bound(rate):
    eps = _episodes(3000, seed=11)
    from handyrl_b200.wire import episode_to_flat
    from handyrl_b200.replay import held_out
    fes = [episode_to_flat(ep) for ep in eps]
    # identical games are one decision: count distinct contents
    distinct = {}
    for fe in fes:
        key = (fe.action.tobytes(), fe.prob.tobytes(), fe.turn.tobytes(), fe.outcome.tobytes())
        distinct[key] = held_out(fe, rate)
    n = len(distinct)
    k = sum(distinct.values())
    assert n > 1000
    assert abs(k - n * rate) <= 5 * math.sqrt(n * rate * (1 - rate)), (k, n, rate)


@pytest.mark.parametrize('value', [1, 1.0, -0.1, 1.5, 'x', True, float('nan')])
def test_rates_outside_the_open_interval_are_refused(value):
    from handyrl_b200.train import validation_rate
    with pytest.raises(ValueError):
        validation_rate({'validation_rate': value})


def test_rate_off_and_needs_the_gpu_replay():
    from handyrl_b200.train import validation_rate
    assert validation_rate({}) is None
    assert validation_rate({'validation_rate': None}) is None
    assert validation_rate({'validation_rate': 0}) is None
    assert validation_rate({'validation_rate': 0.05}) == 0.05
    assert validation_rate({'validation_rate': 0.05, 'gpu_replay': True}) == 0.05
    with pytest.raises(ValueError):
        validation_rate({'validation_rate': 0.05, 'gpu_replay': False})
    assert validation_rate({'validation_rate': 0, 'gpu_replay': False}) is None


def test_trainer_and_learner_step_refuse_a_bad_key():
    """Both constructors check the key before touching a device."""
    import torch
    from handyrl_b200.train import LearnerStep, Trainer
    from handyrl_b200.nets import tictactoe_net
    args = {'batch_size': 4, 'forward_steps': 4, 'gpu_replay': True}
    for bad in ({'validation_rate': 2.0}, {'validation_rate': 0.1, 'gpu_replay': False}):
        with pytest.raises(ValueError):
            Trainer(dict(args, **bad), tictactoe_net())
        with pytest.raises(ValueError):
            LearnerStep(torch.nn.Linear(2, 2), dict(args, **bad), None, lr=1e-3)


def test_validation_lines_and_loss_plot_does_not_take_them():
    from handyrl_b200.train import loss_line
    sums = {'p': 51.2, 'v': 23.1, 'r': 0.0, 'ent': 184.3, 'total': 56.1, 'dcnt': 100.0}
    assert loss_line('validation', sums, HEADS) == 'validation = p:0.512 v:0.231 ent:1.843 total:0.561'
    assert loss_line('validation_ema', sums, HEADS) == 'validation_ema = p:0.512 v:0.231 ent:1.843 total:0.561'
    assert loss_line('loss', sums, HEADS) == 'loss = ' + ' '.join(k + ':' + '%.3f' % (sums[k] / 100.0) for k in HEADS)
    for name in ('validation', 'validation_ema'):
        line = loss_line(name, sums, HEADS)
        assert not line.startswith('loss')          # the reference's scripts/loss_plot.py takes line.startswith('loss')
        m = re.fullmatch(r'(\w+) = ((?:\w+:-?[0-9.]+ ?)+)', line)
        assert m and m.group(1) == name


def test_binding_mirrors_the_header():
    from handyrl_b200 import _capi
    assert 'hrl_loss_fwd' in _capi.SYMBOLS
    assert _capi.SYMBOLS['hrl_loss_fwd'] == _capi.SYMBOLS['hrl_loss_fwd_bwd']
    header = open(os.path.join(ROOT, 'include', 'hrl_b200.h')).read()
    assert re.search(r'\bint hrl_loss_fwd\(const HrlLossArgs \*args, void \*stream\);', header)
    assert _capi.HRL_ABI_VERSION == 3 and '#define HRL_ABI_VERSION 3' in header


def test_loss_fwd_refuses_cpu_tensors():
    from handyrl_b200 import ops, _capi
    from handyrl_b200.synthetic import synthetic_batch, synthetic_outputs
    args = {'turn_based_training': True, 'observation': False, 'gamma': 0.8, 'lambda': 0.7, 'burn_in_steps': 0,
            'entropy_regularization': 0.1, 'entropy_regularization_decay': 0.1, 'policy_target': 'UPGO', 'value_target': 'VTRACE'}
    batch = synthetic_batch(4, 8, 2, 9, seed=0, with_obs=False)
    outs = synthetic_outputs(batch, seed=1)
    with pytest.raises(_capi.HrlError):
        ops.loss_fwd(outs, batch, args)
