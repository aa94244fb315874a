"""Learner diagnostics without a GPU: the float64 reference on a batch with known answers, the host-side summary, and the C ABI
mirror of the new symbols and indices."""
import os
import re
import subprocess
import tempfile

import numpy as np

from diag_oracle import diagnostics

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARGS = {'turn_based_training': False, 'observation': False, 'gamma': 0.8, 'lambda': 0.7, 'burn_in_steps': 0,
        'entropy_regularization': 0.1, 'entropy_regularization_decay': 0.1, 'policy_target': 'MC', 'value_target': 'MC'}


def known_batch(B=2, T=3, P=2, A=4):
    """Uniform pi (zero logits, no illegal action), mu = 1/2 on even steps and 1/8 on odd ones, every player acts and observes.
    MC without a return head: value target = outcome, advantage = (outcome - value) + return (losses.py:64-66)."""
    mu = np.where(np.arange(T)[None, :, None, None] % 2 == 0, 0.5, 0.125) * np.ones((B, T, P, 1))
    ret = np.arange(B * T * P, dtype=np.float64).reshape(B, T, P, 1) / 10.0
    batch = {
        'action_mask': np.zeros((B, T, P, A)), 'action': np.zeros((B, T, P, 1), np.int64), 'selected_prob': mu,
        'reward': np.zeros((B, T, P, 1)), 'return': ret, 'turn_mask': np.ones((B, T, P, 1)),
        'observation_mask': np.ones((B, T, P, 1)), 'episode_mask': np.ones((B, T, 1, 1)), 'progress': np.zeros((B, T, 1)),
        'outcome': np.arange(B * P, dtype=np.float64).reshape(B, 1, P, 1) / 4.0,
    }
    value = np.broadcast_to(0.5 * batch['outcome'] + 0.1, (B, T, P, 1)).copy()   # err = 0.5 outcome - 0.1: explained variance 0.75
    outs = {'policy': np.zeros((B, T, P, A)), 'value': value}
    return batch, outs


def test_oracle_on_a_batch_with_known_answers():
    from handyrl_b200 import ops
    batch, outs = known_batch()
    s, near = diagnostics(batch, outs, ARGS)
    d = dict(zip(ops.DIAG_KEYS, s))
    n = 2 * 3 * 2
    assert d['n_pol'] == n and d['n_val'] == n and near == 0
    # rho = (1/4) / mu: 0.5 on even steps (two of three), 2 on odd ones
    assert np.isclose(d['rho'], n / 3 * (2 * 0.5 + 2.0))
    assert d['rho_clip'] == n / 3
    assert np.isclose(d['logr'], n / 3 * (2 * np.log(0.5) + np.log(2.0)))
    summ = ops.summarize_diagnostics(s)
    assert np.isclose(summ['rho'], 1.0) and np.isclose(summ['clip'], 1 / 3)
    assert np.isclose(summ['kl'], np.log(2) / 3)
    assert np.isclose(summ['ev_v'], 0.75)
    ret, val, oc = batch['return'][..., 0], outs['value'][..., 0], batch['outcome'][..., 0]
    assert np.isclose(d['adv'], ((oc - val + ret) * np.minimum(0.25 / batch['selected_prob'][..., 0], 1)).sum())
    assert 'ev_r' not in summ and 'gnorm' not in summ


def test_summary_never_divides_by_zero():
    from handyrl_b200 import ops
    assert ops.summarize_diagnostics([0.0] * ops.NUM_DIAG) == {}
    assert ops.summarize_diagnostics({}) == {}
    s = dict.fromkeys(ops.DIAG_KEYS, 0.0)
    s.update(gnorm=10.0, gnorm2=52.0, gclip=1.0, steps=2.0)
    out = ops.summarize_diagnostics(s)
    assert out == {'gnorm': 5.0, 'gnorm_sd': 1.0, 'gclip': 0.5}
    # a value head whose target is constant: no explained variance, but the policy-side fields are there
    s = dict.fromkeys(ops.DIAG_KEYS, 0.0)
    s.update(n_pol=4.0, rho=4.0, n_val=4.0, tv=4.0, tv2=4.0, ev=1.0, ev2=1.0)
    out = ops.summarize_diagnostics(s)
    assert 'ev_v' not in out and out['rho'] == 1.0 and out['clip'] == 0.0
    # a shorter vector (the loss pass's entries only) is padded with zeros
    assert ops.summarize_diagnostics([4.0, 8.0]) == ops.summarize_diagnostics(dict(n_pol=4.0, rho=8.0))


def test_diagnostics_line_is_parseable():
    from handyrl_b200 import ops
    line = ops.format_diagnostics({'rho': 1.0244, 'clip': 0.318, 'kl': 0.041, 'adv': 0.002, 'adv_sd': 0.437, 'ev_v': 0.612,
                                   'gnorm': 57.3, 'gclip': 1.0})
    assert line == 'diagnostics = rho:1.024 clip:0.318 kl:0.041 adv:0.002 adv_sd:0.437 ev_v:0.612 gnorm:57.3 gclip:1.000'
    m = re.fullmatch(r'diagnostics = ((?:\w+:-?[0-9.e+-]+ ?)+)', line)
    assert m and dict(kv.split(':') for kv in m.group(1).split())['gnorm'] == '57.3'


def test_diag_indices_and_symbols_mirror_the_header():
    from handyrl_b200 import _capi
    for name in ('hrl_loss_fwd_bwd_diag', 'hrl_loss_diag_workspace_bytes', 'hrl_clip_adam_step'):
        assert name in _capi.SYMBOLS
    names = ['HRL_DIAG_' + k.upper() for k in _capi.DIAG_KEYS]
    src = ('#include <stdio.h>\n#include "hrl_b200.h"\nint main(){' + ''.join('printf("%%d\\n", (int)%s);' % n for n in names) +
           'printf("%d\\n%d\\n", (int)HRL_NUM_LOSS_DIAG, (int)HRL_NUM_DIAG); return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, 'd.c')
        open(c, 'w').write(src)
        exe = os.path.join(d, 'd')
        subprocess.run(['gcc', '-I', os.path.join(ROOT, 'include'), c, '-o', exe], check=True)
        got = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    assert got == list(range(_capi.NUM_DIAG)) + [_capi.NUM_LOSS_DIAG, _capi.NUM_DIAG]


def test_diag_workspace_is_a_superset_of_the_plain_one():
    import __graft_entry__ as g
    g.build()
    from handyrl_b200._capi import lib
    for B in (1, 7, 512):
        plain = lib().hrl_loss_workspace_bytes(B, 32, 2, 1, 9)
        assert lib().hrl_loss_diag_workspace_bytes(B, 32, 2, 1, 9) >= plain + 8 * B * 16 * 4
