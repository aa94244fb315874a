"""CPU checks of prioritised replay (train_args['prioritized_replay']): the key, the host references of the kernels, and the
sampler's argument block against the header."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

from handyrl_b200 import priority

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------- config

@pytest.mark.parametrize('value', [None, False])
def test_off_values(value):
    assert priority.config({'prioritized_replay': value}) is None
    assert priority.config({}) is None


def test_defaults_and_overrides():
    assert priority.config({'prioritized_replay': True}) == {'alpha': 0.6, 'beta': 0.4, 'epsilon': 0.01}
    assert priority.config({'prioritized_replay': {}}) == {'alpha': 0.6, 'beta': 0.4, 'epsilon': 0.01}
    spec = priority.config({'prioritized_replay': {'alpha': 0, 'beta': 1, 'epsilon': 1e-3}, 'gpu_replay': True})
    assert spec == {'alpha': 0.0, 'beta': 1.0, 'epsilon': 1e-3}
    assert all(isinstance(v, float) for v in spec.values())


@pytest.mark.parametrize('value', [
    1, 0, 'yes', [0.6], (0.6, 0.4),                             # other values
    {'alpha': 0.6, 'gamma': 1}, {'temperature': 1}, {1: 2},     # unknown keys
    {'alpha': -0.1}, {'beta': -0.01}, {'beta': 1.5}, {'epsilon': 0}, {'epsilon': -1},       # out of range
    {'alpha': float('nan')}, {'beta': float('inf')}, {'alpha': '0.6'}, {'beta': True}, {'epsilon': None},
])
def test_malformed_values_raise(value):
    with pytest.raises(ValueError):
        priority.config({'prioritized_replay': value})


def test_needs_the_gpu_replay():
    with pytest.raises(ValueError, match='gpu_replay'):
        priority.config({'prioritized_replay': True, 'gpu_replay': False})
    assert priority.config({'prioritized_replay': False, 'gpu_replay': False}) is None


def test_trainer_raises_when_built():
    """The Trainer parses the key in its constructor (before it needs a GPU)."""
    import torch
    from handyrl_b200.train import Trainer
    args = {'prioritized_replay': {'alpha': -1}, 'batch_size': 4, 'forward_steps': 2, 'maximum_episodes': 10}
    with pytest.raises(ValueError):
        Trainer(args, torch.nn.Linear(2, 2))
    with pytest.raises(ValueError):
        Trainer(dict(args, prioritized_replay=True, gpu_replay=False), torch.nn.Linear(2, 2))


# ---------------------------------------------------------------- host references

def test_window_priorities_hand_computed():
    B, T, P = 3, 4, 2
    adv = np.zeros((B, T, P, 1), np.float32)
    tm = np.zeros((B, T, P, 1), np.float32)
    # window 0: burn-in 1; trained cells t = 1..3; turns at (1, 0), (2, 1), (3, 0)
    adv[0, :, :, 0] = [[100, 100], [1, 9], [9, -2], [-3, 9]]
    tm[0, :, :, 0] = [[1, 1], [1, 0], [0, 1], [1, 0]]
    # window 1: no trained turn -> no priority
    tm[1, 0, 0, 0] = 1
    adv[1] = 5
    # window 2: one turn
    adv[2, 2, 1, 0] = -0.5
    tm[2, 2, 1, 0] = 1
    q = priority.window_priorities(adv, tm, burn_in=1, epsilon=0.01)
    assert q[0] == pytest.approx((1 + 2 + 3) / 3 + 0.01)
    assert np.isnan(q[1])
    assert q[2] == pytest.approx(0.5 + 0.01)


def test_alpha_zero_is_the_recency_law():
    prio = np.array([5.0, 0.01, 3.0, 1e4])
    p = priority.draw_probabilities(prio, 0.0)
    np.testing.assert_allclose(p, np.arange(1, 5) / 10.0, rtol=0, atol=1e-15)


def test_draw_probabilities_hand_computed():
    prio = np.array([4.0, 1.0, 0.25])
    p = priority.draw_probabilities(prio, 0.5)
    w = np.array([1 * 2.0, 2 * 1.0, 3 * 0.5])
    np.testing.assert_allclose(p, w / w.sum(), rtol=1e-15)
    p1 = priority.draw_probabilities(prio, 1.0)
    np.testing.assert_allclose(p1, np.array([4.0, 2.0, 0.75]) / 6.75, rtol=1e-15)


def test_importance_weights():
    w = priority.importance_weights([4.0, 1.0, 1.0, 0.25], alpha=1.0, beta=0.5)
    x = np.array([0.5, 1.0, 1.0, 2.0])
    np.testing.assert_allclose(w, 4 * x / x.sum(), rtol=1e-15)
    assert w.mean() == pytest.approx(1.0)
    assert (priority.importance_weights([4.0, 1.0, 7.0], alpha=0.6, beta=0.0) == 1.0).all()
    assert (priority.importance_weights([4.0, 1.0, 7.0], alpha=0.0, beta=1.0) == 1.0).all()


def test_update_rule():
    prio = np.ones(6, np.float32)
    serial = np.array([10, 11, 12, 13, -1, 15], np.int64)
    slots = np.array([0, 2, 0, 3, 1, 4, 5])
    sers = np.array([10, 12, 10, 99, 11, -1, 15])           # window 3's serial is stale, window 5 carries no serial
    q = np.array([0.5, 2.0, 0.75, 8.0, np.nan, 9.0, 0.3])   # window 4 gives no priority
    new, mx = priority.update(prio, serial, 1.0, slots, sers, q)
    assert new[0] == np.float32(0.75)                        # duplicates resolve to the max
    assert new[2] == np.float32(2.0)
    assert new[3] == 1.0 and new[1] == 1.0 and new[4] == 1.0  # stale, no priority, no serial: untouched
    assert new[5] == np.float32(0.3)                          # a priority may fall
    assert mx == np.float32(2.0)                              # max_prio rises to the largest written
    new2, mx2 = priority.update(prio, serial, 3.0, slots, sers, q)
    assert mx2 == 3.0                                         # ...and never falls
    same, mx3 = priority.update(prio, serial, 1.0, slots, sers, q, skip=True)
    assert (same == prio).all() and mx3 == 1.0                # a rejected step writes nothing


def test_refresh_new_slots():
    prio = np.array([0.5, 0.7, 0.9], np.float32)
    ps = np.array([3, 4, -1], np.int64)
    p2, s2 = priority.refresh(prio, ps, np.array([3, 8, 9]), [0, 1, 2], 2.5)
    assert list(p2) == [0.5, 2.5, 2.5] and list(s2) == [3, 8, 9]


def test_replay_serials_and_snapshot():
    """DeviceReplay numbers every stored episode and reports the sampler's (head, count) view."""
    import torch
    from handyrl_b200.replay import DeviceReplay
    from handyrl_b200.synthetic import tictactoe_episodes
    rep = DeviceReplay(10_000, 3, device='cpu')
    eps = tictactoe_episodes(5, seed=0)
    for ep in eps:
        rep.add(ep)
    assert rep.next_serial == 5
    head, count = rep.snapshot(10)
    assert count == 3
    live = [(head + i) % 4 for i in range(count)]
    assert [int(rep._serial[s]) for s in live] == [2, 3, 4]
    assert rep.snapshot(2) == (head, 2)
    assert rep.dir_dev is None
    mir = DeviceReplay(10_000, 3, device='cpu', mirror=True)
    for ep in eps:
        mir.add(ep)
    d = mir.dir_dev.numpy()
    for s in live:
        assert list(d[s]) == list(mir._dir[s]) + [mir._serial[s]]
    assert torch.is_tensor(mir.dir_dev) and mir.dir_dev.dtype == torch.int64


# ---------------------------------------------------------------- ABI

def test_sample_args_layout_matches_header():
    from handyrl_b200 import _capi
    S = _capi.HrlReplaySampleArgs
    fields = [n for n, _ in S._fields_]
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "hrl_b200.h"\nint main(){' +
           'printf("%zu\\n", sizeof(HrlReplaySampleArgs));' +
           ''.join('printf("%%zu\\n", offsetof(HrlReplaySampleArgs, %s));' % f for f in fields) +
           'printf("%zu\\n", offsetof(HrlLossArgs, window_weight));printf("%zu\\n", sizeof(HrlLossArgs));return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, 's.c')
        open(c, 'w').write(src)
        exe = os.path.join(d, 's')
        subprocess.run(['gcc', '-I', os.path.join(ROOT, 'include'), c, '-o', exe], check=True)
        got = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    want = ([ctypes.sizeof(S)] + [getattr(S, f).offset for f in fields] +
            [_capi.HrlLossArgs.window_weight.offset, ctypes.sizeof(_capi.HrlLossArgs)])
    assert got == want, list(zip(['sizeof'] + fields + ['loss.window_weight', 'sizeof(loss)'], got, want))


def test_window_weight_is_the_last_loss_field():
    from handyrl_b200 import _capi
    assert _capi.HrlLossArgs._fields_[-1][0] == 'window_weight'
