"""CPU checks of categorical value heads (train_args['value_bins'], value_bins.py): the key's parsing, the target distributions,
the float64 reference against autograd, the replay's ingest, the drop-in compute_loss refusal and the C struct layout."""
import ctypes
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from handyrl_b200 import value_bins

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

TWO_HOT = {'bins': 51, 'low': -1.0, 'high': 1.0}
HL_GAUSS = {'bins': 101, 'low': -8.0, 'high': 8.0, 'symlog': True, 'sigma': 0.12}


# ----------------------------------------------------------------------------------------------------------- the key

@pytest.mark.parametrize('value', [None, False, 0, 0.0])
def test_off_forms(value):
    assert value_bins.config({}) is None
    assert value_bins.config({'value_bins': value}) is None


def test_defaults_and_values():
    got = value_bins.config({'value_bins': {'value': TWO_HOT, 'return': HL_GAUSS}})
    assert got == {'value': {'bins': 51, 'low': -1.0, 'high': 1.0, 'symlog': False, 'sigma': 0.0},
                   'return': {'bins': 101, 'low': -8.0, 'high': 8.0, 'symlog': True, 'sigma': 0.12}}
    got = value_bins.config({'value_bins': {'return': {'bins': 2, 'low': 0, 'high': 1}}})
    assert list(got) == ['return'] and got['return']['bins'] == 2 and isinstance(got['return']['low'], float)
    assert value_bins.config({'value_bins': {'value': {'bins': 1024, 'low': -1, 'high': 1}}})['value']['bins'] == 1024


@pytest.mark.parametrize('value', [True, 1, 'yes', [], {}, {'policy': TWO_HOT}, {'value': TWO_HOT, 'values': TWO_HOT},
                                   {'value': 51}, {'value': True}])
def test_other_values_raise(value):
    with pytest.raises(ValueError, match='value_bins'):
        value_bins.config({'value_bins': value})


@pytest.mark.parametrize('spec', [
    {'bins': 1, 'low': -1, 'high': 1}, {'bins': 1025, 'low': -1, 'high': 1}, {'bins': 51.0, 'low': -1, 'high': 1},
    {'bins': True, 'low': -1, 'high': 1}, {'bins': 51, 'low': 1, 'high': 1}, {'bins': 51, 'low': 2, 'high': 1},
    {'bins': 51, 'low': float('-inf'), 'high': 1}, {'bins': 51, 'low': -1, 'high': float('nan')},
    {'bins': 51, 'low': True, 'high': 2}, {'bins': 51, 'low': '0', 'high': 1}, {'bins': 51, 'high': 1},
    {'bins': 51, 'low': -1, 'high': 1, 'symlog': 1}, {'bins': 51, 'low': -1, 'high': 1, 'sigma': -0.1},
    {'bins': 51, 'low': -1, 'high': 1, 'sigma': float('inf')}, {'bins': 51, 'low': -1, 'high': 1, 'sigma': True},
    {'bins': 51, 'low': -1, 'high': 1, 'width': 1},
])
def test_bad_entries_raise(spec):
    with pytest.raises(ValueError, match='value_bins'):
        value_bins.config({'value_bins': {'value': spec}})


# ----------------------------------------------------------------------------------------------------------- targets

@pytest.mark.parametrize('spec', [TWO_HOT, {'bins': 2, 'low': -1, 'high': 1}, {'bins': 7, 'low': -3, 'high': 5, 'symlog': True}])
def test_two_hot_reproduces_the_clamped_target(spec):
    spec = value_bins.config({'value_bins': {'value': spec}})['value']
    rng = np.random.default_rng(0)
    y = np.concatenate([rng.uniform(-12, 12, 500), [spec['low'], spec['high'], 0.0, -40.0, 40.0],
                        value_bins.symexp(value_bins.centres(spec)) if spec['symlog'] else value_bins.centres(spec)])
    pi = value_bins.target_distribution(y, spec)
    x = np.clip(value_bins.symlog(y) if spec['symlog'] else y, spec['low'], spec['high'])
    assert (pi >= -1e-12).all() and ((pi > 0).sum(-1) <= 2).all()
    np.testing.assert_allclose(pi.sum(-1), 1.0, rtol=0, atol=1e-12)
    np.testing.assert_allclose(pi @ value_bins.centres(spec), x, rtol=0, atol=1e-12)


def test_hl_gauss_sums_to_one_and_concentrates():
    spec = dict(value_bins.config({'value_bins': {'value': {'bins': 41, 'low': -2, 'high': 2}}})['value'])
    delta = 4 / 40
    y = np.linspace(-1.5, 1.5, 37)
    errs = []
    for sigma in (1.0 * delta, 0.5 * delta, 0.1 * delta, 0.02 * delta):
        spec['sigma'] = sigma
        pi = value_bins.target_distribution(y, spec)
        assert (pi >= 0).all()
        np.testing.assert_allclose(pi.sum(-1), 1.0, rtol=0, atol=1e-12)
        errs.append(np.abs(pi @ value_bins.centres(spec) - y).max())
    # the mean of the binned Gaussian approaches x as sigma -> 0: within half a bin, shrinking toward the nearest centre
    assert errs[0] < 1e-6 and all(e <= 0.5 * delta + 1e-12 for e in errs)
    spec['sigma'] = 0.5 * delta
    far = value_bins.target_distribution(np.array([50.0, -50.0]), spec)     # clamped to the support's ends
    assert far[0].argmax() == 40 and far[1].argmax() == 0


def test_expectation_matches_the_law():
    rng = np.random.default_rng(1)
    for spec in (TWO_HOT, HL_GAUSS):
        spec = value_bins.config({'value_bins': {'value': spec}})['value']
        z = rng.normal(size=(5, 3, spec['bins'])) * 4
        p = np.exp(z - z.max(-1, keepdims=True))
        p /= p.sum(-1, keepdims=True)
        m = p @ value_bins.centres(spec)
        want = np.sign(m) * (np.exp(np.abs(m)) - 1) if spec['symlog'] else m
        np.testing.assert_allclose(value_bins.expectation(z, spec), want, rtol=1e-12, atol=1e-12)
    big = np.zeros((1, 51))
    big[0, 50] = 80.0                       # saturated logits: the last centre
    assert value_bins.expectation(big, value_bins.config({'value_bins': {'value': TWO_HOT}})['value'])[0] == pytest.approx(1.0)


# ----------------------------------------------------------------------------------------------------------- reference

def _law_by_autograd(z, y, om, spec, burn_in, w):
    """The loss written out on its own: every (b, t, p) column, its row q, a plain double loop over the trained cells."""
    B, T, Pa, K = z.shape
    P = y.shape[2]
    pi = torch.from_numpy(value_bins.target_distribution(y.numpy(), spec))
    logp = torch.log_softmax(z, -1)
    total = z.new_zeros(())
    for b in range(B):
        for t in range(T):
            if burn_in > 0 and T > 1 and t < burn_in:
                continue
            for p in range(P):
                q = p if Pa == P else 0
                c = (1.0 if w is None else float(w[b])) * float(om[b, t, p])
                if c != 0:
                    total = total + c * -(pi[b, t, p] * logp[b, t, q]).sum()
    return total


@pytest.mark.parametrize('Pa, P, T, burn_in, sigma, weights', [
    (1, 2, 5, 0, 0.0, False), (2, 2, 5, 3, 0.0, True), (1, 4, 6, 3, 0.75, True), (4, 4, 1, 0, 0.75, False),
    (1, 1, 4, 0, 0.75, True), (1, 2, 1, 3, 0.0, True),
])
def test_reference_gradient_is_autograd(Pa, P, T, burn_in, sigma, weights):
    spec = value_bins.config({'value_bins': {'value': {'bins': 9, 'low': -2, 'high': 2, 'symlog': Pa == 1, 'sigma': sigma}}})['value']
    g = torch.Generator().manual_seed(Pa * 100 + P * 10 + T)
    B, K = 3, 9
    z = (torch.randn(B, T, Pa, K, generator=g, dtype=torch.float64) * 3).requires_grad_(True)
    y = torch.randn(B, T, P, generator=g, dtype=torch.float64) * 3          # some targets outside the support
    om = (torch.rand(B, T, P, generator=g) > 0.3).double()
    w = torch.rand(B, generator=g, dtype=torch.float64) * 2 if weights else None
    loss = _law_by_autograd(z, y, om, spec, burn_in, w)
    (dz_auto,) = torch.autograd.grad(loss, z)
    ref = value_bins.reference(z.detach(), y, om, spec, burn_in=burn_in, window_weight=w)
    assert ref["loss"] == pytest.approx(float(loss.detach()), rel=1e-12, abs=1e-12)
    torch.testing.assert_close(ref['dz'], dz_auto, rtol=0, atol=1e-12)
    assert ref['dz'].shape == (B, T, Pa, K) and ref['pi'].shape == (B, T, P, K) and ref['v'].shape == (B, T, Pa)
    if burn_in > 0 and T > 1:
        assert (ref['dz'][:, :burn_in] == 0).all()


# ----------------------------------------------------------------------------------------------------------- ingest

def _moments(K, steps=6, players=(0, 1), seed=0):
    rng = np.random.default_rng(seed)
    moments = []
    for s in range(steps):
        turn = players[s % len(players)]
        m = {'observation': {}, 'selected_prob': {}, 'action_mask': {}, 'action': {}, 'value': {}, 'reward': {}, 'return': {},
             'turn': [turn]}
        for p in players:
            seen = p == turn or s % 3 == 0
            m['observation'][p] = rng.normal(size=(2, 3, 3)).astype(np.float32) if seen else None
            m['value'][p] = rng.normal(size=(K,)).astype(np.float32) * 3 if seen else None
            m['selected_prob'][p] = 0.5 if p == turn else None
            m['action_mask'][p] = np.zeros(9, np.float32) if p == turn else None
            m['action'][p] = 1 if p == turn else None
            m['reward'][p] = None
            m['return'][p] = None
        moments.append(m)
    return moments


def test_ingest_reduces_logits_to_the_expectation():
    from handyrl_b200.batch import flatten_moments, reduce_values
    bins = value_bins.config({'value_bins': {'value': TWO_HOT}})
    moments = _moments(51)
    fe = flatten_moments(moments, {0: 1.0, 1: -1.0})
    assert fe.value.shape == (6, 2, 51)
    fe = reduce_values(fe, bins)
    assert fe.value.shape == (6, 2, 1) and fe.value.dtype == np.float32
    for s, m in enumerate(moments):
        for p in (0, 1):
            want = 0.0 if m['value'][p] is None else value_bins.expectation(m['value'][p], bins['value'])
            assert fe.value[s, p, 0] == pytest.approx(want, abs=1e-6)
    # scalar values, a categorical return head alone, or the key off: unchanged
    scalar = flatten_moments(_moments(1), {0: 1.0, 1: -1.0})
    assert reduce_values(scalar, bins).value.shape == (6, 2, 1)
    raw = flatten_moments(_moments(51), {0: 1.0, 1: -1.0})
    assert reduce_values(raw, None).value.shape == (6, 2, 51)
    assert reduce_values(raw, value_bins.config({'value_bins': {'return': HL_GAUSS}})).value.shape == (6, 2, 51)
    with pytest.raises(ValueError, match='bins'):
        reduce_values(flatten_moments(_moments(7), {0: 1.0, 1: -1.0}), bins)


def test_net_head_check():
    bins = value_bins.config({'value_bins': {'value': TWO_HOT}})
    value_bins.check_net_heads(bins, {'policy': torch.zeros(2, 9), 'value': torch.zeros(2, 51)})
    with pytest.raises(ValueError, match='1 value'):
        value_bins.check_net_heads(bins, {'policy': torch.zeros(2, 9), 'value': torch.zeros(2, 1)})
    with pytest.raises(ValueError, match="no 'return' head"):
        value_bins.check_net_heads(value_bins.config({'value_bins': {'return': HL_GAUSS}}),
                                   {'policy': torch.zeros(2, 9), 'value': torch.zeros(2, 1)}, bins=False)


def test_drop_in_compute_loss_refuses_the_key():
    from handyrl_b200.train import compute_loss
    with pytest.raises(ValueError, match='value_bins'):
        compute_loss({}, None, None, {'value_bins': {'value': TWO_HOT}})


# ----------------------------------------------------------------------------------------------------------- boundary

def test_struct_layout_matches_header():
    from handyrl_b200 import _capi
    fields = [('HrlValueBinsArgs', f) for f in ('K', 'burn_in', 'low', 'high', 'symlog', 'sigma', 'head', 'logits', 'expect',
                                                'target', 'observation_mask', 'window_weight', 'dlogits', 'losses', 'workspace',
                                                'workspace_bytes')] + [('HrlLossArgs', 'window_weight'), ('HrlLossArgs', 'external_heads')]
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "hrl_b200.h"\nint main(){printf("%zu\\n", sizeof(HrlValueBinsArgs));'
           'printf("%zu\\n", sizeof(HrlLossArgs));' +
           ''.join('printf("%%zu\\n", offsetof(%s, %s));' % f for f in fields) + 'return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, 's.c')
        open(c, 'w').write(src)
        exe = os.path.join(d, 's')
        subprocess.run(['gcc', '-I', os.path.join(ROOT, 'include'), c, '-o', exe], check=True)
        got = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    want = [ctypes.sizeof(_capi.HrlValueBinsArgs), ctypes.sizeof(_capi.HrlLossArgs)] + \
        [getattr(getattr(_capi, s), f).offset for s, f in fields]
    assert got == want


def test_kernels_do_not_spill():
    """Every width of both kernels (lanes per row 4, 8, 16, 32; the cross-entropy with and without its gradient) compiles for
    sm_90a without spills or a stack."""
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    if not (os.path.exists(nvcc) or shutil.which(nvcc)):
        pytest.skip('nvcc is not available')
    with tempfile.TemporaryDirectory() as d:
        cmd = [nvcc, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-c', '-Xptxas', '-v',
               '-o', os.path.join(d, 'value_bins_kernel.o'), os.path.join(ROOT, 'handyrl_b200', 'csrc', 'value_bins_kernel.cu')]
        res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    seen, cur = {}, None
    for line in res.stderr.splitlines():
        if 'Compiling entry function' in line:
            m = re.search(r'(bins_expect_kernel|bins_ce_kernel)ILi(\d+)E(Lb[01])?', line)
            cur = (m.group(1), int(m.group(2)), m.group(3)) if m else None
            continue
        s = re.search(r'(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads', line)
        if s and cur is not None:
            seen[cur] = tuple(int(x) for x in s.groups())
    want = {('bins_expect_kernel', L, None): (0, 0, 0) for L in (4, 8, 16, 32)}
    want.update({('bins_ce_kernel', L, g): (0, 0, 0) for L in (4, 8, 16, 32) for g in ('Lb0', 'Lb1')})
    assert seen == want
