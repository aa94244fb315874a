"""Categorical value heads on the GPU (train_args['value_bins']): the expectation and cross-entropy kernels against the float64
reference, their bits under repeats and graph replays, the fused loss pass with a head left to them, three learner steps
against a float64 CPU learner, and how the key composes with gradient accumulation, prioritised replay, diagnostics, the
non-finite guard, validation, distillation and the GPU replay."""
import copy
import math
import os
import pickle

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from conftest import GOLDEN

pytestmark = pytest.mark.gpu

with open(os.path.join(GOLDEN, 'step_cases.pkl'), 'rb') as f:
    STEP_CASES = pickle.load(f)
with open(os.path.join(GOLDEN, 'rnn_cases.pkl'), 'rb') as f:
    RNN_CASES = pickle.load(f)

ARGS = {'gamma': 0.8, 'lambda': 0.7, 'entropy_regularization': 0.1, 'entropy_regularization_decay': 0.1,
        'policy_target': 'UPGO', 'value_target': 'VTRACE'}


@pytest.fixture(autouse=True)
def default_precision_flags():
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _spec(K, low=-1.0, high=1.0, symlog=False, sigma=0.0):
    return {'bins': K, 'low': float(low), 'high': float(high), 'symlog': symlog, 'sigma': float(sigma)}


def _cuda(tree):
    return {k: v.cuda() for k, v in tree.items()}


# ----------------------------------------------------------------------------------------------------------- expectation

@pytest.mark.parametrize('K', [2, 3, 51, 256, 1024])
@pytest.mark.parametrize('symlog', [False, True])
def test_expectation_matches_float64(K, symlog):
    from handyrl_b200 import ops, value_bins
    spec = _spec(K, -3.0, 5.0, symlog=symlog)
    g = torch.Generator().manual_seed(K)
    z = torch.randn(7, 5, 2, K, generator=g) * 4
    z[0, 0, 0] = 0.0
    z[0, 0, 0, K - 1] = 80.0                    # saturated rows: all mass on one bin
    z[0, 1, 1] = -80.0
    z[0, 1, 1, 0] = 80.0
    z[1, 2, 0] = 80.0                           # equal huge logits: the plain mean of the centres
    got = ops.value_bins_expect(z.cuda(), spec, P=2)
    torch.cuda.synchronize()
    ref = torch.from_numpy(value_bins.expectation(z.double().numpy(), spec))
    got = got.cpu().double().squeeze(-1)
    tol = 2e-6 * max(abs(spec['low']), abs(spec['high'])) * (1 + ref.abs()) * (math.exp(max(abs(spec['low']), abs(spec['high']))) if symlog else 1)
    assert bool(((got - ref).abs() <= tol).all()), float((got - ref).abs().max())
    want_top = math.expm1(5.0) if symlog else 5.0
    assert float(got[0, 0, 0]) == pytest.approx(want_top, rel=1e-5)


# ----------------------------------------------------------------------------------------------------------- cross-entropy

CE_CASES = {    # name: P, Pa, T, burn_in, sigma (in bins), symlog, weights
    'alt_p2': (2, 1, 6, 0, 0.0, False, False),
    'pa_eq_p2': (2, 2, 6, 3, 0.75, True, True),
    'alt_p4': (4, 1, 5, 3, 0.0, True, True),
    'pa_eq_p4': (4, 4, 5, 0, 0.75, False, True),
    'solo': (1, 1, 4, 0, 0.75, False, False),
    't1': (2, 2, 1, 0, 0.0, False, True),
    'alt_t1': (4, 1, 1, 0, 0.75, True, False),
}


def _ce_case(name, K=51, B=24, seed=0):
    from handyrl_b200 import ops
    P, Pa, T, bi, sig, symlog, weights = CE_CASES[name]
    low, high = (-3.0, 3.0) if symlog else (-1.0, 1.0)
    spec = _spec(K, low, high, symlog, sig * (high - low) / (K - 1))
    g = torch.Generator().manual_seed(seed + K)
    z = torch.randn(B, T, Pa, K, generator=g) * 3
    y = torch.randn(B, T, P, 1, generator=g) * 2.5 * (8 if symlog else 1)         # many targets outside the support
    om = (torch.rand(B, T, P, 1, generator=g) > 0.25).float()
    w = (torch.rand(B, generator=g) * 2).float() if weights else None
    buf = ops.LossBuffers(B, T, P, Pa, 3, True, False, 'cuda', value_bins={'value': spec})
    ops.bins_targets(buf)['value'].copy_(y)
    batch = {'observation_mask': om.cuda()}
    args = {'burn_in_steps': bi}
    return spec, z, y, om, w, buf, batch, args


def _ce(z, spec, batch, args, buf, w=None, forward_only=False):
    from handyrl_b200 import ops
    buf.losses.zero_()
    return ops.value_bins_fwd_bwd(z, 'value', spec, batch, args, buf, window_weight=w, forward_only=forward_only)


@pytest.mark.parametrize('name', sorted(CE_CASES))
@pytest.mark.parametrize('K', [51, 7])
def test_cross_entropy_matches_the_reference(name, K):
    from handyrl_b200 import value_bins
    spec, z, y, om, w, buf, batch, args = _ce_case(name, K)
    from handyrl_b200 import ops
    zc = z.cuda()
    wc = w.cuda() if w is not None else None
    buf.losses.zero_()
    buf.losses[4] = 2.5         # the pass adds to the total
    dz = ops.value_bins_fwd_bwd(zc, 'value', spec, batch, args, buf, window_weight=wc)
    torch.cuda.synchronize()
    ref = value_bins.reference(z, y, om, spec, burn_in=args['burn_in_steps'], window_weight=w)
    L = float(buf.losses[1])
    assert L == pytest.approx(ref['loss'], rel=1e-5, abs=1e-5)
    assert float(buf.losses[4]) == pytest.approx(2.5 + L, rel=1e-6)
    assert float(buf.losses[0]) == 0 and float(buf.losses[2]) == 0
    wmax = 1.0 if w is None else float(w.max())
    scale = wmax * (CE_CASES[name][0] if CE_CASES[name][1] == 1 else 1)
    err = float((dz.cpu().double() - ref['dz']).abs().max())
    assert err <= 1e-6 * scale, (err, scale)
    bi, T = args['burn_in_steps'], z.shape[1]
    if bi > 0 and T > 1:
        assert bool((dz[:, :bi] == 0).all())
    # the forward-only form: the same sums as the form with the gradient, when both are unweighted
    full = _ce(zc, spec, batch, args, buf).clone()
    s_full = buf.losses.clone()
    _ce(zc, spec, batch, args, buf, forward_only=True)
    torch.cuda.synchronize()
    assert torch.equal(buf.losses, s_full)
    assert full.shape == z.shape


@pytest.mark.parametrize('name', ['alt_p2', 'pa_eq_p2'])
def test_unit_weights_are_null_and_repeats_and_replays_are_bit_identical(name):
    from handyrl_b200 import ops
    spec, z, y, om, w, buf, batch, args = _ce_case(name, 51, seed=3)
    zc = z.cuda()
    ones = torch.ones(z.shape[0], device='cuda')
    a = _ce(zc, spec, batch, args, buf).clone()
    la = buf.losses.clone()
    b = _ce(zc, spec, batch, args, buf, ones).clone()
    lb = buf.losses.clone()
    assert torch.equal(a, b) and torch.equal(la, lb)
    results = []
    for _ in range(2):
        buf.losses.zero_()
        ops.value_bins_fwd_bwd(zc, 'value', spec, batch, args, buf)
        torch.cuda.synchronize()
        results.append((buf.losses.clone(), buf.dlogits['value'].clone()))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            buf.losses.zero_()
            ops.value_bins_fwd_bwd(zc, 'value', spec, batch, args, buf)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        results.append((buf.losses.clone(), buf.dlogits['value'].clone()))
    for r in results:
        assert torch.equal(r[0], la) and torch.equal(r[1], a)


def test_refusals():
    from handyrl_b200 import ops
    from handyrl_b200._capi import HrlError
    spec, z, y, om, w, buf, batch, args = _ce_case('alt_p2', 51)
    with pytest.raises(ValueError, match='51 bins'):
        ops.value_bins_fwd_bwd(z[..., :7].contiguous().cuda(), 'value', spec, batch, args, buf)
    with pytest.raises(HrlError, match='contiguous'):
        ops.value_bins_expect(z.cuda().transpose(0, 1), spec)
    with pytest.raises(HrlError, match='K=1025'):
        ops.value_bins_expect(torch.zeros(1, 1, 1, 1025, device='cuda'), _spec(1025))


# ----------------------------------------------------------------------------------------------------------- the loss pass

VARIANTS = ['rows-direct', 'rows-staged', 'bulk', 'element', 'group']


@pytest.mark.parametrize('A', [9, 384])
@pytest.mark.parametrize('form', ['fwd_bwd', 'diag', 'fwd'])
@pytest.mark.parametrize('heads', [1, 2, 3])
def test_external_heads_leave_the_rest_of_the_pass_bit_identical(A, form, heads):
    from handyrl_b200 import ops
    from handyrl_b200.synthetic import synthetic_batch, synthetic_outputs
    B, T, P = (16, 8, 2) if A == 9 else (8, 8, 2)
    batch = _cuda(synthetic_batch(B, T, P, A, turn_based=True, observation=A == 9, seed=4, with_obs=False))
    outs = _cuda(synthetic_outputs(batch, has_return=True, seed=5))
    Pa = outs['policy'].shape[2]
    args = dict(ARGS, turn_based_training=True, burn_in_steps=2)
    cat = {h: _spec(5) for bit, h in ((1, 'value'), (2, 'return')) if heads & bit}
    for variant in VARIANTS:
        tuning = {'variant': variant}
        got = []
        for bins in (None, cat):
            buf = ops.LossBuffers(B, T, P, Pa, A, True, True, 'cuda', taps=True, grads=form != 'fwd', value_bins=bins,
                                  diagnostics=form == 'diag')
            if form == 'fwd':
                ops.loss_fwd(outs, batch, args, buffers=buf, tuning=tuning)
            else:
                ops.loss_fwd_bwd(outs, batch, args, buffers=buf, tuning=tuning, diagnostics=form == 'diag')
            torch.cuda.synchronize()
            got.append(buf)
        plain, ext = got
        for i in (0, 3, 5):
            assert torch.equal(plain.losses[i], ext.losses[i]), (variant, i)
        term = 0.0
        for i, bit in ((1, 1), (2, 2)):
            if heads & bit:
                assert float(ext.losses[i]) == 0.0
                term += float(plain.losses[i])
            else:
                assert torch.equal(plain.losses[i], ext.losses[i])
        assert float(ext.losses[4]) == pytest.approx(float(plain.losses[4]) - term, rel=1e-6, abs=1e-5 * (1 + abs(term)))
        for k in plain.taps:
            assert torch.equal(plain.taps[k], ext.taps[k]), (variant, k)
        if form != 'fwd':
            assert torch.equal(plain.dpolicy, ext.dpolicy), variant
            assert (ext.dvalue is None) == bool(heads & 1) and (ext.dreturn is None) == bool(heads & 2)
            if not heads & 1:
                assert torch.equal(plain.dvalue, ext.dvalue)
            if not heads & 2:
                assert torch.equal(plain.dreturn, ext.dreturn)
        if form == 'diag':
            assert torch.equal(plain.diagnostics, ext.diagnostics), variant


def test_external_head_needs_its_target_tap_and_no_gradient():
    import ctypes as C
    from handyrl_b200 import _capi, ops
    from handyrl_b200.synthetic import synthetic_batch, synthetic_outputs
    batch = _cuda(synthetic_batch(4, 4, 2, 9, seed=1, with_obs=False))
    outs = _cuda(synthetic_outputs(batch, seed=2))
    buf = ops.LossBuffers(4, 4, 2, 1, 9, True, False, 'cuda', value_bins={'value': _spec(5)})
    ops.loss_fwd_bwd(outs, batch, dict(ARGS, turn_based_training=True), buffers=buf)
    a = buf._cached_fwd_bwd[1]
    bad = type(a).from_buffer_copy(a)
    bad.tap_target_value = None
    assert _capi.lib().hrl_loss_fwd_bwd(C.byref(bad), ops._stream_ptr()) == -1
    bad.tap_target_value = a.tap_target_value
    bad.dvalue_raw = buf.dpolicy.data_ptr()
    assert _capi.lib().hrl_loss_fwd_bwd(C.byref(bad), ops._stream_ptr()) == -1
    bad.dvalue_raw = None
    bad.external_heads = 4
    assert _capi.lib().hrl_loss_fwd_bwd(C.byref(bad), ops._stream_ptr()) == -1
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------------------------- learner steps

class CatBoardNet(nn.Module):
    """A TicTacToe-shaped feed-forward net (3 planes on 3x3, 9 actions) whose value head outputs K logits."""

    def __init__(self, bins=51, width=16):
        super().__init__()
        self.conv1 = nn.Conv2d(3, width, 3, padding=1)
        self.conv2 = nn.Conv2d(width, width, 3, padding=1)
        self.p_out = nn.Linear(9 * width, 9)
        self.v_out = nn.Linear(9 * width, bins)

    def forward(self, x, hidden=None):
        h = F.relu(self.conv2(F.relu(self.conv1(x)))).flatten(1)
        return {'policy': self.p_out(h), 'value': self.v_out(h)}


class CatGatedNet(nn.Module):
    """The small recurrent net of nets.GatedBoardNet with both heads categorical."""

    def __init__(self, value_bins=21, return_bins=31):
        super().__init__()
        from handyrl_b200.nets import GatedBoardNet
        self.core = GatedBoardNet()
        cells = 16 * self.core.width
        self.core.v_out = nn.Linear(cells, value_bins)
        self.core.r_out = nn.Linear(cells, return_bins)

    def init_hidden(self, batch_size=None):
        return self.core.init_hidden(batch_size)

    def forward(self, x, hidden):
        c = self.core
        s = c.embed(x['scalar'])[:, :, None, None].expand(-1, -1, *c.board)
        h_in = F.relu(c.norm(c.inp(torch.cat([x['board'], s], 1))))
        h, cs = hidden
        i, f, o, g = c.gates(torch.cat([h_in, h], 1)).chunk(4, 1)
        cs = torch.sigmoid(f) * cs + torch.sigmoid(i) * torch.tanh(g)
        h = torch.sigmoid(o) * torch.tanh(cs)
        flat = h.flatten(1)
        return {'policy': c.p_out(flat), 'value': c.v_out(flat), 'return': c.r_out(flat), 'hidden': (h, cs)}


def _board_batch(s):
    from handyrl_b200.synthetic import synthetic_batch
    c = STEP_CASES['alt']
    B, T, P, A = c['dims']
    return synthetic_batch(B, T, P, A, turn_based=c['args']['turn_based_training'], observation=c['args']['observation'], seed=40 + s)


def _rnn_batch(s):
    from handyrl_b200.batch import tree_map
    c = RNN_CASES[sorted(RNN_CASES)[0]]
    batch = tree_map(lambda a: torch.from_numpy(a).clone(), c['batch'])
    if s:
        g = torch.Generator().manual_seed(s)
        batch['observation'] = tree_map(lambda o: o + 0.1 * torch.randn(o.shape, generator=g), batch['observation'])
    return batch


def _setups():
    return {
        'board': (lambda: CatBoardNet(51), _board_batch, dict(STEP_CASES['alt']['args']),
                  {'value': {'bins': 51, 'low': -1.0, 'high': 1.0}}),
        'gated': (CatGatedNet, _rnn_batch, dict(RNN_CASES[sorted(RNN_CASES)[0]]['args']),
                  {'value': {'bins': 21, 'low': -1.0, 'high': 1.0, 'sigma': 0.075},
                   'return': {'bins': 31, 'low': -3.0, 'high': 3.0, 'symlog': True, 'sigma': 0.15}}),
    }


def _targets(raw, batch, args):
    """targets['value'] / targets['return'] of oracle/torch_learner.loss_from_raw, from its own target code, on heads that
    are already the expectations (B, T, Pa, 1); returned (B, T', P) after the burn-in cut."""
    from oracle.torch_learner import _target
    bi = args.get('burn_in_steps', 0)

    def cut(x):
        return x[:, bi:] if (bi > 0 and x.size(1) > 1) else x
    tm4, om4 = batch['turn_mask'], batch['observation_mask']
    pol = raw['policy'] * tm4
    if pol.size(2) > 1 and batch['action'].size(2) == 1:
        pol = pol.sum(2, keepdim=True)
    pol = cut(pol - batch['action_mask'])
    heads = {k: cut(raw[k] * om4) for k in ('value', 'return') if k in raw}
    om = cut(om4).squeeze(-1)
    em = cut(batch['episode_mask']).squeeze(-1)
    act, mu = cut(batch['action']), cut(batch['selected_prob'])
    oc = batch['outcome'].squeeze(-1)
    rew, ret = cut(batch['reward']).squeeze(-1), cut(batch['return']).squeeze(-1)
    logp = F.log_softmax(pol, -1).gather(-1, act).squeeze(-1) * em
    rho = torch.exp(logp - torch.log(mu.clamp(1e-16, 1)).squeeze(-1) * em).clamp(0, 1)
    out = {}
    if 'value' in heads:
        v = heads['value'].squeeze(-1)
        v_mask = om
        if args['turn_based_training'] and v.size(2) == 2:
            v_opp, om_opp = -v.flip(2), om.flip(2)
            v = (v * om + v_opp * om_opp) / (om + om_opp + 1e-8)
            v_mask = (om + om_opp).clamp(0, 1)
        out['value'] = _target(args['value_target'], v * em + oc * (1 - em), oc, None, args['lambda'], 1.0, rho, rho, v_mask)[0]
    if 'return' in heads:
        out['return'] = _target(args['value_target'], heads['return'].squeeze(-1), ret, rew, args['lambda'], args['gamma'],
                                rho, rho, om)[0]
    return {k: v.expand_as(om) for k, v in out.items()}


def _reference_step(net, opt, batch, args, bins):
    """One float64 step of the law on the host: forward, the expectations in place of the categorical heads for the loss and
    the targets, the cross-entropy against their two-hot / HL-Gauss distributions, autograd, clip 4.0, Adam."""
    from handyrl_b200 import value_bins
    from oracle.torch_learner import _walk, loss_from_raw, recurrent_raw_outputs
    B, T, Pa = batch['action'].shape[:3]
    P = batch['turn_mask'].shape[2]
    if hasattr(net, 'init_hidden'):
        raw = recurrent_raw_outputs(net, _walk(lambda h: h.double(), net.init_hidden([B, P])), batch, args)
    else:
        outs = net(_walk(lambda o: o.flatten(0, 2), batch['observation']), None)
        raw = {k: v.unflatten(0, (B, T, Pa)) for k, v in outs.items() if v is not None and k != 'hidden'}
    fed = dict(raw)
    for h, spec in bins.items():
        fed[h] = torch.from_numpy(value_bins.expectation(raw[h].detach().numpy(), spec)).unsqueeze(-1)
    losses, _ = loss_from_raw(fed, batch, args)
    tg = _targets(fed, batch, args)
    bi = args.get('burn_in_steps', 0)
    total = losses['total']
    for h, spec in bins.items():
        total = total - losses['v' if h == 'value' else 'r']
        z = raw[h][:, bi:] if (bi > 0 and T > 1) else raw[h]
        om = batch['observation_mask'][:, bi:] if (bi > 0 and T > 1) else batch['observation_mask']
        pi = torch.from_numpy(value_bins.target_distribution(tg[h].detach().numpy(), spec))
        lp = F.log_softmax(z, -1)
        lp = lp.expand(-1, -1, P, -1) if z.size(2) == 1 else lp
        total = total + (om * -(pi * lp).sum(-1, keepdim=True)).sum()
    opt.zero_grad()
    total.backward()
    torch.nn.utils.clip_grad_norm_(list(net.parameters()), 4.0)
    opt.step()
    return float(total.detach())


@pytest.mark.parametrize('use_graph', [False, True], ids=['eager', 'graph'])
@pytest.mark.parametrize('which', ['board', 'gated'])
def test_three_learner_steps_match_a_float64_learner(which, use_graph):
    from handyrl_b200.batch import tree_map
    from handyrl_b200.train import LearnerStep
    make, batch_fn, args, bins = _setups()[which]
    torch.manual_seed(1)
    net = make()
    ref = copy.deepcopy(net).double()
    opt = torch.optim.Adam(ref.parameters(), lr=1e-3, weight_decay=1e-5)
    stepper = LearnerStep(net, dict(args, value_bins=bins), batch_fn(0), lr=1e-3, use_graph=use_graph)
    assert stepper.engine is None
    for s in range(3):
        batch = batch_fn(s)
        b64 = tree_map(lambda t: t.double() if t.is_floating_point() else t, batch)
        ref_total = _reference_step(ref, opt, b64, args, value_bins_config(bins))
        stepper.step(stepper.new_packed().fill(batch))
        got = stepper.read_losses()
        assert got['total'] == pytest.approx(ref_total, rel=1e-4, abs=1e-4), s
    state = stepper.cpu_state_dict()
    for k, v in ref.state_dict().items():
        # the bias of the convolution that feeds BatchNorm has a gradient of exactly 0: its Adam steps follow rounding noise
        # (conftest.noise_driven), and only that BatchNorm's running mean sees it
        if v.is_floating_point() and k not in ('core.inp.bias', 'core.norm.running_mean'):
            np.testing.assert_allclose(state[k].double().numpy(), v.numpy(), rtol=1e-4, atol=2e-5, err_msg=k)


def value_bins_config(bins):
    from handyrl_b200 import value_bins
    return value_bins.config({'value_bins': bins})


def _stepper(which, steps=1, **extra):
    from handyrl_b200.train import LearnerStep
    make, batch_fn, args, bins = _setups()[which]
    torch.manual_seed(1)
    stepper = LearnerStep(make(), dict(args, value_bins=bins, **extra), batch_fn(0), lr=1e-3)
    for s in range(steps):
        stepper.step(stepper.new_packed().fill(batch_fn(s)))
    stepper.stream.synchronize()
    return stepper


def test_launches_and_the_net_check():
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.train import LearnerStep
    on = _stepper('board')
    make, batch_fn, args, bins = _setups()['board']
    assert on.launches_per_step > 0
    assert float(on.loss_accum[1]) > 0      # the cross-entropy took the value head's place
    # a one-output tanh head (the fused tower's BoardNet) is refused at warm-up; a missing head when built
    torch.manual_seed(1)
    stepper = LearnerStep(tictactoe_net(), dict(args, value_bins=bins), batch_fn(0), lr=1e-3)
    with pytest.raises(ValueError, match='51 bins'):
        stepper.warm_up()
    with pytest.raises(ValueError, match="no 'return' head"):
        LearnerStep(make(), dict(args, value_bins={'return': bins['value']}), batch_fn(0), lr=1e-3)


def test_gradient_accumulation_matches_one_micro_batch():
    one = _stepper('board', steps=2)
    two = _stepper('board', steps=2, gradient_accumulation=2)
    a, b = one.cpu_state_dict(), two.cpu_state_dict()
    for k in a:
        if a[k].is_floating_point():
            torch.testing.assert_close(b[k], a[k], rtol=1e-4, atol=2e-5, msg=k)
    torch.testing.assert_close(two.loss_accum, one.loss_accum, rtol=1e-5, atol=1e-5)


def test_prioritised_replay_and_diagnostics_together():
    st = _stepper('board', steps=2, diagnostics=True, prioritized_replay={'alpha': 0.6, 'beta': 0.4}, maximum_episodes=64)
    assert st.prio_state is not None and st.diag_accum is not None
    assert bool(torch.isfinite(st.accum).all())
    assert float(st.diag_accum[7]) > 0          # n_val: the value-fit sums, on the expectation


def test_nonfinite_value_logit_is_rejected():
    from handyrl_b200.train import LearnerStep
    make, batch_fn, args, bins = _setups()['board']
    torch.manual_seed(1)
    net = make()
    with torch.no_grad():
        net.v_out.bias[3] = float('nan')
    stepper = LearnerStep(net, dict(args, value_bins=bins, skip_nonfinite=True), batch_fn(0), lr=1e-3)
    for s in range(2):
        stepper.step(stepper.new_packed().fill(batch_fn(s)))
    stepper.stream.synchronize()
    assert int(stepper.skipped) == 2 and int(stepper.opt.step_count) == 0


def test_validation_equals_the_training_forward_sums():
    from handyrl_b200.train import LearnerStep
    make, batch_fn, args, bins = _setups()['board']
    torch.manual_seed(1)
    stepper = LearnerStep(make(), dict(args, value_bins=bins), batch_fn(0), lr=1e-3, validation=True)
    stepper.warm_up()
    packed = stepper.new_packed().fill(batch_fn(1))
    stepper.dev_buffer.copy_(packed.buffer.to('cuda'))
    torch.cuda.synchronize()
    stepper.validate_in_place()
    val = stepper.pop_validation()['validation']
    stepper.step(packed)
    got = stepper.read_losses()
    stepper.stream.synchronize()
    for k in ('p', 'v', 'ent', 'total'):
        assert val[k] == pytest.approx(got[k], rel=1e-6, abs=1e-6), k
    assert val['v'] > 0


def test_distillation_adds_only_its_own_term(tmp_path):
    make, batch_fn, args, bins = _setups()['board']
    torch.manual_seed(11)
    path = str(tmp_path / 'teacher.pth')
    torch.save(make().state_dict(), path)
    off = _stepper('board', steps=1)
    on = _stepper('board', steps=1, distill={'teacher': path, 'coef': 0.0})
    assert torch.equal(on.loss_accum, off.loss_accum)
    on = _stepper('board', steps=1, distill={'teacher': path, 'coef': 0.5})
    kl, term = on.distill_accum.tolist()
    assert kl > 0 and term == pytest.approx(0.5 * kl, rel=1e-6)
    for i in (0, 1, 3, 5):
        assert float(on.loss_accum[i]) == float(off.loss_accum[i]), i
    assert float(on.loss_accum[4]) == pytest.approx(float(off.loss_accum[4]) + term, rel=1e-5)


def test_episodes_with_value_logits_train_through_the_gpu_replay():
    from handyrl_b200.batch import reduce_values
    from handyrl_b200.replay import DeviceReplay
    from handyrl_b200 import value_bins
    from handyrl_b200.wire import episode_to_flat
    from test_value_bins_cpu import _moments
    import bz2
    bins = value_bins.config({'value_bins': {'value': {'bins': 51, 'low': -1.0, 'high': 1.0}}})
    eps = []
    for seed in range(4):
        m = _moments(51, steps=8, seed=seed)
        eps.append({'moment': [bz2.compress(pickle.dumps(m))], 'outcome': {0: 1.0, 1: -1.0}, 'steps': 8, 'args': {}})
    replay = DeviceReplay(256, 16, device='cuda')
    fes = [reduce_values(episode_to_flat(ep), bins) for ep in eps]
    replay.add_flat_many(fes)
    torch.cuda.synchronize()
    got = replay.st_value[:32].cpu().numpy()
    want = np.concatenate([fe.value[..., 0] for fe in fes])
    np.testing.assert_array_equal(got, want)
    with pytest.raises(ValueError, match='scalar'):
        DeviceReplay(256, 16, device='cuda').add_flat_many([episode_to_flat(eps[0])])
