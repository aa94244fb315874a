"""Policy distillation on the GPU (train_args['distill'], LearnerStep(distill=..., teacher=...)): the kernel against the float64
reference at the flagship shapes, its bits next to the fused loss kernel, graph replay and a coefficient of 0; the learner step
with a zero coefficient against the key off; the step's gradient against the reference learner with the term added; the
annealing, the prioritised weights, the non-finite guard and the teacher's shape check."""
import os
import pickle

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from test_distill_cpu import _kl_by_autograd_law

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


# ----------------------------------------------------------------------------------------------------------- the kernel

SHAPES = {      # name: B, T, P, A, turn_based, observation, burn_in
    'cfg2': (512, 32, 2, 9, True, False, 0),
    'pa_eq_p': (64, 16, 2, 9, True, True, 0),
    'cfg3_like': (32, 16, 2, 214, True, True, 4),
    'cfg4_like': (64, 16, 4, 4, False, False, 0),
    'wide': (16, 64, 2, 512, True, False, 0),
}


def _kernel_case(name, seed=0):
    from handyrl_b200.synthetic import synthetic_batch, synthetic_outputs
    B, T, P, A, tb, obs, bi = SHAPES[name]
    batch = synthetic_batch(B, T, P, A, turn_based=tb, observation=obs, burn_in=bi, seed=seed, with_obs=False)
    outs = synthetic_outputs(batch, seed=seed + 1)
    g = torch.Generator().manual_seed(seed + 2)
    teacher = outs['policy'] + 0.7 * torch.randn(outs['policy'].shape, generator=g)
    w = (torch.rand(B, generator=g) * 2).float()
    args = dict(ARGS, turn_based_training=tb, observation=obs, burn_in_steps=bi)
    return batch, outs, teacher, w, args


def _cuda(tree):
    return {k: v.cuda() for k, v in tree.items()}


def _k1(outs, batch, args, w):
    from handyrl_b200 import ops
    buf = ops.loss_fwd_bwd(outs, batch, args, window_weight=w)
    return buf


def _bound(student, teacher, batch, args, w):
    """Sum f * w * sum_a pT * (|log pT| + |log pS|) over the trained rows: the scale of the sums' rounding."""
    from handyrl_b200.distill import _epilogue
    bi = args['burn_in_steps']
    zs, zt = _epilogue(student, batch, bi), _epilogue(teacher, batch, bi)
    lps, lpt = torch.log_softmax(zs, -1), torch.log_softmax(zt, -1)
    pt = lpt.exp()
    row = (pt * (lpt.abs() + lps.abs())).nan_to_num(0.0).sum(-1)
    tm = batch['turn_mask'].double()
    tm = (tm[:, bi:] if bi > 0 and tm.size(1) > 1 else tm).squeeze(-1)
    f = tm.sum(-1, keepdim=True) if row.size(2) == 1 else tm
    return float((row * f * w.double().view(-1, 1, 1)).sum())


@pytest.mark.parametrize('name', sorted(SHAPES))
def test_kernel_matches_the_reference(name):
    from handyrl_b200 import distill, ops
    batch, outs, teacher, w, args = _kernel_case(name)
    db, do, dt, dw = _cuda(batch), _cuda(outs), teacher.cuda(), w.cuda()
    c = 0.8
    step = torch.zeros(1, dtype=torch.int64, device='cuda')
    alone = _k1(do, db, args, dw)
    losses1, dpol1 = alone.losses.clone(), alone.dpolicy.clone()
    buf = _k1(do, db, args, dw)
    sums = ops.distill_fwd_bwd(do['policy'], dt, db, args, buf, step, c, 0, window_weight=dw)
    torch.cuda.synchronize()
    kl_ref, g_ref = distill.reference(outs['policy'], teacher, batch, args, c, window_weight=w)
    # the loss pass's own sums are untouched, the total carries the term
    l1, l2 = losses1.cpu(), buf.losses.cpu()
    for i in (0, 1, 2, 3, 5):
        assert l1[i].item() == l2[i].item() or (np.isnan(l1[i].item()) and np.isnan(l2[i].item())), i
    s = sums.cpu().double()
    bound = _bound(outs['policy'], teacher, batch, args, w)
    assert abs(float(s[0]) - float(kl_ref)) <= 1e-5 * bound + 1e-6, (float(s[0]), float(kl_ref), bound)
    assert float(s[1]) == pytest.approx(c * float(s[0]), rel=1e-6)
    assert float(l2[4]) == pytest.approx(float(l1[4]) + c * float(s[0]), rel=1e-6, abs=1e-4)
    # dpolicy = the loss pass's + the reference's term, per element within 1e-5 * c * w * f^2
    bi = args['burn_in_steps']
    tm = batch['turn_mask'].double().squeeze(-1)
    f = tm.sum(-1, keepdim=True) if outs['policy'].shape[2] == 1 else tm
    tol = (1e-5 * c * w.double().view(-1, 1, 1) * f * f).unsqueeze(-1) + 1e-7 * dpol1.cpu().double().abs()
    diff = buf.dpolicy.cpu().double() - dpol1.cpu().double() - g_ref
    assert bool((diff.abs() <= tol + 1e-9).all()), float((diff.abs() - tol).max())
    if bi > 0:
        assert torch.equal(buf.dpolicy[:, :bi], dpol1[:, :bi])


@pytest.mark.parametrize('name', ['cfg2', 'cfg3_like'])
def test_graph_replays_and_repeats_are_bit_identical(name):
    from handyrl_b200 import ops
    batch, outs, teacher, w, args = _kernel_case(name, seed=5)
    db, do, dt, dw = _cuda(batch), _cuda(outs), teacher.cuda(), w.cuda()
    step = torch.full((1,), 3, dtype=torch.int64, device='cuda')
    results = []
    buf = _k1(do, db, args, dw)
    for _ in range(2):
        ops.loss_fwd_bwd(do, db, args, buffers=buf, window_weight=dw)
        ops.distill_fwd_bwd(do['policy'], dt, db, args, buf, step, 0.5, 10, window_weight=dw)
        torch.cuda.synchronize()
        results.append((buf.losses.clone(), buf.dpolicy.clone(), buf.distill_sums.clone()))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            ops.loss_fwd_bwd(do, db, args, buffers=buf, window_weight=dw)
            ops.distill_fwd_bwd(do['policy'], dt, db, args, buf, step, 0.5, 10, window_weight=dw)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        results.append((buf.losses.clone(), buf.dpolicy.clone(), buf.distill_sums.clone()))
    for r in results[1:]:
        for a, b in zip(results[0], r):
            assert torch.equal(a, b)


@pytest.mark.parametrize('coef, n, N', [(0.0, 0, 0), (1.0, 10, 10), (1.0, 25, 10)])
def test_zero_coefficient_reports_kl_and_writes_nothing(coef, n, N):
    from handyrl_b200 import distill, ops
    batch, outs, teacher, w, args = _kernel_case('cfg2', seed=7)
    db, do, dt, dw = _cuda(batch), _cuda(outs), teacher.cuda(), w.cuda()
    alone = _k1(do, db, args, dw)
    losses1, dpol1 = alone.losses.clone(), alone.dpolicy.clone()
    buf = _k1(do, db, args, dw)
    sums = ops.distill_fwd_bwd(do['policy'], dt, db, args, buf, torch.full((1,), n, dtype=torch.int64, device='cuda'),
                               coef, N, window_weight=dw)
    torch.cuda.synchronize()
    assert torch.equal(buf.losses, losses1) and torch.equal(buf.dpolicy, dpol1)
    kl_ref, _ = distill.reference(outs['policy'], teacher, batch, args, 0.0, window_weight=w)
    assert float(sums[1]) == 0.0
    assert float(sums[0]) == pytest.approx(float(kl_ref), rel=1e-5)


def test_refusals():
    from handyrl_b200 import ops
    from handyrl_b200._capi import HrlError
    batch, outs, teacher, w, args = _kernel_case('cfg4_like')
    db, do = _cuda(batch), _cuda(outs)
    buf = _k1(do, db, args, None)
    step = torch.zeros(1, dtype=torch.int64, device='cuda')
    with pytest.raises(HrlError, match='float32'):
        ops.distill_fwd_bwd(do['policy'], teacher.cuda().bfloat16(), db, args, buf, step, 1.0)
    with pytest.raises(ValueError, match='teacher policy is shaped'):
        ops.distill_fwd_bwd(do['policy'], teacher.cuda()[..., :3].contiguous(), db, args, buf, step, 1.0)


# ----------------------------------------------------------------------------------------------------------- learner steps

def _tictactoe_batch(s, name='alt'):
    from handyrl_b200.synthetic import synthetic_batch
    c = STEP_CASES[name]
    B, T, P, A = c['dims']
    return synthetic_batch(B, T, P, A, turn_based=c['args']['turn_based_training'], observation=c['args']['observation'], seed=40 + s)


def _rnn_batch(s):
    from handyrl_b200.batch import tree_map
    c = RNN_CASES[sorted(RNN_CASES)[0]]
    batch = tree_map(lambda a: torch.from_numpy(a).clone(), c['batch'])
    if s:       # other steps: the same episode layout, other observations
        g = torch.Generator().manual_seed(s)
        batch['observation'] = tree_map(lambda o: o + 0.1 * torch.randn(o.shape, generator=g), batch['observation'])
    return batch


def _geese_batch(s):
    from handyrl_b200.synthetic import synthetic_geese_batch
    return synthetic_geese_batch(8, 4, 4, 4, seed=60 + s)


def _nets():
    from handyrl_b200.nets import BoardNet, GatedBoardNet, TorusNet, tictactoe_net
    return {
        'boardnet': (tictactoe_net, _tictactoe_batch, dict(STEP_CASES['alt']['args'])),
        'torus': (lambda: TorusNet(width=16, depth=2), _geese_batch,
                  dict(ARGS, turn_based_training=False, observation=False, burn_in_steps=0, forward_steps=4)),
        'gated': (GatedBoardNet, _rnn_batch, dict(RNN_CASES[sorted(RNN_CASES)[0]]['args'])),
    }


def _seeded(make, seed):
    torch.manual_seed(seed)
    return make()


def _teacher_file(tmp_path, make, seed=11, poison=False):
    net = _seeded(make, seed)
    state = net.state_dict()
    if poison:
        k = next(k for k, v in state.items() if v.is_floating_point())
        state[k] = state[k].clone()
        state[k].view(-1)[0] = float('nan')
    path = str(tmp_path / ('teacher%d.pth' % seed))
    torch.save(state, path)
    return path


def _run(make, batch_fn, args, steps=3, **kw):
    from handyrl_b200.train import LearnerStep
    net = _seeded(make, 1)
    stepper = LearnerStep(net, args, batch_fn(0), lr=1e-3, **kw)
    out = []
    for s in range(steps):
        stepper.step(stepper.new_packed().fill(batch_fn(s)))
        out.append(stepper.read_losses())
    return stepper, out


@pytest.mark.parametrize('which', ['boardnet', 'torus', 'gated'])
def test_zero_coefficient_is_the_step_without_the_key(which, tmp_path):
    make, batch_fn, args = _nets()[which]
    off, out_off = _run(make, batch_fn, args)
    on, out_on = _run(make, batch_fn, dict(args, distill={'teacher': _teacher_file(tmp_path, make), 'coef': 0.0}))
    assert off.distill_col is None and on.distill_col is not None
    assert (off.engine is not None) == (on.engine is not None) == (which == 'boardnet')
    if which == 'torus':
        # two learners of this module-path net built alike with the key off already differ in the last bits from the second
        # step on (measured on the H100), so only the first step is compared bit for bit and the rest to fp32 rounding
        assert out_on[0] == out_off[0]
        for a, b in zip(out_on[1:], out_off[1:]):
            assert a == pytest.approx(b, rel=1e-5)
        for (k, a), (_, b) in zip(off.cpu_state_dict().items(), on.cpu_state_dict().items()):
            if not k.endswith(('conv.bias', 'bn.running_mean')):     # conftest.noise_driven: zero-gradient biases before BatchNorm
                torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5, msg=k)
    else:
        assert out_on == out_off
        for (k, a), (_, b) in zip(off.cpu_state_dict().items(), on.cpu_state_dict().items()):
            assert torch.equal(a, b), k
        assert torch.equal(on.loss_accum, off.loss_accum)
    assert float(on.distill_accum[0]) > 0 and float(on.distill_accum[1]) == 0
    assert on.launches_per_step == off.launches_per_step + on.micro_batches * (on.launches_per_teacher + 1)


def _reference_gradient(stepper, make, teacher_cpu, batch, args, c):
    """d(total + c kl) / d params of the reference learner at the learner's current state (weights and BatchNorm buffers)."""
    from handyrl_b200.train import forward_raw
    from oracle.torch_learner import _walk, loss_from_raw, recurrent_raw_outputs
    net = make()
    state = stepper.cpu_state_dict()
    net.load_state_dict({k: state[k] for k in net.state_dict()})
    net.train()
    B, T, Pa = batch['action'].shape[:3]
    P = batch['turn_mask'].shape[2]
    if hasattr(net, 'init_hidden'):
        raw = recurrent_raw_outputs(net, net.init_hidden([B, P]), batch, args)
    else:
        outs = net(_walk(lambda o: o.flatten(0, 2), batch['observation']), None)
        raw = {k: v.unflatten(0, (B, T, Pa)) for k, v in outs.items() if v is not None and k != 'hidden'}
    with torch.no_grad():
        hidden = teacher_cpu.init_hidden([B, P]) if hasattr(teacher_cpu, 'init_hidden') else None
        t_raw = forward_raw(teacher_cpu, hidden, batch, args, train=False)['policy']
    losses, _ = loss_from_raw(raw, batch, args)
    kl = _kl_by_autograd_law(raw['policy'], t_raw, batch, args, None)
    params = list(net.parameters())
    grads = torch.autograd.grad(losses['total'] + c * kl, params)
    return torch.cat([g.reshape(-1) for g in grads]).double(), float((losses['total'] + c * kl).detach())


@pytest.mark.parametrize('which, tc, tol', [('boardnet', True, 2e-3), ('boardnet', False, 2e-4), ('gated', True, 2e-3),
                                            ('narrow_teacher', True, 2e-3)])
def test_step_gradient_matches_the_reference_learner(which, tc, tol, tmp_path):
    from handyrl_b200 import distill
    from handyrl_b200.nets import BoardNet
    nets = _nets()
    make, batch_fn, args = nets['gated' if which == 'gated' else 'boardnet']
    spec = {'coef': 0.5, 'anneal_steps': 10}
    if which == 'narrow_teacher':
        small = lambda: BoardNet(width=8, depth=1)      # noqa: E731
        spec.update(teacher=_teacher_file(tmp_path, small), net='test_distill_gpu:narrow_board_net')
        teacher_make = small
    else:
        spec['teacher'] = _teacher_file(tmp_path, make)
        teacher_make = make
    teacher_cpu = teacher_make()
    teacher_cpu.load_state_dict(torch.load(spec['teacher']))
    teacher_cpu.eval()
    from handyrl_b200.train import LearnerStep
    stepper = LearnerStep(_seeded(make, 1), dict(args, distill=spec, tensor_cores=tc), batch_fn(0), lr=1e-3)
    for s in range(3):
        batch = batch_fn(s)
        n = int(stepper.opt.step_count)
        c = distill.coefficient(spec, n)
        ref, ref_total = _reference_gradient(stepper, make, teacher_cpu, batch, args, c)
        stepper.step(stepper.new_packed().fill(batch))
        got = stepper.read_losses()
        stepper.stream.synchronize()
        grad = stepper.opt.flat_grad[:stepper.opt.n].double().cpu()
        scale = float(ref.abs().max())
        assert float((grad - ref).abs().max()) <= tol * scale, (s, float((grad - ref).abs().max()), scale)
        assert got['total'] == pytest.approx(ref_total, rel=tol, abs=tol)


def narrow_board_net():
    from handyrl_b200.nets import BoardNet
    return BoardNet(width=8, depth=1)


def test_annealing_and_prioritised_weights(tmp_path):
    """term / kl is c_n at n = 0, 1, ...; with N = 4 it reaches 0 at n = 4 and stays there."""
    make, batch_fn, args = _nets()['boardnet']
    stepper, _ = _run(make, batch_fn, dict(args, distill={'teacher': _teacher_file(tmp_path, make), 'coef': 2.0, 'anneal_steps': 4}),
                      steps=0)
    for n in range(6):
        stepper.step(stepper.new_packed().fill(batch_fn(n)))
        stepper.stream.synchronize()
        kl, term = stepper.opt.extra_slots[stepper.distill_col:stepper.n_tail].tolist()
        assert kl > 0
        assert term / kl == pytest.approx(2.0 * max(0.0, 1 - n / 4), rel=1e-6, abs=1e-7), n
    # the window weights of prioritised replay multiply the term: all weights 2 give twice the sums
    from handyrl_b200 import ops
    batch = {k: v.cuda() for k, v in batch_fn(0).items() if k != 'observation'}
    outs = {'policy': torch.randn(batch['action_mask'].shape, device='cuda')}
    teacher = torch.randn(batch['action_mask'].shape, device='cuda')
    step = torch.zeros(1, dtype=torch.int64, device='cuda')
    sums = []
    for w in (None, torch.full((batch['action'].shape[0],), 2.0, device='cuda')):
        buf = ops.loss_fwd_bwd(outs, batch, args, window_weight=w)
        sums.append(ops.distill_fwd_bwd(outs['policy'], teacher, batch, args, buf, step, 1.0, window_weight=w).clone())
    torch.cuda.synchronize()
    assert torch.equal(sums[1], 2 * sums[0])


def test_gradient_accumulation_sums_the_micro_batches(tmp_path):
    """k = 2: the step's distillation sums are those of its two halves, each by the kernel alone."""
    from handyrl_b200 import ops
    make, batch_fn, args = _nets()['torus']
    spec = {'teacher': _teacher_file(tmp_path, make), 'coef': 1.0}
    stepper, _ = _run(make, batch_fn, dict(args, distill=spec, gradient_accumulation=2), steps=1)
    stepper.stream.synchronize()
    rows = stepper.loss_rows[:, stepper.distill_col:stepper.n_tail].double()
    assert torch.allclose(stepper.opt.extra_slots[stepper.distill_col:stepper.n_tail].double(), rows.sum(0), rtol=1e-6)
    assert (rows[:, 0] > 0).all()
    assert stepper.launches_per_step > 0


def test_nonfinite_teacher_is_rejected_by_the_guard(tmp_path):
    make, batch_fn, args = _nets()['torus']
    spec = {'teacher': _teacher_file(tmp_path, make, poison=True), 'coef': 1.0, 'anneal_steps': 2}
    stepper, out = _run(make, batch_fn, dict(args, distill=spec, skip_nonfinite=True), steps=3)
    before = _seeded(make, 1).state_dict()
    stepper.stream.synchronize()
    # c_n > 0 at n = 0: rejected, n stays 0, so every step is rejected
    assert int(stepper.skipped) == 3 and int(stepper.opt.step_count) == 0
    assert float(stepper.loss_accum.abs().sum()) == 0 and float(stepper.distill_accum.abs().sum()) == 0
    state = stepper.cpu_state_dict()
    for k, v in before.items():
        if v.is_floating_point():
            assert torch.equal(state[k], v), k


def test_teacher_of_another_action_count_fails_at_warm_up(tmp_path):
    from handyrl_b200.nets import BoardNet
    from handyrl_b200.train import LearnerStep
    make, batch_fn, args = _nets()['boardnet']
    other = lambda: BoardNet(actions=4)         # noqa: E731
    stepper = LearnerStep(_seeded(make, 1), args, batch_fn(0), lr=1e-3, teacher=_seeded(other, 2))
    with pytest.raises(ValueError, match='teacher policy is shaped'):
        stepper.warm_up()
