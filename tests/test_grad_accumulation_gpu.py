"""Gradient accumulation on the GPU (train_args['gradient_accumulation'] / LearnerStep(gradient_accumulation=k)): the step of k
micro-batches against the micro-batched reference (test_grad_accumulation_cpu.micro_batched_reference), the accumulate forms
of the fused tower, determinism, the keys it composes with, memory and the Trainer."""
import copy
import gc
import os
import pickle
import threading

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from test_grad_accumulation_cpu import micro_batched_reference

pytestmark = pytest.mark.gpu

with open(os.path.join(GOLDEN, 'step_cases.pkl'), 'rb') as f:
    STEP_CASES = pickle.load(f)
with open(os.path.join(GOLDEN, 'net_step_cases.pkl'), 'rb') as f:
    NET_CASES = pickle.load(f)


@pytest.fixture(autouse=True)
def default_precision_flags():
    """PyTorch's defaults (cuDNN TF32 allowed): LearnerStep itself must switch to full fp32."""
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _grad(stepper):
    """The pre-optimiser gradient the last step left in the bucket (the optimiser reads it, never writes it)."""
    stepper.stream.synchronize()
    return stepper.opt.flat_grad[:stepper.opt.n].double().cpu()


def _tictactoe(name, s):
    from handyrl_b200.synthetic import synthetic_batch
    c = STEP_CASES[name]
    B, T, P, A = c['dims']
    return synthetic_batch(B, T, P, A, turn_based=c['args']['turn_based_training'], observation=c['args']['observation'], seed=40 + s)


def _reference_gradient(stepper, make_net, batch, args, k):
    """The micro-batched reference's pre-optimiser gradient at the learner's current state (weights and BatchNorm buffers), so
    that the gradient check does not depend on where Adam's sign-like first updates took the two trajectories."""
    net = make_net()
    state = stepper.cpu_state_dict()
    net.load_state_dict({key: state[key] for key in net.state_dict()})
    return micro_batched_reference(net, batch, args, k, torch.optim.SGD(net.parameters(), lr=0.0))[2]


def _run_tictactoe(name, k, steps=3, reference_grads=False, **kw):
    from handyrl_b200.nets import tictactoe_net, load_state_by_order
    from handyrl_b200.train import LearnerStep
    c = STEP_CASES[name]
    args = dict(c['args'], **kw.pop('args', {}))
    net = load_state_by_order(tictactoe_net(), c['state0'])
    stepper = LearnerStep(net, args, _tictactoe(name, 0), lr=c['lr'], gradient_accumulation=k, **kw)
    out = []
    for s in range(steps):
        ref = _reference_gradient(stepper, tictactoe_net, _tictactoe(name, s), c['args'], k or 1) if reference_grads else None
        stepper.step(stepper.new_packed().fill(_tictactoe(name, s)))
        out.append((stepper.read_losses(), float(stepper.opt.grad_norm), _grad(stepper)) + ((ref,) if reference_grads else ()))
    return stepper, out


def _reference_tictactoe(name, k, steps=3):
    from handyrl_b200.nets import tictactoe_net, load_state_by_order
    c = STEP_CASES[name]
    net = load_state_by_order(tictactoe_net(), c['state0'])
    opt = torch.optim.Adam(net.parameters(), lr=c['lr'], weight_decay=1e-5)
    out = [micro_batched_reference(net, _tictactoe(name, s), c['args'], k, opt) for s in range(steps)]
    return net, out


# The golden TicTacToe batches hold B = 16 windows, so at k = 4 a micro-batch is 4 windows (32 samples).  On one of them the
# learner's k = 1 step alone already differs from the float64-accurate reference by 2.7e-3 of max |g| in one element (BatchNorm
# over so few samples); the k = 4 bucket equals the sum of those four k = 1 steps to 1e-7 (test_micro_batches_add_up_to_
# their k_equals_one_steps).  The gradient bound is therefore 5e-3 of max |g| at k = 4.
GRAD_TOL_K4 = 5e-3


def _compare(got, ref, net_ref, stepper, k, loss_tol, gnorm_tol, grad_tol):
    if k == 4:
        grad_tol = max(grad_tol, GRAD_TOL_K4)
    for s, ((g_losses, g_norm, g_grad, r_grad), (r_losses, r_norm, _)) in enumerate(zip(got, ref)):
        # the two trajectories part after Adam's sign-like first updates: later steps' sums may differ by more
        scale = max(abs(v) for n, v in r_losses.items() if n != 'dcnt')
        for n, v in r_losses.items():
            if n == 'dcnt':
                assert g_losses['dcnt'] == v
            else:
                assert abs(g_losses[n] - v) <= (1 + s) * loss_tol * scale + loss_tol, (s, n, g_losses[n], v)
        assert abs(g_norm - r_norm) <= (1 + s) * gnorm_tol * r_norm, (s, g_norm, r_norm)
        scale = float(r_grad.abs().max())
        assert float((g_grad - r_grad).abs().max()) <= grad_tol * scale, (s, float((g_grad - r_grad).abs().max()), scale)
    # weights of the two independent trajectories: Adam moves an element by ~lr * sign(g) per step, and an element whose
    # gradient is near zero may take the other sign (more often than at k = 1: micro-batches of 4 windows normalise 32 samples)
    lr = STEP_CASES['alt']['lr']
    state = stepper.cpu_state_dict()
    for key, want in net_ref.state_dict().items():
        if key.endswith('num_batches_tracked'):
            assert int(state[key]) == int(want) == k * len(got), key       # k forwards per step
        else:
            np.testing.assert_allclose(state[key].numpy(), want.numpy(), rtol=1e-3, atol=2 * lr * len(got) + 5e-5, err_msg=key)


# ---------------------------------------------------------------- off is off


def test_key_absent_is_k_equals_one_bit_for_bit():
    """Absent and 1 run the same captured step: the same launches, bit-identical loss sums, gradients and weights."""
    name = sorted(STEP_CASES)[0]
    a, out_a = _run_tictactoe(name, None)
    b, out_b = _run_tictactoe(name, 1)
    assert a.micro_batches == b.micro_batches == 1 and a.launches_per_step == b.launches_per_step
    for (la, na, ga), (lb, nb, gb) in zip(out_a, out_b):
        assert la == lb and na == nb and torch.equal(ga, gb)
    for (k, va), (_, vb) in zip(a.cpu_state_dict().items(), b.cpu_state_dict().items()):
        assert torch.equal(va, vb), k


# ---------------------------------------------------------------- against the micro-batched reference


@pytest.mark.parametrize('k', [2, 4])
@pytest.mark.parametrize('name', sorted(STEP_CASES))
def test_strict_fp32_matches_the_micro_batched_reference(name, k):
    stepper, got = _run_tictactoe(name, k, reference_grads=True, args={'tensor_cores': False})
    assert stepper.engine is None and stepper.micro_batches == k
    net, ref = _reference_tictactoe(name, k)
    # (k = 4: the trajectories part at the first step -- see GRAD_TOL_K4 -- so the later sums get the 3xTF32 bounds)
    _compare(got, ref, net, stepper, k, loss_tol=2e-5 if k == 2 else 1e-4, gnorm_tol=1e-4 if k == 2 else 1e-3, grad_tol=1e-4)


@pytest.mark.parametrize('form', ['fused-graph', 'fused-eager', 'modules'])
@pytest.mark.parametrize('k', [2, 4])
@pytest.mark.parametrize('name', sorted(STEP_CASES))
def test_tensor_cores_match_the_micro_batched_reference(name, k, form):
    """3xTF32, on the fused tower (graph and eager) and on the module path, to the bounds of the whole-batch parity test."""
    stepper, got = _run_tictactoe(name, k, reference_grads=True, use_graph=form != 'fused-eager', fused_tower=form != 'modules')
    assert (stepper.engine is not None) == (form != 'modules')
    net, ref = _reference_tictactoe(name, k)
    _compare(got, ref, net, stepper, k, loss_tol=1e-4, gnorm_tol=1e-3, grad_tol=1e-3)


@pytest.mark.parametrize('name', sorted(NET_CASES))
def test_geister_and_geese_stand_ins_match_the_micro_batched_reference(name):
    """The recurrent DRC net (burn-in, hidden masking; hidden0 of B/k windows, deferred weight gradients flushed per
    micro-batch) and the torus tower, from the net_step_cases.pkl starting weights on its seeded batches, k = 2."""
    from conftest import net_case_setup, noise_driven
    from handyrl_b200.train import LearnerStep
    c = NET_CASES[name]
    k = 2
    net, batches = net_case_setup(c)
    ref_net = copy.deepcopy(net)
    stepper = LearnerStep(net, c['args'], batches[0], lr=c['lr'], gradient_accumulation=k)
    opt = torch.optim.Adam(ref_net.parameters(), lr=c['lr'], weight_decay=1e-5)
    make = lambda: copy.deepcopy(ref_net)
    for s, batch in enumerate(batches):
        r_grad = _reference_gradient(stepper, make, batch, c['args'], k)
        stepper.step(stepper.new_packed().fill(batch))
        got = stepper.read_losses()
        g_grad = _grad(stepper)
        sums, gnorm, _ = micro_batched_reference(ref_net, batch, c['args'], k, opt)
        scale = max(abs(v) for n, v in sums.items() if n != 'dcnt')
        for n, v in sums.items():
            if n == 'dcnt':
                assert got[n] == v
            else:
                assert abs(got[n] - v) <= (1 + s) * 1e-4 * scale + 1e-4, (s, n, got[n], v)
        assert abs(float(stepper.opt.grad_norm) - gnorm) <= 2e-3 * gnorm
        keep = torch.ones_like(r_grad, dtype=torch.bool)
        off = 0
        for key, p in ref_net.named_parameters():
            if noise_driven(c, key):
                keep[off:off + p.numel()] = False
            off += p.numel()
        assert float((g_grad - r_grad)[keep].abs().max()) <= 2e-3 * float(r_grad[keep].abs().max())
    final = stepper.cpu_state_dict()
    for key, vr in ref_net.state_dict().items():
        v = final[key]
        if noise_driven(c, key):
            continue
        if v.dtype.is_floating_point:
            bad = np.abs(v.numpy() - vr.numpy()) > 5e-5 + 1e-3 * np.abs(vr.numpy())
            assert bad.mean() <= 1e-3, '%s: %d of %d elements differ' % (key, bad.sum(), bad.size)
            np.testing.assert_allclose(v.numpy(), vr.numpy(), rtol=1e-3, atol=2 * c['lr'] * len(batches) + 5e-5, err_msg=key)
        else:
            assert int(v) == int(vr), key


@pytest.mark.parametrize('fused', [True, False], ids=['fused', 'modules'])
def test_micro_batches_add_up_to_their_k_equals_one_steps(fused):
    """The k = 4 bucket (gradient and loss sums) is the sum of four k = 1 steps, one on each slice, from the same state."""
    from handyrl_b200.nets import tictactoe_net, load_state_by_order
    from handyrl_b200.train import LearnerStep
    c = STEP_CASES['alt']
    batch = _tictactoe('alt', 0)
    st = LearnerStep(load_state_by_order(tictactoe_net(), c['state0']), c['args'], batch, lr=1e-3, gradient_accumulation=4,
                     fused_tower=fused)
    st.step(st.new_packed().fill(batch))
    g4, l4 = _grad(st), st.read_losses()
    total, sums = torch.zeros_like(g4), {}
    for i in range(4):
        sl = {key: v[4 * i:4 * (i + 1)].contiguous() for key, v in batch.items()}
        one = LearnerStep(load_state_by_order(tictactoe_net(), c['state0']), c['args'], sl, lr=1e-3, fused_tower=fused)
        one.step(one.new_packed().fill(sl))
        total += _grad(one)
        for n, v in one.read_losses().items():
            sums[n] = sums.get(n, 0.0) + v
    assert float((g4 - total).abs().max()) <= 1e-6 * float(total.abs().max())
    for n, v in sums.items():
        assert abs(l4[n] - v) <= 1e-6 * abs(v) + 1e-6, (n, l4[n], v)


def test_batchnorm_free_net_accumulates_to_the_full_batch_gradient():
    """nets.BoardNet(norm=False): the k = 4 bucket is the k = 1 bucket up to fp32 summation order."""
    from handyrl_b200.nets import BoardNet
    from handyrl_b200.synthetic import synthetic_batch
    from handyrl_b200.train import LearnerStep
    args = STEP_CASES['alt']['args']
    batch = synthetic_batch(64, 8, 2, 9, seed=3)
    grads, losses = [], []
    for k in (1, 4):
        torch.manual_seed(0)
        stepper = LearnerStep(BoardNet(norm=False), args, batch, lr=1e-4, gradient_accumulation=k)
        stepper.step(stepper.new_packed().fill(batch))
        grads.append(_grad(stepper))
        losses.append(stepper.read_losses())
    scale = float(grads[0].abs().max())
    assert float((grads[1] - grads[0]).abs().max()) <= 1e-5 * scale
    for n, v in losses[0].items():
        assert abs(losses[1][n] - v) <= 1e-5 * abs(v) + 1e-5, (n, losses[1][n], v)


def test_fused_tower_matches_the_module_path_parameter_by_parameter():
    """k = 4: the fused tower's accumulate forms (heads, BatchNorm finalisation, fold) against autograd over the modules."""
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.synthetic import synthetic_batch
    from handyrl_b200.train import LearnerStep
    args = STEP_CASES['alt']['args']
    batch = synthetic_batch(64, 8, 2, 9, seed=1)
    res = {}
    for fused in (True, False):
        torch.manual_seed(0)
        stepper = LearnerStep(tictactoe_net(), args, batch, lr=1e-4, fused_tower=fused, gradient_accumulation=4)
        assert (stepper.engine is not None) == fused
        stepper.step(stepper.new_packed().fill(batch))
        stepper.stream.synchronize()
        res[fused] = ({k: p.grad.detach().cpu().clone() for k, p in stepper.model.named_parameters()}, stepper.cpu_state_dict())
    for k, gf in res[True][0].items():
        gm = res[False][0][k]
        scale = max(gm.abs().max().item(), 1e-6)
        assert (gf - gm).abs().max().item() <= 1e-3 * scale, k
    for k, v in res[True][1].items():
        if 'running' in k:
            np.testing.assert_allclose(v.numpy(), res[False][1][k].numpy(), rtol=1e-5, atol=1e-6, err_msg=k)
        elif k.endswith('num_batches_tracked'):
            assert int(v) == int(res[False][1][k]) == 4


def test_two_runs_are_bit_identical_and_graph_equals_eager():
    name = sorted(STEP_CASES)[0]
    runs = [_run_tictactoe(name, 4, use_graph=g) for g in (True, True, False)]
    assert runs[0][0].launches_per_step == runs[1][0].launches_per_step
    for stepper, out in runs[1:]:
        for (la, na, ga), (lb, nb, gb) in zip(runs[0][1], out):
            assert la == lb and na == nb and torch.equal(ga, gb)
        for (k, va), (_, vb) in zip(runs[0][0].cpu_state_dict().items(), stepper.cpu_state_dict().items()):
            assert torch.equal(va, vb), k


def test_launches_per_step_count_every_micro_batch():
    """Per micro-batch the fused tower repacks its weights (one launch: the BatchNorm pivots follow the running statistics each
    forward moved), runs its forward and backward and the loss kernel; the k loss-pass sums are folded by one launch."""
    name = sorted(STEP_CASES)[0]
    one = _run_tictactoe(name, 1, steps=1)[0].launches_per_step
    two = _run_tictactoe(name, 2, steps=1)[0].launches_per_step
    four = _run_tictactoe(name, 4, steps=1)[0].launches_per_step
    per_micro = two - one - 1
    assert per_micro > 0 and four == one + 3 * per_micro + 1, (one, two, four)


# ---------------------------------------------------------------- with the other keys


def _state_image(st):
    st.stream.synchronize()
    return [t.clone() for t in (st.state.bytes, st.opt.exp_avg, st.opt.exp_avg_sq, st.opt.step_count)]


def test_nan_in_the_last_micro_batch_rejects_the_whole_step():
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.synthetic import synthetic_batch
    from handyrl_b200.train import LearnerStep
    args = dict(STEP_CASES['alt']['args'], skip_nonfinite=True)
    good, bad = synthetic_batch(16, 8, 2, 9, seed=1), synthetic_batch(16, 8, 2, 9, seed=2)
    bad['observation'][12:, 3] = float('nan')            # only micro-batch 3 of 4
    stepper = LearnerStep(tictactoe_net(), args, good, lr=1e-3, gradient_accumulation=4)
    stepper.step(stepper.new_packed().fill(good))
    before = _state_image(stepper)
    stepper.step(stepper.new_packed().fill(bad))
    after = _state_image(stepper)
    for a, b in zip(before, after):
        assert torch.equal(a, b)
    assert float(stepper.skipped) == 1.0
    stepper.step(stepper.new_packed().fill(good))
    stepper.stream.synchronize()
    assert float(stepper.skipped) == 1.0 and int(stepper.opt.step_count) == 2


def test_diagnostics_sum_the_micro_batches_loss_passes():
    """The diagnostics sums of a step are those of the k loss passes; the last one is recomputed from the fused tower's
    outputs of the last micro-batch (static buffers) by ops.loss_fwd_bwd(..., diagnostics=True)."""
    from handyrl_b200 import ops
    from handyrl_b200._capi import NUM_LOSS_DIAG
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.synthetic import synthetic_batch
    from handyrl_b200.train import LearnerStep
    args = dict(STEP_CASES['alt']['args'], diagnostics=True)
    batch = synthetic_batch(32, 8, 2, 9, seed=5)
    k = 4
    stepper = LearnerStep(tictactoe_net(), args, batch, lr=1e-3, gradient_accumulation=k, use_graph=False)
    stepper.warm_up()
    stepper.pop_diagnostics()
    stepper.step(stepper.new_packed().fill(batch))
    diag = stepper.pop_diagnostics()
    loss_pass_diag = slice(stepper.slots.diag.start, stepper.slots.diag.start + NUM_LOSS_DIAG)
    rows = stepper.loss_rows.double().cpu()
    want = rows[:, loss_pass_diag].sum(0)
    got = torch.tensor([diag[key] for key in list(diag)[:NUM_LOSS_DIAG]], dtype=torch.float64)
    torch.testing.assert_close(got, want, rtol=1e-6, atol=1e-6)
    assert diag['steps'] == 1.0
    with torch.cuda.stream(stepper.stream):
        eng = stepper.engine
        B, T, Pa = stepper._micro[-1]['action'].shape[:3]
        outs = {'policy': eng.policy.view(B, T, Pa, -1), 'value': eng.value.view(B, T, Pa, 1)}
        buf = ops.loss_fwd_bwd(outs, stepper._micro[-1], args, diagnostics=True)
        torch.cuda.current_stream().synchronize()
    assert torch.equal(buf.losses.cpu(), stepper.loss_rows[-1, stepper.slots.loss].cpu())
    assert torch.equal(buf.diagnostics[:NUM_LOSS_DIAG].cpu(), stepper.loss_rows[-1, loss_pass_diag].cpu())


def test_prioritised_replay_stores_each_windows_own_priority():
    """Window b's priority is its q_b from its own micro-batch's advantage tap, with the full batch's importance weights."""
    from handyrl_b200 import ops, priority
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.synthetic import synthetic_batch
    from handyrl_b200.train import LearnerStep
    args = dict(STEP_CASES['alt']['args'], prioritized_replay=True, maximum_episodes=63)
    B, k = 32, 4
    batch = synthetic_batch(B, 8, 2, 9, seed=6)
    stepper = LearnerStep(tictactoe_net(), args, batch, lr=1e-3, gradient_accumulation=k)
    stepper.warm_up()
    ps = stepper.prio_state
    w = torch.rand(B, generator=torch.Generator().manual_seed(0)) + 0.5
    w = w * B / w.sum()
    with torch.cuda.stream(stepper.stream):
        ps.prio_serial[:B].copy_(torch.arange(B))
        ps.win_slot.copy_(torch.arange(B, dtype=torch.int32))
        ps.win_serial.copy_(torch.arange(B))
        ps.win_weight.copy_(w)
    stepper.step(stepper.new_packed().fill(batch))
    stepper.stream.synchronize()
    adv = stepper.advantage.cpu().numpy()
    q = priority.window_priorities(adv, batch['turn_mask'].numpy(), 0, ps.epsilon)
    prio = ps.prio[:B].cpu().numpy()
    fin = np.isfinite(q)
    assert fin.sum() > B // 2
    np.testing.assert_allclose(prio[fin], q[fin], rtol=1e-6)
    Bm = B // k
    with torch.cuda.stream(stepper.stream):
        eng, mb = stepper.engine, stepper._micro[-1]
        outs = {'policy': eng.policy.view(Bm, 8, 1, -1), 'value': eng.value.view(Bm, 8, 1, 1)}
        buf = ops.loss_fwd_bwd(outs, mb, args, taps=True, window_weight=ps.win_weight[-Bm:])
        torch.cuda.current_stream().synchronize()
    assert torch.equal(buf.taps['advantage'].cpu(), stepper.advantage[-Bm:].cpu())
    assert torch.equal(buf.losses.cpu(), stepper.loss_rows[-1, stepper.slots.loss].cpu())


def test_validation_runs_in_micro_batches_and_leaves_the_learner_as_it_was():
    """A validation pass's sums are those of the step's k forwards on the same batch with the same weights, and the pass leaves
    the state bit for bit as it was."""
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.synthetic import synthetic_batch
    from handyrl_b200.train import LearnerStep
    args = STEP_CASES['alt']['args']
    batch = synthetic_batch(32, 8, 2, 9, seed=7)
    stepper = LearnerStep(tictactoe_net(), args, batch, lr=1e-3, gradient_accumulation=4, validation=True)
    stepper.warm_up()
    packed = stepper.new_packed().fill(batch)
    with torch.cuda.stream(stepper.stream):
        stepper.dev_buffer.copy_(packed.buffer.to(stepper.device))
    before = _state_image(stepper)
    stepper.validate_in_place()
    val = stepper.pop_validation()['validation']
    assert all(torch.equal(a, b) for a, b in zip(before, _state_image(stepper)))
    stepper.step_in_place()
    got = stepper.read_losses()
    for n, v in got.items():
        assert abs(val[n] - v) <= 1e-6 * abs(v) + 1e-6, (n, val[n], v)


def test_weight_average_counts_one_update_per_step():
    name = sorted(STEP_CASES)[0]
    stepper, _ = _run_tictactoe(name, 4, args={'weight_ema': 0.9})
    assert int(stepper.opt.step_count) == 3
    assert stepper.ema_state_dict().keys() == stepper.cpu_state_dict().keys()


# ---------------------------------------------------------------- memory


def _peak_bytes(B, k):
    """Peak allocated bytes of building, warming up and capturing the step of nets.WideActionNet (64x64, 512 actions)."""
    from handyrl_b200.nets import WideActionNet
    from handyrl_b200.synthetic import synthetic_batch
    from handyrl_b200.train import LearnerStep
    batch = synthetic_batch(B, 64, 2, 512, seed=0, obs_shape=(1, 64, 64))
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    torch.manual_seed(0)
    stepper = LearnerStep(WideActionNet(), STEP_CASES['alt']['args'], batch, lr=1e-4, gradient_accumulation=k)
    stepper.warm_up()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    packed_bytes = stepper.layout.nbytes
    stepper.close()
    del stepper
    gc.collect()
    torch.cuda.empty_cache()
    return peak, packed_bytes


def test_micro_batches_cut_the_peak_memory_of_the_step():
    """B = 64 windows of T = 64 (4,096 samples): k = 4 needs less than half the memory of k = 1, and no more than the step
    of B = 16 windows plus the buffers that stay B-sized (the packed batch and the advantage tap; the slack allowed is one
    packed batch of 64 windows plus 16 MiB)."""
    for B, k in ((64, 1), (64, 4), (16, 1)):        # cuDNN's autotuner tries its workspaces on the first build of a shape
        _peak_bytes(B, k)
    full, packed64 = _peak_bytes(64, 1)
    micro, _ = _peak_bytes(64, 4)
    small, _ = _peak_bytes(16, 1)
    assert micro < 0.5 * full, (micro, full)
    assert micro <= small + packed64 + (16 << 20), (micro, small, packed64)


# ---------------------------------------------------------------- the Trainer


def test_trainer_trains_with_the_key(capsys):
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.train import Trainer
    with open(os.path.join(GOLDEN, 'batch_cases.pkl'), 'rb') as f:
        case = pickle.load(f)['tictactoe']
    args = dict(case['args'], batch_size=8, minimum_episodes=4, num_batchers=1, **{'lambda': 0.7},
                entropy_regularization=0.1, entropy_regularization_decay=0.1, policy_target='UPGO', value_target='VTRACE',
                gpu_replay=True, num_gpus=1, gradient_accumulation=2)
    tr = Trainer(args, tictactoe_net())
    tr.episodes.extend(case['episodes'])
    th = threading.Thread(target=tr.run, daemon=True)
    th.start()
    model, steps = tr.update()
    assert tr.stepper.micro_batches == 2 and steps >= 1 and not model.training
    model2, steps2 = tr.update()
    assert steps2 > steps
    assert any(not torch.equal(a, b) for a, b in zip(model.state_dict().values(), model2.state_dict().values()))
    tr.stop()
    th.join(timeout=10)
    assert not th.is_alive()
    assert 'loss = ' in capsys.readouterr().out
