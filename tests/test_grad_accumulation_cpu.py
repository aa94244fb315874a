"""Gradient accumulation without a GPU: how train_args['gradient_accumulation'] is read and checked, and the micro-batched
reference the GPU tests compare the learner against (built from oracle/torch_learner.py)."""
import numpy as np
import pytest
import torch

from oracle.torch_learner import CpuLearner, _walk, loss_from_raw, recurrent_raw_outputs

ARGS = {'turn_based_training': True, 'observation': False, 'gamma': 0.8, 'lambda': 0.7, 'burn_in_steps': 0, 'forward_steps': 8,
        'entropy_regularization': 0.1, 'entropy_regularization_decay': 0.1, 'policy_target': 'UPGO', 'value_target': 'VTRACE'}


def micro_batched_reference(net, batch, args, k, opt, max_norm=4.0):
    """One optimiser step of `net` on `batch` trained as k micro-batches: per slice [i*B/k, (i+1)*B/k) the forward in train
    mode, loss_from_raw and backward() into the same .grad; then clip_grad_norm_(max_norm) and opt.step() once.  Returns
    (loss sums {p, v, r?, ent, total, dcnt} as floats, pre-clip gradient norm, the flat pre-optimiser gradient)."""
    B, T, Pa = batch['action'].shape[:3]
    P = batch['turn_mask'].shape[2]
    Bm = B // k
    params = list(net.parameters())
    net.train()
    opt.zero_grad()
    sums = {}
    for i in range(k):
        mb = _walk(lambda t: t[i * Bm:(i + 1) * Bm], batch)
        if hasattr(net, 'init_hidden'):
            raw = recurrent_raw_outputs(net, _walk(lambda h: h.to(mb['action'].device), net.init_hidden([Bm, P])), mb, args)
        else:
            outs = net(_walk(lambda o: o.flatten(0, 2), mb['observation']), None)
            raw = {n: v.unflatten(0, (Bm, T, Pa)) for n, v in outs.items() if v is not None and n != 'hidden'}
        losses, dcnt = loss_from_raw(raw, mb, args)
        losses['total'].backward()
        for n, v in list(losses.items()) + [('dcnt', dcnt)]:
            sums[n] = sums.get(n, 0.0) + float(v.detach())
    grad = torch.cat([p.grad.reshape(-1) for p in params]).detach().clone()
    gnorm = float(torch.nn.utils.clip_grad_norm_(params, max_norm))
    opt.step()
    return sums, gnorm, grad


# ---------------------------------------------------------------- the key


@pytest.mark.parametrize('value, want', [(None, 1), (0, 1), (1, 1), (2, 2), (8, 8), (np.int64(4), 4)])
def test_accepted_values(value, want):
    from handyrl_b200.train import gradient_accumulation
    args = {} if value is None else {'gradient_accumulation': value}
    assert gradient_accumulation(args) == want
    assert gradient_accumulation({'gradient_accumulation': None}) == 1


@pytest.mark.parametrize('value', [True, False, -1, 2.0, 1.5, '2', [2]])
def test_malformed_values_raise(value):
    from handyrl_b200.train import gradient_accumulation
    with pytest.raises(ValueError):
        gradient_accumulation({'gradient_accumulation': value})


def test_learner_step_refuses_bad_keys_before_touching_a_device():
    """LearnerStep checks the key (and the argument of the same name) and its divisibility of the batch first."""
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.synthetic import synthetic_batch
    from handyrl_b200.train import LearnerStep
    batch = synthetic_batch(12, 4, 2, 9, seed=0)
    for kw in ({'gradient_accumulation': 5}, {'gradient_accumulation': True}, {'gradient_accumulation': 'x'}):
        with pytest.raises(ValueError):
            LearnerStep(tictactoe_net(), dict(ARGS, **kw), batch, lr=1e-3)
    with pytest.raises(ValueError, match='does not divide'):
        LearnerStep(tictactoe_net(), ARGS, batch, lr=1e-3, gradient_accumulation=8)
    with pytest.raises(ValueError, match='time_loss_kernel'):
        LearnerStep(tictactoe_net(), ARGS, batch, lr=1e-3, gradient_accumulation=2, time_loss_kernel=True)


def test_trainer_refuses_a_batch_size_the_key_does_not_divide():
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.train import Trainer
    for k in (3, -2, 2.5):
        with pytest.raises(ValueError):
            Trainer(dict(ARGS, batch_size=16, gradient_accumulation=k), tictactoe_net())


# ---------------------------------------------------------------- the micro-batched reference


def _setup(norm, seed=0, B=16, T=8):
    from handyrl_b200.nets import BoardNet
    from handyrl_b200.synthetic import synthetic_batch
    torch.manual_seed(seed)
    net = BoardNet(norm=norm)
    return net, synthetic_batch(B, T, 2, 9, seed=40 + seed)


def test_reference_without_batchnorm_is_the_full_batch_step():
    """BoardNet(norm=False): the micro-batched step of 4 slices is CpuLearner's whole-batch step up to fp32 summation order --
    loss sums, gradient, norm and weights."""
    import copy
    net, batch = _setup(norm=False)
    twin = copy.deepcopy(net)
    full = CpuLearner(net, ARGS, lr=1e-3)
    losses, dcnt = full.step(batch)
    grad_full = torch.cat([p.grad.reshape(-1) for p in full.params])
    opt = torch.optim.Adam(twin.parameters(), lr=1e-3, weight_decay=1e-5)
    sums, gnorm, grad = micro_batched_reference(twin, batch, ARGS, 4, opt)
    for n, v in losses.items():
        assert abs(sums[n] - v) <= 1e-5 * abs(v) + 1e-5, (n, sums[n], v)
    assert sums['dcnt'] == dcnt
    scale = float(grad_full.abs().max())
    assert float((grad - grad_full).abs().max()) <= 1e-5 * scale
    assert abs(gnorm - full.grad_norm) <= 1e-5 * full.grad_norm
    for a, b in zip(net.parameters(), twin.parameters()):
        torch.testing.assert_close(b, a, rtol=0, atol=2e-3 + 1e-6)        # Adam's first step: ~lr * sign(g) per element
    close = sum(int(torch.isclose(b, a, rtol=0, atol=1e-6).sum()) for a, b in zip(net.parameters(), twin.parameters()))
    assert close >= 0.999 * sum(p.numel() for p in net.parameters())


def test_reference_with_batchnorm_uses_per_micro_batch_statistics():
    """The BN net: the micro-batched step differs from the whole-batch step beyond fp32 reordering (each slice is normalised
    with its own statistics), and the running statistics move once per slice."""
    import copy
    net, batch = _setup(norm=True)
    twin = copy.deepcopy(net)
    full = CpuLearner(net, ARGS, lr=1e-3)
    full.step(batch)
    grad_full = torch.cat([p.grad.reshape(-1) for p in full.params])
    opt = torch.optim.Adam(twin.parameters(), lr=1e-3, weight_decay=1e-5)
    _, _, grad = micro_batched_reference(twin, batch, ARGS, 4, opt)
    assert float((grad - grad_full).abs().max()) > 1e-3 * float(grad_full.abs().max())
    bn_full, bn_micro = net.tower[0][1], twin.tower[0][1]
    assert int(bn_full.num_batches_tracked) == 1 and int(bn_micro.num_batches_tracked) == 4
    assert not torch.allclose(bn_full.running_mean, bn_micro.running_mean, rtol=0, atol=1e-6)
