"""fastnet.BoardBatchNorm2d on CPU tensors against nn.BatchNorm2d in float64 over three training steps: every configuration
the fused kernels do not take must behave exactly as nn.BatchNorm2d does (momentum=None is a cumulative average, eval mode
normalises with the running statistics, no running statistics, no affine parameters) and the CPU var_mean path must match."""
import copy

import pytest
import torch

CASES = {
    'cumulative_average': dict(momentum=None),
    'eval_mode': dict(eval=True),
    'no_running_stats': dict(track_running_stats=False),
    'no_affine': dict(affine=False),
    'var_mean_path': dict(momentum=0.3),
}


@pytest.mark.parametrize('name', sorted(CASES))
def test_board_batchnorm_falls_through_like_nn_batchnorm(name):
    from handyrl_b200 import fastnet
    kw = dict(CASES[name])
    evaluate = kw.pop('eval', False)
    torch.manual_seed(0)
    C = 6
    ref = torch.nn.BatchNorm2d(C, eps=1e-3, **kw).double()
    if ref.affine:
        with torch.no_grad():
            ref.weight.copy_(torch.tensor([1.3, -0.7, 0.0, 2.0, 0.5, 1.0]))
            ref.bias.uniform_(-0.5, 0.5)
    if ref.track_running_stats:
        ref.running_mean.normal_(0, 0.1)
        ref.running_var.uniform_(0.5, 2.0)
    fast = torch.nn.Sequential(copy.deepcopy(ref))
    assert fastnet.optimize_small_boards(fast) == 1 and type(fast[0]) is fastnet.BoardBatchNorm2d
    ref.train(not evaluate)
    fast.train(not evaluate)
    for step in range(3):
        x = torch.randn(17, C, 3, 3, dtype=torch.float64) * torch.tensor([1.0, 3.0, 0.2, 1.0, 5.0, 1.0]).view(1, C, 1, 1) + 0.5 * step
        dy = torch.randn_like(x)
        xr, xf = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
        yr, yf = ref(xr), fast(xf)
        yr.backward(dy)
        yf.backward(dy)
        torch.testing.assert_close(yf, yr, rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(xf.grad, xr.grad, rtol=1e-12, atol=1e-12)
        for (k, a), (_, b) in zip(ref.named_parameters(), fast[0].named_parameters()):
            torch.testing.assert_close(b.grad, a.grad, rtol=1e-12, atol=1e-12, msg=k)
        for (k, a), (_, b) in zip(ref.named_buffers(), fast[0].named_buffers()):
            if a.dtype.is_floating_point:
                torch.testing.assert_close(b, a, rtol=1e-12, atol=1e-12, msg=k)
            else:
                assert int(b) == int(a) == (0 if evaluate else step + 1), k
