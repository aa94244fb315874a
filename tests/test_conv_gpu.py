"""Convolutions over a board as implicit tensor-core products (ops.conv_implicit) inside the nets: zero `same` padding (Geister's
ConvLSTM cells, reference geister.py:18-56) and wrap-around padding (Hungry Geese's TorusConv2d, reference hungry_geese.py:20-37),
fastnet's routing of board convolutions, deferred weight gradients, and batches past 2^22 pixels.  The products themselves,
element by element against float64 on every shape they admit, are test_conv_products_gpu.py."""
import pytest
import torch
import torch.nn.functional as F

from tower_ref import _close, conv_ref, conv_ref_input, conv_ref_weight, conv_src

pytestmark = pytest.mark.gpu

def test_rewritten_modules_use_the_implicit_products():
    """fastnet routes nn.Conv2d (zeros / circular `same` padding) over boards too large for the dense form to conv_implicit."""
    from handyrl_b200 import fastnet, ops
    torch.manual_seed(0)
    for mode in ('zeros', 'circular'):
        conv = torch.nn.Conv2d(16, 24, 3, padding=1, padding_mode=mode).cuda()
        ref = torch.nn.Conv2d(16, 24, 3, padding=1, padding_mode=mode).cuda().double()
        ref.load_state_dict({k: v.double() for k, v in conv.state_dict().items()})
        net = torch.nn.Sequential(conv)
        assert fastnet.optimize_small_boards(net) == 1
        x = torch.randn(11, 16, 6, 6, device='cuda')
        before = ops.LAUNCHES['n']
        fastnet.new_step()
        y = net(x)
        assert ops.LAUNCHES['n'] > before
        assert (y.double() - ref(x.double())).abs().max().item() < 1e-4


ROUTES = {        # route, kernel, board, Cin, padding_mode, tensor_cores
    'dense_1x3': ('dense', (1, 3), (3, 3), 8, 'zeros', True),                 # at most 16 cells: one dense product
    'dense_5x1': ('dense', (5, 1), (4, 4), 8, 'zeros', True),
    'implicit_3x1': ('implicit', (3, 1), (6, 6), 8, 'zeros', True),
    'implicit_1x5_torus': ('implicit', (1, 5), (7, 11), 8, 'circular', True),
    'implicit_1x3_small_torus': ('implicit', (1, 3), (3, 3), 8, 'circular', True),   # the dense form is zero padding only
    'conv_same_cin6': ('conv_same', (1, 3), (6, 6), 6, 'zeros', True),        # Cin % 4 != 0: no implicit product
    'conv_same_fp32': ('conv_same', (3, 1), (6, 6), 8, 'zeros', False),       # tensor_cores=False
    'cudnn_torus_cin6': ('cudnn', (1, 3), (6, 6), 6, 'circular', True),       # wrap-around padding the implicit path refuses
    'cudnn_1x1': ('cudnn', (1, 1), (6, 6), 8, 'zeros', True),                 # nothing to gain over a plain product
    'cudnn_17x17': ('cudnn', (3, 1), (17, 17), 8, 'zeros', True),             # more than 256 cells
}


@pytest.mark.parametrize('name', list(ROUTES))
def test_board_conv_routes_non_square_kernels(name, monkeypatch):
    """fastnet.BoardConv2d runs a stride-1 `same` convolution over a board as a dense product (at most 16 cells, zero padding),
    as the implicit products (conv_implicit_supported), as _ConvSame (zero padding they refuse, or tensor_cores=False: cuDNN's
    forward with an input gradient by the flipped, channel-transposed kernel) or else as cuDNN.  Each route, with a non-square
    kernel, against float64: output, input, weight and bias gradients."""
    from handyrl_b200 import fastnet
    monkeypatch.setattr(torch.backends.cudnn, 'allow_tf32', False)
    route, (kh, kw), (H, W), Cin, mode, tensor_cores = ROUTES[name]
    Cout, N = 12, 5
    torch.manual_seed(sum(map(ord, name)))
    conv = torch.nn.Conv2d(Cin, Cout, (kh, kw), padding=(kh // 2, kw // 2), padding_mode=mode).cuda()
    assert fastnet.optimize_small_boards(torch.nn.Sequential(conv), tensor_cores=tensor_cores) == 1
    x = torch.randn(N, Cin, H, W, device='cuda')
    dy = torch.randn(N, Cout, H, W, device='cuda')
    xs = x.clone().requires_grad_(True)
    fastnet.new_step()
    dense_before = fastnet.BoardConv2d.dense_calls
    y = conv(xs)
    y.backward(dy)
    fn = type(y.grad_fn).__name__
    taken = ('dense' if fastnet.BoardConv2d.dense_calls > dense_before else 'implicit' if fn.startswith('_ConvImplicit')
             else 'conv_same' if fn.startswith('_ConvSame') else 'cudnn' if fn.startswith('Convolution') else fn)
    assert taken == route, (taken, fn)

    src = conv_src(H, W, kh, kw, mode == 'circular')
    xd, wd, bd, dyd = x.double(), conv.weight.detach().double(), conv.bias.detach().double(), dy.double()

    def bound(mag):          # fp32-class products (3xTF32, or cuDNN fp32 in any algorithm) with room to spare
        return 2e-5 * mag + 1e-6 * mag.max()
    _close(y, conv_ref(xd, wd, src, bd), bound(conv_ref(xd.abs(), wd.abs(), src, bd.abs())), 'output')
    _close(xs.grad, conv_ref_input(dyd, wd, src), bound(conv_ref_input(dyd.abs(), wd.abs(), src)), 'input gradient')
    _close(conv.weight.grad, conv_ref_weight(dyd, xd, src, kh, kw), bound(conv_ref_weight(dyd.abs(), xd.abs(), src, kh, kw)),
           'weight gradient')
    _close(conv.bias.grad, dyd.sum((0, 2, 3)), bound(dyd.abs().sum((0, 2, 3))), 'bias gradient')


def test_reference_style_torus_convolution_is_recognised():
    """The reference writes the wrap-around convolution as edge concatenation + an unpadded convolution (hungry_geese.py:24-37);
    fastnet recognises the module by structure and runs it as the wrap-around implicit product, forward and backward."""
    import torch.nn as nn
    from handyrl_b200 import fastnet, ops

    class TorusConv2d(nn.Module):          # restated from the reference's forward (not imported: no kaggle_environments here)
        def __init__(self, input_dim, output_dim, kernel_size, bn):
            super().__init__()
            self.edge_size = (kernel_size[0] // 2, kernel_size[1] // 2)
            self.conv = nn.Conv2d(input_dim, output_dim, kernel_size=kernel_size)
            self.bn = nn.BatchNorm2d(output_dim) if bn else None

        def forward(self, x):
            h = torch.cat([x[:, :, :, -self.edge_size[1]:], x, x[:, :, :, :self.edge_size[1]]], dim=3)
            h = torch.cat([h[:, :, -self.edge_size[0]:], h, h[:, :, :self.edge_size[0]]], dim=2)
            h = self.conv(h)
            return self.bn(h) if self.bn is not None else h

    torch.manual_seed(3)
    ref = TorusConv2d(32, 32, (3, 3), False).cuda().double()
    net = TorusConv2d(32, 32, (3, 3), False).cuda()
    net.load_state_dict({k: v.float() for k, v in ref.state_dict().items()})
    assert fastnet.optimize_small_boards(net) >= 1
    x = torch.randn(9, 32, 7, 11, device='cuda')
    xs, xd = x.clone().requires_grad_(True), x.double().requires_grad_(True)
    dy = torch.randn(9, 32, 7, 11, device='cuda')
    before = ops.LAUNCHES['n']
    fastnet.new_step()
    y = net(xs)
    y.backward(dy)
    assert ops.LAUNCHES['n'] >= before + 3
    yd = ref(xd)
    yd.backward(dy.double())
    assert (y.double() - yd).abs().max().item() < 1e-4
    assert (xs.grad.double() - xd.grad).abs().max().item() < 1e-4
    assert (net.conv.weight.grad.double() - ref.conv.weight.grad).abs().max().item() < 2e-3 * ref.conv.weight.grad.abs().max().item()
    fastnet.restore(net)
    assert type(net) is TorusConv2d


@pytest.mark.parametrize('wrap,bias,steps', [(False, True, 5), (True, False, 5), (False, True, 70)])
def test_deferred_weight_gradients_of_a_shared_convolution(wrap, bias, steps):
    """A recurrent cell applies ONE convolution several times per backward pass.  Inside ops.deferred_weight_gradients() the
    applications only record their (dy, x) pairs; one segmented product per weight (+ its ones row for the bias) then adds the
    summed gradient into weight.grad / bias.grad: same result as per-application products, and as float64 autograd."""
    from handyrl_b200 import ops
    g = torch.Generator(device='cuda').manual_seed(21)
    N, Cin, Cout, H, W = 23, 16, 16, 6, 6
    w = torch.nn.Parameter(torch.randn(Cout, Cin, 3, 3, device='cuda', generator=g) * 0.2)
    b = torch.nn.Parameter(torch.randn(Cout, device='cuda', generator=g)) if bias else None
    x0 = torch.randn(N, Cin, H, W, device='cuda', generator=g)

    def run(conv, x):
        if steps > 10:        # many applications side by side (a long chain of them is chaotic: nothing to compare)
            return sum(torch.tanh(conv(x * (0.5 + i / steps))) for i in range(steps))
        for _ in range(steps):                       # the output of one application feeds the next (as h does in a ConvLSTM)
            x = torch.tanh(conv(x))
        return x

    dy = torch.randn(N, Cout, H, W, device='cuda', generator=g)
    grads = {}
    for mode in ('immediate', 'deferred'):
        w.grad = torch.full_like(w, 0.5)                         # the flush must ADD to what is there (other uses of the weight)
        if bias:
            b.grad = None
        ops.conv_weights_changed()
        y = run(lambda t: ops.conv_implicit(t, w, b, wrap), x0)
        before = ops.LAUNCHES['n']
        if mode == 'deferred':
            with ops.deferred_weight_gradients():
                y.backward(dy)
        else:
            y.backward(dy)
        grads[mode] = (w.grad.clone(), None if not bias else b.grad.clone(), ops.LAUNCHES['n'] - before)
    assert grads['deferred'][2] < grads['immediate'][2]          # `steps` products + reductions became 1 + 1 (2 + 2 beyond 64 pairs)
    wd = w.detach().double().requires_grad_(True)
    bd = b.detach().double().requires_grad_(True) if bias else None

    def conv64(t):
        if wrap:
            return torch.nn.functional.conv2d(torch.nn.functional.pad(t, (1, 1, 1, 1), mode='circular'), wd, bd)
        return torch.nn.functional.conv2d(t, wd, bd, padding=1)
    run(conv64, x0.double()).backward(dy.double())
    scale = wd.grad.abs().max().item()
    for mode in grads:
        assert (grads[mode][0].double() - 0.5 - wd.grad).abs().max().item() <= 3e-5 * scale, mode
        if bias:
            assert (grads[mode][1].double() - bd.grad).abs().max().item() <= 3e-5 * bd.grad.abs().max().item(), mode
    assert (grads['deferred'][0] - grads['immediate'][0]).abs().max().item() <= 2e-5 * scale


def test_conv_implicit_beyond_four_million_pixels():
    """A product's rows are pixels: a Geese-sized batch (7x11 torus boards) of more than 2^22 pixels must convolve every board,
    including those whose pixel index needs more than 22 bits, exactly like the first ones (forward and input gradient,
    checked board by board against float64 on both ends of the batch)."""
    from handyrl_b200 import ops
    N, C, H, W = 55_000, 32, 7, 11                         # 4.24 M pixels, 540 MB per activation tensor
    assert N * H * W > 1 << 22
    g = torch.Generator(device='cuda').manual_seed(22)
    x = torch.randn(N, C, H, W, device='cuda', generator=g).contiguous(memory_format=torch.channels_last)
    w = torch.randn(C, C, 3, 3, device='cuda', generator=g) * 0.2
    dy = torch.randn(N, C, H, W, device='cuda', generator=g).contiguous(memory_format=torch.channels_last)
    xs = x.clone().requires_grad_(True)
    ops.conv_weights_changed()
    y = ops.conv_implicit(xs, w, None, True)
    y.backward(dy)
    torch.cuda.synchronize()
    for lo, hi in ((0, 64), ((1 << 22) // (H * W) - 32, N)):
        xd = x[lo:hi].double().requires_grad_(True)
        yd = F.conv2d(F.pad(xd, (1, 1, 1, 1), mode='circular'), w.double())
        yd.backward(dy[lo:hi].double())
        for got, want, red in ((y[lo:hi], yd, C * 9), (xs.grad[lo:hi], xd.grad, C * 9)):
            scale = want.abs().max().item()
            err = (got.double() - want).abs().max().item()
            assert err <= 3e-6 * scale * (1 + red ** 0.5 / 8), (lo, hi, err, scale)
