"""Rewrite pass for nets that convolve over tiny boards (TicTacToe 3x3, Geister 6x6, ...).

cuDNN has no efficient kernels for N ~ 10^4, H x W <= ~6x6: its heuristics pick FFT or
"grouped direct" kernels that leave most of the GPU idle, which makes the user's net -- not the loss --
most of a learner step.  A stride-1 "same" convolution over a
board with HW cells is exactly a dense linear map (Cin*HW -> Cout*HW) whose matrix is a fixed 0/1
re-indexing of the kernel weights, so the layer runs as ONE matrix product per direction on the flattened
(N, Cin*HW) activations (NCHW-contiguous, no layout change) -- on CUDA through the hand-written wgmma
3xTF32 GEMM (csrc/gemm_kernel.cu: tensor cores at fp32-class accuracy) with the dense matrix and its adjoint produced by one kernel each (csrc/net_kernel.cu) -- and BatchNorm2d
as fused reductions.  ConvLSTM cells (reference geister.py:18-56) get their gate arithmetic fused the same way.

`optimize_small_boards(model)` swaps the class of eligible nn.Conv2d / nn.BatchNorm2d modules in place:
parameters, buffers and state_dict keys are untouched (reference checkpoints keep loading, workers keep
unpickling a plain nn.Module after `restore`), the arithmetic is the same fp32 multiply-adds in a
different summation order.  Inputs whose board is larger than `max_cells` fall through to cuDNN.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

MAX_CELLS = 256           # BatchNorm: fused coalesced passes for boards up to 16x16 (NCHW or channels-last)
DENSE_MAX_CELLS = 16      # convolution as a dense product: only while the board is about as small as the kernel
DENSE_MAX_ELEMS = 1 << 20   # ... and the dense matrix stays small (4 MB)


def _selection(kh, kw, H, W, ph, pw, device, dtype):
    """S[k, q, p] = 1 iff kernel tap k of output cell q reads input cell p (zero padding drops the rest)."""
    S = torch.zeros(kh * kw, H * W, H * W, dtype=dtype)
    for a in range(kh):
        for b in range(kw):
            for oh in range(H):
                for ow in range(W):
                    ih, iw = oh + a - ph, ow + b - pw
                    if 0 <= ih < H and 0 <= iw < W:
                        S[a * kw + b, oh * W + ow, ih * W + iw] = 1
    return S.to(device)


class _SplitKLinear(torch.autograd.Function):
    """y = x @ W^T with the weight gradient computed split-K: for N ~ 10^4 rows and a (C*HW)^2 weight the plain
    wgrad GEMM (dy^T @ x, reduction over N) has only ~80 output tiles -- fewer than H100's 132 SMs, each looping
    over all N rows.  Splitting N into chunks turns it into a batched GEMM with chunks x 80 tiles plus a tiny sum."""

    CHUNKS = int(__import__('os').environ.get('HRL_SPLITK', '32'))

    @staticmethod
    def forward(ctx, x, w):
        ctx.save_for_backward(x, w)
        return x @ w.t()

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        dx = dw = None
        if ctx.needs_input_grad[0]:
            dx = dy @ w
        if ctx.needs_input_grad[1]:
            N = x.shape[0]
            S = _SplitKLinear.CHUNKS
            if N % S == 0 and N // S >= 256:
                dw = torch.bmm(dy.reshape(S, N // S, -1).transpose(1, 2), x.reshape(S, N // S, -1)).sum(0)
            else:
                dw = dy.t() @ x
        return dx, dw


# Adjoint weights of the step in flight: {(data_ptr, shape, memory format): flipped/transposed copy}.  A recurrent net calls
# each convolution T times per step; the copy is made once.  The learner clears the cache at the start of every step
# and ops.FlatAdam after every update (new_step): it writes the parameters from its own kernel, which no version counter sees.
_ADJOINT = {}


def new_step():
    _ADJOINT.clear()
    from . import ops
    ops.conv_weights_changed()


def _adjoint_weight(w, channels_last):
    key = (w.data_ptr(), tuple(w.shape), channels_last, w._version)      # (_version: in-place updates by torch optimisers)
    wt = _ADJOINT.get(key)
    if wt is None:
        wt = w.detach().transpose(0, 1).flip(2, 3)
        wt = wt.contiguous(memory_format=torch.channels_last) if channels_last else wt.contiguous()
        _ADJOINT[key] = wt
    return wt


class _ConvSame(torch.autograd.Function):
    """Stride-1 "same" convolution whose INPUT gradient is computed as what it is -- the same kind of convolution of dy with
    the spatially flipped, channel-transposed kernel -- i.e. by cuDNN's forward kernels.  At the shapes of the board games
    (N = 512..16384 positions of 6x6, 64 -> 128 channels, fp32 without TF32) cuDNN's backward-data choice is
    `dgrad2d_grouped_direct_kernel`, several times slower than the forward `implicit_convolve_sgemm` of the same shape.
    Same multiply-adds, other order.
    The weight gradient stays with cuDNN (convolution_backward, weight only)."""

    @staticmethod
    def forward(ctx, x, w, b):
        ctx.save_for_backward(x, w)
        ctx.has_bias = b is not None
        return F.conv2d(x, w, b, padding=(w.shape[2] // 2, w.shape[3] // 2))

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        pad = (w.shape[2] // 2, w.shape[3] // 2)
        dx = dw = db = None
        cl = x.is_contiguous(memory_format=torch.channels_last) and not x.is_contiguous()
        if cl:
            dy = dy.contiguous(memory_format=torch.channels_last)
        if ctx.needs_input_grad[0]:
            dx = F.conv2d(dy, _adjoint_weight(w, cl), None, padding=pad)
        if ctx.needs_input_grad[1]:
            dw = torch.ops.aten.convolution_backward(dy, x, w, None, (1, 1), pad, (1, 1), False, (0, 0), 1, (False, True, False))[1]
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = dy.sum((0, 2, 3))
        return dx, dw, db


class BoardConv2d(nn.Conv2d):
    """nn.Conv2d whose forward runs as a dense GEMM when the board is tiny."""

    dense_calls = 0       # how often the dense path ran (LearnerStep probes this to pick the memory format)

    def _eligible(self, x):
        kh, kw = self.kernel_size
        cells = x.shape[2] * x.shape[3] if x.dim() == 4 else 0
        return (x.dim() == 4 and cells <= DENSE_MAX_CELLS
                and self.out_channels * cells * self.in_channels * cells <= DENSE_MAX_ELEMS and self.stride == (1, 1)
                and self.dilation == (1, 1) and self.groups == 1 and self.padding_mode == 'zeros'
                and self.padding == (kh // 2, kw // 2) and kh % 2 == 1 and kw % 2 == 1)

    def _sel(self, H, W, device, dtype):
        cache = self.__dict__.setdefault('_sel_cache', {})
        key = (H, W, device, dtype)
        if key not in cache:
            kh, kw = self.kernel_size
            cache[key] = _selection(kh, kw, H, W, self.padding[0], self.padding[1], device, dtype)
        return cache[key]

    def _same(self, x, wrap=False):
        kh, kw = self.kernel_size
        return (x.dim() == 4 and x.is_cuda and x.shape[2] * x.shape[3] <= MAX_CELLS and self.stride == (1, 1)
                and self.dilation == (1, 1) and self.groups == 1 and self.padding_mode == ('circular' if wrap else 'zeros')
                and kh % 2 == 1 and kw % 2 == 1 and tuple(self.padding) == (kh // 2, kw // 2) and kh * kw > 1)

    def forward(self, x):
        if not self._eligible(x):
            wrap = self.padding_mode == 'circular'
            if self._same(x, wrap):
                from . import ops
                if getattr(self, 'tensor_cores', True) and ops.conv_implicit_supported(x, self.weight):
                    # tensor cores: the convolution as an implicit product over (tap, channel), no dense matrix, no im2col
                    return ops.conv_implicit(x, self.weight, self.bias, wrap, bf16=_bf16(self))
                if torch.is_grad_enabled() and not wrap:
                    return _ConvSame.apply(x, self.weight, self.bias)
            return super().forward(x)
        N, Cin, H, W = x.shape
        HW = H * W
        Cout = self.out_channels
        BoardConv2d.dense_calls += 1
        if x.is_cuda and x.dtype == torch.float32 and getattr(self, 'tensor_cores', True):
            # tensor cores: dense matrix by one kernel, then forward / input-gradient / weight-gradient as wgmma products
            from . import ops
            y = ops.board_conv(x, self.weight, bf16=_bf16(self))
            if self.bias is not None:
                y = y + self.bias.view(1, Cout, 1, 1)
            return y
        S = self._sel(H, W, x.device, x.dtype)                                        # (K, HW, HW)
        # dense matrix of the layer: Wb[(o,q),(i,p)] = sum_k w[o,i,k] S[k,q,p]
        Wb = (self.weight.reshape(Cout * Cin, -1) @ S.reshape(S.shape[0], HW * HW))
        Wb = Wb.reshape(Cout, Cin, HW, HW).permute(0, 2, 1, 3).reshape(Cout * HW, Cin * HW)
        y = _SplitKLinear.apply(x.reshape(N, Cin * HW), Wb)
        y = y.reshape(N, Cout, H, W)
        if self.bias is not None:
            y = y + self.bias.view(1, Cout, 1, 1)
        return y


class BoardBatchNorm2d(nn.BatchNorm2d):
    """nn.BatchNorm2d with training-mode statistics as two fused reductions over (N, HW) on tiny boards
    (cuDNN's spatial BN kernels launch one CTA per channel: ~1 ms at N=16384, C=32)."""

    def forward(self, x):
        if not (self.training and x.dim() == 4 and x.shape[2] * x.shape[3] <= MAX_CELLS and self.track_running_stats
                and self.momentum is not None):      # (momentum None: a cumulative average, left to nn.BatchNorm2d)
            return super().forward(x)
        N, C, H, W = x.shape
        if x.is_cuda and x.dtype == torch.float32 and self.affine:
            # fused kernels (csrc/bn_kernel.cu): 3 coalesced passes forward, 3 backward
            from . import ops
            with torch.no_grad():
                self.num_batches_tracked.add_(1)
            return ops.batch_norm_train(x, self.weight, self.bias, self.running_mean, self.running_var, self.eps, self.momentum)
        x3 = x.reshape(N, C, H * W)
        var, mean = torch.var_mean(x3, dim=(0, 2), unbiased=False, keepdim=True)
        with torch.no_grad():
            n = N * H * W
            self.num_batches_tracked.add_(1)
            self.running_mean.mul_(1 - self.momentum).add_(mean.reshape(C), alpha=self.momentum)
            self.running_var.mul_(1 - self.momentum).add_(var.reshape(C) * (n / max(n - 1, 1)), alpha=self.momentum)
        scale = torch.rsqrt(var + self.eps)
        if self.affine:
            scale = scale * self.weight.view(1, C, 1)
            y = (x3 - mean) * scale + self.bias.view(1, C, 1)
        else:
            y = (x3 - mean) * scale
        return y.reshape(N, C, H, W)


_SWAPS = {nn.Conv2d: BoardConv2d, nn.BatchNorm2d: BoardBatchNorm2d}
_UNSWAPS = {v: k for k, v in _SWAPS.items()}
_CELL_CLASSES = {}        # original ConvLSTM cell class -> fused subclass


def _is_conv_lstm_cell(m):
    """Duck-typed ConvLSTM cell: one convolution `conv` over [input, h] whose output holds the four gate maps of
    `hidden_dim` (reference geister.py:18-35) / `state_maps` (nets.ConvLstmCell) channels, called as cell(x, (h, c))."""
    conv = getattr(m, 'conv', None)
    maps = getattr(m, 'hidden_dim', None) or getattr(m, 'state_maps', None)
    return (isinstance(conv, nn.Conv2d) and isinstance(maps, int) and conv.out_channels == 4 * maps
            and len(list(m.children())) == 1 and not isinstance(m, nn.Conv2d))


def _is_torus_conv(m):
    """Duck-typed wrap-around convolution as the reference writes it (hungry_geese.py:24-37): `edge_size` = half the kernel, an
    unpadded `conv`, an optional `bn`; forward = concatenate the opposite edges on both axes, convolve, normalise."""
    conv, edge = getattr(m, 'conv', None), getattr(m, 'edge_size', None)
    return (isinstance(conv, nn.Conv2d) and isinstance(edge, tuple) and len(edge) == 2 and not isinstance(m, nn.Conv2d)
            and tuple(conv.padding) == (0, 0) and conv.kernel_size == (2 * edge[0] + 1, 2 * edge[1] + 1) and conv.stride == (1, 1)
            and conv.dilation == (1, 1) and conv.groups == 1 and hasattr(m, 'bn')
            and all(name in ('conv', 'bn') for name, _ in m.named_children()))


_TORUS_CLASSES = {}


def _fused_torus_class(cls):
    if cls not in _TORUS_CLASSES:
        original = cls.forward

        def forward(self, x):
            from . import ops
            if (x.dim() == 4 and x.is_cuda and x.shape[2] * x.shape[3] <= MAX_CELLS and getattr(self.conv, 'tensor_cores', True)
                    and ops.conv_implicit_supported(x, self.conv.weight)):
                h = ops.conv_implicit(x, self.conv.weight, self.conv.bias, True, bf16=_bf16(self.conv))      # the wrap lives in the neighbour table
                return self.bn(h) if self.bn is not None else h
            return original(self, x)
        _TORUS_CLASSES[cls] = type('Fused' + cls.__name__, (cls,), {'forward': forward, '_hrl_original': cls})
    return _TORUS_CLASSES[cls]


def _fused_cell_class(cls):
    if cls not in _CELL_CLASSES:
        def forward(self, x, state):
            h, c = state
            gates = self.conv(torch.cat([x, h], dim=-3))
            if gates.is_cuda and gates.dtype == torch.float32 and gates.dim() == 4:
                from . import ops
                return ops.lstm_gates(gates, c)           # one kernel forward, one backward (csrc/net_kernel.cu)
            i, f, o, g = gates.chunk(4, dim=-3)
            c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
            return torch.sigmoid(o) * torch.tanh(c), c
        _CELL_CLASSES[cls] = type('Fused' + cls.__name__, (cls,), {'forward': forward, '_hrl_original': cls})
    return _CELL_CLASSES[cls]


def _bf16(conv):
    return getattr(conv, 'tensor_cores', True) == 'bf16'


def optimize_small_boards(model, tensor_cores=True):
    """Swap eligible modules to their board-aware subclasses, in place.  Returns how many were swapped.
    tensor_cores=False keeps the dense products on cuBLAS fp32 SIMT kernels (bit-for-bit fp32 summation; the tensor-core
    3xTF32 products truncate their fp32 accumulator and are ~1e-5 relative per product, see DESIGN.md).
    tensor_cores='bf16' runs the same tensor-core products on bf16 operands (rounded after their fp32 transform, fp32
    accumulation): faster, ~2^-8 relative per product."""
    n = 0
    for m in model.modules():
        if type(m) in _SWAPS:
            m.__class__ = _SWAPS[type(m)]
            if isinstance(m, BoardConv2d):
                m.__dict__['tensor_cores'] = 'bf16' if tensor_cores == 'bf16' else bool(tensor_cores)
            n += 1
        elif _is_conv_lstm_cell(m) and not hasattr(type(m), '_hrl_original'):
            m.__class__ = _fused_cell_class(type(m))
            n += 1
        elif _is_torus_conv(m) and not hasattr(type(m), '_hrl_original'):
            m.__class__ = _fused_torus_class(type(m))
            n += 1
    return n


def restore(model):
    """Undo optimize_small_boards (e.g. before pickling a model for CPU workers)."""
    for m in model.modules():
        if type(m) in _UNSWAPS:
            m.__dict__.pop('_sel_cache', None)
            m.__class__ = _UNSWAPS[type(m)]
        elif hasattr(type(m), '_hrl_original'):
            m.__class__ = type(m)._hrl_original
    return model
