"""Fused training engine for conv -> BatchNorm -> ReLU towers over a tiny board (nets.BoardNet: the architecture of the
reference's TicTacToe net, handyrl/envs/tictactoe.py:52-69).

The generic path runs such a net as PyTorch modules whose convolutions / BatchNorms are swapped for this library's
kernels one module at a time (fastnet.py): ~100 launches per learner step, every activation crossing memory several
times (product, statistics, normalise, ReLU, their four backward passes).  Here the whole net is scheduled by hand on the
fused tensor-core product `hrl_gemm_fused` (csrc/gemm_kernel.cu): a layer is ONE launch per direction --

  forward   Y_l = relu(bn_{l-1}(Y_{l-1})) @ Wd_l^T      BatchNorm-apply + ReLU of the previous layer happen while the A operand
                                                          is staged; the epilogue leaves this layer's batch statistics
  backward  dZ_{l-1} = (dY_l @ Wd_l) * (Z_{l-1} > 0)    dY_l = BatchNorm backward of dZ_l, formed while the operand is staged;
                                                          the epilogue applies the ReLU mask and leaves the two batch sums
                                                          of the next BatchNorm backward
            dWd_l = dY_l^T @ relu(bn(Y_{l-1}))           both operands transformed on the fly, split over samples, folded
                                                          onto the 3x3 taps by hrl_board_fold

with `Wd` the dense matrix of a convolution over the board (hrl_board_expand), tiny kernels finalising the BatchNorm
statistics between the products (csrc/tower_kernel.cu), and the 1x1-conv + LeakyReLU + Linear heads in two row kernels.
Nothing here goes through autograd: `backward` writes straight into the parameters' .grad (views of the learner's flat
gradient bucket).  Semantics are those of the module version (checked parameter by parameter in tests/test_tower_gpu.py and
by the reference's own 3-step golden): nn.BatchNorm2d training statistics incl. running buffers, ReLU / LeakyReLU(0.1)
masks, tanh value.
"""
import ctypes as C

import torch

from . import _capi, nets
from ._capi import MAX_BOARD_JOBS, MAX_BOARD_ROWS, HrlFoldJob, HrlPackJob, check, lib
from .ops import _count, _operand, _ptr, _stream_ptr, gemm_fused, k_splits  # noqa: F401 (_operand: the operand dicts of _gemm)


def supports(model):
    """The engine covers nets.BoardNet as it stands (3x3 convolutions with BatchNorm in the tower, 1x1 squeeze heads) when every
    convolution's packed image fits (width x cells <= MAX_BOARD_ROWS rows) and the heads fit their kernels (at most 16 cells,
    64 squeeze outputs and 32 actions).  Each tower BatchNorm must be affine, track running statistics and have a numeric
    momentum: the engine reads its weight, bias and running buffers and applies the momentum update."""
    if type(model) is not nets.BoardNet or len(model.tower) == 0:
        return False
    if not all(len(blk) == 2 and isinstance(blk[1], torch.nn.BatchNorm2d) for blk in model.tower):
        return False
    if not all(bn.affine and bn.track_running_stats and isinstance(bn.momentum, (int, float)) for bn in (blk[1] for blk in model.tower)):
        return False
    if model.stem.kernel_size != (3, 3) or any(blk[0].kernel_size != (3, 3) or blk[0].bias is not None for blk in model.tower):
        return False
    cells = model.p_out.in_features // model.p_squeeze.out_channels
    dense = model.stem.out_channels * cells
    heads = (model.p_squeeze.out_channels + model.v_squeeze.out_channels +
             (model.r_squeeze.out_channels if model.r_squeeze is not None else 0)) * cells
    return cells <= 16 and dense % 4 == 0 and dense <= MAX_BOARD_ROWS and heads <= 64 and model.p_out.out_features <= 32


class FusedBoardNet:
    """Forward / backward of a nets.BoardNet in training mode on (M, planes, H, W) observations with static buffers
    (CUDA-graph friendly).  The module keeps owning the parameters and BatchNorm buffers; this object only reads them and
    writes their gradients."""

    def __init__(self, model, M, device, bf16=False):
        assert supports(model)
        self.model, self.M, self.device = model, int(M), device
        # bf16: every product runs on bf16 operands (HrlGemmArgs.bf16, fp32 accumulation) with bf16 weight images; the heads,
        # BatchNorm finalisation and fold kernels stay fp32
        self.bf16 = bool(bf16)
        st = model.stem
        self.planes, self.width = st.in_channels, st.out_channels
        self.pmaps = model.p_squeeze.out_channels
        self.vmaps = model.v_squeeze.out_channels
        self.rmaps = model.r_squeeze.out_channels if model.r_squeeze is not None else 0
        self.cells = model.p_out.in_features // self.pmaps
        self.A = model.p_out.out_features
        self.H = self.W = None
        self.D = self.width * self.cells
        self.K0 = self.planes * self.cells
        self.NH = (self.pmaps + self.vmaps + self.rmaps) * self.cells
        self.ldh = (self.NH + 3) // 4 * 4
        self.depth = len(model.tower)
        self.tiles = (self.M + 127) // 128
        f = dict(dtype=torch.float32, device=device)
        M_, D = self.M, self.D
        # weights as packed B-operand images (pre-split TF32 hi/lo, or bf16 in a quarter of the bytes; pre-swizzled, one bulk copy
        # per stage): `f` for the forward product (rows = output features), `b` for the input-gradient product (rows = input features)
        img = lambda rows, K: torch.zeros(lib().hrl_board_pack_floats(rows, K) // (4 if self.bf16 else 1), **f)
        self.W0f = img(D, self.K0)
        self.Wf = [img(D, D) for _ in range(self.depth)]
        self.Wb = [img(D, D) for _ in range(self.depth)]
        self.Whf = img(self.NH, D)
        self.Whb = img(D, self.NH)
        self.b0 = torch.empty(D, **f)
        self.bh = torch.empty(self.NH, **f)
        self.A0 = torch.empty((M_, D), **f)
        self.Y = [torch.empty((M_, D), **f) for _ in range(self.depth)]
        self.dZ = [torch.empty((M_, D), **f) for _ in range(self.depth)]
        self.dZ0 = torch.empty((M_, D), **f)
        self.Hpre = torch.zeros((M_, self.ldh), **f)
        self.dHpre = torch.zeros((M_, self.ldh), **f)
        self.policy = torch.empty((M_, self.A), **f)
        self.value = torch.empty((M_, 1), **f)
        self.ret = torch.empty((M_, 1), **f) if self.rmaps else None
        self.cp = torch.empty((self.tiles, 2, D), **f)
        cols = lambda: torch.empty(D, **f)
        self.bn = [dict(mean=cols(), rstd=cols(), scale=cols(), shift=cols(), p=cols(), q=cols(), r=cols()) for _ in range(self.depth)]
        n_out = self.A * self.pmaps * self.cells + (self.vmaps + self.rmaps) * self.cells + self.pmaps + self.vmaps + self.rmaps
        self.heads_ws = torch.empty(lib().hrl_heads_num_blocks(M_) * n_out, **f)
        # weight-gradient products: split over samples so that (row tiles x slices) fills the GPU
        # (each product keeps its slice partials in a region of its own: ALL of them are folded onto the convolution
        #  weights by one launch at the end of the backward pass)
        self.splits, self.ws_at = {}, {}
        ws_floats = 0
        for name, rows, colsn, count in (('stem', D, self.K0, 1), ('tower', D, D, self.depth), ('heads', self.NH, D, 1)):
            s = self.splits[name] = k_splits(rows, colsn, M_)
            for i in range(count):
                self.ws_at[(name, i)] = ws_floats
                ws_floats += s * rows * colsn
        self.ws = torch.empty(ws_floats, **f)
        self.fold_jobs = []
        self.slope = 0.1

    # ------------------------------------------------------------------ helpers
    def _gemm(self, a, b, out, K, N, M=None, bias=None, epilogue='store', splits=1, partial=False, ep=None, ws=None):
        """partial: leave the product in `ws` as its K-slice partials (gemm_fused with no output)."""
        gemm_fused(a, b, self.M if M is None else M, N, K, out=None if partial else out, ws=ws, splits=splits, bias=bias, epilogue=epilogue,
                   ep=ep, col_partials=self.cp if epilogue in ('stats', 'mask_stats') else None, bf16=self.bf16)

    def _pack_all(self, jobs):
        """jobs: dicts of HrlPackJob fields with tensors for the pointers -- one launch for up to MAX_BOARD_JOBS convolutions.
        The same launches write each tower layer's BatchNorm statistics pivot into its `mean` (up to MAX_BOARD_JOBS layers per
        launch; there are fewer tower layers than jobs): the running mean where |running mean| >> running std, else 0.  The
        statistics epilogue sums y - pivot and hrl_bn_finalize_fwd adds the pivot back, so that fp32 sums of y and y^2 do not
        cancel when |mean| >> std.  The running statistics are saved state: a step's arithmetic depends on nothing a
        checkpoint or a rejected step leaves out."""
        bns = [(blk[1], st) for blk, st in zip(self.model.tower, self.bn)]
        pivots = lambda ts: C.cast((C.c_void_p * max(1, len(ts)))(*[t.data_ptr() for t in ts]), C.c_void_p)
        for i in range(0, len(jobs), MAX_BOARD_JOBS):
            chunk = jobs[i:i + MAX_BOARD_JOBS]
            piv = bns[i:i + MAX_BOARD_JOBS]
            arr = (HrlPackJob * len(chunk))()
            for j, kw in zip(arr, chunk):
                w = kw['w']
                j.w, (j.Cout, j.Cin, j.kh, j.kw), j.H, j.W = _ptr(w), w.shape, self.H, self.W
                j.image_fwd, j.fwd_rows, j.fwd_row0 = _ptr(kw.get('fwd')), kw.get('fwd_rows', 0), kw.get('fwd_row0', 0)
                j.image_bwd, j.bwd_rows, j.bwd_k0 = _ptr(kw.get('bwd')), kw.get('bwd_rows', 0), kw.get('bwd_k0', 0)
                j.bias, j.bias_cells = _ptr(kw.get('bias')), _ptr(kw.get('bias_cells'))
                j.bf16 = int(self.bf16)
            check(lib().hrl_board_pack_many_pivot(C.byref(arr), len(chunk), pivots([b.running_mean for b, _ in piv]),
                                                  pivots([b.running_var for b, _ in piv]), pivots([st['mean'] for _, st in piv]),
                                                  len(piv), self.width, self.cells, _stream_ptr()))
            _count()

    def _fold_all(self, accumulate):
        """Every weight-gradient product of the backward pass onto its convolution's taps, in one launch (added to the
        gradients when `accumulate`)."""
        jobs, self.fold_jobs = self.fold_jobs, []
        for i in range(0, len(jobs), MAX_BOARD_JOBS):
            chunk = jobs[i:i + MAX_BOARD_JOBS]
            arr = (HrlFoldJob * len(chunk))()
            for j, (src, splits, stride, grad) in zip(arr, chunk):
                j.ddense, j.splits, j.split_stride, j.dw = _ptr(src), splits, stride, _ptr(grad)
                (j.Cout, j.Cin, j.kh, j.kw), j.H, j.W = grad.shape, self.H, self.W
                j.accumulate = int(accumulate)
            check(lib().hrl_board_fold_many(C.byref(arr), len(chunk), _stream_ptr()))
            _count()

    def _wgrad(self, a, b, rows, cols, region, grads):
        """dense gradient (rows x cols) = A_op^T-style product over the samples, left as slice partials in the product's
        workspace region; queued for the fold onto the conv weights.  grads: list of (weight.grad tensor, first dense row)."""
        s = self.splits[region[0]]
        ws = self.ws[self.ws_at[region]:]
        self._gemm(a, b, None, K=self.M, N=cols, M=rows, splits=s, partial=True, ws=ws)
        for grad, row0 in grads:
            self.fold_jobs.append((ws[row0 * cols:], s, rows * cols if s > 1 else 0, grad))

    # ------------------------------------------------------------------ forward
    def forward(self, x):
        """x (M, planes, H, W) -> {'policy': (M, A), 'value': (M, 1)[, 'return': (M, 1)]} (static buffers)."""
        m = self.model
        M_, D = self.M, self.D
        assert x.shape[0] == M_ and x.is_contiguous() and x.dtype == torch.float32
        H, W = x.shape[2], x.shape[3]
        self.H, self.W = H, W
        self.x2d = x.view(M_, self.K0)
        with torch.no_grad():
            # every convolution's weights (and the biases of the stem / squeeze convolutions, one copy per cell) in one launch
            jobs = [dict(w=m.stem.weight, fwd=self.W0f, fwd_rows=D, bias=m.stem.bias, bias_cells=self.b0)]
            for l, blk in enumerate(m.tower):
                jobs.append(dict(w=blk[0].weight, fwd=self.Wf[l], fwd_rows=D, bwd=self.Wb[l], bwd_rows=D))
            heads = [(m.p_squeeze, 0), (m.v_squeeze, self.pmaps * self.cells)] + \
                ([(m.r_squeeze, (self.pmaps + self.vmaps) * self.cells)] if self.rmaps else [])
            for sq_, row0 in heads:       # the squeeze convolutions side by side in ONE operand
                jobs.append(dict(w=sq_.weight, fwd=self.Whf, fwd_rows=self.NH, fwd_row0=row0, bwd=self.Whb, bwd_rows=D, bwd_k0=row0,
                                 bias=sq_.bias, bias_cells=self.bh[row0:]))
            self._pack_all(jobs)          # (and the BatchNorm statistics pivots)
            # stem: bias + ReLU in the epilogue
            self._gemm(dict(t=self.x2d), dict(t=self.W0f, packed=True), self.A0, K=self.K0, N=D, bias=self.b0, epilogue='relu')
            src = dict(t=self.A0)
            for l, blk in enumerate(m.tower):
                bnm, st = blk[1], self.bn[l]
                self._gemm(src, dict(t=self.Wf[l], packed=True), self.Y[l], K=D, N=D, epilogue='stats', ep=dict(mean=st['mean']))
                check(lib().hrl_bn_finalize_fwd(_ptr(self.cp), self.tiles, self.width, self.cells, M_, _ptr(bnm.weight), _ptr(bnm.bias),
                                                float(bnm.eps), float(bnm.momentum), _ptr(bnm.running_mean), _ptr(bnm.running_var),
                                                _ptr(bnm.num_batches_tracked), _ptr(st['mean']), _ptr(st['rstd']), _ptr(st['scale']),
                                                _ptr(st['shift']), _stream_ptr()))
                _count()
                src = dict(t=self.Y[l], consts=(st['scale'], st['shift']), relu=True)
            self._gemm(src, dict(t=self.Whf, packed=True), self.Hpre, K=D, N=self.NH, bias=self.bh)
            check(lib().hrl_heads_fwd(_ptr(self.Hpre), self.ldh, M_, self.cells, self.pmaps, self.vmaps, self.rmaps, self.A, self.slope,
                                      _ptr(m.p_out.weight), _ptr(m.v_out.weight), _ptr(m.r_out.weight) if self.rmaps else None,
                                      _ptr(self.policy), _ptr(self.value), _ptr(self.ret), _stream_ptr()))
            _count()
        out = {'policy': self.policy, 'value': self.value}
        if self.rmaps:
            out['return'] = self.ret
        return out

    # ------------------------------------------------------------------ backward
    def backward(self, dpolicy, dvalue, dreturn=None, accumulate=False):
        """Gradients of every parameter from the output gradients, written into param.grad (which must exist), or added to
        what param.grad holds when `accumulate` (the micro-batches after the first of a gradient-accumulation step)."""
        m = self.model
        M_, D, H, W = self.M, self.D, self.H, self.W
        L = self.depth
        with torch.no_grad():
            g = lambda p_: p_.grad
            # (named: a temporary copy freed before the launch could be handed to the next .contiguous())
            dpolicy, dvalue = dpolicy.contiguous(), dvalue.contiguous()
            dreturn = dreturn.contiguous() if self.rmaps else None
            acc = int(accumulate)
            check(lib().hrl_heads_bwd(_ptr(self.Hpre), self.ldh, M_, self.cells, self.pmaps, self.vmaps, self.rmaps, self.A, self.slope,
                                      _ptr(m.p_out.weight), _ptr(m.v_out.weight), _ptr(m.r_out.weight) if self.rmaps else None,
                                      _ptr(self.value), _ptr(dpolicy), _ptr(dvalue),
                                      _ptr(dreturn), _ptr(self.dHpre),
                                      _ptr(g(m.p_out.weight)), _ptr(g(m.v_out.weight)), _ptr(g(m.r_out.weight)) if self.rmaps else None,
                                      _ptr(g(m.p_squeeze.bias)), _ptr(g(m.v_squeeze.bias)), _ptr(g(m.r_squeeze.bias)) if self.rmaps else None,
                                      _ptr(self.heads_ws), acc, _stream_ptr()))
            _count(2)
            top = self.bn[L - 1]
            a_top = dict(t=self.Y[L - 1], consts=(top['scale'], top['shift']), relu=True)          # A_L = relu(bn_L(Y_L))
            # squeeze convolutions: weight gradient, then the gradient entering the tower with the last ReLU mask + BN sums
            heads = [(g(m.p_squeeze.weight), 0), (g(m.v_squeeze.weight), self.pmaps * self.cells)]
            if self.rmaps:
                heads.append((g(m.r_squeeze.weight), (self.pmaps + self.vmaps) * self.cells))
            self._wgrad(dict(t=self.dHpre, kmajor=False), dict(a_top, kmajor=False, by_row=True), self.NH, D, ('heads', 0), heads)
            self._gemm(dict(t=self.dHpre), dict(t=self.Whb, packed=True), self.dZ[L - 1], K=self.NH, N=D, epilogue='mask_stats',
                       ep=dict(y=self.Y[L - 1], scale=top['scale'], shift=top['shift'], mean=top['mean'], rstd=top['rstd']))
            for l in range(L - 1, -1, -1):
                blk, st = m.tower[l], self.bn[l]
                bnm = blk[1]
                check(lib().hrl_bn_finalize_bwd(_ptr(self.cp), self.tiles, self.width, self.cells, M_, _ptr(bnm.weight),
                                                _ptr(st['mean']), _ptr(st['rstd']), _ptr(g(bnm.weight)), _ptr(g(bnm.bias)),
                                                _ptr(st['p']), _ptr(st['q']), _ptr(st['r']), acc, _stream_ptr()))
                _count()
                dy = dict(t=self.dZ[l], t2=self.Y[l], consts=(st['p'], st['q'], st['r']))            # dY_l from dZ_l on the fly
                if l > 0:
                    below = self.bn[l - 1]
                    a_in = dict(t=self.Y[l - 1], consts=(below['scale'], below['shift']), relu=True)
                else:
                    a_in = dict(t=self.A0)
                self._wgrad(dict(dy, kmajor=False, by_row=True), dict(a_in, kmajor=False, by_row=True), D, D, ('tower', l),
                            [(g(blk[0].weight), 0)])
                if l > 0:
                    self._gemm(dy, dict(t=self.Wb[l], packed=True), self.dZ[l - 1], K=D, N=D, epilogue='mask_stats',
                               ep=dict(y=self.Y[l - 1], scale=below['scale'], shift=below['shift'], mean=below['mean'], rstd=below['rstd']))
                else:
                    self._gemm(dy, dict(t=self.Wb[0], packed=True), self.dZ0, K=D, N=D, epilogue='mask_stats', ep=dict(y=self.A0))
            # stem: bias gradient from the column sums of dZ0, weight gradient over the raw observations
            check(lib().hrl_bn_finalize_bwd(_ptr(self.cp), self.tiles, self.width, self.cells, M_, None, None, None, None,
                                            _ptr(g(m.stem.bias)), None, None, None, acc, _stream_ptr()))
            _count()
            self._wgrad(dict(t=self.dZ0, kmajor=False), dict(t=self.x2d, kmajor=False), D, self.K0, ('stem', 0), [(g(m.stem.weight), 0)])
            self._fold_all(accumulate)
