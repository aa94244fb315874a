"""The fused tower engine (tower.FusedBoardNet) in its default 3xTF32 precision, stage by stage against float64, and the
kernels it chains between its products (csrc/tower_kernel.cu, csrc/net_kernel.cu) on their own.

Each float64 stage takes its inputs from the engine's own buffers of the stage before (the previous layer's output, the
BatchNorm constants the finalise kernels left), so every bound below belongs to one stage's arithmetic:

* a 3xTF32 product of K terms is within U32 (K_slice + 8) of sum|a||b| (the bound test_gemm_tower_gpu.py holds the kernels
  to).  The fp32 accumulator truncates, and with ReLU'd operands the errors do not cancel: the bound is linear in K.  The
  operand transforms (BatchNorm-apply + ReLU, the BatchNorm backward) are fmaf's in fp32; tower_ref._transform_ref gives that
  fp32 operand exactly, and the products split it into hi and lo with no further rounding, so no transform term is needed;
* a sum of n fp32 terms in any order is within (n + 1) U32 of sum|terms|;
* a weight gradient is its K slices' products, then hrl_board_fold's fp32 sums over the slices and the output cells
  (tower_ref._wgrad_bound);
* the batch statistics, rstd and running buffers take the bounds of test_bf16_gpu.py, of the sums of y - pivot.
"""
import copy
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from tower_ref import U32, _close, _conv, _conv_in, _conv_w, _transform_ref, _wgrad_bound, traced_gemms

pytestmark = pytest.mark.gpu


def tf32x3_bound(K, splits=1):
    """a 3xTF32 product over K terms in `splits` K slices of whole 32-element chunks, relative to sum|a||b|"""
    from handyrl_b200._capi import lib
    chunks = -(-K // 32)
    per = -(-chunks // lib().hrl_gemm_effective_splits(K, splits))
    return U32 * (min(K, 32 * per) + 8)


CFG2 = dict(planes=3, board=(3, 3), width=32, depth=3, actions=9)
CASES = {         # net (nets.BoardNet kwargs), M, and what the case reaches
    'cfg2': (CFG2, 16384),                 # the benchmark's shapes: tower kernel, many weight-gradient K slices, heads K = 27
    'ragged300': (CFG2, 300),              # a partial last row tile
    'ragged100': (CFG2, 100),              # one K slice: the weight gradients write C directly, fold stride 0
    'narrow': (dict(planes=3, board=(3, 3), width=16, depth=2, actions=9, return_head=True), 515),      # D = 144: wgmma kernel
    'below_floor': (dict(planes=3, board=(3, 3), width=28, depth=2, actions=9), 1000),                # D = 252 < 257
    'non_square': (dict(planes=3, board=(2, 5), width=28, depth=2, actions=32), 1000),                # D = 280, 10 cells
    # 16 cells, D = 288, 64 squeeze outputs and 32 actions (the heads' limits), stem K0 = 320 in 16-byte rows
    'limits': (dict(planes=20, board=(4, 4), width=18, depth=2, actions=32, return_head=True), 1000),
    'deep': (dict(planes=3, board=(3, 3), width=8, depth=9, actions=9), 515),                          # 12 pack / fold jobs
    'pivot': (CFG2, 1000),                 # a nonzero BatchNorm statistics pivot in layer 1
}


def _make(name):
    from handyrl_b200 import nets, tower
    kw, M = CASES[name]
    torch.manual_seed(sum(map(ord, name)))
    net = nets.BoardNet(**kw).cuda().train()
    for blk in net.tower:                # non-trivial affine parameters and running statistics
        blk[1].weight.data.uniform_(0.5, 1.5)
        blk[1].bias.data.normal_(0, 0.3)
        blk[1].running_mean.normal_(0, 0.1)
        blk[1].running_var.uniform_(0.5, 2.0)
    if name == 'pivot':
        net.tower[1][1].running_var.fill_(1e-4)
        net.tower[1][1].running_mean.fill_(1.0)
    assert tower.supports(net)
    x = (torch.rand(M, kw['planes'], *kw['board'], device='cuda') < 0.4).float()
    return net, tower.FusedBoardNet(net, M, torch.device('cuda')), x


def _routes(name, net, eng, x, monkeypatch):
    """The route the case is there for: the pack and fold launches of one forward and backward, and the GEMM kernels of traced
    ones (the net's state is restored afterwards)."""
    from handyrl_b200 import _capi
    from handyrl_b200._capi import MAX_BOARD_JOBS
    state = copy.deepcopy(net.state_dict())
    calls = {'hrl_board_pack_many_pivot': [], 'hrl_board_fold_many': []}
    lib = _capi.lib()
    for fn in calls:
        real = getattr(lib, fn)
        monkeypatch.setattr(lib, fn, lambda *a, _real=real, _n=calls[fn]: (_n.append(a[1]), _real(*a))[1])
    for p in net.parameters():
        p.grad = torch.zeros_like(p)

    def step():
        out = eng.forward(x)
        eng.backward(*[torch.ones_like(out[k]) for k in ('policy', 'value')], torch.ones_like(out['return']) if eng.rmaps else None)
    step()
    monkeypatch.undo()
    seen = traced_gemms(step, runs=3, repeat=2)
    net.load_state_dict(state)
    tower_kernel = {a for k, a in seen if k == 'gemm_tower_kernel'}
    wgmma = {a for k, a in seen if k == 'gemm_tf32x3_kernel'}
    assert bool(tower_kernel) == (257 <= eng.D <= 288), seen
    if eng.D > 256:
        assert tower_kernel == {'0', '1', '2'}, seen
    if name == 'cfg2':
        assert min(eng.splits.values()) > 1 and eng.splits['tower'] > 8
    if name == 'ragged100':
        assert set(eng.splits.values()) == {1}
    if name == 'limits':
        assert eng.NH == 64 and eng.A == 32 and eng.cells == 16 and eng.K0 == 320 and eng.D == 288
        assert len(wgmma) == 1, seen                     # the heads' forward only: the stem's forward is on the tower kernel
        assert ('gemm_wgrad_kernel', '0,0') in seen      # the stem's weight gradient, two plain operands
    n_jobs = 1 + eng.depth + 2 + (eng.rmaps > 0)
    assert sum(calls['hrl_board_pack_many_pivot']) == n_jobs and sum(calls['hrl_board_fold_many']) == n_jobs
    assert max(calls['hrl_board_pack_many_pivot'] + calls['hrl_board_fold_many']) <= MAX_BOARD_JOBS
    if name == 'deep':
        assert calls['hrl_board_pack_many_pivot'] == [8, 4] and calls['hrl_board_fold_many'] == [8, 4]


@pytest.mark.parametrize('name', list(CASES))
def test_fused_tower_products_against_float64(name, monkeypatch):
    net, eng, x = _make(name)
    _routes(name, net, eng, x, monkeypatch)
    run0 = [(blk[1].running_mean.clone(), blk[1].running_var.clone(), int(blk[1].num_batches_tracked)) for blk in net.tower]
    for p in net.parameters():
        p.grad = torch.full_like(p, float('nan'))       # backward must overwrite every element
    out = eng.forward(x)
    g = torch.Generator().manual_seed(5)
    dout = {k: torch.randn(v.shape, generator=g).cuda() for k, v in out.items()}
    eng.backward(dout['policy'], dout['value'], dout.get('return'))
    torch.cuda.synchronize()
    M, (H, W) = eng.M, CASES[name][0]['board']
    L, C_, NH, D, cells = eng.depth, eng.width, eng.NH, eng.D, eng.cells
    n = M * cells
    img = lambda t, ch: t.double().reshape(M, ch, H, W)
    w64 = lambda w: w.detach().double()
    wabs = lambda w: w.detach().double().abs()

    def act(l):
        """the operand the engine builds from layer l's output: relu(fmaf(Y_l, scale, shift)) in fp32 (l = -1: A0)"""
        if l < 0:
            return eng.A0.double()
        st = eng.bn[l]
        return _transform_ref(eng.Y[l], st['scale'][None], st['shift'][None], relu=True, bf16=False)[0]

    def mask(l):
        if l < 0:
            return eng.A0.double() > 0
        st = eng.bn[l]
        return (eng.Y[l].double() * st['scale'].double() + st['shift'].double()).float() > 0          # fmaf in fp32

    # ---- forward: stem (bias + ReLU in the epilogue)
    w0, b0 = net.stem.weight, net.stem.bias.detach().double()
    xd = x.double()
    _close(eng.A0.view(M, C_, H, W), F.relu(_conv(xd, w64(w0), b0)), tf32x3_bound(eng.K0) * _conv(xd, wabs(w0), b0.abs()), 'A0')
    # ---- tower layers: product, batch statistics, finalised constants, running buffers
    for l, blk in enumerate(net.tower):
        a, wl, bn, st = act(l - 1), blk[0].weight, blk[1], eng.bn[l]
        _close(eng.Y[l].view(M, C_, H, W), _conv(img(a, C_), w64(wl)), tf32x3_bound(D) * _conv(img(a.abs(), C_), wabs(wl)), 'Y%d' % l)
        rm0, rv0, nbt0 = run0[l]
        # the statistics pivot hrl_board_pack_many_pivot chose from the running buffers on entry (fp32 comparison)
        pivot = torch.where(rm0 * rm0 > 1024 * rv0, rm0, torch.zeros_like(rm0)).double()
        assert (pivot != 0).any() == (name == 'pivot' and l == 1)
        y = eng.Y[l].double().view(M, C_, cells)
        d = y - pivot[None, :, None]
        mean, var = y.mean((0, 2)), y.var((0, 2), unbiased=False)
        # column partials: fp32 sums of d = y - pivot (one rounding each) over a 128-row tile, summed over the tiles in double
        e_mean = 128 * U32 * d.abs().mean((0, 2))
        e_var = 4 * 128 * U32 * (d * d).mean((0, 2))
        _close(st['mean'].view(C_, cells), mean[:, None].expand(C_, cells), (e_mean + U32 * mean.abs())[:, None] + 1e-30, 'mean%d' % l)
        rstd = (var + bn.eps).rsqrt()
        _close(st['rstd'].view(C_, cells), rstd[:, None].expand(C_, cells), (rstd * (e_var / (var + bn.eps) + 4 * U32))[:, None], 'rstd%d' % l)
        gamma, beta = bn.weight.detach().repeat_interleave(cells), bn.bias.detach().repeat_interleave(cells)
        assert torch.equal(st['scale'], gamma * st['rstd']), 'scale%d' % l                    # one fp32 product
        sh = beta.double() - st['mean'].double() * st['scale'].double()
        _close(st['shift'], sh, 2 * U32 * (beta.double().abs() + (st['mean'].double() * st['scale'].double()).abs()), 'shift%d' % l)
        m_ = bn.momentum
        rm0, rv0 = rm0.double(), rv0.double()
        _close(bn.running_mean, (1 - m_) * rm0 + m_ * mean, m_ * e_mean + 4 * U32 * (rm0.abs() + mean.abs()), 'running_mean%d' % l)
        _close(bn.running_var, (1 - m_) * rv0 + m_ * var * n / (n - 1), m_ * e_var * n / (n - 1) + 4 * U32 * (rv0 + var), 'running_var%d' % l)
        assert int(bn.num_batches_tracked) == nbt0 + 1
    # ---- squeeze convolutions side by side, bias in the epilogue
    sq = [net.p_squeeze, net.v_squeeze] + ([net.r_squeeze] if eng.rmaps else [])
    wsq = torch.cat([s.weight for s in sq])
    bsq = torch.cat([s.bias for s in sq]).detach().double()
    a_top = act(L - 1)
    bound = tf32x3_bound(D) * _conv(img(a_top.abs(), C_), wabs(wsq), bsq.abs())
    _close(eng.Hpre[:, :NH], _conv(img(a_top, C_), w64(wsq), bsq).reshape(M, NH), bound.reshape(M, NH), 'Hpre')
    # ---- heads (fp32 kernels): LeakyReLU, the Linear layers (fmaf chains), tanh on the value
    pre = eng.Hpre[:, :NH].double()
    pc, vc = eng.pmaps * cells, eng.vmaps * cells
    parts = {'policy': (slice(0, pc), net.p_out), 'value': (slice(pc, pc + vc), net.v_out)}
    if eng.rmaps:
        parts['return'] = (slice(pc + vc, NH), net.r_out)
    for k, (cols, lin) in parts.items():
        h = F.leaky_relu(pre[:, cols], eng.slope)
        wl = w64(lin.weight)
        z, za = h @ wl.t(), h.abs() @ wl.abs().t()
        _close(out[k], torch.tanh(z) if k == 'value' else z, (h.shape[1] + 2) * U32 * za + (4 * U32 if k == 'value' else 0), k)

    # ---- backward: heads (dHpre and the Linear weights' gradients)
    for k, (cols, lin) in parts.items():
        wl = w64(lin.weight)
        dk = dout[k].double()
        dz = dk * (1 - eng.value.double() ** 2) if k == 'value' else dk
        slope = torch.where(pre[:, cols] > 0, 1.0, eng.slope)        # LeakyReLU's gradient at 0 is the slope, as in PyTorch
        h = F.leaky_relu(pre[:, cols], eng.slope)
        dza = dz.abs() + (4 * U32 * dk.abs() if k == 'value' else 0)
        _close(eng.dHpre[:, cols], slope * (dz @ wl), (wl.shape[0] + 2) * U32 * slope * (dza @ wl.abs()), 'dpre_' + k)
        _close(lin.weight.grad, dz.t() @ h, (M + 2) * U32 * (dza.t() @ h.abs()), k + '_out.grad')
    dh = eng.dHpre[:, :NH].double()
    dhi, dhai = img(dh, NH // cells), img(dh.abs(), NH // cells)
    # squeeze convolutions: bias gradients (column sums of dHpre), weight gradient over the samples, folded over the cells
    dw_ref = _conv_w(img(a_top, C_), wsq.shape, dhi)
    dw_bound = _wgrad_bound(M, eng.splits['heads'], cells, tf32x3_bound) * _conv_w(img(a_top.abs(), C_), wsq.shape, dhai)
    row = 0
    for s in sq:
        o = s.out_channels
        _close(s.weight.grad, dw_ref[row:row + o], dw_bound[row:row + o], 'squeeze.weight.grad')
        seg = eng.dHpre[:, row * cells:(row + o) * cells].double().view(M, o, cells)
        _close(s.bias.grad, seg.sum((0, 2)), (n + 1) * U32 * seg.abs().sum((0, 2)), 'squeeze.bias.grad')
        row += o
    # the gradient entering the tower: dHpre through the squeeze convolutions' adjoint image, the last ReLU mask applied
    dz_ref = _conv_in((M, C_, H, W), w64(wsq), dhi).reshape(M, -1) * mask(L - 1)
    _close(eng.dZ[L - 1], dz_ref, tf32x3_bound(NH) * _conv_in((M, C_, H, W), wabs(wsq), dhai).reshape(M, -1), 'dZ%d' % (L - 1))

    # ---- backward: tower layers
    for l in range(L - 1, -1, -1):
        blk, st = net.tower[l], eng.bn[l]
        bn, wl = blk[1], blk[0].weight
        dz = eng.dZ[l].double().view(M, C_, cells)
        xh = ((eng.Y[l] - st['mean']) * st['rstd']).double().view(M, C_, cells)          # the epilogue's fp32 xhat
        _close(bn.bias.grad, dz.sum((0, 2)), (n + 1) * U32 * dz.abs().sum((0, 2)), 'bn%d.bias.grad' % l)
        _close(bn.weight.grad, (dz * xh).sum((0, 2)), (n + 2) * U32 * (dz * xh).abs().sum((0, 2)), 'bn%d.weight.grad' % l)
        # the BatchNorm backward as dY = dZ p + Y q + r, from the batch sums the weight and bias gradients hold
        gamma = bn.weight.detach().repeat_interleave(cells)
        p = st['p'].double()
        assert torch.equal(st['p'], gamma * st['rstd']), 'p%d' % l
        rs, mu = st['rstd'].double(), st['mean'].double()
        mdz = bn.bias.grad.double().repeat_interleave(cells) / n
        mdzx = bn.weight.grad.double().repeat_interleave(cells) / n
        _close(st['q'], -p * rs * mdzx, 3 * U32 * (p * rs * mdzx).abs() + 1e-30, 'q%d' % l)
        _close(st['r'], p * (rs * mu * mdzx - mdz), 4 * U32 * p.abs() * ((rs * mu * mdzx).abs() + mdz.abs()) + 1e-30, 'r%d' % l)
        dy = _transform_ref(eng.dZ[l], st['p'][None], st['r'][None], y=eng.Y[l], q=st['q'][None], bf16=False)[0]
        a = act(l - 1)
        dyi, dyai, ai, aai = img(dy, C_), img(dy.abs(), C_), img(a, C_), img(a.abs(), C_)
        bound = _wgrad_bound(M, eng.splits['tower'], cells, tf32x3_bound) * _conv_w(aai, wl.shape, dyai)
        _close(wl.grad, _conv_w(ai, wl.shape, dyi), bound, 'tower%d.weight.grad' % l)
        target = eng.dZ[l - 1] if l > 0 else eng.dZ0
        want = _conv_in((M, C_, H, W), w64(wl), dyi).reshape(M, -1) * mask(l - 1)
        _close(target, want, tf32x3_bound(D) * _conv_in((M, C_, H, W), wabs(wl), dyai).reshape(M, -1), 'dZ%d' % (l - 1))
    # ---- backward: stem
    dz0 = eng.dZ0.double().view(M, C_, cells)
    _close(net.stem.bias.grad, dz0.sum((0, 2)), (n + 1) * U32 * dz0.abs().sum((0, 2)), 'stem.bias.grad')
    bound = _wgrad_bound(M, eng.splits['stem'], cells, tf32x3_bound) * _conv_w(xd, w0.shape, dz0.abs().view(M, C_, H, W))
    _close(w0.grad, _conv_w(xd, w0.shape, dz0.view(M, C_, H, W)), bound, 'stem.weight.grad')
    for p in net.parameters():
        assert torch.isfinite(p.grad).all()

    # ---- accumulate: the same backward again adds the same deterministic values, exactly doubling every gradient
    first = {k: p.grad.clone() for k, p in net.named_parameters()}
    eng.backward(dout['policy'], dout['value'], dout.get('return'), accumulate=True)
    torch.cuda.synchronize()
    for k, p in net.named_parameters():
        assert torch.equal(p.grad, 2 * first[k]), k


def test_learner_step_keeps_nets_past_the_packed_rows_on_the_module_path():
    """BoardNet(board=(4, 4), width=32) has D = 512 rows per convolution image: no engine, and a step on the module path."""
    from handyrl_b200.nets import BoardNet
    from handyrl_b200.synthetic import synthetic_batch
    from handyrl_b200.train import LearnerStep
    args = {'turn_based_training': True, 'observation': False, 'gamma': 0.8, 'lambda': 0.7, 'burn_in_steps': 0, 'forward_steps': 4,
            'entropy_regularization': 0.1, 'entropy_regularization_decay': 0.1, 'policy_target': 'UPGO', 'value_target': 'VTRACE'}
    torch.manual_seed(1)
    net = BoardNet(planes=3, board=(4, 4), width=32, depth=2, actions=16)
    mk = lambda s: synthetic_batch(16, 4, 2, 16, seed=s, obs_shape=(3, 4, 4))
    stepper = LearnerStep(net, args, mk(0), lr=1e-3)
    assert stepper.engine is None
    before = {k: v.clone() for k, v in stepper.cpu_state_dict().items()}
    stepper.step(stepper.new_packed().fill(mk(1)))
    losses = stepper.read_losses()
    assert all(torch.isfinite(torch.tensor(v)) for v in losses.values())
    after = stepper.cpu_state_dict()
    assert any(not torch.equal(before[k], after[k]) for k in before if 'weight' in k)


# ---- the heads' kernels on their own ------------------------------------------------------------------------------------
def _heads(pre, ld, M, cells, maps, A, W, slope, dout, acc, grads):
    from handyrl_b200._capi import check, lib
    from handyrl_b200.ops import _ptr, _stream_ptr
    pm, vm, rm = maps
    policy = torch.full((M, A), float('nan'), device='cuda')
    value = torch.full((M, 1), float('nan'), device='cuda') if vm else None
    ret = torch.full((M, 1), float('nan'), device='cuda') if rm else None
    check(lib().hrl_heads_fwd(_ptr(pre), ld, M, cells, pm, vm, rm, A, slope, _ptr(W['p']), _ptr(W.get('v')), _ptr(W.get('r')),
                              _ptr(policy), _ptr(value), _ptr(ret), _stream_ptr()))
    dpre = torch.full((M, ld), -3.0, device='cuda')
    ws = torch.empty(lib().hrl_heads_num_blocks(M) * sum(t.numel() for t in grads.values()), device='cuda')
    g = lambda k: _ptr(grads.get(k))
    check(lib().hrl_heads_bwd(_ptr(pre), ld, M, cells, pm, vm, rm, A, slope, _ptr(W['p']), _ptr(W.get('v')), _ptr(W.get('r')),
                              _ptr(value), _ptr(dout['p']), _ptr(dout.get('v')), _ptr(dout.get('r')), _ptr(dpre),
                              g('wp'), g('wv'), g('wr'), g('bp'), g('bv'), g('br'), _ptr(ws), int(acc), _stream_ptr()))
    torch.cuda.synchronize()
    return policy, value, ret, dpre


@pytest.mark.parametrize('M', [1, 127, 128, 129])
@pytest.mark.parametrize('maps,A', [((4, 0, 0), 32), ((2, 1, 1), 32), ((2, 1, 0), 9)])
def test_heads_kernels_against_float64(maps, A, M):
    """hrl_heads_fwd and hrl_heads_bwd over 16 cells: LeakyReLU(0.1), the bias-free Linear heads and tanh, and their
    gradients, with exact zeros in the squeeze outputs and NaN in the padding columns of `pre` (ld > NH)."""
    cells, slope = 16, 0.1
    pm, vm, rm = maps
    NH = (pm + vm + rm) * cells
    ld = NH + 4
    g = torch.Generator(device='cuda').manual_seed(M * 10 + A + pm)
    rnd = lambda *s: torch.randn(*s, device='cuda', generator=g)
    pre = torch.full((M, ld), float('nan'), device='cuda')
    pre[:, :NH] = rnd(M, NH) * (rnd(M, NH).abs() > 0.3)               # about a quarter exact zeros
    W = {'p': rnd(A, pm * cells) * 0.3}
    dout = {'p': rnd(M, A)}
    if vm:
        W['v'], dout['v'] = rnd(1, vm * cells) * 0.3, rnd(M, 1)
    if rm:
        W['r'], dout['r'] = rnd(1, rm * cells) * 0.3, rnd(M, 1)
    shapes = {'wp': (A, pm * cells), 'wv': (1, vm * cells), 'wr': (1, rm * cells), 'bp': (pm,), 'bv': (vm,), 'br': (rm,)}
    shapes = {k: s for k, s in shapes.items() if s[-1] > 0}
    grads = {k: torch.full(s, float('nan'), device='cuda') for k, s in shapes.items()}
    policy, value, ret, dpre = _heads(pre, ld, M, cells, maps, A, W, slope, dout, False, grads)
    x = pre[:, :NH].double()
    spans = {'p': slice(0, pm * cells), 'v': slice(pm * cells, (pm + vm) * cells), 'r': slice((pm + vm) * cells, NH)}
    outs = {'p': policy, 'v': value, 'r': ret}
    want_dpre = torch.zeros_like(x)
    for k in [k for k in 'pvr' if k in W]:
        cols, wk = spans[k], W[k].double()
        h = F.leaky_relu(x[:, cols], slope)
        z, za = h @ wk.t(), h.abs() @ wk.abs().t()
        # fmaf chains of n terms (n + 1 roundings) on h rounded once; tanhf within 2 ulp
        _close(outs[k], torch.tanh(z) if k == 'v' else z, (h.shape[1] + 2) * U32 * za + (4 * U32 if k == 'v' else 0), k)
        dk = dout[k].double()
        dz = dk * (1 - value.double() ** 2) if k == 'v' else dk              # the kernel's (1 - v*v) on its own value
        dza = dz.abs() + (4 * U32 * dk.abs() if k == 'v' else 0)
        gain = torch.where(x[:, cols] > 0, 1.0, slope)                     # slope at exact zeros, as torch's leaky_relu
        want_dpre[:, cols] = gain * (dz @ wk)
        _close(dpre[:, cols], want_dpre[:, cols], (wk.shape[0] + 2) * U32 * gain * (dza @ wk.abs()), 'dpre_' + k)
        # weight gradients: per 128-row block fmaf chains, summed over the blocks in double
        _close(grads['w' + k], dz.t() @ h, (min(M, 128) + 2) * U32 * (dza.t() @ h.abs()), 'dW' + k)
        maps_k = {'p': pm, 'v': vm, 'r': rm}[k]
        seg = dpre[:, cols].double().view(M, maps_k, cells)
        _close(grads['b' + k], seg.sum((0, 2)), (min(M, 128) * cells + 1) * U32 * seg.abs().sum((0, 2)), 'db' + k)
    assert (x == 0).any()
    assert torch.equal(dpre[:, NH:], torch.full_like(dpre[:, NH:], -3.0))      # the padding columns are not written
    # accumulate: each gradient becomes what it held plus the same fp32 value
    held = {k: torch.randn(s, device='cuda', generator=g) for k, s in shapes.items()}
    acc = {k: v.clone() for k, v in held.items()}
    _, _, _, dpre2 = _heads(pre, ld, M, cells, maps, A, W, slope, dout, True, acc)
    assert torch.equal(dpre2, dpre)
    for k in shapes:
        assert torch.equal(acc[k], held[k] + grads[k]), k


# ---- hrl_board_fold_many on its own -------------------------------------------------------------------------------------
FOLD_JOBS = [       # Cout, Cin, k, H, W, splits
    (32, 32, 3, 3, 3, 37),
    (3, 32, 1, 3, 3, 7),
    (18, 20, 3, 4, 4, 13),
    (4, 18, 1, 4, 4, 1),
    (28, 28, 3, 2, 5, 37),
    (3, 28, 1, 2, 5, 13),
    (8, 3, 3, 3, 3, 1),
    (8, 8, 3, 4, 4, 7),
]


def _fold(jobs, dws, accumulate):
    from handyrl_b200._capi import HrlFoldJob, check, lib
    from handyrl_b200.ops import _ptr, _stream_ptr
    arr = (HrlFoldJob * len(jobs))()
    for j, (src, splits, stride, H, W), dw, acc in zip(arr, jobs, dws, accumulate):
        j.ddense, j.splits, j.split_stride, j.dw = _ptr(src), splits, stride, _ptr(dw)
        (j.Cout, j.Cin, j.kh, j.kw), j.H, j.W = dw.shape, H, W
        j.accumulate = int(acc)
    check(lib().hrl_board_fold_many(C.byref(arr), len(jobs), _stream_ptr()))
    torch.cuda.synchronize()


def test_board_fold_many_against_float64():
    """One launch of eight jobs: 3x3 and 1x1 kernels over 3x3, 4x4 and 2x5 boards; one slice at stride 0 (the single-part
    branch) and 7, 13 or 37 slices at a stride longer than a slice (the slice-run branch, runs of unequal length, its 4-wide
    loop and tail).  Against float64: the slices summed, then folded onto the taps through the adjoint of the F.unfold form of
    the dense matrix (test_net_kernels_gpu.py).  Then again with every other job accumulating."""
    g = torch.Generator(device='cuda').manual_seed(3)
    jobs, dws, refs = [], [], []
    for Cout, Cin, k, H, W, splits in FOLD_JOBS:
        HW = H * W
        rows, cols_n = Cout * HW, Cin * HW
        stride = 0 if splits == 1 else rows * cols_n + 5
        src = torch.randn(max(1, splits) * max(stride, rows * cols_n), device='cuda', generator=g)
        slices = torch.stack([src[s * stride:s * stride + rows * cols_n] for s in range(splits)]).double().view(splits, Cout, HW, cols_n)
        cols = F.unfold(torch.eye(cols_n, device='cuda', dtype=torch.float64).reshape(-1, Cin, H, W), (k, k), padding=k // 2)
        want = torch.einsum('oqp,pkq->ok', slices.sum(0), cols).reshape(Cout, Cin, k, k)
        mag = torch.einsum('oqp,pkq->ok', slices.abs().sum(0), cols).reshape(Cout, Cin, k, k)
        jobs.append((src, splits, stride, H, W))
        dws.append(torch.full((Cout, Cin, k, k), float('nan'), device='cuda'))
        # fp32 sums over the slices, then over the output cells
        refs.append((want, (splits + HW + 1) * U32 * mag + 1e-30))
    _fold(jobs, dws, [False] * len(jobs))
    for i, (dw, (want, bound)) in enumerate(zip(dws, refs)):
        _close(dw, want, bound, 'job %d %s' % (i, FOLD_JOBS[i]))
    held = [torch.randn(dw.shape, device='cuda', generator=g) for dw in dws]
    again = [h.clone() for h in held]
    flags = [i % 2 == 0 for i in range(len(jobs))]
    _fold(jobs, again, flags)
    for i, (got, h, dw, acc) in enumerate(zip(again, held, dws, flags)):
        assert torch.equal(got, h + dw if acc else dw), (i, acc)
