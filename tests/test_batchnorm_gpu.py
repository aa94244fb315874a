"""Every BatchNorm path of the learner against float64 F.batch_norm (training mode, autograd) on the same fp32 inputs:

(a) hrl_bn_train_fwd / _bwd (fastnet.BoardBatchNorm2d -> ops.batch_norm_train) at shapes that reach each layout branch of
    bn_shape / bn_grid, with channels whose |mean| / std is 300 and 1000, a constant channel, channels scaled by 1e4 and
    1e-4, negative / zero gamma and eps != 1e-5;
(b) the tower engine's hrl_bn_finalize_fwd / _bwd on column partials built from known float64 data;
(c) the tower engine (tower.FusedBoardNet) on a net whose first tower layer sees channels with |mean| / std in the hundreds.

Tolerances are stated per channel with R = |mean| / sqrt(var + eps) and u = 2^-24 (fp32 unit roundoff).  Rounding the mean
to fp32 moves x - mean by up to u * |mean|, i.e. u * R in normalised units: that term grows with R and cannot be avoided
in fp32.  The variance must not lose more than a small multiple of u whatever R is: with unshifted one-pass sums of x and
x^2 it loses about 1e-3 of itself at R = 300 and 1e-2 at R = 1000, which the tests below reject."""
import copy
import ctypes as C
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
VAR_RTOL = 64 * U           # relative error allowed in the batch variance (and rstd), independent of R

# (N, C, H, W, channels_last): the branch of bn_shape / bn_grid each one reaches
SHAPES = {
    'cl_C32_F8': (512, 32, 3, 3, True),            # channels-last, 8 pixels folded per row
    'cl_C3_partial_block': (640, 3, 3, 3, True),   # F*C = 192 columns: a partial column block
    'cl_C256_F1': (300, 256, 3, 3, True),
    'cl_C300_two_blocks': (200, 300, 2, 2, True),
    'cl_C5_odd_rows': (33, 5, 3, 3, True),         # N*HW odd: F = 1
    'nchw_straddle': (700, 32, 3, 3, False),       # C*HW = 288: a channel straddles the 256-column block boundary
    'nchw_HW1': (1000, 6, 1, 1, False),
    'nchw_HW77': (257, 6, 7, 11, False),
    'nchw_HW256': (300, 6, 16, 16, False),         # fastnet.MAX_CELLS
    'nchw_N1': (1, 6, 7, 11, False),
    'cl_N1': (1, 6, 7, 11, True),
    'nchw_N65_ragged_slab': (65, 6, 3, 3, False),
    'cl_slab_cap': (12000, 32, 7, 11, True),       # bn_grid caps the slabs: 110 rows per slab
    'nchw_slab_cap': (2048, 64, 16, 16, False),    # 64 column blocks, 17 slabs of 121 rows
}
GAMMAS = [1.3, -0.7, 0.0, 2.0, 0.5, -1.0]
EPS, MOMENTUM = 1e-3, 0.3


def _channel_data(shape, g):
    """Normal data; per channel (index mod 6): plain, |mean|/std = 300, = 1000, constant, scaled by 1e4, scaled by 1e-4."""
    N, Cn, H, W = shape
    x = torch.randn((N, Cn, H, W), generator=g, dtype=torch.float64) * 2 + 0.5
    for c in range(Cn):
        kind = c % 6
        if kind == 1:                # mean 300, std 1
            x[:, c] = 300.0 + torch.randn((N, H, W), generator=g, dtype=torch.float64)
        elif kind == 2:              # mean -250, std 0.25
            x[:, c] = -250.0 + 0.25 * torch.randn((N, H, W), generator=g, dtype=torch.float64)
        elif kind == 3:
            x[:, c] = 2.5
        elif kind == 4:
            x[:, c] *= 1e4
        elif kind == 5:
            x[:, c] *= 1e-4
    return x.float()


def _worst(err, tol):
    """(worst err / tol, flat index) -- err and tol broadcast; an exact result passes a zero tolerance (gamma = 0)."""
    r = torch.where(err == 0, 0.0, err / tol).flatten()
    i = int(r.argmax())
    return float(r[i]), i


def _check(name, got, want, tol):
    err = (got.double() - want).abs()
    ratio, i = _worst(err, tol.expand_as(err))
    assert ratio <= 1.0, '%s: error %.3g > tolerance %.3g at %d (got %r, want %r)' % (
        name, float(err.flatten()[i]), float(tol.expand_as(err).flatten()[i]), i, float(got.flatten()[i]), float(want.flatten()[i]))


@pytest.mark.parametrize('name', sorted(SHAPES))
def test_bn_train_matches_float64(name):
    from handyrl_b200 import fastnet
    N, Cn, H, W, cl = SHAPES[name]
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    bn = torch.nn.BatchNorm2d(Cn, eps=EPS, momentum=MOMENTUM)
    with torch.no_grad():
        bn.weight.copy_(torch.tensor([GAMMAS[c % len(GAMMAS)] for c in range(Cn)]))
        bn.bias.copy_(torch.rand(Cn, generator=g) - 0.5)
        bn.running_mean.copy_(torch.randn(Cn, generator=g) * 0.1)
        bn.running_var.copy_(torch.rand(Cn, generator=g) * 1.5 + 0.5)
    ref = copy.deepcopy(bn).double().cuda().train()
    fast = torch.nn.Sequential(copy.deepcopy(bn)).cuda().train()
    assert fastnet.optimize_small_boards(fast) == 1
    fmt = torch.channels_last if cl else torch.contiguous_format
    n = N * H * W
    for step in range(2):
        x = _channel_data((N, Cn, H, W), g).cuda().contiguous(memory_format=fmt)
        dy = torch.randn((N, Cn, H, W), generator=g).cuda().contiguous(memory_format=fmt)
        rm0, rv0 = ref.running_mean.clone(), ref.running_var.clone()
        xf = x.clone().requires_grad_(True)
        yf = fast(xf)
        yf.backward(dy)
        assert yf.is_contiguous(memory_format=fmt) and xf.grad.is_contiguous(memory_format=fmt)
        xd = x.double().requires_grad_(True)
        yd = F.batch_norm(xd, ref.running_mean, ref.running_var, ref.weight, ref.bias, True, MOMENTUM, EPS)
        yd.backward(dy.double())
        with torch.no_grad():
            x64 = x.double()
            var, mu = torch.var_mean(x64, dim=(0, 2, 3), unbiased=False)
            sd = (var + EPS).sqrt()
            R = (mu.abs() / sd).view(1, Cn, 1, 1)
            gam = ref.weight.detach().abs().view(1, Cn, 1, 1)
            bet = ref.bias.detach().abs().view(1, Cn, 1, 1)
            xhat = ((x64 - mu.view(1, Cn, 1, 1)) / sd.view(1, Cn, 1, 1)).abs()
            # y: fp32 mean (u R), the subtraction and product (u |xhat|), rstd (VAR_RTOL |xhat|), the add of beta
            _check('y', yf.detach(), yd, gam * (4 * U * (1 + R + xhat) + VAR_RTOL * xhat) + 4 * U * bet)
            # dx = gamma rstd (dy - mean dy - xhat mean(dy xhat)): the same relative errors on the channel's scale gamma rstd |dy|
            dyd = dy.double()
            gmax = dyd.abs().amax(dim=(0, 2, 3)).view(1, Cn, 1, 1)
            _check('dx', xf.grad, xd.grad, gam / sd.view(1, Cn, 1, 1) * gmax * (8 * U * (1 + R + xhat) + 2 * VAR_RTOL * (1 + xhat)))
            # dbeta = sum dy, dgamma = sum dy xhat: fp32 slab sums folded in fp64
            sabs = dyd.abs().sum(dim=(0, 2, 3))
            sxabs = (dyd * xhat).abs().sum(dim=(0, 2, 3))
            _check('dbeta', fast[0].bias.grad, ref.bias.grad, 64 * U * sabs + 1e-30)
            _check('dgamma', fast[0].weight.grad, ref.weight.grad, 4 * U * (1 + R.view(Cn)) * sabs + (64 * U + VAR_RTOL) * sxabs + 1e-30)
            # running statistics (momentum 0.3, unbiased variance)
            _check('running_mean', fast[0].running_mean, ref.running_mean, 8 * U * (rm0.abs() + mu.abs()) + 1e-30)
            _check('running_var', fast[0].running_var, ref.running_var,
                   8 * U * rv0.abs() + MOMENTUM * VAR_RTOL * var * n / max(n - 1, 1) + 1e-30)
            assert int(fast[0].num_batches_tracked) == step + 1
            const = [c for c in range(Cn) if c % 6 == 3]
            if const:                # a constant channel: variance 0, x - mean exactly 0, so y = beta and dgamma = 0 exactly
                assert torch.equal(yf.detach()[:, const], fast[0].bias.detach()[const].view(1, -1, 1, 1).expand(N, -1, H, W))
                assert torch.equal(fast[0].weight.grad[const], torch.zeros(len(const), device='cuda'))
        fast[0].weight.grad = fast[0].bias.grad = None
        ref.weight.grad = ref.bias.grad = None


# ---------------------------------------------------------------------------------------------- (b) the tower's finalize kernels
def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


@pytest.mark.parametrize('tiles', [1, 129])
@pytest.mark.parametrize('HW', [1, 9, 16])
@pytest.mark.parametrize('pivot', [False, True], ids=['raw_sums', 'shifted_sums'])
def test_tower_bn_finalize_fwd(tiles, HW, pivot):
    """hrl_bn_finalize_fwd: column partials of known float64 data (per 128-row tile, as the STATS epilogue leaves them; summed
    less the pivot that mean_col holds on entry) -> per-column mean / rstd / scale / shift, running statistics,
    num_batches_tracked."""
    from handyrl_b200._capi import check, lib
    Cn = 6
    rows = 128 * tiles - (37 if tiles > 1 else 28)
    g = torch.Generator().manual_seed(tiles * 100 + HW)
    mu = torch.tensor([0.5, 300.0, -1000.0, 2.5, 40.0, -3.0], dtype=torch.float64)
    sd = torch.tensor([1.0, 1.0, 1.0, 0.0, 1e3, 1e-3], dtype=torch.float64)
    if not pivot:                 # unshifted sums keep the variance only while |mean| / std is small
        mu = torch.tensor([0.5, 1.0, -1.0, 2.5, 40.0, -1e-3], dtype=torch.float64)
    y = (mu.view(1, Cn, 1) + sd.view(1, Cn, 1) * torch.randn((rows, Cn, HW), generator=g, dtype=torch.float64)).float().double()
    K = (mu + 0.3 * sd).float().double() if pivot else torch.zeros(Cn, dtype=torch.float64)
    d = (y - K.view(1, Cn, 1)).reshape(rows, Cn * HW)
    parts = torch.zeros((tiles, 2, Cn * HW), dtype=torch.float64)
    for t in range(tiles):
        blk = d[t * 128:(t + 1) * 128]
        parts[t, 0], parts[t, 1] = blk.sum(0), (blk * blk).sum(0)
    cp = parts.float().cuda()
    gamma = torch.tensor([1.3, -0.7, 0.0, 2.0, 0.5, -1.0], device='cuda')
    beta = torch.tensor([0.1, -0.2, 0.3, 0.0, -0.5, 0.25], device='cuda')
    rm0 = torch.linspace(-0.2, 0.3, Cn, device='cuda')
    rv0 = torch.linspace(0.5, 2.0, Cn, device='cuda')
    rm, rv = rm0.clone(), rv0.clone()
    nbt = torch.tensor([5], dtype=torch.int64, device='cuda')
    mean_col = K.float().repeat_interleave(HW).cuda()            # the pivot, read before the batch mean overwrites it
    rstd_col, scale_col, shift_col = (torch.full((Cn * HW,), float('nan'), device='cuda') for _ in range(3))
    check(lib().hrl_bn_finalize_fwd(_p(cp), tiles, Cn, HW, rows, _p(gamma), _p(beta), EPS, MOMENTUM, _p(rm), _p(rv), _p(nbt),
                                    _p(mean_col), _p(rstd_col), _p(scale_col), _p(shift_col), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    # float64 reference from the fp32 partials the kernel reads (what it can know), and from the data itself
    n = rows * HW
    p64 = cp.double().cpu().view(tiles, 2, Cn, HW).sum(dim=(0, 3))
    dm = p64[0] / n
    m_ref, var_ref = K + dm, (p64[1] / n - dm * dm).clamp_min(0)
    var_data, mu_data = torch.var_mean(y, dim=(0, 2), unbiased=False)
    assert ((m_ref - mu_data).abs() <= 4 * U * (mu_data.abs() + sd)).all(), (m_ref, mu_data)
    rs_ref = 1 / (var_ref + EPS).sqrt()
    sc_ref = gamma.double().cpu() * rs_ref
    sh_ref = beta.double().cpu() - m_ref * sc_ref
    cols = lambda v: v.repeat_interleave(HW)
    got = lambda t: t.double().cpu()
    np.testing.assert_allclose(got(mean_col), cols(m_ref), rtol=U, atol=1e-30)
    np.testing.assert_allclose(got(rstd_col), cols(rs_ref), rtol=2 * U, atol=0)
    np.testing.assert_allclose(got(scale_col), cols(sc_ref), rtol=3 * U, atol=0)
    # shift = beta - mean * scale in fp32: |mean * scale| = R |gamma| carries the rounding
    np.testing.assert_allclose(got(shift_col), cols(sh_ref), rtol=0, atol=float(4 * U * (m_ref.abs() * sc_ref.abs() + beta.abs().cpu()).max()))
    # the variance from the data itself: fp32 tile sums less the pivot keep it to a small multiple of u
    np.testing.assert_allclose(var_ref.numpy(), var_data.numpy(), rtol=VAR_RTOL, atol=1e-12)
    np.testing.assert_allclose(got(rm), (1 - MOMENTUM) * rm0.double().cpu() + MOMENTUM * m_ref, rtol=4 * U, atol=4 * U)
    np.testing.assert_allclose(got(rv), (1 - MOMENTUM) * rv0.double().cpu() + MOMENTUM * var_ref * n / max(n - 1, 1), rtol=4 * U, atol=1e-30)
    assert int(nbt) == 6


@pytest.mark.parametrize('layers', [1, 8])
@pytest.mark.parametrize('with_jobs', [False, True], ids=['pivots_alone', 'with_pack_jobs'])
def test_tower_bn_pivot(layers, with_jobs):
    """hrl_board_pack_many_pivot's pivots: per column the running mean where |running mean| > 32 running std, exactly 0
    elsewhere (the sums then stay those of the unshifted statistics, bit for bit); alone and behind the blocks of pack jobs."""
    from handyrl_b200._capi import check, lib
    Cn, HW = 7, 9
    ratios = torch.tensor([0.0, 3.0, -31.5, 32.5, -40.0, 300.0, -1000.0], dtype=torch.float64)
    g = torch.Generator().manual_seed(layers)
    rms, rvs, cols = [], [], []
    for l in range(layers):
        sd = torch.rand(Cn, generator=g, dtype=torch.float64) * 10 + 0.01
        rms.append((ratios.roll(l) * sd).float().cuda())
        rvs.append((sd * sd).float().cuda())
        cols.append(torch.full((Cn * HW,), float('nan'), device='cuda'))
    arr = lambda ts: C.cast((C.c_void_p * len(ts))(*[t.data_ptr() for t in ts]), C.c_void_p)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    jobs, n_jobs, images = None, 0, []
    if with_jobs:                 # two convolutions packed in the same launch, against hrl_board_pack one at a time
        from handyrl_b200._capi import HrlPackJob
        n_jobs = 2
        jobs = (HrlPackJob * n_jobs)()
        for j in jobs:
            w = torch.randn((4, 3, 3, 3), generator=g).cuda()
            img = torch.zeros(lib().hrl_board_pack_floats(4 * 9, 3 * 9), device='cuda')
            j.w, (j.Cout, j.Cin, j.kh, j.kw), j.H, j.W = C.c_void_p(w.data_ptr()), w.shape, 3, 3
            j.image_fwd, j.fwd_rows = C.c_void_p(img.data_ptr()), 4 * 9
            images.append((w, img))
        jobs = C.byref(jobs)
    check(lib().hrl_board_pack_many_pivot(jobs, n_jobs, arr(rms), arr(rvs), arr(cols), layers, Cn, HW, stream))
    torch.cuda.synchronize()
    for w, img in images:
        want = torch.zeros_like(img)
        check(lib().hrl_board_pack(C.c_void_p(w.data_ptr()), 4, 3, 3, 3, 3, 3, C.c_void_p(want.data_ptr()), 4 * 9, 0, None, 0, 0, stream))
        torch.cuda.synchronize()
        assert torch.equal(img, want)
    for l in range(layers):
        big = ratios.roll(l).abs() > 32
        want = torch.where(big, rms[l].cpu(), torch.zeros(Cn)).repeat_interleave(HW)
        assert torch.equal(cols[l].cpu(), want), l


@pytest.mark.parametrize('tiles', [1, 129])
@pytest.mark.parametrize('HW', [1, 9, 16])
@pytest.mark.parametrize('stem', [False, True], ids=['batchnorm', 'stem_bias'])
def test_tower_bn_finalize_bwd(tiles, HW, stem):
    """hrl_bn_finalize_bwd: column sums of dZ and dZ * xhat -> dbeta, dgamma and the per-column constants of
    dY = dZ p + Y q + r, the BatchNorm backward gamma rstd (dZ - mean dZ - xhat mean(dZ xhat)) with xhat = (Y - mean) rstd.
    The stem form (gamma NULL) writes dbeta only."""
    from handyrl_b200._capi import check, lib
    Cn = 6
    rows = 128 * tiles - (37 if tiles > 1 else 28)
    n = rows * HW
    g = torch.Generator().manual_seed(tiles * 1000 + HW)
    cp = (torch.randn((tiles, 2, Cn * HW), generator=g) * torch.tensor([1.0, 1e3, 1e-3, 10.0, 1.0, 5.0]).repeat_interleave(HW)).cuda()
    gamma = torch.tensor([1.3, -0.7, 0.0, 2.0, 0.5, -1.0], device='cuda')
    mu = torch.tensor([0.5, 300.0, -1000.0, 2.5, 40.0, -3.0], device='cuda')
    rstd = torch.tensor([1.0, 0.5, 2.0, 31.6, 1e-3, 3.0], device='cuda')
    mean_col, rstd_col = mu.repeat_interleave(HW), rstd.repeat_interleave(HW)
    dgamma, dbeta = torch.full((Cn,), float('nan'), device='cuda'), torch.full((Cn,), float('nan'), device='cuda')
    pqr = [torch.full((Cn * HW,), 7.0, device='cuda') for _ in range(3)]
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    if stem:
        check(lib().hrl_bn_finalize_bwd(_p(cp), tiles, Cn, HW, rows, None, None, None, None, _p(dbeta), *map(_p, pqr), 0, stream))
    else:
        check(lib().hrl_bn_finalize_bwd(_p(cp), tiles, Cn, HW, rows, _p(gamma), _p(mean_col), _p(rstd_col), _p(dgamma), _p(dbeta),
                                        *map(_p, pqr), 0, stream))
    torch.cuda.synchronize()
    p64 = cp.double().cpu().view(tiles, 2, Cn, HW)
    s, q = p64[:, 0].sum(dim=(0, 2)), p64[:, 1].sum(dim=(0, 2))
    sabs = p64[:, 0].abs().sum(dim=(0, 2))
    qabs = p64[:, 1].abs().sum(dim=(0, 2))
    np.testing.assert_array_less((dbeta.double().cpu() - s).abs().numpy(), (2 * U * sabs + 1e-30).numpy())
    if stem:
        assert torch.isnan(dgamma).all()
        assert all(torch.equal(t, torch.full_like(t, 7.0)) for t in pqr)          # no BatchNorm: the constants stay untouched
        return
    np.testing.assert_array_less((dgamma.double().cpu() - q).abs().numpy(), (2 * U * qabs + 1e-30).numpy())
    G, M, RS = gamma.double().cpu(), mu.double().cpu(), rstd.double().cpu()
    p_ref = G * RS
    mdz, mdzx = s / n, q / n
    q_ref = -p_ref * RS * mdzx
    r_ref = p_ref * (RS * M * mdzx - mdz)
    cols = lambda v: v.repeat_interleave(HW).numpy()
    got = lambda t: t.double().cpu().numpy()
    np.testing.assert_allclose(got(pqr[0]), cols(p_ref), rtol=2 * U, atol=0)
    np.testing.assert_allclose(got(pqr[1]), cols(q_ref), rtol=8 * U, atol=1e-30)
    # r = p (rstd mean mean(dZ xhat) - mean dZ): fp32, so the error scales with the larger of the two terms
    tol_r = 8 * U * p_ref.abs() * ((RS * M * mdzx).abs() + mdz.abs())
    np.testing.assert_array_less(np.abs(got(pqr[2]) - cols(r_ref)), cols(tol_r) + 1e-30)


# ------------------------------------------------------------------------------------- (c) the tower engine, large-mean channels
@pytest.mark.parametrize('M', [100, 1025], ids=['one_tile', 'ragged_tiles'])
def test_fused_tower_large_mean_channels(M):
    """A BoardNet whose stem bias is large on every third channel, read by the first tower convolution through its centre tap
    only (so the offset is the same in every cell): that layer's pre-BatchNorm channels have |mean| / std of about 320
    (computed here in float64 and required to be >= 300).  The net is restored with running statistics near
    the batch statistics, as a trained net has them; the engine takes its statistics pivot from the running mean where
    |running mean| > 32 running std (written by hrl_board_pack_many_pivot).  Two
    steps against the float64 module: outputs, parameter gradients, running buffers."""
    from handyrl_b200 import nets, tower
    torch.manual_seed(11)
    ref = nets.BoardNet(planes=3, board=(3, 3), width=32, depth=3, actions=9).double().cuda().train()
    with torch.no_grad():
        ref.stem.bias[::3] = 300.0
        w0 = ref.tower[0][0].weight
        w0[:, ::3] = 0.0
        w0[:, ::3, 1, 1] = 0.05
        for blk in ref.tower:
            blk[1].weight.uniform_(0.5, 1.5)
            blk[1].bias.normal_(0, 0.3)
    g = torch.Generator().manual_seed(M)
    xs = [(torch.rand((M, 3, 3, 3), generator=g) < 0.4).float().cuda() for _ in range(2)]
    pre = {}
    ref.tower[0][0].register_forward_hook(lambda mod, inp, out: pre.__setitem__('y', out.detach()))

    def first_layer_stats():        # the first step's batch statistics of that layer, float64
        with torch.no_grad():
            copy.deepcopy(ref)(xs[0].double())
        var, mu = torch.var_mean(pre['y'], dim=(0, 2, 3), unbiased=False)
        return var, mu, (mu.abs() / (var + ref.tower[0][1].eps).sqrt()).max().item()

    with torch.no_grad():           # the mean is proportional to the bias, the spread does not depend on it: aim at R = 320
        ref.stem.bias[::3] *= 320.0 / first_layer_stats()[2]
    var0, mu0, ratio = first_layer_stats()
    assert ratio >= 300, ratio
    ref.tower[0][0]._forward_hooks.clear()
    with torch.no_grad():
        bn0 = ref.tower[0][1]
        bn0.running_mean.copy_(mu0 + 0.5 * var0.sqrt())
        bn0.running_var.copy_(var0 * 1.1 + 1e-3)
        for blk in ref.tower[1:]:
            blk[1].running_mean.normal_(0, 0.1)
            blk[1].running_var.uniform_(0.5, 2.0)
    fast = copy.deepcopy(ref).float()
    assert tower.supports(fast)
    eng = tower.FusedBoardNet(fast, M, torch.device('cuda'))
    for step, x in enumerate(xs):
        for p in list(fast.parameters()) + list(ref.parameters()):
            p.grad = torch.full_like(p, 7.0) if p.dtype == torch.float32 else None
        out = eng.forward(x)
        want = ref(x.double())
        # outputs: 3e-5 (3xTF32 products, as test_tower_gpu) plus the apply-form rounding the tower's operand transform keeps:
        # y * scale + shift cancels terms of size R |gamma| -- u R |gamma| per activation of the first layer
        gmax = max(float(b[1].weight.abs().max()) for b in ref.tower)
        atol = 3e-5 + 16 * U * ratio * gmax
        for k in want:
            np.testing.assert_allclose(out[k].double().cpu().numpy(), want[k].detach().cpu().numpy(), rtol=0, atol=atol,
                                       err_msg='step %d %s' % (step, k))
        gr = torch.Generator().manual_seed(5 + step)
        dout = {k: torch.randn(v.shape, generator=gr).cuda() for k, v in out.items()}
        sum((want[k] * dout[k].double()).sum() for k in want).backward()
        eng.backward(dout['policy'], dout['value'], dout.get('return'))
        torch.cuda.synchronize()
        # parameter gradients: 5e-2 as test_tower_gpu, plus the first layer's 3xTF32 product error, about 1e-5 of its output
        # |Y| ~ R std (the shrink of the truncating accumulator is not uniform over elements): ~1e-5 R in xhat downstream
        for (k, pr), (_, pf) in zip(ref.named_parameters(), fast.named_parameters()):
            scale = pr.grad.abs().max().item() + 1e-6
            assert (pf.grad.double() - pr.grad).abs().max().item() <= (5e-2 + 1e-4 * ratio) * scale, ('step', step, k, 'fused vs float64')
        # running buffers: rtol 1e-5 as test_tower_gpu.  The large-mean layer's own statistics are held to it exactly (unshifted
        # fp32 tile sums miss its variance by ~3e-3); the layers after it see the product error above in their inputs
        for (k, br), (_, bf) in zip(ref.named_buffers(), fast.named_buffers()):
            if br.dtype.is_floating_point:
                atol = 1e-6 if k.startswith('tower.0.') else 1e-6 + 1e-8 * ratio
                np.testing.assert_allclose(bf.double().cpu().numpy(), br.cpu().numpy(), rtol=1e-5, atol=atol, err_msg='step %d %s' % (step, k))
            else:
                assert int(bf) == int(br) == step + 1, k
