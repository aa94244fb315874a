"""How the tensor-core products are launched, without a GPU: ops.k_splits against the split rule written out, and the
HrlGemmArgs that ops.gemm_fused hands to hrl_gemm_fused (stubbed) for each form of product, with the launches it counts."""
import ctypes

import pytest
import torch


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as g
    g.build()
    from handyrl_b200._capi import lib
    return lib()


def _rule(rows, cols, K, segments):
    """128 x 288 output tiles, one CTA per tile, slice and segment on 132 SMs, at least 64 of K per slice; then only as many
    slices as whole 32-element chunks of K give without an empty one"""
    tiles = ((rows + 127) // 128) * ((cols + 287) // 288)
    want = max(1, min(K // 64, 132 // (tiles * segments)))
    chunks = (K + 31) // 32
    per = -(-chunks // min(want, chunks))
    return -(-chunks // per)


SHAPES = ([(288, cols, M) for cols in (27, 288) for M in (100, 300, 515, 2048, 16384, 32768)]          # TicTacToe stem and tower
          + [(27, 288, M) for M in (100, 2048, 32768)]                                                   # its squeeze heads
          + [(rows, cols, n * 36) for rows, cols in ((128, 576), (128, 577), (8, 288), (8, 289))         # Geister cells, move head
             for n in (1, 2, 7, 256, 512)]
          + [(rows, cols, K) for rows in (4, 129, 300) for cols in (12, 289, 2593) for K in (1, 5, 31, 32, 33, 63, 64, 65, 4097)])


@pytest.mark.parametrize('segments', [1, 2, 3, 9, 20, 64])
def test_k_splits_follows_the_written_out_rule(lib, segments):
    from handyrl_b200 import ops
    for rows, cols, K in SHAPES:
        assert ops.k_splits(rows, cols, K, segments) == _rule(rows, cols, K, segments), (rows, cols, K, segments)
        if K <= 32:
            assert ops.k_splits(rows, cols, K, segments) == 1


def _fields(s):
    return {name: (_fields(getattr(s, name)) if isinstance(getattr(s, name), ctypes.Structure) else getattr(s, name))
            for name, _ in s._fields_}


@pytest.fixture
def launches(lib, monkeypatch):
    """every hrl_gemm_fused call's arguments (with the segment pointers read while the call lasts), nothing launched"""
    from handyrl_b200 import ops
    got = []

    def stub(ref, stream):
        g = ref._obj
        f = _fields(g)
        seg = ctypes.POINTER(ctypes.c_void_p)
        f['seg_a'] = [ctypes.cast(g.seg_a, seg)[i] for i in range(g.segments)]
        f['seg_b'] = [ctypes.cast(g.seg_b, seg)[i] for i in range(g.segments)]
        got.append(f)
        return 0
    monkeypatch.setattr(lib, 'hrl_gemm_fused', stub)
    monkeypatch.setattr(ops, '_stream_ptr', lambda: None)
    return got


def _expect(**kw):
    """an all-zero HrlGemmArgs as _fields reads it, with the given fields set"""
    from handyrl_b200._capi import HrlGemmArgs
    f = _fields(HrlGemmArgs())
    f['seg_a'] = f['seg_b'] = []
    for k, v in kw.items():
        if isinstance(v, dict):
            f[k].update(v)
        else:
            f[k] = v
    return f


def _count(fn):
    from handyrl_b200 import ops
    before = ops.LAUNCHES['n']
    fn()
    return ops.LAUNCHES['n'] - before


def test_dense_product_with_and_without_split(launches):
    from handyrl_b200 import ops
    M, N, K = 200, 96, 4096
    a, b, out, bias = torch.zeros(K, M), torch.zeros(N, K), torch.zeros(M, N + 4)[:, :N], torch.zeros(N)
    ws = torch.zeros(8 * M * N)
    A, B = dict(ptr=a.data_ptr(), ld=M, kmajor=0), dict(ptr=b.data_ptr(), ld=K, kmajor=1)
    dense = dict(a=A, b=B, M=M, N=N, K=K)
    # one slice: the product into `out` (with bias), or into the workspace when there is no output
    assert _count(lambda: ops.gemm_fused(dict(t=a, kmajor=False), dict(t=b), M, N, K, out=out, ws=ws, bias=bias)) == 1
    assert launches[-1] == _expect(**dense, C=out.data_ptr(), ldc=N + 4, splits=1, bias=bias.data_ptr())
    assert _count(lambda: ops.gemm_fused(dict(t=a, kmajor=False), dict(t=b), M, N, K, ws=ws, bf16=True)) == 1
    assert launches[-1] == _expect(**dense, C=ws.data_ptr(), ldc=N, splits=1, bf16=1)
    # split: the partials and their sum into `out`, two launches; or the partials left in the workspace, one
    assert _count(lambda: ops.gemm_fused(dict(t=a, kmajor=False), dict(t=b), M, N, K, out=out, ws=ws, splits=8)) == 2
    assert launches[-1] == _expect(**dense, C=out.data_ptr(), ldc=N + 4, splits=8, workspace=ws.data_ptr())
    assert _count(lambda: ops.gemm_fused(dict(t=a, kmajor=False), dict(t=b), M, N, K, ws=ws, splits=8)) == 1
    assert launches[-1] == _expect(**dense, C=None, ldc=N, splits=8, workspace=ws.data_ptr())
    # a split asked of a K of one 32-element chunk runs as one slice: no sum
    assert _count(lambda: ops.gemm_fused(dict(t=a, kmajor=False), dict(t=b), M, N, 32, out=out, ws=ws, splits=8)) == 1
    assert launches[-1]['splits'] == 8 and launches[-1]['workspace'] == ws.data_ptr()


@pytest.mark.parametrize('bf16', [False, True])
def test_tower_products(launches, bf16):
    """FusedBoardNet's forward product on a packed weight image with the statistics epilogue, and its weight gradients split
    over K slices (M = 300) or not (M = 100), left in their workspace regions for the fold"""
    from handyrl_b200 import nets, tower
    for M in (300, 100):
        eng = tower.FusedBoardNet(nets.tictactoe_net(), M, torch.device('cpu'), bf16=bf16)
        D, st = eng.D, eng.bn[0]
        assert eng.splits == {'stem': 1 if M == 100 else 4, 'tower': 1 if M == 100 else 4, 'heads': 1 if M == 100 else 4}
        src = dict(t=eng.A0, consts=(st['scale'], st['shift']), relu=True)
        assert _count(lambda: eng._gemm(src, dict(t=eng.Wf[0], packed=True), eng.Y[0], K=D, N=D, epilogue='stats',
                                        ep=dict(mean=st['mean']))) == 1
        assert launches[-1] == _expect(
            a=dict(ptr=eng.A0.data_ptr(), p=st['scale'].data_ptr(), r=st['shift'].data_ptr(), ld=D, kmajor=1, relu=1),
            b=dict(ptr=eng.Wf[0].data_ptr(), ld=0, kmajor=1, packed=1), C=eng.Y[0].data_ptr(), ldc=D, M=M, N=D, K=D, splits=1,
            epilogue=2, ep_mean=st['mean'].data_ptr(), col_partials=eng.cp.data_ptr(), bf16=int(bf16))
        grad = torch.zeros(32, 32, 3, 3)
        dy = dict(t=eng.dZ[1], t2=eng.Y[1], consts=(st['p'], st['q'], st['r']), kmajor=False, by_row=True)
        assert _count(lambda: eng._wgrad(dy, dict(t=eng.A0, kmajor=False, by_row=True), D, D, ('tower', 1), [(grad, 0)])) == 1
        s, ws = eng.splits['tower'], eng.ws.data_ptr() + 4 * eng.ws_at[('tower', 1)]
        assert launches[-1] == _expect(
            a=dict(ptr=eng.dZ[1].data_ptr(), ptr2=eng.Y[1].data_ptr(), p=st['p'].data_ptr(), q=st['q'].data_ptr(),
                   r=st['r'].data_ptr(), ld=D, feature_is_row=1),
            b=dict(ptr=eng.A0.data_ptr(), ld=D, feature_is_row=1), M=D, N=D, K=M, splits=s, ldc=D, bf16=int(bf16),
            **(dict(C=None, workspace=ws) if s > 1 else dict(C=ws)))
        src_, s_, stride, g_ = eng.fold_jobs[-1]
        assert (src_.data_ptr(), s_, stride) == (ws, s, D * D if s > 1 else 0) and g_ is grad


def test_implicit_convolution_forward(launches):
    """conv_mode 1: pixels (channels-last rows) times a packed image over taps x channels padded to 32"""
    from handyrl_b200 import ops
    pix, image, table, bias = torch.zeros(2 * 36, 40), torch.zeros(4096), torch.zeros(36 * 9, dtype=torch.int16), torch.zeros(24)
    out = []
    assert _count(lambda: out.append(ops._conv_product(pix, image, 24, 40, 9, table, 36, bias=bias))) == 1
    assert out[0].shape == (72, 24)
    assert launches[-1] == _expect(a=dict(ptr=pix.data_ptr(), ld=40, kmajor=1), b=dict(ptr=image.data_ptr(), kmajor=1, packed=1),
                                   bias=bias.data_ptr(), C=out[0].data_ptr(), ldc=24, M=72, N=24, K=9 * 64, splits=1,
                                   conv_off=table.data_ptr(), conv_mode=1, conv_hw=36, conv_taps=9, conv_cin=40)


def test_segmented_weight_gradient_with_the_ones_row(launches, lib, monkeypatch):
    """conv_mode 2 over three (dy, x) pairs of one weight, with the bias gradient as a ones-row column: one segmented product
    and one reduction into .grad"""
    from handyrl_b200 import ops
    reduced = []
    monkeypatch.setattr(lib, 'hrl_conv_wgrad_reduce2', lambda *a: (reduced.append(a), 0)[1])
    Cout, Cin, pixels = 16, 8, 4 * 36
    w, b = torch.nn.Parameter(torch.zeros(Cout, Cin, 3, 3)), torch.nn.Parameter(torch.zeros(Cout))
    pairs = [(torch.zeros(pixels, Cout), torch.zeros(pixels, Cin)) for _ in range(3)]
    table = torch.zeros(36 * 9, dtype=torch.int16)
    job = {'w': w, 'b': b, 'pairs': pairs, 'geom': (table, 36), 'bf16': False}
    assert _count(lambda: ops._flush_weight_gradient(job)) == 2
    per = ops.k_splits(Cout, 9 * Cin + 1, pixels, 3)
    assert per > 1
    f = launches[-1]
    ws = f['workspace']
    assert f == _expect(a=dict(ptr=pairs[0][0].data_ptr(), ld=Cout), b=dict(ptr=pairs[0][1].data_ptr(), ld=Cin), C=None,
                        ldc=9 * Cin + 1, M=Cout, N=9 * Cin + 1, K=pixels, splits=per, workspace=ws, conv_off=table.data_ptr(),
                        conv_mode=2, conv_hw=36, conv_taps=9, conv_cin=Cin, segments=3, conv_ones_row=1,
                        seg_a=[dy.data_ptr() for dy, _ in pairs], seg_b=[x.data_ptr() for _, x in pairs])
    assert ws is not None and len(reduced) == 1
    assert [reduced[0][i] for i in (1, 2, 5, 6, 7, 8)] == [3 * per, 9 * Cin + 1, Cout, Cin, 9, 1]
    assert reduced[0][0].value == ws and reduced[0][3].value == w.grad.data_ptr() and reduced[0][4].value == b.grad.data_ptr()
