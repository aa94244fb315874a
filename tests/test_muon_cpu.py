"""The Muon optimiser without a GPU: the train_args key, the split of hrl_muon_plan on the shipped nets' parameter shapes,
the float64 restatement (tests/muon_ref.py) against closed forms, the optimiser file format, and the kernel's compile."""
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from muon_ref import matrix_view, muon_step, ns_polynomial, orthogonalise

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')

BAD = ['Muon', 'MUON', 'sgd', '', 0, ['muon'], {'name': 'Muon'}, {'lr_scale': 2.0}, {'name': 'muon', 'mu': 0.9},
       {'name': 'muon', 'ns_steps': 3}, {'name': 'muon', 'lr_scale': 0.0}, {'name': 'muon', 'lr_scale': -1.0},
       {'name': 'muon', 'lr_scale': float('nan')}, {'name': 'muon', 'lr_scale': float('inf')},
       {'name': 'muon', 'lr_scale': True}, {'name': 'muon', 'lr_scale': '2'}, {'name': 'muon', 'lr_scale': None}]


# ---------------------------------------------------------------- the key


def test_both_muon_forms_are_accepted():
    from handyrl_b200.train import optimizer_config
    assert optimizer_config('muon') == {'name': 'muon', 'lr_scale': 1.0}
    assert optimizer_config({'name': 'muon'}) == {'name': 'muon', 'lr_scale': 1.0}
    assert optimizer_config({'name': 'muon', 'lr_scale': 3}) == {'name': 'muon', 'lr_scale': 3.0}
    assert optimizer_config({'name': 'muon', 'lr_scale': 0.25}) == {'name': 'muon', 'lr_scale': 0.25}


@pytest.mark.parametrize('value', BAD, ids=[repr(v) for v in BAD])
def test_bad_values_raise_at_build(value):
    from handyrl_b200.train import LearnerStep, Trainer, optimizer_config
    with pytest.raises(ValueError):
        optimizer_config(value)
    with pytest.raises(ValueError):
        LearnerStep(None, {'optimizer': value}, None, lr=1e-3)
    with pytest.raises(ValueError):
        Trainer({'optimizer': value}, None)


def test_helper_ranks_get_the_key(monkeypatch):
    """multigpu.Fleet hands each helper rank the train_args its LearnerStep parses the key from (no process is started)."""
    import torch.multiprocessing as mp
    from handyrl_b200 import multigpu

    class Conn:
        def send(self, msg):
            pass

    started = []

    class Context:
        def Pipe(self):
            return Conn(), Conn()

        def Process(self, target, args, daemon):
            started.append((target, args))
            return type('P', (), {'start': lambda self: None})()

    monkeypatch.setattr(mp, 'get_context', lambda method: Context())
    monkeypatch.setattr(multigpu, '_init_group', lambda rank, world, port: None)
    monkeypatch.setattr(multigpu, 'pin_to_gpu_numa', lambda device: None)
    args = {'optimizer': {'name': 'muon', 'lr_scale': 0.5}, 'maximum_episodes': 10}
    multigpu.Fleet(3, args, torch.nn.Linear(2, 2), [], 1e-3)
    assert [t for t, _ in started] == [multigpu._helper_main] * 2
    assert all(a[3]['optimizer'] == {'name': 'muon', 'lr_scale': 0.5} for _, a in started)


# ---------------------------------------------------------------- the split

# the matrices (r, k) of each shipped net that Muon owns, in parameter order
TABLE = {
    'tictactoe': [(32, 27), (32, 288), (32, 288), (32, 288), (2, 32), (9, 18)],
    'geister': [(32, 225), (128, 576), (128, 576), (128, 576), (8, 288), (4, 8), (2, 32), (2, 32)],
    'geese': [(32, 153)] + [(32, 288)] * 12 + [(4, 32)],
    'wide': [(32, 9), (32, 288), (64, 288), (64, 576)],
}


def _net(name):
    from handyrl_b200 import nets
    torch.manual_seed(0)
    return {'tictactoe': nets.tictactoe_net, 'geister': nets.geister_net, 'geese': nets.geese_net,
            'wide': nets.WideActionNet}[name]()


@pytest.mark.parametrize('name', sorted(TABLE))
def test_split_of_the_shipped_nets(name):
    from handyrl_b200.ops import muon_plan
    net = _net(name)
    shapes = [tuple(p.shape) for p in net.parameters()]
    kinds, mats, spans = muon_plan(shapes)
    got = [matrix_view(s) for s, k in zip(shapes, kinds) if k == 'matrix']
    assert got == TABLE[name]
    too_large = [(n, tuple(p.shape)) for (n, p), k in zip(net.named_parameters(), kinds) if k == 'too_large']
    assert too_large == ([('p_out.weight', (512, 1024))] if name == 'wide' else [])
    for s, k in zip(shapes, kinds):                    # everything else is Adam-owned: no matrix with a side >= 2 left
        if k == 'adam':
            assert len(s) < 2 or min(matrix_view(s)) < 2, s
    # the table: every bucket word owned exactly once, padding never
    numels = [int(np.prod(s)) for s in shapes]
    offsets = np.cumsum([0] + numels)
    n = int(offsets[-1])
    seen = np.zeros(n + 3, np.int64)
    matrix_idx = [i for i, k in enumerate(kinds) if k == 'matrix']
    assert mats.shape == (len(matrix_idx), 4)
    for (off, r, k, tr), i in zip(mats.tolist(), matrix_idx):
        assert off == offsets[i] and (r, k) == matrix_view(shapes[i]) and tr == (1 if r > k else 0)
        seen[off:off + r * k] += 1
    for start, words in spans.tolist():
        assert 0 < words <= 4096
        seen[start:start + words] += 1
    assert (seen[:n] == 1).all() and (seen[n:] == 0).all()
    for i, k in enumerate(kinds):
        if k != 'matrix':
            assert (seen[offsets[i]:offsets[i + 1]] == 1).all()
    assert list(spans[:, 0]) == sorted(spans[:, 0].tolist())


def test_envelope_edges():
    """m_p <= 128 and m_p * n_p <= 128 * 576 (sides rounded up to 16); the smaller side must be >= 2."""
    from handyrl_b200.ops import muon_plan
    cases = {(2, 2): 'matrix', (128, 576): 'matrix', (576, 128): 'matrix', (16, 4608): 'matrix', (16, 4609): 'too_large',
             (128, 577): 'too_large', (129, 129): 'too_large', (1, 64): 'adam', (64, 1): 'adam', (70, 1): 'adam',
             (64,): 'adam', (): 'adam', (32, 1, 3, 3): 'matrix', (1, 32, 3, 3): 'adam', (2, 1, 1, 1): 'adam'}
    kinds, mats, spans = muon_plan(list(cases))
    assert dict(zip(cases, kinds)) == cases


def test_plan_refuses_bad_shapes():
    from handyrl_b200 import _capi
    from handyrl_b200.ops import muon_plan
    with pytest.raises(_capi.HrlError):
        muon_plan([])
    with pytest.raises(_capi.HrlError):
        muon_plan([(3, 0)])


# ---------------------------------------------------------------- the restatement against closed forms


@pytest.mark.parametrize('shape', [(2, 2), (9, 18), (32, 288), (18, 9), (128, 40)])
def test_iterations_act_on_the_singular_values(shape):
    """N = U diag(s) V^T -> U diag(p^5(s / |s|)) V^T: the normalisation divides by |N|_F = |s|, and each iteration maps
    every singular value through p(x) = a x + b x^3 + c x^5 and keeps the singular vectors."""
    g = np.random.default_rng(sum(shape))
    n = g.standard_normal(shape) * np.linspace(0.05, 3.0, shape[1])
    u, s, vt = np.linalg.svd(n, full_matrices=False)
    want = u @ np.diag(ns_polynomial(s / (np.sqrt((s * s).sum()) + 1e-7))) @ vt
    np.testing.assert_allclose(orthogonalise(n), want, rtol=0, atol=1e-12)


def test_polynomial_reaches_the_band_muon_is_known_for():
    """Five iterations take a normalised singular value anywhere in [0.01, 1] into roughly [0.7, 1.2] (not to 1: the
    quintic trades exactness for speed)."""
    p = ns_polynomial(np.linspace(0.01, 1.0, 1000))
    assert p.min() > 0.65 and p.max() < 1.25


@pytest.mark.parametrize('bf16', [False, True])
@pytest.mark.parametrize('shape', [(40, 9), (576, 128), (3, 2)])
def test_tall_matrix_is_the_transpose_of_the_wide_one(shape, bf16):
    n = np.random.default_rng(3).standard_normal(shape)
    np.testing.assert_array_equal(orthogonalise(n, bf16=bf16), orthogonalise(n.T, bf16=bf16).T)


def test_bf16_mode_rounds_every_stored_matrix():
    from muon_ref import round_bf16
    o = orthogonalise(np.random.default_rng(4).standard_normal((8, 24)), bf16=True)
    assert np.array_equal(round_bf16(o), o)
    assert np.abs(o - orthogonalise(np.random.default_rng(4).standard_normal((8, 24)))).max() < 2 ** -4


def test_step_combines_momentum_muon_and_adam():
    """A matrix and a bias with zero momentum at t = 1: M = G, N = (1 + mu) G, so O is the orthogonalisation of G; the bias
    takes Adam's step; the clip scales G but not O (O does not depend on the scale of N)."""
    g = np.random.default_rng(5)
    w, b = g.standard_normal((4, 6)), g.standard_normal(4)
    gw, gb = 10 * g.standard_normal((4, 6)), g.standard_normal(4)
    lr, wd = 1e-2, 1e-5
    out_w, out_m, out_v, out_o, norm = muon_step([w, b], [gw, gb], [np.zeros_like(w), np.zeros_like(b)],
                                                 [np.zeros_like(w), np.zeros_like(b)], ['matrix', 'adam'], 1, lr, lr_scale=2.0)
    c = min(1.0, 4.0 / (norm + 1e-6))
    assert c < 1.0
    np.testing.assert_allclose(out_m[0], c * gw, rtol=1e-15)
    assert (out_v[0] == 0).all()
    o = orthogonalise(1.95 * c * gw)
    np.testing.assert_allclose(out_o[0], o, rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(out_w[0], w - lr * (2.0 * 0.2 * np.sqrt(6) * o + wd * w), rtol=1e-13)
    gb2 = c * gb + wd * b
    np.testing.assert_allclose(out_w[1], b - lr * gb2 / (np.abs(gb2) + 1e-8), rtol=1e-9)
    assert out_o[1] is None


# ---------------------------------------------------------------- the file format


def _format(optimizer=None, name='geister'):
    from handyrl_b200.train import OptimizerStateFormat
    kw = {} if optimizer is None else {'optimizer': optimizer}
    return OptimizerStateFormat(_net(name).named_parameters(), **kw)


def _dict(fmt):
    m = torch.arange(fmt.n_pad, dtype=torch.float32)
    return fmt.to_dict(m, m + 1, 7, 1e-3, 512.0, 7)


def test_muon_dict_carries_its_entries():
    from handyrl_b200.train import optimizer_config
    adam = _dict(_format())
    muon = _dict(_format(optimizer_config({'name': 'muon', 'lr_scale': 2.0})))
    assert sorted(muon) == sorted(list(adam) + ['algorithm', 'lr_scale', 'muon_params'])
    assert muon['algorithm'] == 'muon' and muon['lr_scale'] == 2.0
    assert muon['muon_params'] == ['stem.weight', 'cells.0.conv.weight', 'cells.1.conv.weight', 'cells.2.conv.weight',
                                   'move_head.reduce.weight', 'move_head.project.weight', 'value_head.reduce.weight',
                                   'return_head.reduce.weight']
    assert sorted(_dict(_format(optimizer_config('adam')))) == sorted(adam)
    assert sorted(_dict(_format(optimizer_config('lamb')))) == sorted(list(adam) + ['algorithm', 'lr_scale'])


def test_cross_loading_raises_in_every_direction():
    from handyrl_b200.train import optimizer_config
    fmts = {k: _format(optimizer_config(k)) for k in ('adam', 'lamb', 'muon')}
    dicts = {k: _dict(f) for k, f in fmts.items()}
    for have, fmt in fmts.items():
        for got, d in dicts.items():
            if have == got:
                fmt.unpack(d)
            else:
                with pytest.raises(ValueError):
                    fmt.unpack(d)
    muon = _dict(_format(optimizer_config({'name': 'muon', 'lr_scale': 5.0})))
    m, v, step, lr, ema, steps = fmts['muon'].unpack(muon)               # lr_scale is not compared
    assert step == 7
    for bad in (muon['muon_params'][:-1], muon['muon_params'] + ['set_head.weight'], list(reversed(muon['muon_params']))):
        with pytest.raises(ValueError, match='Muon owns'):
            fmts['muon'].unpack(dict(muon, muon_params=bad))
    with pytest.raises(ValueError):
        fmts['muon'].unpack({k: v for k, v in muon.items() if k != 'muon_params'})


# ---------------------------------------------------------------- the kernel's compile


@pytest.fixture(scope='module')
def compiled():
    """(ptxas -v report per instantiation, SASS) of csrc/muon_kernel.cu built for sm_90a."""
    if not (os.path.exists(NVCC) or shutil.which(NVCC)):
        pytest.skip('nvcc is not available')
    with tempfile.TemporaryDirectory() as d:
        cubin = os.path.join(d, 'muon_kernel.cubin')
        res = subprocess.run([NVCC, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-cubin', '-Xptxas', '-v',
                              '-o', cubin, os.path.join(ROOT, 'handyrl_b200', 'csrc', 'muon_kernel.cu')],
                             capture_output=True, text=True)
        assert res.returncode == 0, res.stdout + res.stderr
        cuobjdump = os.path.join(os.path.dirname(shutil.which(NVCC) or NVCC), 'cuobjdump')
        sass = subprocess.run([cuobjdump, '-sass', cubin], capture_output=True, text=True)
        assert sass.returncode == 0, sass.stderr
    out, cur = {}, None
    for line in res.stderr.splitlines():
        if 'Compiling entry function' in line:
            m = re.search(r'clip_muon_kernelILb(\d)ELb(\d)EE', line)
            cur = (int(m.group(1)), int(m.group(2))) if m else None
            continue
        s = re.search(r'(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads', line)
        if s and cur is not None:
            out[cur] = dict(stack=int(s.group(1)), spill_stores=int(s.group(2)), spill_loads=int(s.group(3)))
    return out, sass.stdout


def test_kernel_builds_without_spills(compiled):
    report, _ = compiled
    assert sorted(report) == [(0, 0), (0, 1), (1, 0), (1, 1)]
    for key, r in report.items():
        assert r['spill_stores'] == 0 and r['spill_loads'] == 0 and r['stack'] == 0, (key, r)


def test_kernel_runs_its_products_on_the_tensor_cores(compiled):
    _, sass = compiled
    assert re.search(r'\bHMMA\.16816\.F32\.BF16\b', sass) or re.search(r'\bHGMMA\b', sass)
