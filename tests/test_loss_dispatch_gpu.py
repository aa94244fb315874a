"""GPU parity of every kernel the dispatcher of hrl_loss_fwd_bwd (csrc/loss_kernel.cu) can launch, against the float64 C oracle.

The fused loss is not one kernel: the dispatcher picks a group, element, rows or bulk kernel (and a template instantiation of it)
from A, T - burn_in, Pa, B, pointer alignment and shared-memory size, and each of them runs the serial or the suffix-scan
recurrence.  The cases below are chosen so that every instantiation serves at least one shape under both recurrences, packed
grids end with a partial CTA, cluster splits of the time axis are ragged, and inputs reach the clamps and underflows of the
softmax.  Each launch is traced with torch.profiler (CUPTI activity records), so a case fails if the dispatcher routes its shape
to another kernel than the one it declares, and the last test checks that the traced set equals KERNELS x RECURRENCES.
"""
import re
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ATOL = 1e-5            # per element, as test_loss_gpu.py
RTOL = 1e-5            # loss sums
ORACLE_ERR_FACTOR = 8  # extreme inputs: kernel error <= 8 x the float32 oracle's own error + ATOL

# every kernel the dispatcher can launch: template arguments without the trailing <DIAG, GRAD> of the form
KERNELS = frozenset(
    ['group<%d>' % rl for rl in (1, 2, 4, 8, 16, 32)] + ['elem', 'bulk'] +
    ['rows<%d,%d,false,%s>' % (lpr, npl, ios)
     for lpr, npl in ((1, 1), (1, 2), (1, 4), (1, 8), (1, 16), (2, 16), (4, 16), (8, 16), (16, 16), (32, 16), (32, 32))
     for ios in ('false', 'true')] +
    ['rows<32,16,true,false>', 'rows<32,32,true,false>'])
RECURRENCES = ('serial', 'scan')
COVERAGE = frozenset((k, r) for k in KERNELS for r in RECURRENCES)

LAYOUTS = {            # turn_based, observation, P  ->  Pa
    'alt': (True, False, 2),     # Pa = 1, two players taking turns
    'alt4': (True, False, 4),    # Pa = 1, four players
    'obs': (True, True, 2),      # Pa = P = 2
    'sim4': (False, False, 4),   # Pa = P = 4
}
TARGETS = [('UPGO', 'VTRACE'), ('TD', 'TD'), ('VTRACE', 'UPGO'), ('MC', 'VTRACE'), ('UPGO', 'TD')]   # (policy, value)


def case(kernel, A, layout, B, T, bi=0, heads='v', variant='auto', bf16=False, **tuning):
    """One shape.  heads: which of the value ('v') and return ('r') heads the net has."""
    return dict(kernel=kernel, A=A, layout=layout, B=B, T=T, bi=bi, heads=heads, variant=variant, bf16=bf16, tuning=tuning)


def _named(cases):
    out = []
    for i, c in enumerate(cases):
        c['seed'] = 1000 + 17 * i + c['A']
        tune = ''.join('-%s%d' % (k[:2], v) for k, v in sorted(c['tuning'].items()))
        c['id'] = '%s-A%d-%s-B%dT%dbi%d-%s-%s%s%s' % (c['kernel'], c['A'], c['layout'], c['B'], c['T'], c['bi'], c['heads'] or 'noheads',
                                                   c['variant'], tune, '-bf16' if c['bf16'] else '')
        out.append(c)
    return out


# Shape matrix: every NPL / LPR step of the row mapping, Pa = 1 and Pa = P (P = 2, 4), heads present and absent.  The packing
# kernels (group, element, rows) get small windows and a prime B, so that the last CTA owns fewer episodes than the others
# (tests/test_loss_dispatch_cpu.py recomputes EPB and checks it).
MATRIX = _named([
    case('group<1>', 1, 'obs', 37, 8),
    case('group<2>', 2, 'sim4', 13, 6, heads='vr'),
    case('group<4>', 3, 'alt', 37, 7, bi=2, heads='vr'),
    case('group<8>', 8, 'obs', 13, 6, bi=1, heads=''),
    case('group<16>', 16, 'alt4', 13, 6, heads='r'),
    case('group<32>', 17, 'alt', 13, 6, bi=2),
    case('group<32>', 24, 'obs', 7, 3, heads='vr'),
    case('group<32>', 32, 'alt', 7, 5),
    case('elem', 3, 'sim4', 13, 5, variant='element'),
    case('elem', 17, 'alt', 13, 6, bi=2, heads='r', variant='element'),
    case('elem', 32, 'obs', 7, 2, variant='element'),
    case('rows<1,1,false,false>', 1, 'alt', 37, 6, variant='rows-direct'),
    case('rows<1,2,false,false>', 2, 'obs', 37, 5, bi=1, variant='rows-direct'),
    case('rows<1,4,false,false>', 3, 'sim4', 13, 4, heads='vr', variant='rows-direct'),
    case('rows<1,8,false,false>', 8, 'alt4', 13, 7, heads='', variant='rows-direct'),
    case('rows<1,16,false,false>', 16, 'alt', 13, 9, bi=3, variant='rows-direct'),
    case('rows<1,1,false,true>', 1, 'obs', 13, 6, variant='rows-staged'),
    case('rows<1,2,false,true>', 2, 'alt', 37, 6, bi=2, heads='vr', variant='rows-staged'),
    case('rows<1,4,false,true>', 4, 'alt4', 13, 6, variant='rows-staged'),
    case('rows<1,8,false,true>', 5, 'sim4', 13, 3, heads='r', variant='rows-staged'),
    case('rows<1,16,false,true>', 9, 'obs', 13, 6, bi=1, variant='rows-staged'),
    case('rows<2,16,false,false>', 17, 'alt', 13, 6, variant='rows-direct'),
    case('rows<2,16,false,true>', 32, 'obs', 13, 5, bi=1, heads='vr', variant='rows-staged'),
    case('rows<2,16,false,true>', 24, 'sim4', 7, 4, variant='rows-staged'),
    case('rows<4,16,false,true>', 33, 'alt', 7, 6),
    case('rows<4,16,false,true>', 64, 'obs', 7, 12, bi=2, heads='r'),
    case('rows<4,16,false,false>', 48, 'alt4', 13, 4, variant='rows-direct'),
    case('rows<8,16,false,true>', 65, 'alt', 7, 3, heads='vr'),
    case('rows<8,16,false,true>', 100, 'obs', 7, 10, bi=3),
    case('rows<8,16,false,true>', 128, 'sim4', 5, 5, heads=''),
    case('rows<8,16,false,false>', 100, 'alt', 7, 5, bi=1, variant='rows-direct'),
    case('rows<16,16,false,false>', 129, 'alt', 7, 3, bi=1),
    case('rows<16,16,false,false>', 256, 'obs', 5, 9, heads='vr'),
    case('rows<16,16,false,true>', 200, 'alt', 7, 3, bi=1, variant='rows-staged'),
    case('rows<32,16,false,false>', 257, 'obs', 5, 6),
    case('rows<32,16,false,false>', 257, 'alt', 7, 3, bi=2, heads='r'),
    case('rows<32,16,false,true>', 257, 'alt4', 5, 5, variant='rows-staged'),
    case('rows<32,16,true,false>', 300, 'sim4', 5, 4, heads='r', variant='rows-direct'),
    case('rows<32,16,true,false>', 512, 'alt', 7, 3, bi=2, variant='rows-direct'),
    case('rows<32,32,false,false>', 513, 'alt', 5, 6, bi=1),
    case('rows<32,32,false,false>', 999, 'alt', 7, 2, bi=1, heads='vr'),
    case('rows<32,32,false,true>', 513, 'obs', 5, 4, heads='vr', variant='rows-staged'),
    case('rows<32,32,true,false>', 700, 'alt', 5, 7, bi=2),
    case('rows<32,32,true,false>', 1024, 'sim4', 3, 3, heads=''),
    case('rows<32,32,true,false>', 1024, 'alt', 7, 2, bi=1),
    case('bulk', 300, 'alt', 5, 20, bi=3),
    case('bulk', 508, 'obs', 5, 16, bi=2, heads='vr'),
    case('bulk', 512, 'sim4', 3, 8, heads='r'),
    case('bulk', 512, 'obs', 7, 40, bi=5),           # default path: a 2-CTA cluster, with burn-in
])

# Bulk (TMA) kernel forced with 1, 2, 4 or 8 CTAs per window: time axes that the cluster does not divide (down to CTAs that own
# no step at all), burn-in 0 and 3, 1 to 17 consumer warps, Pa = 2 and Pa = 1, bf16 logits.
BULK = _named([
    case('bulk', 512, 'obs', 5, 29, bi=0, variant='bulk', cluster=8, consumers=5),
    case('bulk', 512, 'obs', 5, 29, bi=3, heads='vr', variant='bulk', bf16=True, cluster=8, consumers=16),
    case('bulk', 320, 'obs', 7, 9, bi=0, variant='bulk', cluster=8, consumers=1),
    case('bulk', 512, 'obs', 3, 37, bi=0, heads='r', variant='bulk', cluster=8, consumers=17),
    case('bulk', 512, 'obs', 5, 37, bi=3, variant='bulk', cluster=4, consumers=16),
    case('bulk', 512, 'obs', 5, 9, bi=3, heads='vr', variant='bulk', cluster=4, consumers=1),
    case('bulk', 320, 'obs', 5, 37, bi=3, variant='bulk', bf16=True, cluster=2, consumers=17),
    case('bulk', 508, 'obs', 3, 37, bi=3, heads='', variant='bulk', cluster=2, consumers=5),
    case('bulk', 512, 'obs', 3, 23, bi=3, variant='bulk', cluster=1, consumers=17),
    case('bulk', 300, 'alt', 5, 29, bi=3, heads='vr', variant='bulk', cluster=1, consumers=1),
    case('bulk', 300, 'alt', 5, 29, bi=0, variant='bulk', cluster=4, consumers=5),
])

# windows of >= 96 trained steps: the scan recurrence is the default there
LONG = _named([
    case('group<32>', 19, 'alt', 5, 100, bi=2, heads='vr'),
    case('rows<4,16,false,true>', 40, 'alt', 3, 100, bi=2),
    case('bulk', 320, 'alt', 3, 100, bi=2, heads='r'),
])

# extreme but legal inputs (see _make_extreme), one small-A and one wide shape per family
EXTREME = _named([
    case('group<8>', 5, 'alt', 13, 8, bi=2, heads='vr'),
    case('rows<8,16,false,true>', 100, 'obs', 7, 6, bi=2),
    case('bulk', 512, 'obs', 5, 12, bi=2, heads='vr'),
    case('rows<32,32,true,false>', 1024, 'alt', 5, 6, bi=2),
])

_BY_ID = {c['id']: c for c in MATRIX + BULK + LONG + EXTREME}
assert len(_BY_ID) == len(MATRIX + BULK + LONG + EXTREME)
_EXTREME_IDS = {c['id'] for c in EXTREME}


# ------------------------------------------------------------------------------------------------------------------ helpers
_KERNEL_RE = re.compile(r'loss_(rows|group|elem|bulk)_kernel<([^>]*)>')
_FORMS = {('false', 'true'): 'fwd_bwd', ('true', 'true'): 'diag', ('false', 'false'): 'fwd'}
OBSERVED = set()       # (kernel, recurrence) pairs traced in this session


def kernel_key(name):
    """(kernel, form) of a traced loss kernel name, e.g. 'void hrl::loss_rows_kernel<32, 16, true, false, false, true>(...)'
    -> ('rows<32,16,true,false>', 'fwd_bwd'); None for any other kernel."""
    m = _KERNEL_RE.search(name)
    if not m:
        return None
    fam, params = m.group(1), [p.strip() for p in m.group(2).split(',')]
    form = _FORMS[tuple(params[-2:])]
    if fam == 'rows':
        return 'rows<%s>' % ','.join(params[:4]), form
    if fam == 'group':
        return 'group<%s>' % params[0], form
    return fam, form


def traced(fn, attempts=3):
    """Run fn() under torch.profiler (CUPTI activity tracing) and return (its result, the set of loss kernels it launched).
    A trace that holds no loss kernel at all (the tracer can drop the activity record of a kernel that ends just before the
    profiling window closes) is taken again: the launch is deterministic, a dispatch to the wrong kernel still shows."""
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    for _ in range(attempts):
        with torch.profiler.profile(activities=acts) as prof:
            out = fn()
            torch.cuda.synchronize()
            time.sleep(0.002)
        names = set()
        for e in prof.events():
            names.add(e.name)
            names.update(k.name for k in getattr(e, 'kernels', []))
        seen = {k for k in map(kernel_key, names) if k is not None}
        if seen:
            break
    return out, seen


def recurrence_of(c, rec):
    """The recurrence a launch runs: forced, or the default of the dispatcher (the suffix scan from 96 trained steps on)."""
    return rec if rec != 'auto' else ('scan' if c['T'] - c['bi'] >= 96 else 'serial')


def make_inputs(c):
    from handyrl_b200.synthetic import synthetic_batch, synthetic_outputs
    turn_based, observation, P = LAYOUTS[c['layout']]
    batch = synthetic_batch(c['B'], c['T'], P, c['A'], turn_based=turn_based, observation=observation, reward_kind='step',
                            gamma=0.9, burn_in=c['bi'], seed=c['seed'], with_obs=False)
    outs = synthetic_outputs(batch, has_value='v' in c['heads'], has_return='r' in c['heads'], seed=c['seed'] + 1)
    pol, val = TARGETS[c['seed'] % len(TARGETS)]
    args = {'turn_based_training': turn_based, 'observation': observation, 'gamma': 0.9, 'lambda': 0.7,
            'burn_in_steps': c['bi'], 'entropy_regularization': 0.1, 'entropy_regularization_decay': 0.1,
            'policy_target': pol, 'value_target': val}
    if c['bf16']:       # bf16-representable logits: the oracle sees exactly what the kernel reads
        outs['policy'] = outs['policy'].to(torch.bfloat16).float()
    return batch, outs, args


def _make_extreme(batch, outs, seed):
    """In place, on CPU tensors: behaviour probabilities of 1e-30 (below the 1e-16 clamp), 1e-7 and exactly 1; rows with a single
    legal action; rows whose legal logits spread over >= 100 (one action at +70, the taken one at -50, so that its probability
    underflows and its importance ratio sits far below the clamp); and window 0 all padding after the burn-in steps."""
    g = np.random.default_rng(seed)
    am = batch['action_mask'].numpy()
    act = batch['action'].numpy()[..., 0]
    prob = batch['selected_prob'].numpy()[..., 0]
    pol = outs['policy'].numpy()
    live = am[..., 0] == 0           # synthetic batches keep action 0 legal on live rows and mask every action of a dead row
    kind = np.where(live, g.integers(0, 4, live.shape), -1)
    pick = g.integers(0, 4, live.shape)
    prob[live & (pick == 0)] = 1e-30
    prob[live & (pick == 1)] = 1e-7
    prob[live & (pick == 2)] = 1.0
    one = np.nonzero(kind == 1)
    am[one] = 1e32
    am[one + (act[one],)] = 0.0
    for idx in zip(*np.nonzero(kind >= 2)):
        legal = np.nonzero(am[idx] == 0)[0]
        hi = g.choice(legal)
        pol[idx][hi] += 70.0
        if kind[idx] == 3 and hi != act[idx]:
            pol[idx][act[idx]] -= 50.0
        else:
            pol[idx][g.integers(0, pol.shape[-1])] -= 50.0
    return kind, prob


def _pad_after_burn_in(batch, bi):
    """Window 0: every step from the burn-in on is padding (the layout make_batch gives the steps after an episode's end)."""
    for k in ('episode_mask', 'turn_mask', 'observation_mask', 'reward', 'return'):
        batch[k][0, bi:] = 0.0
    batch['action_mask'][0, bi:] = 1e32
    batch['action'][0, bi:] = 0
    batch['selected_prob'][0, bi:] = 1.0
    batch['progress'][0, bi:] = 1.0


def extreme_inputs(c):
    batch, outs, args = make_inputs(c)
    kind, prob = _make_extreme(batch, outs, c['seed'] + 2)
    assert {1, 2, 3} <= set(np.unique(kind).tolist())
    assert {float(np.float32(p)) for p in (1e-30, 1e-7, 1.0)} <= set(np.unique(prob).tolist())
    _pad_after_burn_in(batch, c['bi'])
    return batch, outs, args


def to_dev(d):
    return {k: v.cuda() for k, v in d.items()}


def to_np(d):
    return {k: v.numpy() for k, v in d.items()}


def bf16_half_ulp(x):
    """Half the spacing of bf16 numbers (8 significant bits) at |x|: the rounding error of a bf16 store of x."""
    ax = np.abs(np.asarray(x, np.float64))
    e = np.floor(np.log2(np.where(ax > 0, ax, 1.0)))
    return np.where(ax > 0, np.exp2(e - 8), 0.0)


def assert_close(got, ref, what, err32=None, rtol=0.0, extra=None):
    """|got - ref| <= ATOL + rtol |ref| (+ ORACLE_ERR_FACTOR x err32, the float32 oracle's own error, + extra, where given)."""
    got = np.asarray(got, np.float64)
    ref = np.asarray(ref, np.float64)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    bound = ATOL + rtol * np.abs(ref)
    if err32 is not None:
        bound = bound + ORACLE_ERR_FACTOR * np.asarray(err32, np.float64)
    if extra is not None:
        bound = bound + extra
    err = np.abs(got - ref)
    bad = ~(err <= bound)
    if bad.any():
        i = np.unravel_index(np.argmax(np.where(bad, err - bound, -np.inf)), err.shape)
        raise AssertionError('%s: %d of %d elements outside the bound; worst at %s: got %r, oracle %r, bound %r'
                             % (what, bad.sum(), bad.size, i, got[i], ref[i], bound[i]))


def check_against_oracle(res, batch, outs, args, extreme=False, bf16=False, taps=True):
    from oracle import oracle
    nb, no = to_np(batch), to_np(outs)
    o64 = oracle.loss(nb, no, args, dtype=np.float64)
    o32 = oracle.loss(nb, no, args, dtype=np.float32) if extreme else None
    err = (lambda k: np.abs(o32[k].astype(np.float64) - o64[k])) if extreme else (lambda k: None)
    assert_close(res.losses.cpu().numpy(), o64['losses'], 'losses', err('losses'), rtol=RTOL)
    dpol = res.dpolicy.float().cpu().numpy()
    if bf16:    # gradients leave as bf16: half a bf16 ulp of each element on top of ATOL
        assert_close(dpol, o64['dpolicy_raw'], 'dpolicy', extra=bf16_half_ulp(o64['dpolicy_raw']))
    else:
        assert_close(dpol, o64['dpolicy_raw'], 'dpolicy', err('dpolicy_raw'))
    for k, key in (('dvalue', 'dvalue_raw'), ('dreturn', 'dreturn_raw')):
        if o64[key] is None:
            assert getattr(res, k) is None
        else:
            assert_close(getattr(res, k).cpu().numpy(), o64[key], k, err(key))
    if taps:
        for k in ('target_value', 'target_return', 'advantage', 'logp', 'rho', 'entropy'):
            assert_close(res.taps[k].cpu().numpy(), o64[k], 'tap ' + k, err(k))
    return o64


def tuning_of(c, rec):
    t = dict(c['tuning'], recurrence=rec)
    if c['variant'] != 'auto':
        t['variant'] = c['variant']
    return t


def launch(c, rec, batch, outs, args, **kw):
    """Fused loss of case c on the device; asserts that the declared kernel served it and records (kernel, recurrence)."""
    from handyrl_b200 import ops
    db, do = to_dev(batch), to_dev(outs)
    if c['bf16']:
        do['policy'] = do['policy'].to(torch.bfloat16)
    form = kw.pop('form', 'fwd_bwd')
    fn = ops.loss_fwd if form == 'fwd' else ops.loss_fwd_bwd
    res, seen = traced(lambda: fn(do, db, args, tuning=tuning_of(c, rec), **kw))
    OBSERVED.update((k, recurrence_of(c, rec)) for k, _ in seen)
    # a trace without any loss kernel (dropped record) proves nothing either way; the coverage test relaunches what is missing
    assert seen <= {(c['kernel'], form)}, (c['id'], 'traced', sorted(seen))
    return res


# -------------------------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize('rec', RECURRENCES)
@pytest.mark.parametrize('cid', [c['id'] for c in MATRIX])
def test_shape_matrix_against_oracle(cid, rec):
    c = _BY_ID[cid]
    batch, outs, args = make_inputs(c)
    res = launch(c, rec, batch, outs, args, taps=True)
    check_against_oracle(res, batch, outs, args)


@pytest.mark.parametrize('rec', RECURRENCES)
@pytest.mark.parametrize('cid', [c['id'] for c in BULK])
def test_bulk_cluster_splits_against_oracle(cid, rec):
    """Each CTA of a cluster owns ceil(Tt / cluster) steps of the window, the last ones fewer or none; burn-in steps are zeroed
    by CTA 0 only.  bf16 logits are checked against the float32 oracle on the same (bf16-representable) logits."""
    c = _BY_ID[cid]
    batch, outs, args = make_inputs(c)
    res = launch(c, rec, batch, outs, args, taps=True)
    check_against_oracle(res, batch, outs, args, bf16=c['bf16'])
    if c['bi']:
        assert not res.dpolicy[:, :c['bi']].float().any()


@pytest.mark.parametrize('rec', ['auto', 'serial'])
@pytest.mark.parametrize('cid', [c['id'] for c in LONG])
def test_long_windows_default_scan_and_forced_serial(cid, rec):
    c = _BY_ID[cid]
    assert c['T'] - c['bi'] >= 96
    batch, outs, args = make_inputs(c)
    res = launch(c, rec, batch, outs, args, taps=True)
    check_against_oracle(res, batch, outs, args)


@pytest.mark.parametrize('cid', [c['id'] for c in EXTREME])
def test_extreme_inputs_against_oracle(cid):
    c = _BY_ID[cid]
    batch, outs, args = extreme_inputs(c)
    res = launch(c, 'auto', batch, outs, args, taps=True)
    check_against_oracle(res, batch, outs, args, extreme=True)
    # the padded window: nothing of it is trained, every gradient of it is exactly zero
    assert not res.dpolicy[0].any() and (res.dvalue is None or not res.dvalue[0].any())


SENTINEL = 7.25


def _offset_copy(t, offset, tail=64):
    """t copied into a fresh buffer at `offset` floats (not 16-byte aligned), SENTINEL before and after: (view, buffer)."""
    buf = torch.full((offset + t.numel() + tail,), SENTINEL, dtype=t.dtype, device=t.device)
    view = buf[offset:offset + t.numel()].view(t.shape)
    view.copy_(t)
    return view, buf


@pytest.mark.parametrize('which', ['inputs_and_output', 'output'])
@pytest.mark.parametrize('rec', RECURRENCES)
@pytest.mark.parametrize('A,kernel', [(512, 'rows<32,16,false,false>'), (1024, 'rows<32,32,false,false>')])
def test_misaligned_tensors_take_the_scalar_rows_kernel(A, kernel, rec, which):
    """Logits / action masks at a storage offset of 1 float, and a gradient buffer at 33 floats with guard bands: the vector and
    bulk kernels need 16-byte alignment, so the scalar rows kernel serves; results match the oracle and nothing outside the
    gradient view is written."""
    from handyrl_b200 import ops
    c = _named([case(kernel, A, 'obs', 7, 6, bi=1, heads='vr')])[0]
    batch, outs, args = make_inputs(c)
    db, do = to_dev(batch), to_dev(outs)
    if which == 'inputs_and_output':
        do['policy'], _ = _offset_copy(do['policy'], 1)
        db['action_mask'], _ = _offset_copy(db['action_mask'], 1)
        assert do['policy'].data_ptr() % 16 and db['action_mask'].data_ptr() % 16
    B, T, Pa, _ = do['policy'].shape
    buf = ops.LossBuffers(B, T, 2, Pa, A, True, True, 'cuda', taps=True)
    buf.dpolicy, dpol_buf = _offset_copy(buf.dpolicy, 33)
    buf.dvalue, dval_buf = _offset_copy(buf.dvalue, 1)
    res, seen = traced(lambda: ops.loss_fwd_bwd(do, db, args, buffers=buf, tuning={'recurrence': rec}))
    OBSERVED.update((k, rec) for k, _ in seen)
    assert seen <= {(kernel, 'fwd_bwd')}, sorted(seen)
    check_against_oracle(res, batch, outs, args)
    n = res.dpolicy.numel()
    for name, b, lo, hi in (('dpolicy', dpol_buf, 33, 33 + n), ('dvalue', dval_buf, 1, 1 + res.dvalue.numel())):
        guard = torch.cat([b[:lo], b[hi:]]).cpu()
        assert torch.all(guard == SENTINEL), (name, 'written outside the view')


# one shape per kernel family, ragged and extreme
def _first(cases, **kw):
    return next(c['id'] for c in cases if all(c[k] == v for k, v in kw.items()))


FORM_CASES = [_first(MATRIX, kernel='group<32>', A=17), _first(MATRIX, kernel='elem', A=17),
              _first(MATRIX, kernel='rows<8,16,false,false>'), _first(BULK, bf16=True, tuning={'cluster': 8, 'consumers': 16}),
              _first(BULK, T=9, tuning={'cluster': 4, 'consumers': 1})] + [c['id'] for c in EXTREME]


@pytest.mark.parametrize('cid', FORM_CASES)
def test_forward_only_and_diagnostics_sums_are_bit_identical(cid):
    c = _BY_ID[cid]
    batch, outs, args = (extreme_inputs if cid in _EXTREME_IDS else make_inputs)(c)
    plain = launch(c, 'auto', batch, outs, args)
    fwd_losses = launch(c, 'auto', batch, outs, args, form='fwd')
    diag = launch(c, 'auto', batch, outs, args, form='diag', diagnostics=True)
    assert torch.equal(fwd_losses, plain.losses), (fwd_losses, plain.losses)
    assert torch.equal(diag.losses, plain.losses)
    assert torch.equal(diag.dpolicy, plain.dpolicy)
    assert torch.isfinite(diag.diagnostics).all()


@pytest.mark.parametrize('cid', FORM_CASES)
def test_window_weights_scale_each_window_of_the_oracle(cid):
    """window_weight[b] scales every loss term and gradient of window b; dcnt is not weighted."""
    from oracle import oracle
    c = _BY_ID[cid]
    extreme = cid in _EXTREME_IDS
    batch, outs, args = (extreme_inputs if extreme else make_inputs)(c)
    B = c['B']
    w = np.random.default_rng(c['seed']).uniform(0.25, 2.0, B).astype(np.float32)
    res = launch(c, 'auto', batch, outs, args, window_weight=torch.from_numpy(w).cuda())
    nb, no = to_np(batch), to_np(outs)
    want = np.zeros(6)
    err = np.zeros(6)
    for b in range(B):
        sl = lambda d: {k: v[b:b + 1] for k, v in d.items()}
        lb = oracle.loss(sl(nb), sl(no), args, dtype=np.float64)['losses']
        scale = np.array([w[b]] * 5 + [1.0])
        want += scale * lb
        if extreme:
            err += scale * np.abs(oracle.loss(sl(nb), sl(no), args, dtype=np.float32)['losses'] - lb)
    assert_close(res.losses.cpu().numpy(), want, 'weighted losses', err if extreme else None, rtol=RTOL)
    o64 = oracle.loss(nb, no, args, dtype=np.float64)
    o32 = oracle.loss(nb, no, args, dtype=np.float32) if extreme else None
    wb = w.astype(np.float64).reshape(B, 1, 1, 1)
    for k, key in (('dpolicy', 'dpolicy_raw'), ('dvalue', 'dvalue_raw'), ('dreturn', 'dreturn_raw')):
        if o64[key] is None:
            continue
        got = getattr(res, k).float().cpu().numpy()
        e32 = wb * np.abs(o32[key] - o64[key]) if extreme else None
        if c['bf16'] and k == 'dpolicy':
            assert_close(got, wb * o64[key], 'weighted ' + k, extra=bf16_half_ulp(wb * o64[key]))
        else:
            assert_close(got, wb * o64[key], 'weighted ' + k, e32)


def test_every_instantiation_ran_under_both_recurrences():
    """The traced (kernel, recurrence) pairs equal COVERAGE.  Pairs that no earlier test of this session traced (the file run in
    part, or a dropped trace record) are launched here from the matrix cases declaring the kernel."""
    for kernel, rec in sorted(COVERAGE - OBSERVED):
        for c in [c for c in MATRIX if c['kernel'] == kernel] * 2:
            if (kernel, rec) in OBSERVED:
                break
            batch, outs, args = make_inputs(c)
            launch(c, rec, batch, outs, args)
    assert OBSERVED == COVERAGE, ('traced but not declared', sorted(OBSERVED - COVERAGE), 'declared but not traced',
                                  sorted(COVERAGE - OBSERVED))
