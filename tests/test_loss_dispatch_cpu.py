"""The kernel instantiations the fused loss dispatcher can launch, read from csrc/loss_kernel.cu, are exactly the ones the GPU
parity file declares (test_loss_dispatch_gpu.KERNELS): a new instantiation without a parity case fails on any machine.  Also
checks, from the dispatcher's packing rules, that the packed shapes of that file end their grid with a partial CTA."""
import os
import re

from conftest import ROOT
from test_loss_dispatch_gpu import BULK, KERNELS, LAYOUTS, LONG, MATRIX

SRC = os.path.join(ROOT, 'handyrl_b200', 'csrc', 'loss_kernel.cu')


def _dispatch_source():
    with open(SRC) as f:
        src = f.read()
    start = src.index('static int loss_fwd_bwd(')
    return src[start:src.index('\n}\n', start)]


def dispatched_instantiations():
    body = _dispatch_source()
    b = lambda x: 'true' if x == 'true' else 'false'
    found = set()
    # rows kernel: HRL_CASE(l, n, v, s) and HRL_CASE2(l, n) == HRL_CASE(l, n, false, false) HRL_CASE(l, n, false, true)
    lines = [ln for ln in body.splitlines() if not ln.lstrip().startswith('#define')]
    text = '\n'.join(lines)
    for l, n, v, s in re.findall(r'\bHRL_CASE\(\s*(\d+)\s*,\s*(\d+)\s*,\s*(\w+)\s*,\s*(\w+)\s*\)', text):
        found.add('rows<%s,%s,%s,%s>' % (l, n, b(v), b(s)))
    for l, n in re.findall(r'\bHRL_CASE2\(\s*(\d+)\s*,\s*(\d+)\s*\)', text):
        found.update('rows<%s,%s,false,%s>' % (l, n, s) for s in ('false', 'true'))
    # group kernel: the switch over RL
    found.update('group<%s>' % rl for rl in re.findall(r'loss_group_kernel<\s*(\d+)\s*,\s*DIAG\s*,\s*GRAD\s*>', body))
    if re.search(r'loss_elem_kernel<\s*DIAG\s*,\s*GRAD\s*>', body):
        found.add('elem')
    if re.search(r'launch_bulk<\s*DIAG\s*,\s*GRAD\s*>', body):
        found.add('bulk')
    return found


def test_dispatcher_instantiations_equal_the_declared_coverage():
    found = dispatched_instantiations()
    assert len(found) >= 30, sorted(found)    # the parser still sees the dispatcher
    assert found == set(KERNELS), ('dispatched, no parity case', sorted(found - KERNELS), 'declared, not dispatched',
                                   sorted(KERNELS - found))


def test_every_declared_kernel_has_a_matrix_case():
    assert {c['kernel'] for c in MATRIX} == set(KERNELS)
    assert {c['kernel'] for c in BULK} == {'bulk'} and {1, 2, 4, 8} == {c['tuning']['cluster'] for c in BULK}
    assert {c['kernel'].split('<')[0] for c in LONG} == {'group', 'rows', 'bulk'}


def _pow2_ceil(x):
    p = 1
    while p < x:
        p <<= 1
    return p


def episodes_per_cta(c):
    """EPB of a packing kernel for case c: the rules of loss_fwd_bwd (group, element, rows)."""
    P = LAYOUTS[c['layout']][2]
    Pa = 1 if LAYOUTS[c['layout']][0] and not LAYOUTS[c['layout']][1] else P
    R, A, B = (c['T'] - c['bi']) * Pa, c['A'], c['B']
    fam = c['kernel'].split('<')[0]
    if fam in ('group', 'elem'):
        per_ep = R * (_pow2_ceil(A) if fam == 'group' else A)
        epb = 1 if per_ep >= 256 else -(-256 // per_ep)
        return min(epb, B)
    lpr = 1
    while lpr < 32 and -(-A // lpr) > 16:
        lpr <<= 1
    lanes = R * lpr
    return 1 if lanes >= 64 else min(64 // lanes, B)


def test_packed_shapes_end_with_a_partial_cta():
    """Each packing family has cases whose last CTA owns fewer episodes than EPB (B % EPB != 0), and EPB > 1 wherever B is
    packed at all."""
    ragged = set()
    for c in MATRIX:
        fam = c['kernel'].split('<')[0]
        if fam == 'bulk':
            continue
        epb = episodes_per_cta(c)
        if epb > 1:
            assert c['B'] % epb != 0, (c['id'], epb)
            ragged.add(fam)
    assert ragged == {'group', 'elem', 'rows'}
