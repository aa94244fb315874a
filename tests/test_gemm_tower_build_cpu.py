"""Compile-time guard of the tower's forward / input-gradient GEMM (csrc/gemm_tower_kernel.cu), no GPU needed.  Template
argument: the A operand kind (0 plain, 1 x*p + r with optional ReLU, 2 two sources); cfg2 runs all three.  Each must fit the
128 registers of a 512-thread block without spills, keep the wgmma chain unserialised (no C75xx warning from ptxas), and
issue HGMMA.64x144x8.F32.TF32 with its A operand in registers.
"""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'handyrl_b200', 'csrc')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
CUOBJDUMP = os.path.join(os.path.dirname(NVCC), 'cuobjdump')


@pytest.fixture(scope='module')
def build():
    """(ptxas -v output, cuobjdump -sass output) of the unit."""
    if not (os.path.exists(NVCC) or shutil.which(NVCC)):
        pytest.skip('nvcc is not available')
    with tempfile.TemporaryDirectory() as d:
        obj = os.path.join(d, 'gemm_tower_kernel.o')
        cmd = [NVCC, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-c', '-Xptxas', '-v',
               '-o', obj, os.path.join(CSRC, 'gemm_tower_kernel.cu')]
        res = subprocess.run(cmd, capture_output=True, text=True)
        assert res.returncode == 0, res.stdout + res.stderr
        sass = None
        if os.path.exists(CUOBJDUMP):
            dump = subprocess.run([CUOBJDUMP, '-sass', obj], capture_output=True, text=True)
            assert dump.returncode == 0, dump.stderr
            sass = dump.stdout
    return res.stderr, sass


def report(log):
    """{kind: {'regs', 'stack', 'spill_stores', 'spill_loads'}} per gemm_tower_kernel instantiation."""
    pat = re.compile(r'gemm_tower_kernelILi(\d)EE')
    out, cur = {}, None
    for line in log.splitlines():
        if 'Compiling entry function' in line:
            m = pat.search(line)
            cur = int(m.group(1)) if m else None
            continue
        if cur is None:
            continue
        s = re.search(r'(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads', line)
        if s:
            out.setdefault(cur, {}).update(stack=int(s.group(1)), spill_stores=int(s.group(2)), spill_loads=int(s.group(3)))
        r = re.search(r'Used (\d+) registers', line)
        if r:
            out.setdefault(cur, {})['regs'] = int(r.group(1))
    return out


def test_every_operand_kind_is_instantiated(build):
    assert sorted(report(build[0])) == [0, 1, 2]


@pytest.mark.parametrize('kind', [0, 1, 2])
def test_no_spills_and_at_most_128_registers(build, kind):
    r = report(build[0])[kind]
    assert r['spill_stores'] == 0 and r['spill_loads'] == 0 and r['stack'] == 0, r
    assert r['regs'] <= 128, r


def test_wgmma_chain_is_not_serialised(build):
    warnings = [line for line in build[0].splitlines() if re.search(r'\(C75\d\d\)', line) or 'serialized' in line]
    assert not warnings, warnings


def test_sass_issues_hgmma_with_register_a(build):
    sass = build[1]
    if sass is None:
        pytest.skip('cuobjdump is not available')
    hgmma = re.findall(r'HGMMA\.64x144x8\.F32\.TF32 (R\d+), (\S+), gdesc', sass)
    assert hgmma, 'no HGMMA.64x144x8.F32.TF32 in the SASS'
    assert all(re.fullmatch(r'R\d+', a) for _, a in hgmma), hgmma
