"""Compile-time guard of the tensor-core GEMM (csrc/gemm_kernel.cu), no GPU needed: ptxas must keep every wgmma chain
unserialised and the flagship workload's instantiations free of register spills.

* C7519 ("warpgroup.arrive is injected ... to allow use of registers in GMMA") means ptxas could not keep the accumulators
  in fixed registers across the wgmma of a stage and waits between them: the three-product chain runs partly serialised.
  It returns as soon as the MMA width stops being a compile-time constant of the kernel.
* The instantiations the TicTacToe tower runs at B=512 T=32 (bench.py's cfg2) must not spill: the packed-weight forward and
  input gradient <A k-major, B k-major, packed, width 144>, the weight gradient <both transposed, width 144> and the stem's
  weight gradient <both transposed, width 16>.
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

# (A k-major, B k-major, packed B, MMA width)
CFG2 = [(True, True, True, 144), (False, False, False, 144), (False, False, False, 16)]


def ptxas_report():
    """{(a_k, b_k, packed, width): {'spill_stores': bytes, 'spill_loads': bytes, 'stack': bytes, 'c7519': count}}."""
    if not (os.path.exists(NVCC) or shutil.which(NVCC)):
        pytest.skip('nvcc is not available')
    with tempfile.TemporaryDirectory() as d:
        cmd = [NVCC, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-c', '-Xptxas', '-v',
               '-o', os.path.join(d, 'gemm_kernel.o'), os.path.join(CSRC, 'gemm_kernel.cu')]
        res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    pat = re.compile(r'gemm_tf32x3_kernelILb([01])ELb([01])ELb([01])ELi(\d+)E')
    report, cur = {}, None
    for line in res.stderr.splitlines():
        m = pat.search(line)
        if 'C7519' in line:
            assert m, line
            key = tuple(bool(int(x)) for x in m.groups()[:3]) + (int(m.group(4)),)
            report.setdefault(key, {'c7519': 0})
            report[key]['c7519'] += 1
            continue
        if 'Compiling entry function' in line:
            cur = None
            if m:
                cur = tuple(bool(int(x)) for x in m.groups()[:3]) + (int(m.group(4)),)
                report.setdefault(cur, {'c7519': 0})
            continue
        s = re.search(r'(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads', line)
        if s and cur is not None:
            report[cur].update(stack=int(s.group(1)), spill_stores=int(s.group(2)), spill_loads=int(s.group(3)))
    return report


@pytest.fixture(scope='module')
def report():
    return ptxas_report()


def test_every_width_is_instantiated(report):
    widths = sorted({k[3] for k in report})
    assert widths == list(range(8, 129, 8)) + [144]
    for w in widths:        # four operand layouts of plain B, two of a packed (k-major) B image
        assert sum(1 for k in report if k[3] == w) == 6, w


def test_no_injected_warpgroup_arrive(report):
    bad = {k: v['c7519'] for k, v in report.items() if v['c7519']}
    assert not bad, 'ptxas serialised the wgmma chain (C7519) in %s' % bad


@pytest.mark.parametrize('key', CFG2, ids=lambda k: 'a%d_b%d_packed%d_n%d' % k)
def test_flagship_instantiations_do_not_spill(report, key):
    r = report[key]
    assert r['spill_stores'] == 0 and r['spill_loads'] == 0 and r['stack'] == 0, r
