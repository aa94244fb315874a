"""Compile-time guard of the weight-gradient GEMM on warp-level MMAs (csrc/gemm_wgrad_kernel.cu), no GPU needed: the
instantiations the TicTacToe tower runs at B=512 T=32 (bench.py's cfg2) must not spill.  Template arguments are the
operand kinds (A: 0 plain, 1 x*p + r, 2 two sources; B: 0 plain, 1 x*p + r): <2, 1> the tower layers after the first,
<2, 0> the first tower layer (the stem's output is a plain operand), <0, 1> the heads.
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

CFG2 = [(2, 1), (2, 0), (0, 1)]


@pytest.fixture(scope='module')
def report():
    """{(a_kind, b_kind): {'spill_stores': bytes, 'spill_loads': bytes, 'stack': bytes}} from ptxas -v."""
    if not (os.path.exists(NVCC) or shutil.which(NVCC)):
        pytest.skip('nvcc is not available')
    with tempfile.TemporaryDirectory() as d:
        cmd = [NVCC, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-c', '-Xptxas', '-v',
               '-o', os.path.join(d, 'gemm_wgrad_kernel.o'), os.path.join(CSRC, 'gemm_wgrad_kernel.cu')]
        res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    pat = re.compile(r'gemm_wgrad_kernelILi(\d)ELi(\d)EE')
    out, cur = {}, None
    for line in res.stderr.splitlines():
        if 'Compiling entry function' in line:
            m = pat.search(line)
            cur = (int(m.group(1)), int(m.group(2))) if m else None
            continue
        s = re.search(r'(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads', line)
        if s and cur is not None:
            out[cur] = dict(stack=int(s.group(1)), spill_stores=int(s.group(2)), spill_loads=int(s.group(3)))
    return out


def test_every_operand_kind_is_instantiated(report):
    assert sorted(report) == [(a, b) for a in range(3) for b in range(2)]


@pytest.mark.parametrize('key', CFG2, ids=lambda k: 'a%d_b%d' % k)
def test_flagship_instantiations_do_not_spill(report, key):
    r = report[key]
    assert r['spill_stores'] == 0 and r['spill_loads'] == 0 and r['stack'] == 0, r
