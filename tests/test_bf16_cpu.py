"""The bf16 mode of the net's tensor-core products without a GPU: the train_args key, the ABI fields it adds, and a compile-time
guard of the bf16 GEMM translation unit (csrc/gemm_bf16_kernel.cu) in the manner of test_gemm_build_cpu.py."""
import ctypes
import os
import re
import shutil
import subprocess
import tempfile

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'handyrl_b200', 'csrc')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')

# (A k-major, B k-major, packed B, MMA width) of the TicTacToe tower at B=512 T=32 (bench.py's cfg2)
CFG2 = [(True, True, True, 144), (False, False, False, 144), (False, False, False, 16)]


@pytest.mark.parametrize('value,mode', [(True, True), (False, False), ('bf16', 'bf16'), ('tf32', True), ('', False), (1, True),
                                        (0, False), (None, False)])
def test_tensor_core_key(value, mode):
    from handyrl_b200.train import tensor_core_mode
    got = tensor_core_mode(value)
    assert got == mode and type(got) is type(mode)


def test_tensor_core_key_absent_is_the_default():
    from handyrl_b200.train import tensor_core_mode
    assert tensor_core_mode({}.get('tensor_cores', True)) is True


def test_optimize_small_boards_marks_the_mode():
    from handyrl_b200 import fastnet
    for mode, mark in ((True, True), (False, False), ('bf16', 'bf16')):
        net = torch.nn.Sequential(torch.nn.Conv2d(4, 8, 3, padding=1), torch.nn.BatchNorm2d(8))
        assert fastnet.optimize_small_boards(net, tensor_cores=mode) == 2
        assert net[0].tensor_cores == mark and fastnet._bf16(net[0]) == (mark == 'bf16')


def test_appended_abi_fields():
    """HrlGemmArgs.bf16 and HrlPackJob.bf16 sit at the end of their structs (zero = the 3xTF32 behaviour), at the offsets
    the C compiler gives them."""
    from handyrl_b200 import _capi
    fields = [('HrlGemmArgs', 'bf16'), ('HrlPackJob', 'bf16'), ('HrlGemmArgs', 'conv_ones_row'), ('HrlPackJob', 'bias_cells')]
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "hrl_b200.h"\nint main(){' +
           'printf("%zu\\n", sizeof(HrlGemmArgs));printf("%zu\\n", sizeof(HrlPackJob));' +
           ''.join('printf("%%zu\\n", offsetof(%s, %s));' % f for f in fields) + 'return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, 's.c')
        open(c, 'w').write(src)
        exe = os.path.join(d, 's')
        subprocess.run(['gcc', '-I', os.path.join(ROOT, 'include'), c, '-o', exe], check=True)
        got = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    want = [ctypes.sizeof(_capi.HrlGemmArgs), ctypes.sizeof(_capi.HrlPackJob)] + \
        [getattr(getattr(_capi, n), f).offset for n, f in fields]
    assert got == want
    for n in ('HrlGemmArgs', 'HrlPackJob'):
        assert getattr(_capi, n)._fields_[-1][0] == 'bf16'
    assert _capi.SYMBOLS['hrl_conv_pack_bf16'] == _capi.SYMBOLS['hrl_conv_pack']
    assert _capi.HRL_ABI_VERSION == 3


def ptxas_report():
    """{(a_k, b_k, packed, width): {'spill_stores', 'spill_loads', 'stack', 'c7519'}} of the bf16 translation unit."""
    if not (os.path.exists(NVCC) or shutil.which(NVCC)):
        pytest.skip('nvcc is not available')
    with tempfile.TemporaryDirectory() as d:
        cmd = [NVCC, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-c', '-Xptxas', '-v',
               '-o', os.path.join(d, 'gemm_bf16_kernel.o'), os.path.join(CSRC, 'gemm_bf16_kernel.cu')]
        res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    assert 'gemm_tf32x3_kernel' not in res.stderr          # the 3xTF32 instantiations live in gemm_kernel.cu alone
    pat = re.compile(r'gemm_bf16_kernelILb([01])ELb([01])ELb([01])ELi(\d+)E')
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


def test_every_bf16_width_is_instantiated(report):
    widths = sorted({k[3] for k in report})
    assert widths == list(range(8, 129, 8)) + [144]
    for w in widths:        # four operand layouts of plain B, two of a packed (k-major) B image
        assert sum(1 for k in report if k[3] == w) == 6, w


def test_no_injected_warpgroup_arrive_bf16(report):
    bad = {k: v['c7519'] for k, v in report.items() if v['c7519']}
    assert not bad, 'ptxas serialised the wgmma chain (C7519) in %s' % bad


@pytest.mark.parametrize('key', CFG2, ids=lambda k: 'a%d_b%d_packed%d_n%d' % k)
def test_flagship_bf16_instantiations_do_not_spill(report, key):
    r = report[key]
    assert r['spill_stores'] == 0 and r['spill_loads'] == 0 and r['stack'] == 0, r
