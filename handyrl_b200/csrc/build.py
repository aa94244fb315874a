"""Build handyrl_b200/libhrl_b200.so from the .cu sources with nvcc for sm_90a (in-tree)."""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(os.path.dirname(HERE), 'libhrl_b200.so')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
         '-Xcompiler', '-fPIC', '-shared', '--ptxas-options=-v',
         '--threads', '0']          # the translation units compile in parallel (two of them are the GEMM's 102 instantiations each)


def sources():
    return sorted(glob.glob(os.path.join(HERE, '*.cu')))


def needs_build():
    if not os.path.exists(OUT):
        return True
    deps = sources() + glob.glob(os.path.join(HERE, '*.cuh')) + [os.path.join(HERE, '..', '..', 'include', 'hrl_b200.h'),
                                                                os.path.abspath(__file__)]      # the flags live here
    return any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return OUT
    cmd = [NVCC] + FLAGS + ['-o', OUT] + sources()
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError('nvcc failed: ' + ' '.join(cmd))
    if verbose:
        sys.stderr.write(res.stderr)
    with open(os.path.join(HERE, 'ptxas.log'), 'w') as f:
        f.write(res.stderr)
    return OUT


if __name__ == '__main__':
    print(build(force='-f' in sys.argv, verbose=True))
