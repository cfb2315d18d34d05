"""Build libnmarl.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python -m deeprl_network_b200.build [--force]

The shared library lands next to this file (git-ignored, but it travels to the GPU box with
the repo snapshot).  env.cu is compiled with --fmad=false: the CACC dynamics must reproduce the
reference's NumPy float64 arithmetic, which never contracts a*b+c.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libnmarl.so')
SOURCES = [('api.cu', []), ('env.cu', ['--fmad=false']), ('cell_fwd.cu', []), ('train.cu', []), ('tc_gemm.cu', []), ('tc_cell.cu', []), ('tc_bwd.cu', []), ('tc_wgrad.cu', []), ('eval.cu', [])]
ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
COMMON = ['-O3', '-lineinfo', '-std=c++17', '-Xcompiler', '-fPIC', '-Xcompiler', '-fvisibility=hidden']


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, '..', 'include', 'nmarl.h')]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not _stale():
        return LIB
    nvcc = os.environ.get('NVCC', 'nvcc')
    objdir = os.path.join(HERE, 'build')
    os.makedirs(objdir, exist_ok=True)
    procs, objs = [], []
    for src, extra in SOURCES:
        obj = os.path.join(objdir, src.replace('.cu', '.o'))
        cmd = [nvcc] + ARCH + COMMON + extra + ['-c', os.path.join(CSRC, src), '-o', obj]
        if verbose:
            print(' '.join(cmd))
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(obj)
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError('nvcc failed on %s:\n%s' % (src, out.decode()))
    cmd = [nvcc] + ARCH + ['-shared', '-o', LIB] + objs + ['-Xcompiler', '-fvisibility=hidden']
    subprocess.check_call(cmd)
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose=True))
