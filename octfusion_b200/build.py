"""Compile the CUDA sources in csrc/ for sm_90a into octfusion_b200/lib/liboctfusion_b200.so.

Plain nvcc, in-tree output next to the package, so that the built tree is importable as it stands (a read-only
tree included).  Cross-compiles without a GPU.  Re-runs only when a source is newer than the .so.
"""
from __future__ import annotations
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIBDIR = os.path.join(HERE, 'lib')
LIB = os.path.join(LIBDIR, 'liboctfusion_b200.so')
SOURCES = ['runtime.cu', 'gemm_simt.cu', 'gemm_tc.cu', 'norm.cu', 'attention.cu', 'misc.cu', 'graph.cu', 'mpu.cu', 'metrics.cu',
           'mesh.cu', 'points.cu', 'mesh_components.cu']
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
              '-Xcompiler', '-fPIC', '--expt-relaxed-constexpr', '--extended-lambda']


def _nvcc():
    for c in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return 'nvcc'


def have_nvcc() -> bool:
    import shutil
    c = _nvcc()
    return os.path.exists(c) if os.path.isabs(c) else shutil.which(c) is not None


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + ['common.cuh', 'mc_table.inc']] + [
            os.path.join(HERE, '..', 'include', 'octfusion_b200.h'), os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    os.makedirs(LIBDIR, exist_ok=True)
    objdir = os.path.join(HERE, 'build')
    os.makedirs(objdir, exist_ok=True)
    nvcc = _nvcc()
    procs = []
    for s in SOURCES:
        obj = os.path.join(objdir, s.replace('.cu', '.o'))
        cmd = [nvcc, *NVCC_FLAGS, '-c', os.path.join(CSRC, s), '-o', obj]
        if verbose:
            cmd.insert(1, '-Xptxas'); cmd.insert(2, '-v')
        procs.append((s, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    objs = []
    for s, obj, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError('nvcc failed on %s:\n%s' % (s, out))
        if verbose and out:
            print(out)
        objs.append(obj)
    cmd = [nvcc, '-shared', '-o', LIB, *objs, '-lcudart']
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError('link failed:\n' + r.stdout)
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
