"""TEST INFRASTRUCTURE.  Builds oracle/_ref/libref_structural.so: the reference's own structural-loss kernels
(metrics/pytorch_structural_losses/src/approxmatch.cu and nndistance.cu, the CUDA behind `match_cost` and
`nn_distance` of reference metrics/evaluation_metrics.py), compiled IN PLACE from the reference checkout named by
OCTFUSION_REFERENCE for sm_90a, plus the C wrapper oracle/ref_structural.cu.  No torch is needed; the library is loaded
with ctypes by oracle/ref_metrics.py and is the reference arm of tests/test_gpu_metrics.py and
tools/bench_metrics.py.

Without a reference checkout this does nothing and keeps whatever oracle/_ref already holds.

    python -m oracle.build_ref
"""
from __future__ import annotations
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
OUT_DIR = os.path.join(HERE, '_ref')
LIB = os.path.join(OUT_DIR, 'libref_structural.so')
WRAPPER = os.path.join(HERE, 'ref_structural.cu')
REFERENCE_ROOT = os.environ.get('OCTFUSION_REFERENCE', '/root/reference')
FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-Xcompiler', '-fPIC']


def reference_src() -> str:
    return os.path.join(REFERENCE_ROOT, 'metrics', 'pytorch_structural_losses', 'src')


def build(verbose: bool = False) -> str | None:
    """compile the reference kernels into LIB; returns its path, or None when the reference tree is absent"""
    src = reference_src()
    units = [os.path.join(src, 'approxmatch.cu'), os.path.join(src, 'nndistance.cu'), WRAPPER]
    if not all(os.path.exists(u) for u in units):
        return None
    from octfusion_b200.build import _nvcc
    nvcc = _nvcc()
    os.makedirs(OUT_DIR, exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:
        objs, procs = [], []
        for u in units:
            obj = os.path.join(tmp, os.path.basename(u) + '.o')
            cmd = [nvcc, *FLAGS, '-I', src, '-c', u, '-o', obj]
            procs.append((u, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
            objs.append(obj)
        for u, p in procs:
            out, _ = p.communicate()
            if p.returncode != 0:
                raise RuntimeError('nvcc failed on %s:\n%s' % (u, out))
            if verbose and out:
                print(out)
        tmp_lib = os.path.join(tmp, os.path.basename(LIB))
        r = subprocess.run([nvcc, '-shared', '-o', tmp_lib, *objs, '-lcudart'], stdout=subprocess.PIPE,
                           stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            raise RuntimeError('link failed:\n' + r.stdout)
        os.replace(tmp_lib, LIB)
    return LIB


if __name__ == '__main__':
    sys.path.insert(0, os.path.dirname(HERE))
    print(build(verbose='-v' in sys.argv) or 'reference tree not found at %s: nothing built' % REFERENCE_ROOT)
