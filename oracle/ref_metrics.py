"""TEST INFRASTRUCTURE.  The reference arm of the shape metrics: the reference's own CUDA kernels (approxmatch,
matchcost, nndistance; oracle/_ref/libref_structural.so, built by oracle/build_ref.py) driven the way reference
metrics/evaluation_metrics.py drives them:

  - nn_distance / match_cost: one call of the reference launchers per batch of pairs (the match matrix
    [B, m, n] and the scratch are allocated here, as pytorch_structural_losses does);
  - pairwise_emd_cd(a, b): `_pairwise_EMD_CD_` (:111-154): for each cloud a_i, b in batches of up to 256 clouds,
    a_i copied once per pair of the batch, CD = mean(dist1) + mean(dist2), EMD = match cost / N.

Used by tests/test_gpu_metrics.py and tools/bench_metrics.py; never by the product.
"""
from __future__ import annotations
import ctypes as C
import os
import torch

LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), '_ref', 'libref_structural.so')
_lib = None


class ReferenceLibraryMissing(RuntimeError):
    pass


def load():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ReferenceLibraryMissing(
                '%s is missing: __graft_entry__.build() compiles it from the reference checkout '
                '(oracle/build_ref.py, OCTFUSION_REFERENCE)' % LIB_PATH)
        lib = C.CDLL(LIB_PATH)
        vp, i = C.c_void_p, C.c_int
        lib.ref_approxmatch.argtypes = [i, i, i, vp, vp, vp, vp, vp]
        lib.ref_matchcost.argtypes = [i, i, i, vp, vp, vp, vp, vp]
        lib.ref_nndistance.argtypes = [i, i, vp, i, vp, vp, vp, vp, vp, vp]
        for f in (lib.ref_approxmatch, lib.ref_matchcost, lib.ref_nndistance):
            f.restype = i
        _lib = lib
    return _lib


def _p(t):
    return C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _check(rc, what):
    if rc != 0:
        raise RuntimeError('reference %s failed' % what)


@torch.no_grad()
def nn_distance(x, y):
    """(dist1 [B, n], dist2 [B, m]) from the reference nndistance"""
    lib = load()
    x, y = x.contiguous(), y.contiguous()
    b, n, m = x.shape[0], x.shape[1], y.shape[1]
    d1 = torch.empty(b, n, device=x.device)
    d2 = torch.empty(b, m, device=x.device)
    i1 = torch.empty(b, n, dtype=torch.int32, device=x.device)
    i2 = torch.empty(b, m, dtype=torch.int32, device=x.device)
    _check(lib.ref_nndistance(b, n, _p(x), m, _p(y), _p(d1), _p(i1), _p(d2), _p(i2), _stream()), 'nndistance')
    return d1, d2


@torch.no_grad()
def match_cost(x, y):
    """[B] un-normalised cost from the reference approxmatch + matchcost"""
    lib = load()
    x, y = x.contiguous(), y.contiguous()
    b, n, m = x.shape[0], x.shape[1], y.shape[1]
    match = torch.empty(b, m, n, device=x.device)
    temp = torch.empty(b, 2 * (n + m), device=x.device)
    out = torch.empty(b, device=x.device)
    _check(lib.ref_approxmatch(b, n, m, _p(x), _p(y), _p(match), _p(temp), _stream()), 'approxmatch')
    _check(lib.ref_matchcost(b, n, m, _p(x), _p(y), _p(match), _p(out), _stream()), 'matchcost')
    return out


@torch.no_grad()
def pairwise_emd_cd(a, b, batch_size=256, rows=None):
    """(cd [R, Nb], emd [R, Nb]) for the rows `rows` of a (all rows when None), as `_pairwise_EMD_CD_` computes them"""
    rows = range(a.shape[0]) if rows is None else rows
    all_cd, all_emd = [], []
    n = a.shape[1]
    for i in rows:
        cd_row, emd_row = [], []
        for j0 in range(0, b.shape[0], batch_size):
            bj = b[j0:j0 + batch_size]
            ai = a[i].view(1, -1, 3).expand(bj.shape[0], -1, -1).contiguous()
            d1, d2 = nn_distance(ai, bj)
            cd_row.append(d1.mean(dim=1) + d2.mean(dim=1))
            emd_row.append(match_cost(ai, bj) / float(n))
        all_cd.append(torch.cat(cd_row))
        all_emd.append(torch.cat(emd_row))
    return torch.stack(all_cd), torch.stack(all_emd)
