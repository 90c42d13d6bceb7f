"""TEST INFRASTRUCTURE -- restatement of the exact EMD of the OctFusion evaluation (reference
metrics/evaluation_metrics.py `emd_approx`, :35-52, which solves the fp32 distance matrix with scipy's
linear_sum_assignment) and of the integer problem csrc/emd_exact.cu solves in its place.  It is the checker for
csrc/emd_exact.cu and the exact arm of octfusion_b200.metrics; never shipped, never timed as the product (except as the
host `port` arm of tools/bench_emd_exact.py).

Pinning: tests/golden/metrics_emd_exact.npz (oracle/gen_golden_emd_exact.py) holds the unmodified reference's exact-arm
outputs on seeded inputs; tests/test_emd_exact_oracle.py compares against it.
"""
from __future__ import annotations
import math
import numpy as np
import torch
from scipy.optimize import linear_sum_assignment


def emd_exact(x, y):
    """[B] exact EMD of (x[i], y[i]) as reference `emd_approx` (metrics/evaluation_metrics.py:35-52) computes it: the
    distance matrix (x - y).norm(dim=-1) in the clouds' dtype, scipy's linear_sum_assignment on it, the mean of the
    matched distances"""
    assert x.shape[1] == y.shape[1]
    dist = (x[:, :, None, :] - y[:, None, :, :]).norm(dim=-1).cpu().numpy()
    out = []
    for d in dist:
        r, c = linear_sum_assignment(d)
        out.append(d[r, c].mean())
    return torch.from_numpy(np.stack(out).reshape(-1)).to(x)


def emd_exact_distances(x, y):
    """[n, n] fp32 distances of one pair as csrc/emd_exact.cu forms them: sqrt((dx*dx + dy*dy) + dz*dz) with every
    operation rounded to fp32 on its own (numpy does not contract)"""
    x, y = np.asarray(x, np.float32), np.asarray(y, np.float32)
    dx, dy, dz = (x[:, None, a] - y[None, :, a] for a in range(3))
    return np.sqrt((dx * dx + dy * dy) + dz * dz)


def emd_exact_exponent(x, y):
    """k of the cost quantum q = 2^(k - 24): the smallest power of two s = 2^k >= the diagonal of the joint bounding
    box of the pair (squared in fp64 as (ex*ex + ey*ey) + ez*ez from the fp32 extremes), at least 2^-100"""
    pts = np.concatenate([np.asarray(x, np.float32), np.asarray(y, np.float32)])
    e = pts.max(0).astype(np.float64) - pts.min(0).astype(np.float64)
    d2 = (e[0] * e[0] + e[1] * e[1]) + e[2] * e[2]
    if d2 == 0.0:
        return -100
    m, ex = math.frexp(d2)
    t = ex - 1 if m == 0.5 else ex                   # smallest t with 2^t >= d2
    return max(-100, -((-t) // 2))                   # ceil(t / 2)


def emd_exact_quantized(x, y):
    """per pair (emd, cstar, k) of the integer problem csrc/emd_exact.cu solves: c = rint(d / q) with q = 2^(k - 24),
    cstar = the optimal assignment cost of c (scipy, exact on integers below 2^53) and emd = fp32(cstar q / n) in fp64.
    emd is what the kernel returns bit for bit."""
    out = []
    for xi, yi in zip(np.asarray(x, np.float32), np.asarray(y, np.float32)):
        k = emd_exact_exponent(xi, yi)
        c = np.rint(emd_exact_distances(xi, yi).astype(np.float64) * 2.0 ** (24 - k)).astype(np.int64)
        r, col = linear_sum_assignment(c)
        cstar = int(c[r, col].sum())
        out.append((np.float32(math.ldexp(float(cstar), k - 24) / xi.shape[0]), cstar, k))
    return out
