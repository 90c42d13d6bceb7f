"""TEST INFRASTRUCTURE -- torch restatement of the shape metrics of the OctFusion evaluation (reference
metrics/evaluation_metrics.py and metrics/pytorch_structural_losses): nearest-neighbour distances, the approximate
EMD cost (float64 by default, vectorised per level), and the MMD / COV and k-NN reductions.  It is the checker for
csrc/metrics.cu and octfusion_b200.metrics; never shipped, never timed as the product.

Pinning: tests/golden/metrics.npz (oracle/gen_golden_metrics.py) holds the unmodified reference's outputs on seeded
inputs; tests/test_metrics_oracle.py compares against it.  All citations are file:line under the reference tree.
"""
from __future__ import annotations
import torch
def pc_sqdist(x, y):
    """[B, n, m] squared distances |y_l - x_k|^2 from coordinate differences (no |x|^2 + |y|^2 - 2xy expansion)"""
    return ((y[:, None, :, :] - x[:, :, None, :]) ** 2).sum(-1)


def nn_distance(x, y):
    """(dist1 [B, n], dist2 [B, m]): nearest-neighbour squared distances both ways (nndistance, distChamfer :11-21)"""
    d = pc_sqdist(x, y)
    return d.min(2).values, d.min(1).values


def approx_match_cost(x, y, dtype=torch.float64):
    """un-normalised approximate-EMD cost [B] of (xyz1 = x, xyz2 = y), n == m: the progressive matching of
    pytorch_structural_losses/src/approxmatch.cu (approxmatchkernel :3-182; levels -4^j for j = 7 .. -1, the j = -2
    branch is unreachable) followed by its cost (matchcostkernel :184-224), each level vectorised over all (k, l)."""
    x, y = x.to(dtype), y.to(dtype)
    d = pc_sqdist(x, y)                                   # [B, k, l]
    rem_l = torch.ones(x.shape[:2], dtype=dtype)
    rem_r = torch.ones(y.shape[:2], dtype=dtype)
    dist = d.sqrt()
    cost = torch.zeros(x.shape[0], dtype=dtype)
    for j in range(7, -2, -1):
        e = torch.exp(-(4.0 ** j) * d)
        ratio_l = rem_l / (1e-9 + (e * rem_r[:, None, :]).sum(2))
        sum_r = (e * ratio_l[:, :, None]).sum(1) * rem_r
        ratio_r = torch.clamp(rem_r / (sum_r + 1e-9), max=1.0) * rem_r
        rem_r = torch.clamp(rem_r - sum_r, min=0.0)
        w = e * ratio_l[:, :, None] * ratio_r[:, None, :]
        rem_l = torch.clamp(rem_l - w.sum(2), min=0.0)
        cost = cost + (w * dist).sum((1, 2))
    return cost


def lgan_mmd_cov(all_dist):
    """lgan_mmd_cov (metrics/evaluation_metrics.py:189-201) of a [N_sample, N_ref] matrix"""
    smp_min, nearest_ref = torch.min(all_dist, dim=1)
    ref_min = torch.min(all_dist, dim=0).values
    cov = torch.tensor(float(nearest_ref.unique().numel()) / float(all_dist.shape[1])).to(all_dist)
    return {'lgan_mmd': ref_min.mean(), 'lgan_cov': cov, 'lgan_mmd_smp': smp_min.mean()}


def knn(Mxx, Mxy, Myy, k, sqrt=False):
    """knn (metrics/evaluation_metrics.py:157-186): k-NN two-sample classifier over x (label 1) then y (label 0),
    each point's own entry excluded; a point is predicted x when at least k/2 of its k nearest points are x.
    Neighbours come from a stable sort of each column of the joint matrix."""
    n0, n1 = Mxx.shape[0], Myy.shape[0]
    is_x = torch.arange(n0 + n1) < n0
    joint = torch.vstack([torch.hstack([Mxx, Mxy]), torch.hstack([Mxy.T, Myy])]).clone()
    if sqrt:
        joint = joint.abs().sqrt()
    joint.fill_diagonal_(float('inf'))
    neighbours = torch.argsort(joint, dim=0, stable=True)[:k]
    pred_x = 2 * is_x.to(joint.device)[neighbours].sum(0) >= k
    label, pred = is_x.to(Mxx), pred_x.to(Mxx)
    tp, tn = (label * pred).sum(), ((1 - label) * (1 - pred)).sum()
    fp, fn = ((1 - label) * pred).sum(), (label * (1 - pred)).sum()
    return {'tp': tp, 'fp': fp, 'fn': fn, 'tn': tn,
            'precision': tp / (tp + fp + 1e-10), 'recall': tp / (tp + fn + 1e-10),
            'acc_t': tp / (tp + fn + 1e-10), 'acc_f': tn / (tn + fp + 1e-10),
            'acc': (is_x.to(joint.device) == pred_x).float().mean()}
