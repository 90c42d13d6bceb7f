"""Point-cloud shape metrics of the OctFusion evaluation on the GPU: MMD, COV and 1-NNA with Chamfer distance (CD)
and EMD, approximate (the default) or exact (`accelerated_emd=False`).

Drop-in for reference metrics/evaluation_metrics.py (and the `nn_distance` / `match_cost` functions of
metrics/pytorch_structural_losses): the names, argument order, orientation and dict keys are the reference's, so its
callers can swap modules.  The all-pairs distance matrices, the O(N^2 P^2) part, are computed by the kernels of
csrc/metrics.cu and csrc/emd_exact.cu, one launch per matrix; the O(N^2) reductions over finished matrices (min,
unique, top-k) are torch ops on the device.

Inputs are contiguous fp32 CUDA tensors [N, P, 3]; anything else raises (there is no CPU path).  `batch_size`
arguments are accepted for signature compatibility and ignored: every matrix is computed in one launch without
copying any cloud.  Results carry no gradient.

The reference has two EMDs.  `accelerated_emd=True` (the default everywhere here) is the approximate match cost of
pytorch_structural_losses (`emd_approx_cuda`).  `accelerated_emd=False` is the exact EMD that the reference's
`emd_approx` computes with scipy's linear_sum_assignment, and that its metrics fall back to when the structural-loss
extension is not importable; CD is the same in both arms.  The exact EMD is the optimal assignment cost of distances
quantised to q = 2^-24 times the pair's bounding-box scale (include/octfusion_b200.h, of_emd_exact): within q/2 of
the optimum of the fp32 distance matrix, and bit-reproducible.
"""
from __future__ import annotations
import torch

from ._lib import lib, ptr, stream, check, EMD_MAX_POINTS, CD_PAIRWISE_MAX_POINTS

__all__ = ['nn_distance', 'match_cost', 'paired_emd_cd', 'emd_approx', 'emd_exact', 'pairwise_emd_exact', 'EMD_CD',
           'pairwise_cd', 'pairwise_emd_cd', 'lgan_mmd_cov', 'knn', 'compute_cov_mmd', 'compute_1_nna', 'compute_all_metrics']


def _clouds(x, name):
    if not isinstance(x, torch.Tensor) or not x.is_cuda:
        raise RuntimeError('octfusion_b200.metrics: %s must be a CUDA tensor -- there is no CPU path' % name)
    if x.dtype != torch.float32:
        raise TypeError('octfusion_b200.metrics: %s must be float32, got %s' % (name, x.dtype))
    if x.dim() != 3 or x.shape[2] != 3 or x.shape[1] < 1:
        raise ValueError('octfusion_b200.metrics: %s must have shape [N, P >= 1, 3], got %s' % (name, tuple(x.shape)))
    if not x.is_contiguous():
        raise ValueError('octfusion_b200.metrics: %s must be contiguous' % name)
    return x


def _same_device(x, y):
    if x.device != y.device:
        raise ValueError('octfusion_b200.metrics: clouds on %s and %s' % (x.device, y.device))
    torch.cuda.set_device(x.device)


def _equal_sizes(x, y, what='approximate EMD'):
    n = x.shape[1]
    if y.shape[1] != n:
        raise ValueError('octfusion_b200.metrics: %s needs clouds of equal size, got %d and %d' % (what, n, y.shape[1]))
    if n > EMD_MAX_POINTS:
        raise ValueError('octfusion_b200.metrics: %s supports up to %d points per cloud, got %d'
                         % (what, EMD_MAX_POINTS, n))
    return n


@torch.no_grad()
def nn_distance(x, y):
    """(dist1 [B, P], dist2 [B, Q]): squared distance of every point of x[i] to its nearest point of y[i] and back
    (reference pytorch_structural_losses/nn_distance.py, `distChamferCUDA`)."""
    _clouds(x, 'x'); _clouds(y, 'y'); _same_device(x, y)
    if x.shape[0] != y.shape[0]:
        raise ValueError('octfusion_b200.metrics: batch sizes differ (%d, %d)' % (x.shape[0], y.shape[0]))
    b, p, q = x.shape[0], x.shape[1], y.shape[1]
    d1 = torch.empty(b, p, device=x.device)
    d2 = torch.empty(b, q, device=x.device)
    check(lib.of_nn_distance(ptr(x), ptr(y), b, p, q, ptr(d1), ptr(d2), None, stream()), 'nn_distance')
    return d1, d2


def _paired_emd(x, y, want_cd):
    _clouds(x, 'x'); _clouds(y, 'y'); _same_device(x, y)
    if x.shape[0] != y.shape[0]:
        raise ValueError('octfusion_b200.metrics: batch sizes differ (%d, %d)' % (x.shape[0], y.shape[0]))
    n = _equal_sizes(x, y)
    cost = torch.empty(x.shape[0], device=x.device)
    cd = torch.empty(x.shape[0], device=x.device) if want_cd else None
    check(lib.of_match_cost(ptr(x), ptr(y), x.shape[0], n, ptr(cost), ptr(cd), stream()), 'match_cost')
    return cost, cd


@torch.no_grad()
def match_cost(x, y):
    """[B] un-normalised approximate-EMD cost of (x[i], y[i]) (reference pytorch_structural_losses/match_cost.py;
    `emd_approx_cuda` divides it by the number of points)."""
    return _paired_emd(x, y, False)[0]


@torch.no_grad()
def paired_emd_cd(x, y):
    """(cd [B], emd [B]) of the pairs (x[i], y[i]) from one launch: the values pairwise_emd_cd stores for a pair."""
    cost, cd = _paired_emd(x, y, True)
    return cd, cost / x.shape[1]


_EXACT_FAILURES = {1: (RuntimeError, 'the auction reached its round cap (a solver defect; please report the input)'),
                   2: (ValueError, 'a coordinate is not finite'),
                   3: (ValueError, 'the bounding-box diagonal exceeds 2^62, beyond fp32 squared distances')}


def _check_exact(status, what):
    """raise on the first failed pair; reading the statuses is the call's one host synchronisation"""
    code = status.cpu() & 15
    if code.any():
        idx = tuple(int(i) for i in torch.nonzero(code)[0])
        exc, why = _EXACT_FAILURES.get(int(code[idx]), (RuntimeError, 'status %d' % int(code[idx])))
        raise exc('octfusion_b200.metrics: %s: pair %s: %s' % (what, idx[0] if len(idx) == 1 else idx, why))


@torch.no_grad()
def emd_exact(x, y, details=False):
    """[B] exact EMD of (x[i], y[i]): the mean matched distance of an optimal assignment (of_emd_exact).  With
    details=True returns (emd, gap, status): gap [B] int64 is the primal-dual gap of the final auction prices
    (0 <= gap <= n certifies optimality), status [B] int32 the solver's status word (bits 4-7 phases, 8-31 rounds)."""
    _clouds(x, 'x'); _clouds(y, 'y'); _same_device(x, y)
    if x.shape[0] != y.shape[0]:
        raise ValueError('octfusion_b200.metrics: batch sizes differ (%d, %d)' % (x.shape[0], y.shape[0]))
    n = _equal_sizes(x, y, 'exact EMD')
    b = x.shape[0]
    emd = torch.empty(b, device=x.device)
    gap = torch.empty(b, dtype=torch.int64, device=x.device)
    status = torch.zeros(b, dtype=torch.int32, device=x.device)
    check(lib.of_emd_exact(ptr(x), ptr(y), b, n, ptr(emd), ptr(gap), ptr(status), stream()), 'emd_exact')
    _check_exact(status, 'emd_exact')
    return (emd, gap, status) if details else emd


@torch.no_grad()
def emd_approx(x, y):
    """[B] exact EMD of (x[i], y[i]) under the reference's name: reference `emd_approx`, despite the name, solves the
    distance matrix exactly (metrics/evaluation_metrics.py:35-52)."""
    return emd_exact(x, y)


@torch.no_grad()
def pairwise_emd_exact(a, b, details=False):
    """emd [Na, Nb]: exact EMD of every pair (a[i], b[j]), each entry equal to emd_exact of the pair.  When `a is b`
    only i < j is solved and mirrored (the exact EMD is symmetric bit for bit) and the diagonal is 0.  details=True
    returns (emd, gap, status) as emd_exact does."""
    _clouds(a, 'a'); _clouds(b, 'b'); _same_device(a, b)
    n = _equal_sizes(a, b, 'exact EMD')
    emd = torch.empty(a.shape[0], b.shape[0], device=a.device)
    gap = torch.empty(a.shape[0], b.shape[0], dtype=torch.int64, device=a.device)
    status = torch.zeros(a.shape[0], b.shape[0], dtype=torch.int32, device=a.device)
    check(lib.of_emd_exact_pairwise(ptr(a), a.shape[0], ptr(b), b.shape[0], n, 1 if a is b else 0, ptr(emd), ptr(gap),
                                    ptr(status), stream()), 'pairwise_emd_exact')
    _check_exact(status, 'pairwise_emd_exact')
    return (emd, gap, status) if details else emd


@torch.no_grad()
def EMD_CD(sample_pcs, ref_pcs, batch_size=None, reduced=True, accelerated_emd=True):
    """{'MMD-CD', 'MMD-EMD'} of the matched pairs (sample_pcs[i], ref_pcs[i]) (reference EMD_CD).  accelerated_emd
    selects the approximate EMD (True, fused with the CD) or the exact one (False, CD from nn_distance)."""
    if sample_pcs.shape[0] != ref_pcs.shape[0]:
        raise ValueError('octfusion_b200.metrics: REF:%d SMP:%d' % (ref_pcs.shape[0], sample_pcs.shape[0]))
    if accelerated_emd:
        cd, emd = paired_emd_cd(sample_pcs, ref_pcs)
    else:
        emd = emd_exact(sample_pcs, ref_pcs)
        cd = torch.empty_like(emd)
        d1 = torch.empty(sample_pcs.shape[:2], device=emd.device)
        d2 = torch.empty(ref_pcs.shape[:2], device=emd.device)
        check(lib.of_nn_distance(ptr(sample_pcs), ptr(ref_pcs), sample_pcs.shape[0], sample_pcs.shape[1],
                                 ref_pcs.shape[1], ptr(d1), ptr(d2), ptr(cd), stream()), 'EMD_CD')
    if reduced:
        cd, emd = cd.mean(), emd.mean()
    return {'MMD-CD': cd, 'MMD-EMD': emd}


@torch.no_grad()
def pairwise_cd(a, b, batch_size=None):
    """cd [Na, Nb]: Chamfer distance of every pair (a[i], b[j]) (the CD half of pairwise_emd_cd, for any P, Q)."""
    _clouds(a, 'a'); _clouds(b, 'b'); _same_device(a, b)
    if a.shape[1] + b.shape[1] > CD_PAIRWISE_MAX_POINTS:
        raise ValueError('octfusion_b200.metrics: pairwise CD supports P + Q <= %d' % CD_PAIRWISE_MAX_POINTS)
    cd = torch.empty(a.shape[0], b.shape[0], device=a.device)
    check(lib.of_chamfer_pairwise(ptr(a), a.shape[0], a.shape[1], ptr(b), b.shape[0], b.shape[1], ptr(cd), stream()),
          'pairwise_cd')
    return cd


@torch.no_grad()
def pairwise_emd_cd(a, b, batch_size=None, accelerated_emd=True):
    """(cd [Na, Nb], emd [Na, Nb]) of every pair with a[i] as the first cloud (reference `_pairwise_EMD_CD_`).
    Approximate EMD is not symmetric: a matrix of a set against itself is computed in full, not mirrored.  With
    accelerated_emd=False the EMD is exact (pairwise_emd_exact, mirrored when `a is b`) and CD is pairwise_cd."""
    if not accelerated_emd:
        return pairwise_cd(a, b), pairwise_emd_exact(a, b)
    _clouds(a, 'a'); _clouds(b, 'b'); _same_device(a, b)
    n = _equal_sizes(a, b)
    cost = torch.empty(a.shape[0], b.shape[0], device=a.device)
    cd = torch.empty_like(cost)
    check(lib.of_emd_cd_pairwise(ptr(a), a.shape[0], ptr(b), b.shape[0], n, ptr(cost), ptr(cd), stream()),
          'pairwise_emd_cd')
    return cd, cost / n


@torch.no_grad()
def lgan_mmd_cov(all_dist):
    """MMD and COV of a [N_sample, N_ref] distance matrix: lgan_mmd = mean over references of the distance to the
    closest sample, lgan_mmd_smp = mean over samples of the distance to the closest reference, lgan_cov = share of
    references that are the closest reference of at least one sample."""
    n_ref = all_dist.shape[1]
    closest_ref_dist, closest_ref = all_dist.min(dim=1)
    closest_smp_dist = all_dist.min(dim=0).values
    covered = closest_ref.unique().numel()
    return {'lgan_mmd': closest_smp_dist.mean(),
            'lgan_cov': torch.tensor(float(covered) / float(n_ref)).to(all_dist),
            'lgan_mmd_smp': closest_ref_dist.mean()}


@torch.no_grad()
def knn(Mxx, Mxy, Myy, k, sqrt=False):
    """k-nearest-neighbour two-sample classifier over the joint set x (label 1) + y (label 0): each point is
    predicted 1 when at least k/2 of its k nearest other points are x.  Returns tp/fp/fn/tn, precision, recall and
    the accuracies acc_t (on x), acc_f (on y) and acc (all) as device tensors."""
    n0, n1 = Mxx.shape[0], Myy.shape[0]
    label = torch.cat((torch.ones(n0), torch.zeros(n1))).to(Mxx)
    dist = torch.cat((torch.cat((Mxx, Mxy), 1), torch.cat((Mxy.t(), Myy), 1)), 0)
    if sqrt:
        dist = dist.abs().sqrt()
    dist = dist + torch.diag(torch.full((n0 + n1,), float('inf'), dtype=dist.dtype, device=dist.device))
    nearest = dist.topk(k, 0, False).indices                  # [k, n0 + n1]: neighbours of each column
    votes = label[nearest].sum(0)
    pred = (votes >= float(k) / 2).to(label.dtype)
    tp, fp = (pred * label).sum(), (pred * (1 - label)).sum()
    fn, tn = ((1 - pred) * label).sum(), ((1 - pred) * (1 - label)).sum()
    return {'tp': tp, 'fp': fp, 'fn': fn, 'tn': tn,
            'precision': tp / (tp + fp + 1e-10), 'recall': tp / (tp + fn + 1e-10),
            'acc_t': tp / (tp + fn + 1e-10), 'acc_f': tn / (tn + fp + 1e-10),
            'acc': (label == pred).float().mean()}


def _cov_mmd(m_rs_cd, m_rs_emd):
    out = {}
    for metric, m in (('CD', m_rs_cd), ('EMD', m_rs_emd)):
        out.update({'%s-%s' % (k, metric): v for k, v in lgan_mmd_cov(m.t()).items()})
    return out


def _one_nna(m_rs, m_rr, m_ss):
    out = {}
    for metric, i in (('CD', 0), ('EMD', 1)):
        res = knn(m_rr[i], m_rs[i], m_ss[i], 1, sqrt=False)
        out.update({'1-NN-%s-%s' % (metric, k): v for k, v in res.items() if 'acc' in k})
    return out


@torch.no_grad()
def compute_cov_mmd(sample_pcs, ref_pcs, batch_size=None, accelerated_emd=True):
    """lgan_mmd / lgan_cov / lgan_mmd_smp with CD and EMD; the matrix is reference x sample, transposed to
    [N_sample, N_ref] (reference compute_cov_mmd).  accelerated_emd=False: exact EMD."""
    return _cov_mmd(*pairwise_emd_cd(ref_pcs, sample_pcs, accelerated_emd=accelerated_emd))


@torch.no_grad()
def compute_1_nna(sample_pcs, ref_pcs, batch_size=None, accelerated_emd=True):
    """1-NN-{CD,EMD}-{acc_t,acc_f,acc} (reference compute_1_nna).  accelerated_emd=False: exact EMD."""
    return _one_nna(pairwise_emd_cd(ref_pcs, sample_pcs, accelerated_emd=accelerated_emd),
                    pairwise_emd_cd(ref_pcs, ref_pcs, accelerated_emd=accelerated_emd),
                    pairwise_emd_cd(sample_pcs, sample_pcs, accelerated_emd=accelerated_emd))


@torch.no_grad()
def compute_all_metrics(sample_pcs, ref_pcs, batch_size=None, accelerated_emd=True):
    """compute_cov_mmd and compute_1_nna in one call; the reference x sample matrices are computed once.
    accelerated_emd=False: exact EMD."""
    m_rs = pairwise_emd_cd(ref_pcs, sample_pcs, accelerated_emd=accelerated_emd)
    out = _cov_mmd(*m_rs)
    out.update(_one_nna(m_rs, pairwise_emd_cd(ref_pcs, ref_pcs, accelerated_emd=accelerated_emd),
                        pairwise_emd_cd(sample_pcs, sample_pcs, accelerated_emd=accelerated_emd)))
    return out
