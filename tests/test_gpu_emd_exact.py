"""GPU tests (-m gpu) of the exact EMD (csrc/emd_exact.cu, octfusion_b200.metrics emd_exact / emd_approx /
accelerated_emd=False): bit for bit against the restated integer problem (oracle/restate_emd_exact.py
emd_exact_quantized, scipy on the same quantised costs), within the stated bound of the reference's fp32 scipy arm and
of its fixtures (tests/golden/metrics_emd_exact.npz), a certified gap <= n on every pair, and the argument checks."""
import os
import numpy as np
import pytest
import torch

from oracle import restate_emd_exact as R
from tests.test_emd_exact_oracle import emd_bound
from tests.util import GOLDEN

pytestmark = pytest.mark.gpu

CD_RTOL = 1e-6       # as tests/test_gpu_metrics.py: the per-point minima agree, the mean's order differs


@pytest.fixture(scope='module')
def M():
    from octfusion_b200 import metrics
    return metrics


def clouds(n, points, seed):
    from octfusion_b200.synth import synth_point_clouds
    return synth_point_clouds(n, points, seed).cuda()


def solve(M, x, y):
    """(emd, gap, status) of the pairs, with the certificate checked: 0 <= gap <= n, status 0"""
    emd, gap, status = M.emd_exact(x, y, details=True)
    n = x.shape[1]
    assert ((status & 15) == 0).all()
    assert (gap >= 0).all() and (gap <= n).all(), gap
    return emd, gap, status


def check_against_oracles(emd, x, y, ref=None):
    """bit for bit against the quantised restatement; within emd_bound of the reference's fp32 arm (or `ref`)"""
    xc, yc = x.cpu(), y.cpu()
    want = R.emd_exact_quantized(xc, yc)
    ref = R.emd_exact(xc, yc).numpy() if ref is None else ref
    for i, (e, _, k) in enumerate(want):
        got = emd[i].cpu().numpy()
        assert got.tobytes() == e.tobytes(), (i, float(got), float(e))
        max_d = float(R.emd_exact_distances(xc[i], yc[i]).max())
        assert abs(float(got) - float(ref[i])) <= emd_bound(float(ref[i]), max_d, k), (i, float(got), float(ref[i]))


@pytest.mark.parametrize('n', [1, 2, 3, 17, 128, 1000, 2048, 4096])
def test_exact_emd_against_scipy(M, n):
    x, y = clouds(2 if n >= 2048 else 4, n, 30 + n), clouds(2 if n >= 2048 else 4, n, 31 + n)
    emd, _, _ = solve(M, x, y)
    check_against_oracles(emd, x, y)
    assert torch.equal(M.emd_approx(x, y), emd)


@pytest.fixture(scope='module')
def golden():
    from oracle.gen_golden_emd_exact import emd_exact_inputs
    g = np.load(os.path.join(GOLDEN, 'metrics_emd_exact.npz'))
    return g, {k: v.cuda() for k, v in emd_exact_inputs().items()}


@pytest.mark.parametrize('n', [1, 2, 3, 17, 128, 1000, 2048, 4096])
def test_exact_emd_against_reference_fixtures(M, golden, n):
    g, inp = golden
    x, y = inp['x%d' % n], inp['y%d' % n]
    emd, _, _ = solve(M, x, y)
    check_against_oracles(emd, x, y, ref=g['emd%d' % n])


def test_known_answers(M):
    x = clouds(1, 2048, 40)
    perm = torch.randperm(2048, generator=torch.Generator().manual_seed(41)).cuda()
    emd, gap, _ = solve(M, x, x[:, perm].contiguous())
    assert float(emd) == 0.0 and int(gap) == 0
    t = torch.tensor([0.3, -0.2, 0.1], device='cuda')
    y = (x + t).contiguous()
    emd, _, _ = solve(M, x, y)
    check_against_oracles(emd, x, y, ref=[float(t.norm())])
    g = torch.Generator().manual_seed(42)
    a, b = torch.rand(1000, generator=g), torch.rand(1000, generator=g) * 2
    xa = torch.stack([a, torch.zeros_like(a), torch.zeros_like(a)], -1)[None].contiguous().cuda()
    xb = torch.stack([b, torch.zeros_like(b), torch.zeros_like(b)], -1)[None].contiguous().cuda()
    want = float((a.sort().values.double() - b.sort().values.double()).abs().mean())
    emd, _, _ = solve(M, xa, xb)
    check_against_oracles(emd, xa, xb, ref=[want])


def test_degenerate_inputs_finish(M):
    n = 1024
    x = clouds(1, n, 50)
    same = torch.full((1, n, 3), 0.25, device='cuda')
    dup = x[:, :16].repeat(1, n // 16, 1).contiguous()                  # 64 copies of each of 16 points
    g = torch.Generator().manual_seed(51)
    far = torch.rand(1, n, 3, generator=g)
    far[:, n // 2:] += 1000.0                                            # two clusters 1000 apart
    far2 = torch.rand(1, n, 3, generator=g)
    far2[:, : n // 4] += 1000.0
    cases = [(same, same), (same, x), (dup, x), (x, dup), (dup, dup.flip(1).contiguous()),
             (far.cuda(), far2.cuda())]
    for u, v in cases:
        emd, _, _ = solve(M, u, v)
        check_against_oracles(emd, u, v)
    assert float(solve(M, same, same)[0]) == 0.0


def test_pairwise_equals_paired_and_symmetric_mode(M):
    a, b = clouds(12, 512, 60), clouds(9, 512, 61)
    emd, gap, status = M.pairwise_emd_exact(a, b, details=True)
    assert ((status & 15) == 0).all() and (gap >= 0).all() and (gap <= 512).all()
    pe, pg, ps = solve(M, a.repeat_interleave(9, 0).contiguous(), b.repeat(12, 1, 1).contiguous())
    assert torch.equal(pe.view(12, 9), emd) and torch.equal(pg.view(12, 9), gap) and torch.equal(ps.view(12, 9), status)
    sym, sgap, sstat = M.pairwise_emd_exact(a, a, details=True)          # `a is a`: i < j solved and mirrored
    assert torch.equal(sym, sym.t()) and not sym.diagonal().any()
    assert ((sstat & 15) == 0).all() and (sgap >= 0).all() and (sgap <= 512).all()
    full = M.pairwise_emd_exact(a, a.clone())                           # every pair solved in both orders
    assert torch.equal(full, sym)


def test_two_runs_are_identical(M):
    a, b = clouds(6, 2048, 70), clouds(6, 2048, 71)
    r1, r2 = M.emd_exact(a, b, details=True), M.emd_exact(a, b, details=True)
    assert all(torch.equal(u, v) for u, v in zip(r1, r2))
    assert torch.equal(M.pairwise_emd_exact(a, a), M.pairwise_emd_exact(a, a))


def test_exact_arm_of_emd_cd_cov_mmd_1nna_equals_reference_fixtures(M, golden):
    g, inp = golden
    smp, rfc = inp['smp'], inp['ref']
    per_pair = M.EMD_CD(smp, rfc, 3, reduced=False, accelerated_emd=False)
    np.testing.assert_allclose(per_pair['MMD-CD'].cpu().numpy(), g['emd_cd_pairs_MMD-CD'], rtol=CD_RTOL, atol=0)
    check_against_oracles(per_pair['MMD-EMD'], smp, rfc, ref=g['emd_cd_pairs_MMD-EMD'])
    reduced = M.EMD_CD(smp, rfc, 3, accelerated_emd=False)
    assert float(reduced['MMD-CD']) == pytest.approx(float(g['emd_cd_MMD-CD']), rel=CD_RTOL)
    assert float(reduced['MMD-EMD']) == pytest.approx(float(g['emd_cd_MMD-EMD']), rel=1e-5)
    # the matrices of compute_1_nna, entry by entry
    for tag, a, b in (('rs', rfc, smp), ('rr', rfc, rfc), ('ss', smp, smp)):
        cd, emd = M.pairwise_emd_cd(a, b, accelerated_emd=False)
        np.testing.assert_allclose(cd.cpu().numpy(), g['m_%s_cd' % tag], rtol=CD_RTOL, atol=0)
        ref = g['m_%s_emd' % tag]
        for i in range(a.shape[0]):
            for j in range(b.shape[0]):
                k = R.emd_exact_exponent(a[i].cpu().numpy(), b[j].cpu().numpy())
                assert abs(float(emd[i, j]) - float(ref[i, j])) <= emd_bound(float(ref[i, j]), 2.0, k), (tag, i, j)
    got = M.compute_all_metrics(smp, rfc, accelerated_emd=False)
    split = dict(M.compute_cov_mmd(smp, rfc, accelerated_emd=False))
    split.update(M.compute_1_nna(smp, rfc, accelerated_emd=False))
    assert all(torch.equal(got[k], split[k]) for k in got)
    for k, v in got.items():
        want = float(g[('cov_mmd_' if k.startswith('lgan') else '1nna_') + k])
        if 'mmd' in k:
            assert float(v) == pytest.approx(want, rel=1e-5), k
        else:
            assert float(v) == want, k                                 # COV and 1-NNA accuracies: counts


def test_default_arm_is_unchanged(M):
    smp, rfc = clouds(6, 256, 80), clouds(6, 256, 81)
    cd, emd = M.pairwise_emd_cd(rfc, smp)
    cd2, emd2 = M.pairwise_emd_cd(rfc, smp, accelerated_emd=True)
    assert torch.equal(cd, cd2) and torch.equal(emd, emd2)
    exact = M.pairwise_emd_cd(rfc, smp, accelerated_emd=False)[1]
    assert not torch.equal(exact, emd)                                  # a different quantity


def test_bad_inputs_are_rejected(M):
    from octfusion_b200 import _lib
    x = clouds(2, 64, 90)
    with pytest.raises(ValueError, match='equal size'):
        M.emd_exact(x, clouds(2, 65, 91))
    big = torch.zeros(1, _lib.EMD_MAX_POINTS + 1, 3, device='cuda')
    n0 = _lib.launch_count()
    with pytest.raises(ValueError, match='up to'):
        M.emd_exact(big, big)
    assert _lib.launch_count() == n0
    bad = x.clone()
    bad[1, 7, 2] = float('nan')
    with pytest.raises(ValueError, match='pair 1: a coordinate is not finite'):
        M.emd_exact(x, bad)
    bad[1, 7, 2] = float('inf')
    with pytest.raises(ValueError, match=r'pair \(1, 0\): a coordinate is not finite'):
        M.pairwise_emd_exact(bad, x)
    with pytest.raises(TypeError):
        M.emd_exact(x.double(), x.double())
    with pytest.raises(RuntimeError, match='no CPU path'):
        M.emd_exact(x.cpu(), x.cpu())
