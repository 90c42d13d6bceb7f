"""GPU tests (-m gpu) of the shape-metric kernels (csrc/metrics.cu, octfusion_b200.metrics) against the reference's
own CUDA kernels (approxmatch, matchcost, nndistance) compiled into oracle/_ref by __graft_entry__.build(), driven as
reference metrics/evaluation_metrics.py drives them (oracle/ref_metrics.py), and against the restated MMD / COV /
1-NNA reductions (oracle/restate_metrics.py)."""
import os
import pytest
import torch

from oracle import restate_metrics as R

pytestmark = pytest.mark.gpu

CD_RTOL = 1e-6       # per-point distances are bit-identical; only the order of the 2 x P-term mean differs
EMD_RTOL = 1e-4      # same matching; the cost is summed per level instead of through a match matrix


@pytest.fixture(scope='module')
def ref():
    from oracle import ref_metrics
    assert os.path.exists(ref_metrics.LIB_PATH), (
        'the reference kernel library %s is missing: run __graft_entry__.build() on a host with the reference '
        'checkout (OCTFUSION_REFERENCE) to compile it' % ref_metrics.LIB_PATH)
    ref_metrics.load()
    return ref_metrics


@pytest.fixture(scope='module')
def M():
    from octfusion_b200 import metrics
    return metrics


def clouds(n, points, seed):
    from octfusion_b200.synth import synth_point_clouds
    return synth_point_clouds(n, points, seed).cuda()


def max_relerr(a, b):
    return float(((a.double() - b.double()).abs() / b.double().abs().clamp_min(1e-30)).max())


def test_reference_library_is_built(ref):
    assert os.path.getsize(ref.LIB_PATH) > 0


@pytest.mark.parametrize('b,p,q', [(4, 2048, 2048), (3, 1000, 1537), (2, 5000, 300), (2, 1, 7)])
def test_nn_distance_bit_identical_to_reference(ref, M, b, p, q):
    x, y = clouds(b, p, 1), clouds(b, q, 2)
    d1, d2 = M.nn_distance(x, y)
    r1, r2 = ref.nn_distance(x, y)
    assert torch.equal(d1, r1) and torch.equal(d2, r2)


@pytest.mark.parametrize('n', [1, 17, 1000, 2048, 4096])
def test_match_cost_matches_reference(ref, M, n):
    x, y = clouds(3, n, 3), clouds(3, n, 4)
    got, want = M.match_cost(x, y), ref.match_cost(x, y)
    assert max_relerr(got, want) <= EMD_RTOL, (got, want)


def test_match_cost_above_the_limit_is_an_error(M):
    from octfusion_b200 import _lib
    n = _lib.EMD_MAX_POINTS + 1
    x = torch.zeros(1, n, 3, device='cuda')
    cost = torch.empty(1, device='cuda')
    n0 = _lib.launch_count()
    assert _lib.lib.of_match_cost(_lib.ptr(x), _lib.ptr(x), 1, n, _lib.ptr(cost), None, _lib.stream()) == -1
    assert _lib.launch_count() == n0
    with pytest.raises(ValueError):
        M.match_cost(x, x)


@pytest.fixture(scope='module')
def pairwise(ref, M):
    a, b = clouds(40, 2048, 5), clouds(48, 2048, 6)
    cd, emd = M.pairwise_emd_cd(a, b)
    rcd, remd = ref.pairwise_emd_cd(a, b)
    return a, b, cd, emd, rcd, remd


def test_pairwise_emd_cd_matches_reference(pairwise):
    _, _, cd, emd, rcd, remd = pairwise
    assert cd.shape == (40, 48) and emd.shape == (40, 48)
    assert max_relerr(cd, rcd) <= CD_RTOL
    assert max_relerr(emd, remd) <= EMD_RTOL


def test_pairwise_entries_equal_paired_mode_and_repeat(M, pairwise):
    a, b, cd, emd = pairwise[:4]
    na, nb = a.shape[0], b.shape[0]
    pcd, pemd = M.paired_emd_cd(a.repeat_interleave(nb, 0).contiguous(), b.repeat(na, 1, 1).contiguous())
    assert torch.equal(pcd.view(na, nb), cd) and torch.equal(pemd.view(na, nb), emd)
    cd2, emd2 = M.pairwise_emd_cd(a, b)
    assert torch.equal(cd2, cd) and torch.equal(emd2, emd)
    # the Chamfer-only kernel: same per-point minima, its own fixed summation order
    assert max_relerr(M.pairwise_cd(a, b), cd) <= CD_RTOL
    assert torch.equal(M.pairwise_cd(a, b), M.pairwise_cd(a, b))


def test_lgan_mmd_cov_and_knn_equal_restatement_on_identical_matrices(M):
    g = torch.Generator().manual_seed(8)
    m = torch.rand(30, 25, generator=g)
    m[3] = m[7]                                       # exact ties: both sides must break them alike
    got, want = M.lgan_mmd_cov(m.cuda()), R.lgan_mmd_cov(m)
    assert list(got) == ['lgan_mmd', 'lgan_cov', 'lgan_mmd_smp']
    assert float(got['lgan_cov']) == float(want['lgan_cov'])
    for k in ('lgan_mmd', 'lgan_mmd_smp'):
        assert float(got[k]) == pytest.approx(float(want[k]), rel=1e-6)
    mxx, myy, mxy = torch.rand(20, 20, generator=g), torch.rand(16, 16, generator=g), torch.rand(20, 16, generator=g)
    got = M.knn(mxx.cuda(), mxy.cuda(), myy.cuda(), 1)
    want = R.knn(mxx, mxy, myy, 1)
    for k in ('tp', 'fp', 'fn', 'tn', 'acc_t', 'acc_f', 'acc'):
        assert float(got[k]) == float(want[k]), k


def _argmin_disagreements_are_ties(m_got, m_ref, dim, rtol):
    """where the nearest neighbour chosen from the product's matrix differs from the one chosen from the oracle's,
    the oracle's distances to the two candidates are within rtol: a near-tie (two entries within the metric's
    tolerance each can swap order when both are off by it, hence 2 x tolerance at the call sites)"""
    i_got, i_ref = m_got.argmin(dim), m_ref.argmin(dim)
    v_got = m_ref.gather(dim, i_got.unsqueeze(dim)).squeeze(dim)
    v_ref = m_ref.gather(dim, i_ref.unsqueeze(dim)).squeeze(dim)
    differ = i_got != i_ref
    assert ((v_got[differ] - v_ref[differ]).abs() <= rtol * v_ref[differ].abs()).all()
    return bool(differ.any())


def _joint(m_rr, m_rs, m_ss):
    j = torch.cat((torch.cat((m_rr, m_rs), 1), torch.cat((m_rs.t(), m_ss), 1)), 0)
    return j + torch.diag(torch.full((j.shape[0],), float('inf'), device=j.device))


def test_cov_mmd_1nna_end_to_end(ref, M):
    smp, rfc = clouds(24, 512, 10), clouds(20, 512, 11)
    # a few samples close to references, so that COV and 1-NNA are not trivial
    smp[:6] = (rfc[:6] + 0.004 * torch.randn(6, 512, 3, generator=torch.Generator().manual_seed(12)).cuda()).contiguous()
    got = M.compute_all_metrics(smp, rfc)
    assert list(got) == ['lgan_mmd-CD', 'lgan_cov-CD', 'lgan_mmd_smp-CD', 'lgan_mmd-EMD', 'lgan_cov-EMD',
                         'lgan_mmd_smp-EMD', '1-NN-CD-acc_t', '1-NN-CD-acc_f', '1-NN-CD-acc', '1-NN-EMD-acc_t',
                         '1-NN-EMD-acc_f', '1-NN-EMD-acc']
    split = dict(M.compute_cov_mmd(smp, rfc))
    split.update(M.compute_1_nna(smp, rfc))
    assert all(torch.equal(got[k], split[k]) for k in got)
    mats = {'rs': (ref.pairwise_emd_cd(rfc, smp), M.pairwise_emd_cd(rfc, smp)),
            'rr': (ref.pairwise_emd_cd(rfc, rfc), M.pairwise_emd_cd(rfc, rfc)),
            'ss': (ref.pairwise_emd_cd(smp, smp), M.pairwise_emd_cd(smp, smp))}
    for i, (metric, rtol) in enumerate((('CD', CD_RTOL), ('EMD', EMD_RTOL))):
        r_rs, p_rs = mats['rs'][0][i], mats['rs'][1][i]
        want = R.lgan_mmd_cov(r_rs.t())
        for k in ('lgan_mmd', 'lgan_mmd_smp'):
            assert float(got['%s-%s' % (k, metric)]) == pytest.approx(float(want[k]), rel=rtol)
        if not _argmin_disagreements_are_ties(p_rs.t(), r_rs.t(), 1, 2 * rtol):
            assert float(got['lgan_cov-' + metric]) == float(want['lgan_cov'])
        want = R.knn(mats['rr'][0][i], r_rs, mats['ss'][0][i], 1)
        j_got = _joint(mats['rr'][1][i], p_rs, mats['ss'][1][i])
        j_ref = _joint(mats['rr'][0][i], r_rs, mats['ss'][0][i])
        if not _argmin_disagreements_are_ties(j_got, j_ref, 0, 2 * rtol):
            for k in ('acc_t', 'acc_f', 'acc'):
                assert float(got['1-NN-%s-%s' % (metric, k)]) == float(want[k]), k
    emd_cd = M.EMD_CD(smp[:20], rfc, 16)
    assert list(emd_cd) == ['MMD-CD', 'MMD-EMD'] and emd_cd['MMD-CD'].dim() == 0
    per_pair = M.EMD_CD(smp[:20], rfc, 16, reduced=False)
    rd1, rd2 = ref.nn_distance(smp[:20], rfc)
    assert max_relerr(per_pair['MMD-CD'], rd1.mean(1) + rd2.mean(1)) <= CD_RTOL
    assert max_relerr(per_pair['MMD-EMD'], ref.match_cost(smp[:20], rfc) / 512) <= EMD_RTOL


def test_structured_inputs(ref, M):
    n = 2048
    x = clouds(1, n, 20)
    y = clouds(1, n, 21)
    # identical clouds: exactly zero
    d1, d2 = M.nn_distance(x, x)
    assert not d1.any() and not d2.any()
    cd, emd = M.paired_emd_cd(x, x)
    assert float(cd) == 0.0 and float(emd) == pytest.approx(float(ref.match_cost(x, x)) / n, rel=EMD_RTOL, abs=1e-7)
    # every point twice, and a cloud that is one repeated point
    dup = x[:, : n // 2].repeat(1, 2, 1).contiguous()
    single = x[:, :1].expand(1, n, 3).contiguous()
    for c in (dup, single):
        for u, v in ((c, y), (y, c)):
            g1, g2 = M.nn_distance(u, v)
            r1, r2 = ref.nn_distance(u, v)
            assert torch.equal(g1, r1) and torch.equal(g2, r2)
            assert max_relerr(M.match_cost(u, v), ref.match_cost(u, v)) <= EMD_RTOL
    # a permuted second cloud: the same per-point distances, moved
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(22)).cuda()
    yp = y[:, perm].contiguous()
    a1, a2 = M.nn_distance(x, y)
    b1, b2 = M.nn_distance(x, yp)
    assert torch.equal(a1, b1) and torch.equal(a2[:, perm], b2)
    c0, e0 = M.paired_emd_cd(x, y)
    c1, e1 = M.paired_emd_cd(x, yp)
    assert max_relerr(c1, c0) <= CD_RTOL and max_relerr(e1, e0) <= EMD_RTOL
