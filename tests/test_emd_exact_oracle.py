"""CPU tests (-m "not gpu") of the exact-EMD oracle and of the exact-EMD entry points' argument checks: the
restatement of reference `emd_approx` equals the unmodified reference's outputs (tests/golden/metrics_emd_exact.npz,
oracle/gen_golden_emd_exact.py), the quantised problem that csrc/emd_exact.cu solves stays within its stated bound of
them, both give known answers that need no solver, and the C ABI rejects bad arguments before launching anything."""
import ctypes
import os
import numpy as np
import pytest
import torch

from oracle import restate_emd_exact as R
from tests.util import GOLDEN


def emd_bound(ref, max_d, k):
    """|emd - ref| allowed between the quantised exact EMD and the reference's fp32 one:
      q/2             each c_ij q is within q/2 of d_ij, so the optimal mean of c q is within q/2 of the optimum of d;
      2^-21 max d     the reference's distances ((x - y).norm in fp32) and the kernel's (rounded op by op) are each a
                      few ulp (< 4) from the true distance, so entries differ by < 8 ulp = 2^-21 d, and so do optima;
      16 ulp(ref)     the reference's fp32 mean of n matched distances (numpy pairwise summation, < 12 ulp for
                      n <= 4096) plus the final fp32 rounding of the kernel's fp64 result"""
    q = 2.0 ** (k - 24)
    return q / 2 + 2.0 ** -21 * max_d + 16 * float(np.spacing(np.float32(abs(ref))))


@pytest.fixture(scope='module')
def golden():
    from oracle.gen_golden import checksum
    from oracle.gen_golden_emd_exact import emd_exact_inputs
    g = np.load(os.path.join(GOLDEN, 'metrics_emd_exact.npz'))
    inp = emd_exact_inputs()
    for k, v in inp.items():
        assert checksum(v) == pytest.approx(float(g[k + '_sum']), rel=1e-12), k      # generator unchanged
    return g, inp


@pytest.mark.parametrize('n', [1, 2, 3, 17, 128, 1000])
def test_restatement_matches_reference(golden, n):
    g, inp = golden
    got = R.emd_exact(inp['x%d' % n], inp['y%d' % n]).numpy()
    np.testing.assert_allclose(got, g['emd%d' % n], rtol=1e-6, atol=0)


@pytest.mark.parametrize('n', [1, 2, 3, 17, 128, 1000])
def test_quantised_problem_within_bound_of_reference(golden, n):
    g, inp = golden
    x, y = inp['x%d' % n], inp['y%d' % n]
    for i, (emd, cstar, k) in enumerate(R.emd_exact_quantized(x, y)):
        ref = float(g['emd%d' % n][i])
        max_d = float(R.emd_exact_distances(x[i], y[i]).max())
        assert abs(float(emd) - ref) <= emd_bound(ref, max_d, k), (n, i, float(emd), ref)
        assert cstar >= 0 and -100 <= k <= 62


def test_exponent_is_the_smallest_power_of_two_above_the_diagonal():
    x = np.zeros((1, 3), np.float32)
    for diag, k in ((1.0, 0), (1.5, 1), (2.0, 1), (3.0, 2), (0.5, -1), (0.375, -1), (0.25, -2), (0.0, -100)):
        assert R.emd_exact_exponent(x, np.array([[diag, 0, 0]], np.float32)) == k, diag
    x = np.array([[0, 0, 0], [1, 1, 1]], np.float32)          # diagonal sqrt(3): s = 2
    assert R.emd_exact_exponent(x, x) == 1
    assert R.emd_exact_exponent(x * 1e-35, x * 1e-35) == -100                         # clamped below


def _cloud(n, seed):
    return torch.rand(1, n, 3, generator=torch.Generator().manual_seed(seed))


def test_known_answers_without_a_solver():
    x = _cloud(300, 1)
    # a permutation of the cloud: every point has a partner at distance 0
    perm = torch.randperm(300, generator=torch.Generator().manual_seed(2))
    assert float(R.emd_exact(x, x[:, perm])) == 0.0
    assert R.emd_exact_quantized(x, x[:, perm])[0][:2] == (0.0, 0)
    # a translated cloud: no matching beats the identity (triangle inequality), so the EMD is |t|
    t = torch.tensor([0.3, -0.2, 0.1])
    y = x + t
    dn = float(t.norm())
    got = float(R.emd_exact(x, y))
    assert got == pytest.approx(dn, rel=1e-5)
    emd, _, k = R.emd_exact_quantized(x, y)[0]
    assert abs(float(emd) - got) <= emd_bound(got, 1.8, k)
    # collinear clouds: the optimal matching pairs the sorted coordinates
    g = torch.Generator().manual_seed(3)
    a, b = torch.rand(257, generator=g), torch.rand(257, generator=g) * 2
    xa = torch.stack([a, torch.zeros_like(a), torch.zeros_like(a)], -1)[None]
    xb = torch.stack([b, torch.zeros_like(b), torch.zeros_like(b)], -1)[None]
    want = float((a.sort().values.double() - b.sort().values.double()).abs().mean())
    assert float(R.emd_exact(xa, xb)) == pytest.approx(want, rel=1e-6)
    emd, _, k = R.emd_exact_quantized(xa, xb)[0]
    assert abs(float(emd) - want) <= emd_bound(want, 2.0, k)


def test_exact_emd_entry_points_reject_bad_arguments_without_gpu():
    """negative return + error text, no launch, no crash"""
    from octfusion_b200 import _lib
    lib, dummy, other = _lib.lib, ctypes.c_void_p(16), ctypes.c_void_p(32)
    n0 = _lib.launch_count()
    cases = [
        ('of_emd_exact', lib.of_emd_exact(None, dummy, 1, 8, dummy, None, dummy, None)),
        ('of_emd_exact', lib.of_emd_exact(dummy, dummy, 1, 8, dummy, None, None, None)),
        ('of_emd_exact', lib.of_emd_exact(dummy, dummy, 1, 0, dummy, None, dummy, None)),
        ('of_emd_exact', lib.of_emd_exact(dummy, dummy, 1, _lib.EMD_MAX_POINTS + 1, dummy, None, dummy, None)),
        ('of_emd_exact', lib.of_emd_exact(dummy, dummy, -1, 16, dummy, None, dummy, None)),
        ('of_emd_exact_pairwise', lib.of_emd_exact_pairwise(dummy, 2, other, 2, 16, 1, dummy, None, dummy, None)),
        ('of_emd_exact_pairwise', lib.of_emd_exact_pairwise(dummy, 2, dummy, 3, 16, 1, dummy, None, dummy, None)),
        ('of_emd_exact_pairwise', lib.of_emd_exact_pairwise(dummy, 2, dummy, 2, 4097, 0, dummy, None, dummy, None)),
        ('of_emd_exact_pairwise', lib.of_emd_exact_pairwise(dummy, 2, dummy, 2, 16, 0, None, None, dummy, None)),
    ]
    for name, rc in cases:
        assert rc == -1, name
        assert name.encode() in lib.of_last_error()
    assert lib.of_emd_exact(dummy, dummy, 0, 16, dummy, None, dummy, None) == 0             # empty batch
    assert lib.of_emd_exact_pairwise(dummy, 0, dummy, 0, 16, 1, dummy, None, dummy, None) == 0
    assert _lib.launch_count() == n0


def test_exact_emd_refuses_cpu_tensors():
    from octfusion_b200 import metrics as M
    x = torch.rand(2, 16, 3)
    for fn in (M.emd_approx, M.emd_exact, M.pairwise_emd_exact):
        with pytest.raises(RuntimeError, match='no CPU path'):
            fn(x, x)
    with pytest.raises(RuntimeError, match='no CPU path'):
        M.compute_all_metrics(x, x, accelerated_emd=False)
    with pytest.raises(RuntimeError, match='no CPU path'):
        M.EMD_CD(x, x, accelerated_emd=False)
