"""CPU tests (-m "not gpu") of the shape-metric oracle and of the metric entry points' argument checks: the torch
restatements of nn_distance, lgan_mmd_cov and knn equal the unmodified reference's outputs (tests/golden/metrics.npz,
oracle/gen_golden_metrics.py), the restated approximate EMD has the symmetries of a matching, and the C ABI rejects
bad arguments before launching anything."""
import ctypes
import os
import numpy as np
import pytest
import torch

from oracle import restate_metrics as R
from tests.util import GOLDEN


@pytest.fixture(scope='module')
def golden():
    from oracle.gen_golden import checksum
    from oracle.gen_golden_metrics import metrics_inputs
    g = np.load(os.path.join(GOLDEN, 'metrics.npz'))
    inp = metrics_inputs()
    for k, v in inp.items():
        assert checksum(v) == pytest.approx(float(g[k + '_sum']), rel=1e-12), k      # generator unchanged
    return g, inp


def test_nn_distance_restatement_matches_reference(golden):
    g, inp = golden
    d1, d2 = R.nn_distance(inp['x'], inp['y'])
    # the reference's distChamfer expands |x|^2 + |y|^2 - 2 x.y (equal up to float64 rounding) and returns its two
    # directions in the opposite order to nndistance: (per point of y, per point of x)
    np.testing.assert_allclose(d1.numpy(), g['dist2'], rtol=0, atol=1e-12)
    np.testing.assert_allclose(d2.numpy(), g['dist1'], rtol=0, atol=1e-12)


def test_lgan_mmd_cov_and_knn_restatements_match_reference(golden):
    g, inp = golden
    for k, v in R.lgan_mmd_cov(inp['all_dist']).items():
        assert float(v) == float(g['lgan_' + k]), k
    res = R.knn(inp['mxx'], inp['mxy'], inp['myy'], 1)
    assert set(res) == {k[4:] for k in g.files if k.startswith('knn_')}
    for k, v in res.items():
        assert float(v) == float(g['knn_' + k]), k


def test_approx_emd_restatement_is_permutation_invariant():
    gen = torch.Generator().manual_seed(3)
    x = torch.rand(2, 40, 3, generator=gen, dtype=torch.float64)
    y = torch.rand(2, 40, 3, generator=gen, dtype=torch.float64)
    c = R.approx_match_cost(x, y)
    px, py = torch.randperm(40, generator=gen), torch.randperm(40, generator=gen)
    cp = R.approx_match_cost(x[:, px], y[:, py])
    assert torch.allclose(cp, c, rtol=1e-12, atol=0)
    assert (c > 0).all()
    # one point each: the whole mass moves along the single edge
    one = R.approx_match_cost(x[:, :1], y[:, :1])
    assert torch.allclose(one, (x[:, 0] - y[:, 0]).norm(dim=-1), rtol=1e-6)


def test_chamfer_of_a_cloud_with_itself_is_zero():
    x = torch.rand(2, 50, 3, generator=torch.Generator().manual_seed(4))
    d1, d2 = R.nn_distance(x, x)
    assert torch.equal(d1, torch.zeros_like(d1)) and torch.equal(d2, torch.zeros_like(d2))
    assert torch.equal(d1.mean(1) + d2.mean(1), torch.zeros(2))


def test_metric_entry_points_reject_bad_arguments_without_gpu():
    """negative return + error text, no launch, no crash"""
    from octfusion_b200 import _lib
    lib, dummy = _lib.lib, ctypes.c_void_p(16)
    n0 = _lib.launch_count()
    cases = [
        ('of_nn_distance', lib.of_nn_distance(None, dummy, 1, 8, 8, dummy, dummy, None, None)),
        ('of_nn_distance', lib.of_nn_distance(dummy, dummy, 1, 0, 8, dummy, dummy, None, None)),
        ('of_chamfer_pairwise', lib.of_chamfer_pairwise(dummy, 2, 8, dummy, 2, 8, None, None)),
        ('of_chamfer_pairwise', lib.of_chamfer_pairwise(dummy, 2, _lib.CD_PAIRWISE_MAX_POINTS, dummy, 2, 1, dummy, None)),
        ('of_match_cost', lib.of_match_cost(dummy, dummy, 1, _lib.EMD_MAX_POINTS + 1, dummy, None, None)),
        ('of_match_cost', lib.of_match_cost(dummy, dummy, -1, 16, dummy, None, None)),
        ('of_emd_cd_pairwise', lib.of_emd_cd_pairwise(dummy, 2, dummy, 2, 0, dummy, dummy, None)),
        ('of_emd_cd_pairwise', lib.of_emd_cd_pairwise(dummy, 2, dummy, 2, 16, dummy, None, None)),
    ]
    for name, rc in cases:
        assert rc == -1, name
    assert b'of_emd_cd_pairwise' in lib.of_last_error()
    assert lib.of_match_cost(dummy, dummy, 0, 16, dummy, None, None) == 0            # empty batch: nothing to do
    assert _lib.launch_count() == n0


def test_metrics_refuse_cpu_tensors():
    from octfusion_b200 import metrics as M
    x = torch.rand(2, 16, 3)
    for fn in (M.nn_distance, M.match_cost, M.pairwise_emd_cd, M.pairwise_cd, M.compute_all_metrics):
        with pytest.raises(RuntimeError, match='no CPU path'):
            fn(x, x)
