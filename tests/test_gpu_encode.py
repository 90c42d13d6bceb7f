"""-m gpu: the point-cloud encoder path on the device -- Octree.build_octree (csrc/points.cu) against the oracle
restatement (parity UNPINNED at the ocnn boundary), the ND input features, and GraphVAE extract_code / encode_moments /
forward against the oracle and the reference fixture tests/golden/vae_encode_points.npz."""
import numpy as np
import pytest
import torch

from oracle import restate as R
from oracle import restate_encode as RE
from tests import encode_util as E
from tests.util import VAE, relerr, vae_state_dict, build_vae, oracle_child_octree

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def _shell(batch, points, seed):
    from octfusion_b200.synth import synth_shell_points
    return synth_shell_points(batch, points, seed)


def _edge_shapes():
    """duplicates, points exactly on cell faces, unclipped points at +-1.0 and beyond (the mask wraps them), a single
    point, and an empty shape among non-empty ones"""
    g = torch.Generator().manual_seed(4)
    base = torch.rand(300, 3, generator=g) * 1.8 - 0.9
    dup = torch.cat([base, base[:100], base[:100]])
    faces = torch.randint(-32, 32, (400, 3), generator=g).float() / 32           # depth 6: cell faces at k / 32
    wild = torch.tensor([[1.0, 1.0, 1.0], [-1.0, -1.0, -1.0], [1.0, -1.0, 0.0], [1.5, -1.25, 3.0], [-2.0, 0.3, 0.7],
                         [0.999999, -0.999999, 0.0]])
    one = torch.tensor([[0.1, -0.2, 0.3]])
    clouds = [dup, faces, torch.zeros(0, 3), wild, one]
    return [(c, torch.nn.functional.normalize(torch.randn(c.shape[0], 3, generator=g), dim=1)) for c in clouds]


def _check_build(shapes, depth, fd):
    got = E.product_build(shapes, depth, fd)
    want = E.oracle_build(shapes, depth, fd)
    E.assert_same_structure(got, want, depth)
    assert relerr(got.points[depth].cpu(), want.points[depth]) < 1e-6
    assert relerr(got.normals[depth].cpu(), want.normals[depth]) < 1e-6
    feat = RE.InputFeature('ND')(want)
    from octfusion_b200 import InputFeature
    assert relerr(InputFeature('ND')(got).cpu(), feat) < 1e-6
    return got, want


@pytest.mark.parametrize('batch', [1, 5, 32])
@pytest.mark.parametrize('depth,fd', [(6, 2), (8, 4)])
def test_build_matches_oracle(batch, depth, fd):
    _check_build(_shell(batch, 100_000, batch), depth, fd)


def test_build_edge_cases_match_oracle():
    shapes = _edge_shapes()
    got, want = _check_build(shapes, 6, 2)
    assert int(got.children[2].view(len(shapes), -1)[2].max()) == -1          # the empty shape
    _check_build(shapes[3:], 8, 4)


def test_identical_builds_are_equal():
    shapes = _shell(5, 50_000, 1) + _edge_shapes()
    a, b = E.product_build(shapes, 8, 4), E.product_build(shapes, 8, 4)
    E.assert_same_structure(a, b, 8)
    assert torch.equal(a.points[8], b.points[8]) and torch.equal(a.normals[8], b.normals[8])


def test_permuting_the_points_of_a_shape_changes_only_rounding():
    shapes = _shell(3, 50_000, 2)
    g = torch.Generator().manual_seed(0)
    perm = []
    for x, n in shapes:
        p = torch.randperm(x.shape[0], generator=g)
        perm.append((x[p], n[p]))
    a, b = E.product_build(shapes, 8, 4), E.product_build(perm, 8, 4)
    E.assert_same_structure(a, b, 8)
    assert relerr(a.points[8], b.points[8]) < 1e-6 and relerr(a.normals[8], b.normals[8]) < 1e-6


def test_centres_of_a_split_octree_rebuild_it_on_the_device():
    from octfusion_b200 import octree_from_splits
    from octfusion_b200.octree import octree2split_small
    from octfusion_b200.synth import synth_splits
    from tests.test_encode_oracle import _reachable_splits, _centres
    l4, l5 = _reachable_splits(*synth_splits(3, 2))
    want = octree_from_splits(l4, l5, 3, device=DEV)
    got = E.product_build([(p, torch.ones_like(p)) for p in _centres(want, 6)], 6, 4)
    E.assert_same_structure(got, want, 6)
    assert torch.equal(octree2split_small(got, 4), octree2split_small(want, 4))


@pytest.fixture(scope='module')
def encode_case():
    g = E.fixture()
    sd = vae_state_dict()
    shapes = E.fixture_shapes()
    octree = E.oracle_build(shapes, VAE['depth'], VAE['full_depth'])
    doc = R.DualGraph(octree)
    feat = E.oracle_feature(octree, doc)
    moments = R.vae_encode(feat, doc, sd, 8, 6, 2)
    return g, sd, build_vae(sd), shapes, octree, doc, feat, moments


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_input_feature_rows_match_oracle_and_fixture(encode_case, dtype):
    from octfusion_b200 import DualOctree
    g, sd, net, shapes, octree, doc, feat, moments = encode_case
    pdoc = DualOctree(E.product_build(shapes, 8, 4))
    got = pdoc.get_input_feature(dtype=dtype).float().cpu()
    tol = 1e-6 if dtype == torch.float32 else 4e-3
    assert got.shape == feat.shape and relerr(got, feat) < tol
    assert relerr(got[::E.ROW_STEP], torch.from_numpy(g['feature'])) < tol


@pytest.mark.parametrize('dtype,tol', [(torch.float32, 1e-3), (torch.bfloat16, 2e-2)])
def test_extract_code_and_moments_match_oracle_and_fixture(encode_case, dtype, tol):
    g, sd, net, shapes, octree, doc, feat, moments = encode_case
    octree_in = E.product_build(shapes, 8, 4)
    torch.manual_seed(E.CODE_SEED)
    z, pdoc = net.extract_code(octree_in, dtype=dtype)
    want, _ = E.posterior_sample(moments, E.CODE_SEED)
    assert z.shape == want.shape and pdoc.total_num == doc.total_num
    assert relerr(z.cpu(), want) < tol and relerr(z.cpu()[::4], torch.from_numpy(g['code'])) < tol
    got = net.encode_moments(pdoc.get_input_feature(dtype=dtype), pdoc)
    assert relerr(got.float().cpu(), moments) < tol


def _child_octree(octree):
    """GraphVAE.create_child_octree (graph_vae.py:235-244) of the oracle's built octree: its non-empty nodes down to
    depth_stop"""
    import types
    return oracle_child_octree(types.SimpleNamespace(full_depth=octree.full_depth, depth=VAE['depth_stop'],
                                                     batch_size=octree.batch_size, children=octree.children))


@pytest.mark.parametrize('dtype,tol', [(torch.float32, 1e-3), (torch.bfloat16, 2e-2)])
def test_forward_matches_oracle_and_fixture(encode_case, dtype, tol):
    """forward(evaluate=True): kl_loss / code_max / code_min are those of the second posterior sample drawn from the
    product's moments, which match the oracle's; the oracle decodes that same sample on the octree the product grew
    (the labels it chose), and the product may differ from the oracle's own choice only on near-ties (as in
    test_gpu_vae.test_vae_decode_grows_the_same_octree_as_the_oracle)."""
    from octfusion_b200 import DualOctree
    g, sd, net, shapes, octree, doc, feat, moments = encode_case
    octree_in = E.product_build(shapes, 8, 4)
    pdoc = DualOctree(octree_in)
    pm = net.encode_moments(pdoc.get_input_feature(dtype=dtype), pdoc).float().cpu()
    assert relerr(pm, moments) < tol
    z, kl = E.posterior_sample(pm, E.FORWARD_SEED, draws=2)
    zo, klo = E.posterior_sample(moments, E.FORWARD_SEED, draws=2)
    assert relerr(z, zo) < tol and relerr(kl, klo) < tol
    torch.manual_seed(E.FORWARD_SEED)
    out = net.forward(octree_in, evaluate=True, dtype=dtype)
    assert abs(float(out['kl_loss']) - float(kl.mean())) < 1e-4 * abs(float(kl.mean()))
    assert abs(float(out['code_max']) - float(z.max())) < 1e-4 * float(z.abs().max())
    assert abs(float(out['code_min']) - float(z.min())) < 1e-4 * float(z.abs().max())
    for k in ('code_max', 'code_min'):
        assert abs(float(out[k]) - float(g[k])) < tol * max(abs(float(g['code_max'])), abs(float(g['code_min'])))
    mine = {d: out['logits'][d].float().argmax(1).cpu() for d in (6, 7, 8)}
    logits, regs, grown = R.vae_decode(z, R.DualGraph(_child_octree(octree)), sd, 6, 8, 2, update_octree=True,
                                       labels=mine)
    po = out['octree_out']
    assert po.nnum.tolist() == grown.nnum.tolist() and po.nnum_nempty.tolist() == grown.nnum_nempty.tolist()
    for d in (6, 7, 8):
        assert torch.equal(po.keys[d].cpu(), grown.keys[d]) and torch.equal(po.children[d].cpu(), grown.children[d])
        assert relerr(out['logits'][d].float().cpu(), logits[d]) < tol
        assert relerr(out['reg_voxs'][d].float().cpu(), regs[d]) < tol
        flips = logits[d].argmax(1) != mine[d]
        near = tol * float(logits[d].abs().max())
        assert float((logits[d][:, 0] - logits[d][:, 1]).abs()[flips].max() if flips.any() else 0.0) < near
        ref = torch.from_numpy(np.unpackbits(g['label%d' % d])[: int(g['out_nnum'][d])].astype(np.int64))
        if ref.shape == mine[d].shape and torch.equal(ref, mine[d]):
            assert relerr(out['logits'][d].float().cpu()[::E.ROW_STEP], torch.from_numpy(g['logit%d' % d])) < tol
            assert relerr(out['reg_voxs'][d].float().cpu()[::E.ROW_STEP], torch.from_numpy(g['reg%d' % d])) < tol


def test_reconstruction_round_trip_is_structurally_sound(encode_case):
    """points -> forward -> calc_sdf(64) -> point clouds -> metrics against the input points, on random weights: every
    hand-off has the right shape and is finite (no claim about quality)."""
    from octfusion_b200.mpu import calc_sdf
    from octfusion_b200.mesh import pointclouds_from_sdfs
    from octfusion_b200.metrics import compute_all_metrics
    g, sd, net, shapes, octree, doc, feat, moments = encode_case
    torch.manual_seed(0)
    out = net.forward(E.product_build(shapes, 8, 4), evaluate=True)
    sdfs = calc_sdf(out['neural_mpu'], len(shapes), size=64)
    assert sdfs.shape == (len(shapes), 64, 64, 64) and torch.isfinite(sdfs).all()
    grid = torch.stack([torch.arange(8, dtype=torch.float32, device=DEV)] * 3, 1) / 4 - 1.0
    pos = torch.cat([grid, torch.zeros(8, 1, device=DEV)], 1)
    assert torch.isfinite(out['neural_mpu'](pos)).all()
    clouds = torch.cat([pointclouds_from_sdfs(sdfs[b:b + 1], 2048, level=float(sdfs[b].median()))
                        for b in range(len(shapes))])
    ref = torch.stack([x[:2048] for x, _ in shapes]).to(DEV)
    assert clouds.shape == ref.shape and torch.isfinite(clouds).all()
    res = compute_all_metrics(clouds, ref)
    assert res and all(bool(torch.isfinite(torch.as_tensor(v)).all()) for v in res.values())
