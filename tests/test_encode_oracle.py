"""CPU tests of the point-cloud -> octree -> ND feature restatement of ocnn (oracle/restate_encode.py; parity UNPINNED
at the ocnn boundary, SURVEY.md Appendix B) and of the argument checks of the new C entry points."""
import ctypes
import pytest
import torch

from oracle import restate as R
from oracle.octree_util import octree_from_splits as oracle_octree
from octfusion_b200.synth import synth_splits
from oracle import restate_encode as RE
from tests import encode_util as E
from tests.util import VAE, digest, relerr, vae_state_dict


def _centres(octree, depth):
    x, y, z, b = octree.xyzb(depth)
    p = (torch.stack([x, y, z], 1).float() + 0.5) / 2 ** (depth - 1) - 1.0
    return [p[b == i] for i in range(octree.batch_size)]


def _reachable_splits(l4, l5):
    """the synthetic split with every full-layer node that has no subdivided child made empty: a node without points
    below it cannot be non-empty in an octree built from points"""
    keep = l5.view(-1, 8).sum(1) > 0
    l4 = l4.clone()
    l4[l4.nonzero().flatten()[~keep]] = 0
    return l4, l5.view(-1, 8)[keep].flatten()


@pytest.mark.parametrize('batch', [1, 3])
def test_centres_of_a_split_octree_rebuild_it(batch):
    """points at the centres of every depth-6 node of a split octree rebuild it, and octree2split_small of the result
    is the split signal"""
    from octfusion_b200.octree import octree2split_small, split2octree_small
    l4, l5 = _reachable_splits(*synth_splits(batch, 2))
    want = oracle_octree(l4, l5, batch)
    pts = _centres(want, 6)
    got = E.oracle_build([(p, torch.ones_like(p)) for p in pts], 6, 4)
    E.assert_same_structure(got, want, 6)
    split = octree2split_small(got, 4)
    assert torch.equal(split, octree2split_small(want, 4))
    E.assert_same_structure(split2octree_small(split, 6, 4), want, 6)


def test_one_point_per_cell_gives_normal_and_displacement():
    g = torch.Generator().manual_seed(3)
    cells = torch.randperm(8 ** 5, generator=g)[:500]
    x = torch.stack([(cells >> (5 * a)) & 31 for a in range(3)], 1).float()
    off = torch.tensor([0.25, 0.625, 0.875])
    xyz = (x + off) / 16 - 1.0
    n = torch.randn(500, 3, generator=g)
    octree = E.oracle_build([(xyz, n)], 5, 2)
    assert int(octree.nnum_nempty[5]) == 500
    from ocnn.octree import xyz2key
    key = xyz2key(x[:, 0], x[:, 1], x[:, 2], 0, 5)
    rank = torch.searchsorted(octree.key(5, nempty=True), key)
    nhat = torch.nn.functional.normalize(n, dim=1)
    assert torch.allclose(octree.normals[5][rank], nhat, atol=1e-6)
    assert torch.allclose(octree.points[5][rank], x + off, atol=1e-5)
    feat = RE.InputFeature('ND')(octree)
    rows = feat[octree.children[5] >= 0][rank]
    assert torch.allclose(rows[:, :3], nhat, atol=1e-6)
    assert torch.allclose(rows[:, 3], (nhat * (off - 0.5)).sum(1), atol=1e-6)
    assert (feat[octree.children[5] < 0] == 0).all()


def test_batched_build_equals_merged_per_shape_builds():
    from octfusion_b200.synth import synth_shell_points
    shapes = synth_shell_points(3, 3000, 8)
    shapes.insert(1, (torch.zeros(0, 3), torch.zeros(0, 3)))                  # an empty shape among others
    shapes.append((torch.tensor([[1.0, -1.0, 0.5], [1.25, -1.5, 0.0]]), torch.ones(2, 3)))   # unclipped: mask wraps
    batched = E.oracle_build(shapes, 7, 3)
    merged = RE.merge_octrees([E.oracle_build([s], 7, 3) for s in shapes])
    E.assert_same_structure(batched, merged, 7)
    assert torch.equal(batched.points[7], merged.points[7]) and torch.equal(batched.normals[7], merged.normals[7])
    assert int(batched.children[3].view(5, -1)[1].max()) == -1                # the empty shape: no node below fd


def test_clip_keeps_points_strictly_inside():
    p = torch.tensor([[0.0, 0.0, 0.0], [0.99, 0.0, 0.0], [0.0, -0.99, 0.0], [0.9899, -0.9899, 0.5], [1.0, 0.0, 0.0]])
    pts = RE.Points(p, torch.arange(15.).view(5, 3), batch_id=torch.tensor([0, 0, 1, 1, 1]), batch_size=2)
    pts.clip(min=-1, max=1)
    assert pts.points.shape[0] == 2 and torch.equal(pts.batch_id, torch.tensor([0, 1]))
    assert torch.equal(pts.normals, torch.tensor([[0., 1., 2.], [9., 10., 11.]]))


def test_oracle_matches_reference_fixture():
    g = E.fixture()
    shapes = E.fixture_shapes()
    assert abs(sum(float(x.double().abs().sum()) for x, _ in shapes) - float(g['xyz_sum'])) < 1e-6 * float(g['xyz_sum'])
    octree = E.oracle_build(shapes, VAE['depth'], VAE['full_depth'])
    assert octree.nnum.tolist() == g['nnum'].tolist() and octree.nnum_nempty.tolist() == g['nnum_nempty'].tolist()
    for d in range(VAE['full_depth'], VAE['depth'] + 1):
        assert digest(octree.keys[d]) == str(g['keys%d' % d]) and digest(octree.children[d]) == str(g['children%d' % d])
    assert relerr(octree.points[8][::E.ROW_STEP], torch.from_numpy(g['points'])) < 1e-6
    assert relerr(octree.normals[8][::E.ROW_STEP], torch.from_numpy(g['normals'])) < 1e-6
    doc = R.DualGraph(octree)
    feat = E.oracle_feature(octree, doc)
    assert feat.shape[0] == int(g['feature_rows']) == doc.total_num
    assert relerr(feat[::E.ROW_STEP], torch.from_numpy(g['feature'])) < 1e-6
    moments = R.vae_encode(feat, doc, vae_state_dict(), 8, 6, 2)
    z, _ = E.posterior_sample(moments, E.CODE_SEED)
    assert z.shape[0] == int(g['code_rows']) and relerr(z[::4], torch.from_numpy(g['code'])) < 1e-4
    z, kl = E.posterior_sample(moments, E.FORWARD_SEED, draws=2)
    assert abs(float(kl.mean()) - float(g['kl_loss'])) < 1e-4 * abs(float(g['kl_loss']))
    assert abs(float(z.max()) - float(g['code_max'])) < 1e-4 * abs(float(g['code_max']))


def test_input_feature_rejects_other_letters():
    with pytest.raises(NotImplementedError):
        RE.InputFeature('NDF')
    from octfusion_b200 import InputFeature
    for feat, nempty in (('F', False), ('NDF', False), ('ND', True)):
        with pytest.raises(NotImplementedError):
            InputFeature(feat, nempty)


def test_build_entry_points_reject_bad_arguments_without_gpu():
    from octfusion_b200._lib import lib
    ok = lib.of_octree_build_bytes(1000, 32, 8, 4)
    assert ok > 1000 * 24
    for n, b, dep, fd in ((1000, 32, 17, 4), (1000, 1024, 8, 4), (1000, 0, 8, 4), (1000, 2, 8, 8), (1 << 31, 2, 8, 4),
                          (-1, 2, 8, 4)):
        assert lib.of_octree_build_bytes(n, b, dep, fd) == -1
    assert b'of_octree_build_bytes' in lib.of_last_error()
    buf = ctypes.c_void_p(1)
    assert lib.of_octree_build_levels(buf, buf, 10, 2, 17, 4, buf, buf, None) == -1
    assert lib.of_octree_build_levels(buf, None, 10, 2, 8, 4, buf, buf, None) == -1
    assert lib.of_octree_build_fill(buf, 10, 2, 8, 4, 3, 8, buf, buf, None) == -1          # depth below full_depth
    assert lib.of_octree_build_fill(buf, 10, 2, 8, 4, 4, 100, None, buf, None) == -1      # full layer is 2 * 8^4
    assert lib.of_octree_build_signal(buf, 10, 2, 8, 4, buf, buf, buf, None, None) == -1  # normals in without out
    assert lib.of_input_feature_nd(buf, buf, buf, 10, 0, 7, buf, 4, None) == -1
    assert lib.of_input_feature_nd(buf, buf, buf, 10, 0, 0, buf, 3, None) == -1
    assert b'of_input_feature_nd' in lib.of_last_error()


def test_build_octree_refuses_cpu_points():
    if torch.cuda.is_available():
        pytest.skip('only meaningful on a host without a GPU')
    from octfusion_b200 import Octree, Points
    with pytest.raises(RuntimeError):
        Octree(6, 2, 1, 'cpu').build_octree(Points(torch.zeros(4, 3), torch.ones(4, 3)))
    with pytest.raises(ValueError):
        Octree(17, 2, 1, 'cpu').build_octree(Points(torch.zeros(4, 3), torch.ones(4, 3)))
