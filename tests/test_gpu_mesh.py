"""-m gpu tests of the mesh kernels (csrc/mesh.cu, octfusion_b200.mesh): marching cubes equals the numpy restatement
(oracle/restate_mesh.py) bit for bit, keeps its surface properties at 256^3, and surface sampling follows the
area-weighted distribution on the sampled triangles; the metric point clouds of a sphere SDF lie on the sphere."""
import numpy as np
import pytest
import torch

from oracle import restate_mesh as RM
from tests import mesh_util as MU
from tests import util as U

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def _grid(kind, r):
    c = (r - 1) / 2
    if kind == 'noise':
        return MU.noise(r, 7 + r, border=False)
    if kind == 'sphere':
        return MU.sphere(r, 0.35 * r + 0.3)
    if kind == 'torus':
        return MU.torus(r, 0.28 * r, 0.1 * r + 0.3)
    # a plane through grid points: corners at x = c exactly equal the level
    x = np.arange(r, dtype=np.float32)[:, None, None] - np.float32(np.floor(c))
    return np.broadcast_to(x + np.float32(0.25), (r, r, r)).copy()


def _equal(meshes, b, grid, level):
    v, f = meshes.mesh(b)
    wv, wf = RM.marching_cubes(grid, level)
    assert torch.equal(v.cpu(), torch.from_numpy(wv))
    assert torch.equal(f.cpu(), torch.from_numpy(wf))


@pytest.mark.parametrize('r', [2, 3, 17, 64])
@pytest.mark.parametrize('kind', ['noise', 'sphere', 'torus', 'plane'])
def test_marching_cubes_equals_oracle(kind, r):
    from octfusion_b200.mesh import marching_cubes
    grid = _grid(kind, r)
    level = 0.25 if kind == 'plane' else 0.0
    m = marching_cubes(torch.from_numpy(grid).to(DEV), level)
    assert len(m) == 1
    _equal(m, 0, grid, level)
    again = marching_cubes(torch.from_numpy(grid).to(DEV), level)
    assert torch.equal(again.verts, m.verts) and torch.equal(again.faces, m.faces)


def test_marching_cubes_batch_equals_oracle_per_shape():
    from octfusion_b200.mesh import marching_cubes
    r = 17
    grids = [_grid('noise', r), np.ones((r, r, r), np.float32), _grid('torus', r)]     # the middle shape is empty
    m = marching_cubes(torch.from_numpy(np.stack(grids)).to(DEV))
    assert len(m) == 3 and m.vert_offsets.dtype == torch.int64
    assert m.vert_offsets.cpu().tolist()[1] == m.vert_offsets.cpu().tolist()[2]
    for b, g in enumerate(grids):
        _equal(m, b, g, 0.0)
    m2 = marching_cubes(torch.from_numpy(np.stack(grids)).to(DEV))
    assert torch.equal(m2.verts, m.verts) and torch.equal(m2.faces, m.faces)
    assert torch.equal(m2.face_offsets, m.face_offsets)


@pytest.mark.parametrize('kind,chi', [('sphere', 2), ('torus', 0)])
def test_closed_surfaces_at_256(kind, chi):
    from octfusion_b200.mesh import marching_cubes
    r = 256
    grid = MU.sphere(r, 100.0) if kind == 'sphere' else MU.torus(r, 80.0, 30.0)
    v, f = marching_cubes(torch.from_numpy(grid).to(DEV)).mesh(0)
    v, f = v.cpu().numpy(), f.cpu().numpy()
    MU.assert_closed_oriented(f)
    assert MU.euler(v, f) == chi
    assert MU.volume(v, f) > 0


def test_calc_sdf_grid_of_the_golden_octree_equals_oracle():
    """the 256^3 calc_sdf grid of the golden depth-8 VAE octree (random regression values, as test_gpu_mpu)"""
    import os
    from octfusion_b200.mpu import NeuralMPU, calc_sdf
    from octfusion_b200.mesh import marching_cubes
    from octfusion_b200 import graph_vae
    g = np.load(os.path.join(U.GOLDEN, 'vae_decode.npz'))
    labels = {d: torch.from_numpy(np.unpackbits(g['label%d' % d])[: int(g['nnum'][d])].astype(np.int64)) for d in (6, 7, 8)}
    net = graph_vae.GraphVAE(**U.VAE)
    po = net.create_child_octree(U.product_doctree(1, 0).octree)
    for d in (6, 7, 8):
        po.octree_split(labels[d].to(DEV), d)
        if d < 8:
            po.octree_grow(d + 1)
            po.depth += 1
    gen = torch.Generator().manual_seed(33)
    reg = {d: torch.randn(int(po.nnum[4:d + 1].sum()), 4, generator=gen).to(DEV) for d in (6, 7, 8)}
    mpu = NeuralMPU(4, 6, 8)

    def model(pos):
        return mpu(pos, reg, po)[8][0]
    model.mpu_args = (mpu, reg, po)
    sdf = calc_sdf(model, 1, 256, 64 ** 3, -0.9, 0.9)
    m = marching_cubes(sdf)
    assert m.faces.shape[0] > 1000
    _equal(m, 0, sdf[0].cpu().numpy(), 0.0)


def test_all_positive_grid_gives_empty_mesh():
    from octfusion_b200.mesh import marching_cubes, pointclouds_from_sdfs
    g = torch.ones(2, 256, 256, 256, device=DEV)
    m = marching_cubes(g)
    assert m.verts.shape == (0, 3) and m.faces.shape == (0, 3)
    assert m.mesh(1)[0].shape == (0, 3)
    with pytest.raises(ValueError, match=r'\[0, 1\]'):
        pointclouds_from_sdfs(g)


def _mesh_batch(verts, faces):
    from octfusion_b200.mesh import MeshBatch
    v = torch.tensor(verts, dtype=torch.float32, device=DEV)
    f = torch.tensor(faces, dtype=torch.int32, device=DEV)
    return MeshBatch(v, f, [0, len(verts)], [0, len(faces)])


def test_samples_lie_on_their_triangles():
    from octfusion_b200.mesh import marching_cubes, sample_surface
    m = marching_cubes(torch.from_numpy(np.stack([_grid('sphere', 17), _grid('torus', 17)])).to(DEV))
    pts, fi = sample_surface(m, 50000, seed=5)
    assert pts.shape == (2, 50000, 3) and fi.dtype == torch.int32
    for b in range(2):
        v, f = (t.cpu().numpy() for t in m.mesh(b))
        tri = v[f[fi[b].cpu().numpy().astype(np.int64)]].astype(np.float64)
        p = pts[b].cpu().numpy().astype(np.float64)
        e1, e2, d = tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0], p - tri[:, 0]
        # barycentric coordinates by least squares; tolerance scaled by the triangle's conditioning
        g11, g12, g22 = (e1 * e1).sum(1), (e1 * e2).sum(1), (e2 * e2).sum(1)
        det = g11 * g22 - g12 * g12
        a = ((e1 * d).sum(1) * g22 - (e2 * d).sum(1) * g12) / det
        c = ((e2 * d).sum(1) * g11 - (e1 * d).sum(1) * g12) / det
        tol = 1e-5 * np.maximum(1.0, np.maximum(g11, g22) / np.sqrt(det))
        assert (a >= -tol).all() and (c >= -tol).all() and (a + c <= 1 + tol).all()
        off_plane = np.abs((d * np.cross(e1, e2)).sum(1)) / np.sqrt(det)
        assert off_plane.max() < 1e-5


def test_face_frequencies_follow_areas():
    """two triangles with areas 1 : 9 and degenerate faces between them; 10^6 seeded samples, chi-square with one
    degree of freedom below 10.83 (p = 0.001); zero-area faces never chosen"""
    from octfusion_b200.mesh import sample_surface
    verts = [[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [3, 0, 1], [0, 3, 1], [2, 0, 0]]
    faces = [[0, 0, 1], [0, 1, 2], [0, 1, 6], [3, 4, 5], [1, 1, 2]]    # areas 0, 0.5, 0 (collinear), 4.5, 0
    area = RM.face_areas(np.array(verts, np.float32), np.array(faces, np.int64))
    zero = area == 0
    assert zero.tolist() == [True, False, True, False, True]
    m = _mesh_batch(verts, faces)
    n = 10 ** 6
    _, fi = sample_surface(m, n, seed=11)
    counts = np.bincount(fi[0].cpu().numpy(), minlength=len(faces))
    assert counts[zero].sum() == 0
    want = area / area.sum() * n
    live = ~zero
    chi2 = (((counts[live] - want[live]) ** 2) / want[live]).sum()
    assert chi2 < 10.83 * (live.sum() - 1), (counts, want)
    assert area[1] / area[3] == pytest.approx(1 / 9)


def test_sampling_seeds():
    from octfusion_b200.mesh import marching_cubes, sample_surface
    m = marching_cubes(torch.from_numpy(_grid('sphere', 17)).to(DEV))
    a, fa = sample_surface(m, 4096, seed=3)
    b, fb = sample_surface(m, 4096, seed=3)
    c, _ = sample_surface(m, 4096, seed=4)
    assert torch.equal(a, b) and torch.equal(fa, fb)
    assert not torch.equal(a, c)
    # counter-based: the first samples do not depend on how many are drawn
    d, _ = sample_surface(m, 100, seed=3)
    assert torch.equal(d[0], a[0, :100])


def test_to_world_matches_export_mesh_arithmetic():
    from octfusion_b200.mesh import marching_cubes, to_world
    size = 64
    v = marching_cubes(torch.from_numpy(_grid('torus', size)).to(DEV)).verts
    got = to_world(v, size, -0.9, 0.9, 0.5).cpu().numpy()
    vn = v.cpu().numpy()
    want = vn * np.float32((0.9 - -0.9) / size) + np.float32(-0.9)
    want = want * np.float32(0.5)
    assert np.array_equal(got, want)


def test_pointclouds_of_a_sphere_lie_on_the_unit_sphere():
    """pointclouds_from_sdfs on a 128^3 sphere SDF: after scale_to_unit_cube the sphere has radius ~1.  Bounds: every
    point within 0.01 of radius 1; Chamfer distance to 2048 analytic samples below 0.006 (two independent uniform
    samplings of the unit sphere with 2048 points each are ~0.004 apart: 2 / (pi * 2048 / (4 pi)))"""
    from octfusion_b200.mesh import pointclouds_from_sdfs
    from octfusion_b200 import metrics
    r = 128
    sdf = torch.from_numpy(MU.sphere(r, 40.0)).to(DEV)
    pts = pointclouds_from_sdfs(sdf[None].expand(4, -1, -1, -1), n=2048, seed=1)
    assert pts.shape == (4, 2048, 3) and pts.dtype == torch.float32 and pts.is_contiguous()
    rad = pts.norm(dim=-1)
    assert (rad - 1).abs().max() < 0.01
    g = torch.Generator().manual_seed(2)
    ref = torch.randn(4, 2048, 3, generator=g)
    ref = (ref / ref.norm(dim=-1, keepdim=True)).to(DEV).contiguous()
    d1, d2 = metrics.nn_distance(pts, ref)
    cd = d1.mean(1) + d2.mean(1)
    assert (cd < 0.006).all(), cd
    # different seeds per call give different clouds of the same shape
    assert not torch.equal(pts, pointclouds_from_sdfs(sdf[None].expand(4, -1, -1, -1), n=2048, seed=2))
    out = metrics.compute_all_metrics(pts, ref)
    assert all(torch.isfinite(torch.as_tensor(v)).all() for v in out.values())
