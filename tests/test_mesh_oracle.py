"""CPU tests (-m "not gpu") of the marching-cubes table, its numpy restatement (oracle/restate_mesh.py) and the mesh
entry points' argument checks: the generated table cuts every crossing edge exactly once, the committed
csrc/mc_table.inc is the generator's output, the restated meshes are closed, consistently wound 2-manifolds with the
right Euler characteristic, volume and vertex positions, and the C ABI rejects bad arguments before launching."""
import ctypes

import numpy as np
import pytest

from oracle import restate_mesh as RM
from tests import mesh_util as MU

T = RM.T


def _crossing_edges(case):
    return {e for e, (_, a, b) in enumerate(T.EDGES) if (case >> a & 1) != (case >> b & 1)}


@pytest.mark.parametrize('case', range(256))
def test_table_cuts_each_crossing_edge_on_one_loop(case):
    tris = T.table()[case]
    used = {e for t in tris for e in t}
    assert used == _crossing_edges(case)
    loops = T.loops(case)
    flat = [e for loop in loops for e in loop]
    assert sorted(flat) == sorted(_crossing_edges(case))            # each crossing edge on exactly one loop
    assert len(tris) == sum(len(loop) - 2 for loop in loops) <= T.MAX_TRIS
    if case in (0, 255):
        assert tris == []


def test_table_cells_are_closed_and_wound_consistently():
    """per case, the triangles of each loop form a disk: interior edges in two triangles with opposite directions,
    loop edges once; a single inside corner gets the outward triangle (x, y, z edges of corner 0)"""
    for case in range(256):
        for loop in T.loops(case):
            loop = T.fan_start(loop)
            tris = [(loop[0], loop[i], loop[i + 1]) for i in range(1, len(loop) - 1)]
            directed = [(t[i], t[(i + 1) % 3]) for t in tris for i in range(3)]
            assert len(set(directed)) == len(directed)
            boundary = {(loop[i], loop[(i + 1) % len(loop)]) for i in range(len(loop))}
            assert boundary <= set(directed)
            assert all((b, a) in directed for a, b in set(directed) - boundary)
    assert T.table()[1] == [(0, 4, 8)]


def test_committed_table_header_is_generated():
    with open(T.INC_PATH) as f:
        assert f.read() == T.render(), 'csrc/mc_table.inc is stale: run python octfusion_b200/mc_table.py'


@pytest.mark.parametrize('r', [6, 10, 14])
def test_noise_grids_give_closed_oriented_surfaces(r):
    for seed in range(12):
        v, f = RM.marching_cubes(MU.noise(r, 1000 * r + seed))
        MU.assert_closed_oriented(f)
        assert v.dtype == np.float32 and f.dtype == np.int32


@pytest.mark.parametrize('name,grid,chi', [
    ('sphere', lambda: MU.sphere(48, 15.0), 2),
    ('torus', lambda: MU.torus(48, 13.0, 5.0), 0),
    ('two spheres', lambda: MU.two_spheres(48, 8.0), 4),
])
def test_known_shapes_have_their_euler_characteristic(name, grid, chi):
    v, f = RM.marching_cubes(grid())
    MU.assert_closed_oriented(f)
    assert MU.euler(v, f) == chi, name


def test_sphere_volume_and_vertices():
    r, radius = 48, 15.0
    v, f = RM.marching_cubes(MU.sphere(r, radius))
    vol = MU.volume(v, f)
    assert vol > 0
    assert abs(vol / (4 / 3 * np.pi * radius ** 3) - 1) < 0.01
    dist = np.linalg.norm(v.astype(np.float64) - (r - 1) / 2, axis=1)
    assert np.abs(dist - radius).max() < 0.02


def test_vertex_interpolation_expression():
    g = MU.sphere(12, 4.0)
    v, _ = RM.marching_cubes(g, 0.25)
    on_x = v[:, 0] != np.floor(v[:, 0])
    i, j, k = np.floor(v[on_x]).astype(np.int64).T
    fa, fb = g[i, j, k], g[i + 1, j, k]
    t = (np.float32(0.25) - fa) / (fb - fa)
    assert np.array_equal(v[on_x, 0], i.astype(np.float32) + t)
    assert on_x.any()


def test_surface_cut_by_the_grid_boundary_is_open_only_there():
    r = 20
    v, f = RM.marching_cubes(MU.plane(r))
    directed, und, cnt = MU.edge_counts(f)
    assert directed.max() == 1 and cnt.max() == 2
    open_edges = und[cnt == 1]
    assert len(open_edges) > 0
    a, b = v[open_edges[:, 0]], v[open_edges[:, 1]]
    on_boundary = ((a == 0) & (b == 0)) | ((a == r - 1) & (b == r - 1))
    assert on_boundary.any(1).all()


def test_corners_exactly_at_level_keep_the_surface_closed():
    for seed in range(8):
        g = np.random.default_rng(seed).integers(-1, 2, size=(12, 12, 12)).astype(np.float32)
        MU.close(g)
        assert (g == 0).any()
        v, f = RM.marching_cubes(g)
        MU.assert_closed_oriented(f)
        # a level corner is outside: vertices sit on it exactly
        assert (v == np.round(v)).all(1).any()


def test_empty_and_full_grids_give_no_mesh():
    for g in (np.ones((5, 5, 5), np.float32), -np.ones((5, 5, 5), np.float32)):
        v, f = RM.marching_cubes(g)
        assert v.shape == (0, 3) and f.shape == (0, 3)


def test_sampling_restatement():
    verts = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 0], [3, 0, 0], [0, 6, 0]], np.float32)
    faces = np.array([[0, 1, 2], [0, 1, 1], [3, 4, 5]], np.int32)     # areas 0.5, 0, 9
    rng = np.random.default_rng(0)
    n = 20000
    u = 1 - rng.random(n)
    pts, fi = RM.sample_surface(verts, faces, u, rng.random(n), rng.random(n))
    assert not (fi == 1).any()
    assert abs((fi == 0).mean() - 0.5 / 9.5) < 0.01
    assert (pts[:, 2] == 0).all() and (pts[fi == 0].sum(1) <= 1 + 1e-6).all()
    unit = RM.scale_to_unit_cube(pts, verts)                  # vertex box [0, 3] x [0, 6] x 0 -> y spans [-1, 1]
    assert np.abs(unit).max() <= 1 + 1e-6
    assert unit[:, 1].min() < -0.95 and unit[:, 1].max() > 0.95


def test_mesh_entry_points_reject_bad_arguments_without_gpu():
    """negative return + error text, no launch, no crash"""
    from octfusion_b200 import _lib
    lib, dummy = _lib.lib, ctypes.c_void_p(16)
    n0 = _lib.launch_count()
    cases = [
        ('of_mc_count', lambda: lib.of_mc_count(None, 8, 0.0, dummy, dummy, None)),
        ('of_mc_count', lambda: lib.of_mc_count(dummy, 1, 0.0, dummy, dummy, None)),
        ('of_mc_count', lambda: lib.of_mc_count(dummy, _lib.MC_MAX_SIZE + 1, 0.0, dummy, dummy, None)),
        ('of_mc_emit', lambda: lib.of_mc_emit(dummy, 8, 0.0, dummy, None, dummy, dummy, None)),
        ('of_mc_emit', lambda: lib.of_mc_emit(dummy, 0, 0.0, dummy, dummy, dummy, dummy, None)),
        ('of_mesh_bbox', lambda: lib.of_mesh_bbox(dummy, None, 2, dummy, None)),
        ('of_mesh_bbox', lambda: lib.of_mesh_bbox(dummy, dummy, -1, dummy, None)),
        ('of_surface_sample', lambda: lib.of_surface_sample(dummy, dummy, dummy, dummy, -1, 16, 0, dummy, dummy, dummy, None)),
        ('of_surface_sample', lambda: lib.of_surface_sample(dummy, dummy, dummy, dummy, 2, 0, 0, dummy, dummy, dummy, None)),
        ('of_surface_sample', lambda: lib.of_surface_sample(dummy, dummy, None, dummy, 2, 16, 0, dummy, dummy, dummy, None)),
    ]
    for name, call in cases:
        assert call() == -1, name
        assert name.encode() in lib.of_last_error()
    assert lib.of_mesh_bbox(dummy, dummy, 0, dummy, None) == 0                   # empty batch: nothing to do
    assert lib.of_surface_sample(dummy, dummy, dummy, dummy, 0, 16, 0, dummy, dummy, dummy, None) == 0
    assert _lib.launch_count() == n0


def test_mesh_functions_refuse_cpu_tensors():
    import torch
    from octfusion_b200 import mesh as M
    g = torch.from_numpy(MU.sphere(8, 2.0))
    for fn in (M.marching_cubes, M.pointclouds_from_sdfs):
        with pytest.raises(RuntimeError, match='no CPU path'):
            fn(g)
