"""Vectorised numpy restatement of the mesh kernels of csrc/mesh.cu: marching cubes over one [R, R, R] grid with the
table of octfusion_b200/mc_table.py, and area-weighted surface sampling from explicit uniforms.

Same table, same fp32 interpolation expression, same vertex order (grid point linear index, then axis) and face order
(cell linear index, then table order) as the kernels, so `marching_cubes` is compared with the GPU bit for bit.
"""
from __future__ import annotations
import importlib.util
import os
import numpy as np


def _load_table_module():
    """octfusion_b200/mc_table.py is pure Python: load it by path, without importing the package (which loads the
    CUDA library)"""
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'octfusion_b200', 'mc_table.py')
    spec = importlib.util.spec_from_file_location('octfusion_mc_table', path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


T = _load_table_module()

_TAB = T.table()
TRI_COUNT = np.array([len(t) for t in _TAB], dtype=np.int64)
TRI_EDGES = np.full((256, T.MAX_TRIS, 3), -1, dtype=np.int64)
for _c, _tris in enumerate(_TAB):
    if _tris:
        TRI_EDGES[_c, :len(_tris)] = _tris
EDGE_AXIS = np.array([a for a, _, _ in T.EDGES], dtype=np.int64)
EDGE_CORNER = np.array([T.corner_xyz(c) for _, c, _ in T.EDGES], dtype=np.int64)     # [12, 3] lower corner offset


def marching_cubes(sdf, level=0.0):
    """verts [V, 3] fp32 in index space, faces [F, 3] int32 (kernel order)"""
    f = np.ascontiguousarray(sdf, dtype=np.float32)
    r = f.shape[0]
    assert f.shape == (r, r, r) and r >= 2
    lv = np.float32(level)
    inside = f < lv                                       # NaN compares False: outside
    cross = np.zeros((r, r, r, 3), dtype=bool)
    cross[:-1, :, :, 0] = inside[:-1] != inside[1:]
    cross[:, :-1, :, 1] = inside[:, :-1] != inside[:, 1:]
    cross[:, :, :-1, 2] = inside[:, :, :-1] != inside[:, :, 1:]
    flat = cross.reshape(-1)
    vid = np.full(flat.shape, -1, dtype=np.int64)
    vid[flat] = np.arange(int(flat.sum()))
    vid = vid.reshape(r, r, r, 3)

    p = np.argwhere(cross)                                # rows (i, j, k, axis) in (point, axis) order
    i, j, k, ax = p[:, 0], p[:, 1], p[:, 2], p[:, 3]
    step = np.eye(3, dtype=np.int64)[ax]
    fa = f[i, j, k]
    fb = f[i + step[:, 0], j + step[:, 1], k + step[:, 2]]
    t = (lv - fa) / (fb - fa)                             # fp32 sub, sub, div
    verts = np.stack([i, j, k], 1).astype(np.float32)
    verts[np.arange(len(ax)), ax] += t                    # fp32 add
    verts = verts.astype(np.float32)

    case = np.zeros((r - 1,) * 3, dtype=np.int64)
    for c in range(8):
        x, y, z = T.corner_xyz(c)
        case |= inside[x:r - 1 + x, y:r - 1 + y, z:r - 1 + z].astype(np.int64) << c
    cells = np.argwhere(TRI_COUNT[case] > 0)              # cell linear order
    cc = case[cells[:, 0], cells[:, 1], cells[:, 2]]
    edges = TRI_EDGES[cc]                                 # [n, 5, 3]
    valid = np.arange(T.MAX_TRIS)[None, :] < TRI_COUNT[cc][:, None]
    e = np.where(edges < 0, 0, edges)
    q = cells[:, None, None, :] + EDGE_CORNER[e]          # [n, 5, 3, 3]
    ids = vid[q[..., 0], q[..., 1], q[..., 2], EDGE_AXIS[e]]
    faces = ids[valid]
    assert (faces >= 0).all()
    return verts, faces.astype(np.int32).reshape(-1, 3)


def face_areas(verts, faces):
    """fp64 triangle areas of fp32 vertices"""
    v = verts.astype(np.float64)[faces]
    return 0.5 * np.linalg.norm(np.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0]), axis=1)


def sample_surface(verts, faces, u, r1, r2):
    """(points [n, 3] fp32, face_index [n]) for uniforms u in (0, 1] (face choice) and r1, r2 in [0, 1]
    (trimesh sample_surface semantics: searchsorted(side='left') of u * total area in the fp64 cumulative areas)"""
    cum = np.cumsum(face_areas(verts, faces))
    fi = np.searchsorted(cum, u.astype(np.float64) * cum[-1], side='left')
    r1, r2 = r1.astype(np.float32).copy(), r2.astype(np.float32).copy()
    flip = r1 + r2 > 1
    r1[flip], r2[flip] = np.abs(r1[flip] - 1), np.abs(r2[flip] - 1)
    v = verts[faces[fi]]
    pts = v[:, 0] + r1[:, None] * (v[:, 1] - v[:, 0]) + r2[:, None] * (v[:, 2] - v[:, 0])
    return pts.astype(np.float32), fi


def scale_to_unit_cube(points, verts):
    """reference metrics/generate_pointclouds.py:14-21 (padding 0) with the mesh's vertex bounding box"""
    lo, hi = verts.min(0), verts.max(0)
    return ((points - (lo + hi) / 2) * (2 / (hi - lo).max())).astype(np.float32)
