"""Grids and surface checks shared by the mesh tests (numpy, CPU)."""
import numpy as np


def _coords(r):
    x = np.arange(r, dtype=np.float64)
    return np.meshgrid(x, x, x, indexing='ij')


def sphere(r, radius, centre=None):
    c = ((r - 1) / 2,) * 3 if centre is None else centre
    X, Y, Z = _coords(r)
    return (np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2) - radius).astype(np.float32)


def torus(r, major, minor):
    c = (r - 1) / 2
    X, Y, Z = _coords(r)
    return (np.sqrt((np.sqrt((X - c) ** 2 + (Y - c) ** 2) - major) ** 2 + (Z - c) ** 2) - minor).astype(np.float32)


def two_spheres(r, radius):
    c = (r - 1) / 2
    return np.minimum(sphere(r, radius, (r * 0.27, c, c)), sphere(r, radius, (r * 0.73, c, c)))


def plane(r, level=0.0):
    """f = x + 0.5 y - 0.3 z - r / 2 + level: a slanted plane cut by the grid boundary"""
    X, Y, Z = _coords(r)
    return (X + 0.5 * Y - 0.3 * Z - r / 2 + level).astype(np.float32)


def noise(r, seed, border=True):
    g = np.random.default_rng(seed).standard_normal((r, r, r)).astype(np.float32)
    if border:
        close(g)
    return g


def close(g, value=1.0):
    """force the border of the grid outside, so the surface is closed"""
    g[[0, -1]] = value
    g[:, [0, -1]] = value
    g[:, :, [0, -1]] = value
    return g


def edge_counts(faces):
    """(directed-edge multiplicities, undirected edges [E, 2], their multiplicities)"""
    f = np.asarray(faces, dtype=np.int64)
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    directed = np.unique(e, axis=0, return_counts=True)[1]
    und, cnt = np.unique(np.sort(e, 1), axis=0, return_counts=True)
    return directed, und, cnt


def assert_closed_oriented(faces):
    """every undirected edge in exactly two faces, every directed edge in exactly one (consistent winding)"""
    directed, _, cnt = edge_counts(faces)
    assert len(faces) > 0
    assert cnt.min() == 2 and cnt.max() == 2, (cnt.min(), cnt.max())
    assert directed.max() == 1


def euler(verts, faces):
    _, und, _ = edge_counts(faces)
    return len(verts) - len(und) + len(faces)


def volume(verts, faces):
    """enclosed volume by the divergence theorem (positive for outward winding)"""
    v = np.asarray(verts, dtype=np.float64)[np.asarray(faces, dtype=np.int64)]
    return float(np.einsum('ij,ij->i', v[:, 0], np.cross(v[:, 1], v[:, 2])).sum() / 6)
