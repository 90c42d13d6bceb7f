"""Meshes and metric point clouds on the GPU: marching cubes over the `calc_sdf` grid and area-weighted surface sampling.

Connects `mpu.calc_sdf` ([B, R, R, R] fp32 SDF grids on the device) to `metrics.compute_all_metrics` ([B, P, 3] point
clouds) without leaving the device.  Replaces, in the reference,
  skimage.measure.marching_cubes(sdf, level)[:2] + the vertex mapping of export_mesh
      (models/octfusion_model_union.py:435-468)            -> marching_cubes(...).mesh(b), to_world(...)
  scale_to_unit_cube + trimesh mesh.sample(2048)
      (metrics/generate_pointclouds.py:14-37)               -> pointclouds_from_sdfs(...)
The kernels are in csrc/mesh.cu; conventions (inside is f < level, vertex and face order, winding) are stated in
include/octfusion_b200.h.  Inputs must be CUDA tensors: there is no CPU path.
"""
from __future__ import annotations
import ctypes as C
import torch

from ._lib import lib, ptr, stream, check, require_cuda, MC_MAX_SIZE

__all__ = ['MeshBatch', 'marching_cubes', 'to_world', 'sample_surface', 'pointclouds_from_sdfs']


class MeshBatch:
    """Packed meshes of a batch: verts [V, 3] fp32 (index space of the grid), faces [F, 3] int32 with shape-local
    vertex ids, vert_offsets / face_offsets int64 [B + 1] on the device; shape b owns rows
    vert_offsets[b] .. vert_offsets[b + 1] and face_offsets[b] .. face_offsets[b + 1]."""

    def __init__(self, verts, faces, vert_offsets, face_offsets):
        self.verts, self.faces = verts, faces
        self._vo, self._fo = list(vert_offsets), list(face_offsets)
        self.vert_offsets = torch.tensor(self._vo, dtype=torch.int64, device=verts.device)
        self.face_offsets = torch.tensor(self._fo, dtype=torch.int64, device=verts.device)

    def __len__(self):
        return len(self._vo) - 1

    def num_faces(self, b):
        return self._fo[b + 1] - self._fo[b]

    def mesh(self, b):
        """(verts [V_b, 3], faces [F_b, 3]) of shape b, as views"""
        return self.verts[self._vo[b]:self._vo[b + 1]], self.faces[self._fo[b]:self._fo[b + 1]]


def _grids(sdfs):
    if not isinstance(sdfs, torch.Tensor):
        raise TypeError('octfusion_b200.mesh: sdfs must be a tensor')
    require_cuda(sdfs)
    if sdfs.dtype != torch.float32:
        raise TypeError('octfusion_b200.mesh: sdfs must be float32, got %s' % sdfs.dtype)
    if sdfs.dim() == 3:
        sdfs = sdfs.unsqueeze(0)
    if sdfs.dim() != 4 or not sdfs.shape[1] == sdfs.shape[2] == sdfs.shape[3]:
        raise ValueError('octfusion_b200.mesh: sdfs must be [B, R, R, R] or [R, R, R], got %s' % (tuple(sdfs.shape),))
    if not 2 <= sdfs.shape[1] <= MC_MAX_SIZE:
        raise ValueError('octfusion_b200.mesh: grid side must be in [2, %d], got %d' % (MC_MAX_SIZE, sdfs.shape[1]))
    return sdfs.contiguous()


def _at(t, row):
    """pointer to row `row` of a 2-D contiguous tensor"""
    return C.c_void_p(t.data_ptr() + row * t.stride(0) * t.element_size())


@torch.no_grad()
def marching_cubes(sdfs, level=0.0) -> MeshBatch:
    """Isosurface f = level of each [R, R, R] grid (i = x slowest, the layout of calc_sdf).  Vertices are in index
    space, one per grid edge whose ends lie on different sides (inside is f < level), linearly interpolated from the
    lower-index end; faces wind outward for an SDF that is negative inside.  A grid without crossing gives an empty
    mesh.  One host synchronisation per call (the sizes of all meshes are fetched together)."""
    sdfs = _grids(sdfs)
    dev = sdfs.device
    B, R = sdfs.shape[0], sdfs.shape[1]
    n = R ** 3
    lv = float(level)
    with torch.cuda.device(dev):
        st = stream()
        # scratch independent of B, reused shape after shape
        vcnt = torch.empty(n, dtype=torch.int32, device=dev)
        tcnt = torch.empty(n, dtype=torch.int32, device=dev)
        vscan = torch.empty(n + 1, dtype=torch.int32, device=dev)
        tscan = torch.empty(n + 1, dtype=torch.int32, device=dev)
        scratch = torch.empty(int(lib.of_scan_scratch_bytes(n)), dtype=torch.uint8, device=dev)
        totals = torch.empty(B, 2, dtype=torch.int32, device=dev)

        def count_and_scan(b, want_totals):
            g = sdfs[b]
            check(lib.of_mc_count(ptr(g), R, lv, ptr(vcnt), ptr(tcnt), st), 'of_mc_count')
            check(lib.of_exclusive_scan_i32(ptr(vcnt), ptr(vscan), n, _at(totals, b) if want_totals else None,
                                            ptr(scratch), st), 'of_exclusive_scan_i32')
            check(lib.of_exclusive_scan_i32(ptr(tcnt), ptr(tscan), n,
                                            C.c_void_p(_at(totals, b).value + 4) if want_totals else None,
                                            ptr(scratch), st), 'of_exclusive_scan_i32')

        for b in range(B):
            count_and_scan(b, True)
        tot = totals.cpu().tolist()
        vo, fo = [0], [0]
        for nv, nf in tot:
            vo.append(vo[-1] + nv)
            fo.append(fo[-1] + nf)
        verts = torch.empty(vo[-1], 3, dtype=torch.float32, device=dev)
        faces = torch.empty(fo[-1], 3, dtype=torch.int32, device=dev)
        # the scans of the last shape are still in place: emit it first, recount the others
        for b in reversed(range(B)):
            if tot[b][0] == 0:
                continue
            if b != B - 1:
                count_and_scan(b, False)
            check(lib.of_mc_emit(ptr(sdfs[b]), R, lv, ptr(vscan), ptr(tscan), _at(verts, vo[b]), _at(faces, fo[b]), st),
                  'of_mc_emit')
        return MeshBatch(verts, faces, vo, fo)


@torch.no_grad()
def to_world(verts, size, bbmin, bbmax, mesh_scale=1.0):
    """The vertex mapping of export_mesh (models/octfusion_model_union.py:456-457) in fp32 and in its order:
    (verts * ((bbmax - bbmin) / size) + bbmin) * mesh_scale.  bbmin / bbmax are floats or 3-sequences."""
    require_cuda(verts)
    lo = torch.as_tensor(bbmin, dtype=torch.float64)
    step = ((torch.as_tensor(bbmax, dtype=torch.float64) - lo) / size).to(torch.float32).to(verts.device)
    scale = torch.as_tensor(mesh_scale, dtype=torch.float32).to(verts.device)
    return (verts * step + lo.to(torch.float32).to(verts.device)) * scale


def _empty_shapes(meshes):
    return [b for b in range(len(meshes)) if meshes.num_faces(b) == 0]


@torch.no_grad()
def sample_surface(meshes: MeshBatch, count: int, seed: int = 0):
    """(points [B, count, 3] fp32, face_index [B, count] int32): trimesh `sample_surface` on every mesh of the batch
    (faces chosen with probability proportional to their area, zero-area faces never; points uniform on the face).
    Random numbers are Philox keyed by (seed, shape, sample): the same seed gives identical results."""
    if not isinstance(meshes, MeshBatch):
        raise TypeError('octfusion_b200.mesh: sample_surface takes the MeshBatch of marching_cubes')
    count = int(count)
    if count < 1:
        raise ValueError('octfusion_b200.mesh: count must be >= 1, got %d' % count)
    if not 0 <= int(seed) < 2 ** 64:
        raise ValueError('octfusion_b200.mesh: seed must be in [0, 2^64)')
    empty = _empty_shapes(meshes)
    if empty:
        raise ValueError('octfusion_b200.mesh: shapes %s have an empty mesh; there is no surface to sample' % empty)
    B, dev = len(meshes), meshes.verts.device
    with torch.cuda.device(dev):
        cum = torch.empty(meshes.faces.shape[0], dtype=torch.float64, device=dev)
        points = torch.empty(B, count, 3, dtype=torch.float32, device=dev)
        face_index = torch.empty(B, count, dtype=torch.int32, device=dev)
        if B:
            check(lib.of_surface_sample(ptr(meshes.verts), ptr(meshes.vert_offsets), ptr(meshes.faces),
                                        ptr(meshes.face_offsets), B, count, int(seed), ptr(cum), ptr(points),
                                        ptr(face_index), stream()), 'of_surface_sample')
    return points, face_index


@torch.no_grad()
def pointclouds_from_sdfs(sdfs, n: int = 2048, level=0.0, seed: int = 0):
    """[B, n, 3] fp32 metric point clouds of [B, R, R, R] SDF grids: marching_cubes, sample_surface, then
    scale_to_unit_cube (metrics/generate_pointclouds.py:14-21, padding 0: centre of the vertex bounding box to the
    origin, largest extent to 2) applied to the samples.  The normalisation removes any a * v + b map with a > 0, so
    the to_world step of export_mesh is not needed here.  Feeds metrics.compute_all_metrics directly."""
    meshes = marching_cubes(sdfs, level)
    empty = _empty_shapes(meshes)
    if empty:
        raise ValueError('octfusion_b200.mesh: shapes %s have an empty mesh at level %g' % (empty, float(level)))
    points, _ = sample_surface(meshes, n, seed)
    B, dev = len(meshes), points.device
    with torch.cuda.device(dev):
        bbox = torch.empty(B, 6, dtype=torch.float32, device=dev)
        check(lib.of_mesh_bbox(ptr(meshes.verts), ptr(meshes.vert_offsets), B, ptr(bbox), stream()), 'of_mesh_bbox')
    lo, hi = bbox[:, :3], bbox[:, 3:]
    scale = 2.0 / (hi - lo).amax(1)
    return ((points - ((lo + hi) * 0.5)[:, None]) * scale[:, None, None]).contiguous()
