"""Octree container with the field layout the reference reads from `ocnn.octree.Octree`
(third-party, un-vendored; call sites: reference dual_octree.py:28-44, utils/util_dualoctree.py:232-248,
ldm_diffusion_util.py:318-325).  Keys are 64-bit: Morton code (x at bit 3i+2, y at 3i+1, z at 3i,
child index = 4x+2y+z as the reference's lookup tables dual_octree.py:90-112 assume) in bits 0-47,
batch index from bit 48 (dual_octree.py:75).

This is host-side setup that runs once per batch of shapes (SURVEY.md 8f-2 marks the stage-1 ->
stage-2 handoff as a "next" row); the per-step hot path never touches it.

`Points` / `merge_points` / `Octree.build_octree` restate ocnn-pytorch 2.2.x (SURVEY.md Appendix B; parity UNPINNED at
the ocnn boundary): the way into the VAE's latent space (reference models/octfusion_model_vae.py:135-146,
datasets/dualoctree_snet.py:31-45).  The build runs on the CUDA kernels of csrc/points.cu.
"""
from __future__ import annotations
import ctypes as C
import torch

BATCH_SHIFT = 48
KEY_MASK = (1 << 48) - 1
MAX_DEPTH = 16             # 48-bit Morton key
MAX_BATCH = 1024           # batch bits 48..57


class Points:
    """ocnn.octree.Points subset: points [N, 3], normals [N, 3] or None, batch_id [N] int64 (shapes contiguous and in
    order), batch_size."""

    def __init__(self, points, normals=None, batch_id=None, batch_size: int = 1):
        self.points, self.normals, self.batch_size = points, normals, batch_size
        self.batch_id = batch_id if batch_id is not None else torch.zeros(
            points.shape[0], dtype=torch.long, device=points.device)
        self.device = points.device

    def clip(self, min: float = -1.0, max: float = 1.0, esp: float = 0.01):
        """keeps the points with every coordinate strictly inside (min + esp, max - esp), with their normals and
        batch ids."""
        mask = ((self.points > min + esp) & (self.points < max - esp)).all(1)
        self.points = self.points[mask]
        self.normals = self.normals[mask] if self.normals is not None else None
        self.batch_id = self.batch_id[mask]

    def cuda(self):
        return self.to('cuda')

    def to(self, device):
        self.points = self.points.to(device)
        self.normals = self.normals.to(device) if self.normals is not None else None
        self.batch_id = self.batch_id.to(device)
        self.device = self.points.device
        return self


def merge_points(points: list):
    """ocnn.octree.merge_points: the shapes concatenated in order, batch ids 0..B-1."""
    has_normals = all(p.normals is not None for p in points)
    return Points(torch.cat([p.points for p in points]),
                  torch.cat([p.normals for p in points]) if has_normals else None,
                  torch.cat([torch.full((p.points.shape[0],), i, dtype=torch.long, device=p.points.device)
                             for i, p in enumerate(points)]),
                  len(points))


def xyz2key(x, y, z, b=None, depth: int = 16):
    x, y, z = x.long(), y.long(), z.long()
    key = torch.zeros_like(x)
    for i in range(depth):
        key |= (((x >> i) & 1) << (3 * i + 2)) | (((y >> i) & 1) << (3 * i + 1)) | (((z >> i) & 1) << (3 * i))
    if b is not None:
        key = key | (torch.as_tensor(b, device=key.device).long() << BATCH_SHIFT)
    return key


def key2xyz(key, depth: int = 16):
    key = key.long()
    b = key >> BATCH_SHIFT
    k = key & KEY_MASK
    x, y, z = torch.zeros_like(k), torch.zeros_like(k), torch.zeros_like(k)
    for i in range(depth):
        x |= ((k >> (3 * i + 2)) & 1) << i
        y |= ((k >> (3 * i + 1)) & 1) << i
        z |= ((k >> (3 * i)) & 1) << i
    return x, y, z, b


class Octree:
    def __init__(self, depth: int, full_depth: int = 2, batch_size: int = 1, device='cuda'):
        self.depth, self.full_depth, self.batch_size = depth, full_depth, batch_size
        self.device = torch.device(device)
        n = depth + 1
        self.keys = [None] * n
        self.children = [None] * n
        self.nnum = torch.zeros(n, dtype=torch.long)           # host counters (no device sync to read)
        self.nnum_nempty = torch.zeros(n, dtype=torch.long)
        self.points = [None] * n                               # build_octree: per non-empty node of `depth`
        self.normals = [None] * n

    def build_octree(self, point_cloud: Points):
        """ocnn Octree.build_octree (SURVEY.md Appendix B, UNPINNED): the octree of depth `self.depth` of every shape of
        `point_cloud` (batch ids 0..batch_size-1, each shape's points contiguous), full layers up to full_depth, plus
        points[depth] / normals[depth] (mean scaled point, normalised normal sum) per non-empty depth-`depth` node.
        csrc/points.cu; one host synchronisation (the node counts of all depths)."""
        from ._lib import lib, ptr, stream, check, require_cuda
        D, fd, B = self.depth, self.full_depth, self.batch_size
        if not (0 <= fd < D <= MAX_DEPTH and 1 <= B < MAX_BATCH):
            raise ValueError('build_octree: need 0 <= full_depth < depth <= %d and 1 <= batch_size < %d (got %d, %d, %d)'
                             % (MAX_DEPTH, MAX_BATCH, fd, D, B))
        xyz = point_cloud.points
        require_cuda(xyz)
        if xyz.dim() != 2 or xyz.shape[1] != 3:
            raise ValueError('build_octree: points must be [N, 3]')
        xyz = xyz.to(device=self.device, dtype=torch.float32).contiguous()
        nrm = point_cloud.normals
        if nrm is not None:
            if nrm.shape != xyz.shape:
                raise ValueError('build_octree: normals must be [N, 3] like the points')
            nrm = nrm.to(device=self.device, dtype=torch.float32).contiguous()
        n = xyz.shape[0]
        bid = point_cloud.batch_id.to(self.device).reshape(-1).long()
        offsets = torch.searchsorted(bid, torch.arange(B + 1, device=self.device))
        unsorted = (bid[1:] < bid[:-1]).sum().view(1).int()
        nbytes = int(lib.of_octree_build_bytes(n, B, D, fd))
        if nbytes < 0:
            check(nbytes, 'of_octree_build_bytes')
        scratch = torch.empty(max(nbytes, 8), dtype=torch.uint8, device=self.device)
        counts = torch.empty(D + 2, dtype=torch.int32, device=self.device)
        check(lib.of_octree_build_levels(ptr(xyz), ptr(offsets), n, B, D, fd, ptr(scratch), ptr(counts), stream()),
              'of_octree_build_levels')
        got = torch.cat([counts, unsorted]).tolist()                         # the one host synchronisation
        if got[D + 1] or got[D + 2]:
            raise ValueError('build_octree: batch ids must be 0..batch_size-1 with each shape contiguous')
        for d in range(fd + 1):
            self.octree_grow_full(d)
        for d in range(fd, D + 1):
            nnum = B * 8 ** fd if d == fd else 8 * got[d - 1]
            keys = torch.empty(nnum, dtype=torch.long, device=self.device) if d > fd else None
            child = torch.empty(nnum, dtype=torch.int32, device=self.device)
            check(lib.of_octree_build_fill(ptr(scratch), n, B, D, fd, d, nnum, ptr(keys), ptr(child), stream()),
                  'of_octree_build_fill')
            if keys is not None:
                self.keys[d] = keys
            self.children[d] = child
            self.nnum[d], self.nnum_nempty[d] = nnum, got[d]
        self.points[D] = torch.empty((got[D], 3), dtype=torch.float32, device=self.device)
        self.normals[D] = torch.empty((got[D], 3), dtype=torch.float32, device=self.device) if nrm is not None else None
        check(lib.of_octree_build_signal(ptr(scratch), n, B, D, fd, ptr(xyz), ptr(nrm), ptr(self.points[D]),
                                         ptr(self.normals[D]), stream()), 'of_octree_build_signal')
        return self

    # growth: same semantics as the ocnn calls in ldm_diffusion_util.py:318-325 / util_dualoctree.py:238-248
    def octree_grow_full(self, depth: int, update_neigh: bool = False):
        num = 8 ** depth
        k = torch.arange(num, dtype=torch.long, device=self.device)
        b = torch.arange(self.batch_size, dtype=torch.long, device=self.device)
        self.keys[depth] = ((b.unsqueeze(1) << BATCH_SHIFT) | k.unsqueeze(0)).reshape(-1)
        self.children[depth] = torch.arange(num * self.batch_size, dtype=torch.int32, device=self.device)
        self.nnum[depth] = num * self.batch_size
        self.nnum_nempty[depth] = num * self.batch_size

    def octree_split(self, split, depth: int):
        split = split.to(self.device).long()
        rank = torch.cumsum(split, 0) - 1
        self.children[depth] = torch.where(split > 0, rank, torch.full_like(rank, -1)).int()
        self.nnum_nempty[depth] = int(split.sum())

    def octree_grow(self, depth: int, update_neigh: bool = False):
        mask = self.children[depth - 1] >= 0
        kp = self.keys[depth - 1][mask]
        kk = ((kp & KEY_MASK) << 3).unsqueeze(1) + torch.arange(8, device=self.device)
        self.keys[depth] = (((kp >> BATCH_SHIFT).unsqueeze(1) << BATCH_SHIFT) | kk).reshape(-1)
        n = self.keys[depth].numel()
        self.children[depth] = torch.arange(n, dtype=torch.int32, device=self.device)
        self.nnum[depth] = n
        self.nnum_nempty[depth] = n

    def nempty_mask(self, depth: int):
        return self.children[depth] >= 0

    def key(self, depth: int, nempty: bool = False):
        k = self.keys[depth]
        return k[self.nempty_mask(depth)] if nempty else k

    def batch_id(self, depth: int, nempty: bool = False):
        return self.key(depth, nempty) >> BATCH_SHIFT

    def xyzb(self, depth: int, nempty: bool = False):
        return key2xyz(self.key(depth, nempty), depth)

    def to(self, device):
        self.device = torch.device(device)
        self.keys = [k.to(self.device) if k is not None else None for k in self.keys]
        self.children = [c.to(self.device) if c is not None else None for c in self.children]
        self.points = [p.to(self.device) if p is not None else None for p in self.points]
        self.normals = [p.to(self.device) if p is not None else None for p in self.normals]
        return self

    def cuda(self):
        return self.to('cuda')


def create_full_octree(depth: int, full_depth: int, batch_size: int, device):
    """reference ldm_diffusion_util.py:318-325."""
    octree = Octree(depth, full_depth, batch_size, device)
    for d in range(full_depth + 1):
        octree.octree_grow_full(d)
    octree.depth = full_depth
    return octree


def octree_from_splits(label_fd, label_fd1, batch_size: int, full_depth: int = 4, device='cuda'):
    """What reference util_dualoctree.py:225-250 (`split2octree_small`) builds from the stage-1
    split signal: depth = full_depth + 2, split labels at full_depth and full_depth + 1."""
    octree = create_full_octree(full_depth + 2, full_depth, batch_size, device)
    octree.octree_split(label_fd, full_depth)
    octree.octree_grow(full_depth + 1)
    octree.depth += 1
    octree.octree_split(label_fd1, full_depth + 1)
    octree.octree_grow(full_depth + 2)
    octree.depth += 1
    return octree


def split2octree_small(split, input_depth: int, full_depth: int):
    """reference utils/util_dualoctree.py:225-250: the stage-1 output `split` [B, 8, 2^fd, 2^fd, 2^fd] (sign = does
    child k of voxel (x, y, z) exist) -> octree of depth full_depth + 2.  A full-layer voxel is non-empty when any of
    its 8 children is; the children's own split labels are the 8 channels."""
    disc = split > 0
    octree = create_full_octree(input_depth, full_depth, split.shape[0], split.device)
    x, y, z, b = octree.xyzb(full_depth)
    octree.octree_split((disc.sum(1) > 0)[b, x, y, z].long(), full_depth)
    octree.octree_grow(full_depth + 1)
    octree.depth += 1
    x, y, z, b = octree.xyzb(full_depth, nempty=True)
    octree.octree_split(disc[b, :, x, y, z].reshape(-1).long(), full_depth + 1)
    octree.octree_grow(full_depth + 2)
    octree.depth += 1
    return octree


def octree2split_small(octree, full_depth: int):
    """reference utils/util_dualoctree.py:198-211: the inverse -- which children of every full-layer voxel are
    subdivided, as a [B, 8, 2^fd, 2^fd, 2^fd] tensor in {-1, +1}."""
    child = octree.children[full_depth + 1]
    sub = (child >= 0).reshape(-1, 8)                       # per non-empty full-layer node
    n = 2 ** full_depth
    out = torch.zeros((octree.batch_size, n, n, n, 8), dtype=torch.float32, device=child.device)
    x, y, z, b = octree.xyzb(full_depth, nempty=True)
    out[b, x, y, z] = sub.float()
    return 2 * out.permute(0, 4, 1, 2, 3).contiguous() - 1
