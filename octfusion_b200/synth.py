"""Seeded synthetic ShapeNet-shaped octree occupancy (benchmark / test INPUT generator).

No dataset is reachable from the build or the GPU box, so the benchmark workload of
BASELINE.json configs[1] ("depth-6 ShapeNet-shaped random octree") is generated: per shape a
random ellipsoid *shell* (a closed surface, like a ShapeNet mesh) is rasterised at depth 4
and depth 5; a cell is non-empty when it lies within `halfwidth[level]` cells of the surface
(1.55 / 1.1 cells reproduce the node counts SURVEY.md section 8 quotes: N5 ~ 7 k, N6 ~ 20 k per shape).
What comes out is exactly what stage 1 of the reference hands to stage 2
(reference utils/util_dualoctree.py:225-250, `split2octree_small`): a per-node split
label at full_depth and at full_depth+1, in octree (Morton key) order.

Pure torch-CPU integer/float math with an explicit Generator => identical on every host.
"""
from __future__ import annotations
import torch


def _morton_to_xyz(idx: torch.Tensor, depth: int):
    x = torch.zeros_like(idx); y = torch.zeros_like(idx); z = torch.zeros_like(idx)
    for i in range(depth):
        x |= ((idx >> (3 * i + 2)) & 1) << i
        y |= ((idx >> (3 * i + 1)) & 1) << i
        z |= ((idx >> (3 * i)) & 1) << i
    return x, y, z


def _in_shell(x, y, z, depth, centre, axes, halfwidth):
    h = 2.0 / (1 << depth)                                # cell size in [-1,1]^3
    px = (x.double() + 0.5) * h - 1.0
    py = (y.double() + 0.5) * h - 1.0
    pz = (z.double() + 0.5) * h - 1.0
    f = torch.sqrt(((px - centre[0]) / axes[0]) ** 2 + ((py - centre[1]) / axes[1]) ** 2
                   + ((pz - centre[2]) / axes[2]) ** 2)
    amean = float(axes.mean())
    return (f - 1.0).abs() * amean < halfwidth * h


def synth_splits(batch_size: int, seed: int = 0, full_depth: int = 4, halfwidth=(1.55, 1.1)):
    """Returns (label_fd, label_fd1):
    label_fd  [B * 8^fd]         int64 0/1, nodes of the full layer in key order (batch major)
    label_fd1 [8 * sum(label_fd)] int64 0/1, children of the non-empty full-layer nodes.
    Depth = full_depth + 2 octree: every non-empty depth-(fd+1) node gets 8 depth-(fd+2) children.
    """
    g = torch.Generator().manual_seed(seed)
    nfull = 8 ** full_depth
    idx = torch.arange(nfull, dtype=torch.long)
    x4, y4, z4 = _morton_to_xyz(idx, full_depth)
    lab4, lab5 = [], []
    for _ in range(batch_size):
        u = torch.rand(8, generator=g, dtype=torch.float64)
        centre = (u[0:3] * 2 - 1) * 0.15
        r = 0.45 + 0.30 * u[3]
        axes = (0.6 + 0.8 * u[4:7]) * r
        m4 = _in_shell(x4, y4, z4, full_depth, centre, axes, halfwidth[0])
        if not bool(m4.any()):                       # degenerate guard: keep one cell
            m4[0] = True
        lab4.append(m4.long())
        p = idx[m4]
        child = (p.unsqueeze(1) << 3) + torch.arange(8)       # Morton keys at depth fd+1
        x5, y5, z5 = _morton_to_xyz(child.reshape(-1), full_depth + 1)
        m5 = _in_shell(x5, y5, z5, full_depth + 1, centre, axes, halfwidth[1])
        lab5.append(m5.long())
    return torch.cat(lab4), torch.cat(lab5)


def slice_splits(label_fd, label_fd1, lo: int, hi: int, full_depth: int = 4):
    """labels of shapes [lo, hi) out of a synth_splits(B, ...) result (batch sharding: every rank generates the same B
    shapes and keeps its contiguous block)."""
    nfull = 8 ** full_depth
    per = label_fd.view(-1, nfull).sum(1) * 8                  # depth-(fd+1) nodes per shape
    off = torch.cat([torch.zeros(1, dtype=per.dtype), torch.cumsum(per, 0)])
    return label_fd[lo * nfull: hi * nfull], label_fd1[int(off[lo]): int(off[hi])]


def synth_point_clouds(n: int, points: int, seed: int) -> torch.Tensor:
    """[n, points, 3] fp32 surface-like point clouds (the input of the shape metrics): per cloud, points on a random
    ellipsoid shell (semi-axes 0.2 .. 0.45, random centre inside the unit cube) with 1 % radial noise."""
    g = torch.Generator().manual_seed(seed)
    direction = torch.randn(n, points, 3, generator=g)
    direction = direction / direction.norm(dim=-1, keepdim=True)
    axes = 0.2 + 0.25 * torch.rand(n, 1, 3, generator=g)
    centre = 0.45 + 0.1 * torch.rand(n, 1, 3, generator=g)
    radial = 1.0 + 0.01 * torch.randn(n, points, 1, generator=g)
    return (centre + direction * axes * radial).float().contiguous()
