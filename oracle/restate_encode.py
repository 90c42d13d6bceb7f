"""TEST INFRASTRUCTURE.  torch restatement of the ocnn symbols on the way from point clouds into the GraphVAE: `Points`,
`merge_points`, `Octree.build_octree`, `merge_octrees` and `InputFeature('ND')`.  No reference file fixes them: they
are recalled from ocnn-pytorch 2.2.x (SURVEY.md Appendix B) and their parity is UNPINNED at the ocnn boundary.  The
octree class extends the `ocnn_shim` Octree, so the unmodified reference (oracle/ref_import.py) accepts it; the shim
itself has no point-cloud path.  Tensors may live on any device (tools/bench_encode.py runs this on the GPU as the
"port" arm)."""
import torch

from oracle.ref_import import ensure_shim

ensure_shim()
from ocnn.octree import Octree as _ShimOctree, xyz2key     # noqa: E402
from ocnn.nn import octree_pad                             # noqa: E402

_BATCH_SHIFT = 48
_KEY_MASK = (1 << 48) - 1


class Points:
    """ocnn Points (datasets/dualoctree_snet.py:42): points [N, 3], normals [N, 3] or None, batch_id [N]."""

    def __init__(self, points, normals=None, features=None, labels=None, batch_id=None, batch_size=1):
        self.points, self.normals, self.features, self.labels = points, normals, features, labels
        self.batch_size = batch_size
        self.batch_id = batch_id if batch_id is not None else torch.zeros(points.shape[0], dtype=torch.long,
                                                                          device=points.device)

    def clip(self, min=-1.0, max=1.0, esp=0.01):
        """dualoctree_snet.py:45: keep the points with every coordinate strictly inside (min + esp, max - esp)."""
        mask = torch.all(self.points > min + esp, dim=1) & torch.all(self.points < max - esp, dim=1)
        self.points = self.points[mask]
        self.normals = self.normals[mask] if self.normals is not None else None
        self.batch_id = self.batch_id[mask]


def merge_points(points, update_batch_info=True):
    """shapes concatenated in order, batch ids 0..B-1."""
    normals = torch.cat([p.normals for p in points]) if all(p.normals is not None for p in points) else None
    bid = torch.cat([torch.full((p.points.shape[0],), i, dtype=torch.long, device=p.points.device)
                     for i, p in enumerate(points)])
    return Points(torch.cat([p.points for p in points]), normals, batch_id=bid, batch_size=len(points))


class Octree(_ShimOctree):
    """the shim's Octree plus `points[d]` / `normals[d]` and `build_octree`."""

    def __init__(self, depth, full_depth=2, batch_size=1, device='cpu', **kw):
        super().__init__(depth, full_depth, batch_size, device, **kw)
        self.points = [None] * (depth + 1)
        self.normals = [None] * (depth + 1)

    def to(self, device):
        super().to(device)
        self.points = [p.to(self.device) if p is not None else None for p in self.points]
        self.normals = [p.to(self.device) if p is not None else None for p in self.normals]
        return self

    def build_octree(self, point_cloud):
        """ocnn-pytorch 2.2.x Octree.build_octree (models/octfusion_model_vae.py:135-146, octfusion_model_union.py:200-212;
        UNPINNED): p' = (p + 1) * 2^(depth-1) in fp32, cell = long(p') & (2^depth - 1) (truncation toward zero, then the
        mask of xyz2key: +1.0 wraps to cell 0), key = xyz2key(cell, batch).  Depths 0..full_depth are full layers;
        below, the keys of depth d are the 8 children of every distinct depth-(d-1) key, children[d] the rank of each
        among the distinct depth-d keys (-1 where none), and at full_depth children = rank of the non-empty nodes, -1
        elsewhere.  points[depth] = mean of p' per non-empty depth-`depth` node, normals[depth] = F.normalize(sum of
        normals)."""
        D, fd = self.depth, self.full_depth
        pts = point_cloud.points.float()
        dev = pts.device
        scaled = (pts + 1.0) * 2 ** (D - 1)
        cell = scaled.long() & ((1 << D) - 1)
        bid = point_cloud.batch_id.reshape(-1).long()
        key = xyz2key(cell[:, 0], cell[:, 1], cell[:, 2], bid, D)
        for d in range(fd + 1):
            self.octree_grow_full(d)
        uniq = {}
        for d in range(fd, D + 1):
            kd = ((key & _KEY_MASK) >> (3 * (D - d))) | ((key >> _BATCH_SHIFT) << _BATCH_SHIFT)
            uniq[d] = torch.unique(kd)
        u = uniq[fd]
        full = (u >> _BATCH_SHIFT) * 8 ** fd + (u & _KEY_MASK)
        child = torch.full((int(self.nnum[fd]),), -1, dtype=torch.int32, device=dev)
        child[full] = torch.arange(u.numel(), dtype=torch.int32, device=dev)
        self.children[fd] = child
        self.nnum_nempty[fd] = u.numel()
        for d in range(fd + 1, D + 1):
            par, u = uniq[d - 1], uniq[d]
            bb = (par >> _BATCH_SHIFT) << _BATCH_SHIFT
            kk = ((par & _KEY_MASK) << 3).unsqueeze(1) + torch.arange(8, device=dev)
            self.keys[d] = (bb.unsqueeze(1) | kk).reshape(-1)
            parent_of = ((u & _KEY_MASK) >> 3) | ((u >> _BATCH_SHIFT) << _BATCH_SHIFT)
            slot = torch.searchsorted(par, parent_of) * 8 + (u & 7)
            child = torch.full((8 * par.numel(),), -1, dtype=torch.int32, device=dev)
            child[slot] = torch.arange(u.numel(), dtype=torch.int32, device=dev)
            self.children[d] = child
            self.nnum[d], self.nnum_nempty[d] = 8 * par.numel(), u.numel()
        node = torch.searchsorted(uniq[D], key)
        m = uniq[D].numel()
        count = torch.zeros(m, device=dev).index_add_(0, node, torch.ones(node.numel(), device=dev))
        self.points[D] = torch.zeros(m, 3, device=dev).index_add_(0, node, scaled) / count.unsqueeze(1)
        if point_cloud.normals is not None:
            nsum = torch.zeros(m, 3, device=dev).index_add_(0, node, point_cloud.normals.float())
            self.normals[D] = torch.nn.functional.normalize(nsum, dim=1, eps=1e-12)
        return self


def merge_octrees(octrees):
    """models/octfusion_model_vae.py:144: one batched octree from per-shape octrees of the same depth -- per depth the
    keys concatenated with the batch ids shifted, the non-empty ranks offset by the preceding shapes' counts."""
    o0 = octrees[0]
    out = Octree(o0.depth, o0.full_depth, sum(o.batch_size for o in octrees), o0.device)
    for d in range(o0.depth + 1):
        keys, child, b0, r0 = [], [], 0, 0
        for o in octrees:
            c = o.children[d]
            keys.append(o.keys[d] + (b0 << _BATCH_SHIFT))
            child.append(torch.where(c >= 0, c + r0, c))
            b0 += o.batch_size
            r0 += int(o.nnum_nempty[d])
        out.keys[d], out.children[d] = torch.cat(keys), torch.cat(child)
        out.nnum[d] = sum(int(o.nnum[d]) for o in octrees)
        out.nnum_nempty[d] = r0
    for name in ('points', 'normals'):
        parts = [getattr(o, name)[o0.depth] for o in octrees]
        if all(p is not None for p in parts):
            getattr(out, name)[o0.depth] = torch.cat(parts)
    return out


class InputFeature:
    """ocnn-pytorch 2.2.x InputFeature, letters N and D (dual_octree.py:345): [normals[D] | sum((points[D].frac() - 0.5)
    * normals[D])] per non-empty depth-D node, padded with zero rows over all nnum[D] nodes (octree_pad) unless
    nempty."""

    def __init__(self, feature='ND', nempty=False):
        self.feature, self.nempty = feature.upper(), nempty
        if set(self.feature) - set('ND') or not self.feature:
            raise NotImplementedError('InputFeature letters other than N and D are not restated')

    def __call__(self, octree):
        D = octree.depth
        feats = []
        for ch in self.feature:
            if ch == 'N':
                feats.append(octree.normals[D])
            else:
                local = octree.points[D].frac() - 0.5
                feats.append((local * octree.normals[D]).sum(dim=1, keepdim=True))
        out = torch.cat(feats, dim=1)
        return out if self.nempty else octree_pad(out, octree, D)
