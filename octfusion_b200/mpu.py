"""NeuralMPU: evaluates the implicit function defined by the GraphVAE decoder's per-node regression values at
arbitrary query points (SURVEY.md 8f rank 4).  Drop-in for reference models/networks/dualoctree_networks/mpu.py
`NeuralMPU`: same constructor and call signature, returns {depth: (fval [P], flgs [P] bool)}.  One CUDA kernel per
target depth (csrc/mpu.cu) instead of the reference's key search + two sparse-matrix products per depth."""
from __future__ import annotations
import ctypes as C
import torch

from ._lib import lib, ptr, stream, check, OctreeLevels, require_cuda


def _levels(octree, depth):
    lv = OctreeLevels()
    lv.full_depth, lv.depth, lv.batch = octree.full_depth, depth, octree.batch_size
    keep = []
    for d in range(octree.full_depth, depth + 1):
        ch = octree.children[d].contiguous()
        assert ch.dtype == torch.int32 and ch.is_cuda
        lv.children[d] = ch.data_ptr()
        lv.nnum[d] = int(octree.nnum[d])
        keep.append(ch)
    return lv, keep


class NeuralMPU:
    def __init__(self, full_depth, depth_stop, depth):
        self.full_depth, self.depth_stop, self.depth = full_depth, depth_stop, depth

    @torch.no_grad()
    def __call__(self, pos, reg_voxs, octree_out):
        require_cuda(pos)
        pos = pos.float().contiguous()
        assert pos.dim() == 2 and pos.shape[1] == 4
        n = pos.shape[0]
        mpus = {}
        for d in range(self.depth_stop, self.depth + 1):
            reg = reg_voxs[d].float().contiguous()
            want = int(octree_out.nnum[self.full_depth:d + 1].sum())
            assert reg.shape == (want, 4), 'reg_voxs[%d] must hold one row per octree node of depths %d..%d' % (
                d, self.full_depth, d)
            lv, keep = _levels(octree_out, d)
            fval = torch.empty(n, dtype=torch.float32, device=pos.device)
            hit = torch.empty(n, dtype=torch.uint8, device=pos.device)
            check(lib.of_mpu_eval(C.byref(lv), d, ptr(pos), n, ptr(reg), ptr(fval), ptr(hit), stream()), 'of_mpu_eval')
            del keep
            mpus[d] = (fval, hit.bool())
        return mpus


    @torch.no_grad()
    def eval_grid(self, reg_voxs, octree_out, batch_idx: int, size: int, bbmin: float, bbmax: float, head: int, count: int,
                  out: torch.Tensor, depth=None):
        """SDF at depth `depth` (default: the finest) at points [head, head+count) of the size^3 sampling grid of shape
        `batch_idx`, written into out[head:head+count] (of_mpu_eval_grid: coordinates are generated inside the kernel)."""
        d = self.depth if depth is None else depth
        reg = reg_voxs[d].float().contiguous()
        lv, keep = _levels(octree_out, d)
        check(lib.of_mpu_eval_grid(C.byref(lv), d, batch_idx, size, float(bbmin), float(bbmax), head, count, ptr(reg),
                                   ptr(out), stream()), 'of_mpu_eval_grid')
        del keep
        return out


def get_mgrid(size: int, dim: int = 3, device='cuda'):
    """reference utils/util_dualoctree.py:23-42: [size^dim, dim] float32 grid indices, first index slowest."""
    c = torch.arange(size, dtype=torch.float32, device=device)
    return torch.stack(torch.meshgrid(*([c] * dim), indexing='ij'), -1).reshape(size ** dim, dim)


@torch.no_grad()
def calc_sdf(model, batch_size: int = 1, size: int = 256, max_batch: int = 64 ** 3, bbmin: float = -1.0, bbmax: float = 1.0):
    """Drop-in for reference utils/util_dualoctree.py:99-118: the SDF of `batch_size` shapes on a size^3 grid,
    [B, size, size, size] fp32 on the device, evaluated in chunks of `max_batch` points.  `model` maps [P, 4] points
    (x, y, z, batch index) to SDF values.  When it is the `neural_mpu` closure of `GraphVAE.decode_code` or
    `GraphVAE.forward` (it carries `.mpu_args`: the NeuralMPU, reg_voxs, octree and optionally the depth), the grid coordinates are generated inside the evaluation kernel; any other callable gets explicit
    point tensors exactly as in the reference."""
    num = size ** 3
    args = getattr(model, 'mpu_args', None)
    dev = args[2].device if args is not None else 'cuda'
    sdfs = torch.empty((batch_size, num), dtype=torch.float32, device=dev)
    samples = None
    for b in range(batch_size):
        head = 0
        while head < num:
            tail = min(head + max_batch, num)
            if args is not None:
                mpu, reg_voxs, octree_out = args[:3]
                mpu.eval_grid(reg_voxs, octree_out, b, size, bbmin, bbmax, head, tail - head, sdfs[b],
                              depth=args[3] if len(args) > 3 else None)
            else:
                if samples is None:
                    samples = get_mgrid(size, 3, dev) * ((bbmax - bbmin) / size) + bbmin
                pts = torch.cat([samples[head:tail], torch.full((tail - head, 1), float(b), device=dev)], 1)
                sdfs[b, head:tail] = model(pts).reshape(-1)
            head += max_batch
    return sdfs.reshape(batch_size, size, size, size)
