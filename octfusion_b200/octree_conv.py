"""`ocnn.nn.OctreeConv` behind the tap-gather GEMM -- the operator BASELINE.json's north star and configs[0] name
("single OctreeConv 3^3 k=8->8 on one depth-4 synthetic octree").

`ocnn` is a third-party package that is neither vendored nor installable here, and the reference never calls
`OctreeConv` (SURVEY.md section 0: its sparse convolution is the dual-octree `GraphConv`).  The class below keeps ocnn's
constructor / forward signature and parameter layout as recalled from ocnn-pytorch 2.2.x (SURVEY.md Appendix B):

    OctreeConv(in_channels, out_channels, kernel_size=[3], stride=1, nempty=False, direct_method=False,
               use_bias=False, max_buffer=...)      weights [27, Cin, Cout] (+ bias [Cout])
    forward(data [N, Cin], octree, depth) -> [N', Cout]
    neigh = octree.get_neigh(depth, '333', stride, nempty);  out = gather(data, neigh).flatten(1) @ weights.flatten(0, 1)

**Parity is unpinned at the ocnn boundary** (no source, no test of the reference fixes tap order or weight layout).
What IS checked: on a full octree layer the operator equals `torch.nn.functional.conv3d` with zero padding (kernel index
[dx+1, dy+1, dz+1], voxel grid indexed [x, y, z] as `ocnn.nn.octree2voxel`), and on adaptive layers the CUDA path equals
the oracle restatement (oracle/restate.py `octree_conv`).
"""
from __future__ import annotations
import ctypes as C
import math
import torch
import torch.nn as nn

from . import ops
from ._lib import lib, ptr, stream, check, OctreeLevels
from .ops import PreparedWeight, TapTable


def octree_levels(octree):
    """of_octree_levels view of an Octree (keys / children / nnum of depths full_depth..depth)."""
    lv = OctreeLevels()
    lv.full_depth, lv.depth, lv.batch = octree.full_depth, octree.depth, octree.batch_size
    keep = []
    for d in range(octree.full_depth, octree.depth + 1):
        k, c = octree.keys[d].contiguous(), octree.children[d].contiguous()
        assert k.dtype == torch.int64 and c.dtype == torch.int32 and k.is_cuda
        lv.keys[d], lv.children[d], lv.nnum[d] = k.data_ptr(), c.data_ptr(), int(octree.nnum[d])
        keep += [k, c]
    return lv, keep


def octree_neigh(octree, depth: int, stride: int = 1, nempty: bool = False) -> torch.Tensor:
    """`octree.get_neigh(depth, '333', stride, nempty)`: int32 [N', 27], -1 = no neighbour.  stride 2 keeps every 8th
    row (the first child of each octant group: the 3^3 window of the parent cell in child coordinates); nempty=True
    re-indexes rows and entries to the non-empty nodes."""
    if octree.device.type != 'cuda':
        raise RuntimeError('octfusion_b200: the octree must live on a CUDA device (there is no CPU path)')
    cache = octree.__dict__.setdefault('_neigh27', {})
    if depth not in cache:
        lv, keep = octree_levels(octree)
        out = torch.empty((int(octree.nnum[depth]), 27), dtype=torch.int32, device=octree.device)
        check(lib.of_octree_neigh27(C.byref(lv), depth, ptr(out), stream()), 'of_octree_neigh27')
        cache[depth] = out
    neigh = cache[depth]
    if nempty:
        child = octree.children[depth]
        mapped = torch.where(neigh >= 0, child[neigh.clamp(min=0).long()], torch.full_like(neigh, -1))
        neigh = mapped[child >= 0]
    if stride == 2:
        assert not nempty, 'stride 2 with nempty=True is not supported'
        neigh = neigh[::8]
    return neigh.contiguous()


class OctreeConv(nn.Module):
    def __init__(self, in_channels: int, out_channels: int, kernel_size=(3,), stride: int = 1, nempty: bool = False,
                 direct_method: bool = False, use_bias: bool = False, max_buffer: int = int(2e8)):
        super().__init__()
        ks = list(kernel_size) * (3 if len(kernel_size) == 1 else 1)
        if ks != [3, 3, 3] or stride not in (1, 2):
            raise NotImplementedError('octfusion_b200.OctreeConv: kernel 3^3 with stride 1 or 2 (what configs[0] names)')
        self.in_channels, self.out_channels, self.kernel_size, self.stride = in_channels, out_channels, ks, stride
        self.nempty, self.direct_method, self.use_bias, self.max_buffer = nempty, direct_method, use_bias, max_buffer
        self.kdim = 27
        self.weights = nn.Parameter(torch.empty(self.kdim, in_channels, out_channels))
        self.bias = nn.Parameter(torch.zeros(out_channels)) if use_bias else None
        self.reset_parameters()
        self._pw = PreparedWeight(27, in_channels, 0, out_channels)
        self._pw_pad, self._pw_pad_key = None, None

    def reset_parameters(self):
        # xavier-uniform over the [27*Cin, Cout] matrix (ocnn's init, recalled)
        a = math.sqrt(6.0 / float(self.kdim * self.in_channels + self.out_channels))
        nn.init.uniform_(self.weights, -a, a)

    def _padded(self, cpad):
        key = (self.weights.data_ptr(), self.weights._version)
        if self._pw_pad_key != key:
            wp = torch.zeros((27, cpad, self.out_channels), dtype=torch.float32, device=self.weights.device)
            wp[:, : self.in_channels] = self.weights.detach().float()
            self._pw_pad = PreparedWeight(27, cpad, 0, self.out_channels).refresh(wp.view(-1, self.out_channels), 'canon')
            self._pw_pad_src, self._pw_pad_key = wp, key
        return self._pw_pad

    @torch.no_grad()
    def forward(self, data: torch.Tensor, octree, depth: int):
        neigh = octree_neigh(octree, depth, self.stride, self.nempty)
        tap = TapTable(neigh, None, 27)
        x = data.contiguous()
        if x.dtype == torch.bfloat16 and self.in_channels % 64 != 0:
            # tensor-core path wants 64-channel slabs: zero-pad the (narrow) input instead of leaving the tensor cores
            cpad = (self.in_channels + 63) // 64 * 64
            xp = torch.zeros((x.shape[0], cpad), dtype=x.dtype, device=x.device)
            ops.copy_rows(x, xp, x.shape[0], self.in_channels)
            return ops.gather_gemm(xp, self._padded(cpad), tap=tap, bias=self.bias)
        return ops.gather_gemm(x, self._pw.refresh(self.weights.view(-1, self.out_channels), 'canon'), tap=tap,
                               bias=self.bias)

    def extra_repr(self):
        return 'in_channels={}, out_channels={}, kernel_size={}, stride={}, nempty={}, bias={}'.format(
            self.in_channels, self.out_channels, self.kernel_size, self.stride, self.nempty, self.use_bias)
