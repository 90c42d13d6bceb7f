"""Drop-in operator classes: same names, constructor signatures, forward signatures and
state_dict keys as reference models/networks/modules.py (SURVEY.md 8b), every forward executed by
the sm_90a kernels of liboctfusion_b200.so.  Inference only (the hot path is the sampler's
per-step U-Net forward); no autograd through the custom kernels.

Sparse (dual-octree) tensors are [N_d, C] row-major exactly as in the reference.  Dense (LR middle
U-Net) tensors are kept channels-last in *Morton order* [B * 8^r, C] inside the fused network, which
makes `octree2voxel` / the gather back (reference graph_unet_lr.py:175-182) the identity on the full
layer; the module-level `forward(x[B,C,D,H,W])` entry points convert at the boundary.
"""
from __future__ import annotations
import math
import torch
import torch.nn as nn

from . import ops
from .ops import PreparedWeight


def zero_module(module):
    """reference ldm_diffusion_util.py:194-200."""
    for p in module.parameters():
        p.detach().zero_()
    return module


def _norm_groups(channels: int, group: int = 32) -> int:
    """DualOctreeGroupNorm group rule, reference modules.py:271-274."""
    if channels <= 32:
        return channels // 4
    if channels % group != 0:
        return 30
    return group


# =================================================================================================
# sparse (dual-octree) operators
# =================================================================================================
class GraphConv(nn.Module):
    """reference modules.py:163-220."""

    def __init__(self, in_channels, out_channels, n_edge_type=7, avg_degree=7, n_node_type=0, use_bias=False):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.use_bias, self.n_edge_type, self.avg_degree, self.n_node_type = use_bias, n_edge_type, avg_degree, n_node_type
        self.node_channel = n_node_type if n_node_type > 1 else 0
        self.weights = nn.Parameter(torch.empty(n_edge_type * (in_channels + self.node_channel), out_channels))
        if use_bias:
            self.bias = nn.Parameter(torch.empty(out_channels))
        self.reset_parameters()
        self._pw = PreparedWeight(n_edge_type, in_channels, self.node_channel, out_channels)

    def reset_parameters(self):
        std = math.sqrt(2.0 / float(self.avg_degree * self.in_channels + self.avg_degree * self.out_channels))
        a = math.sqrt(3.0) * std
        nn.init.uniform_(self.weights, -a, a)
        if self.use_bias:
            nn.init.zeros_(self.bias)

    def prepared(self):
        return self._pw.refresh(self.weights, 'canon')

    def prepared_padded(self, cpad=64):
        """weights re-laid for an input zero-padded to `cpad` channels (tensor-core path needs C % 64 == 0; the
        3- or 8-channel latent of the first conv is padded instead of falling back to the CUDA cores)."""
        key = (self.weights.data_ptr(), self.weights._version)
        if getattr(self, '_pw_pad_key', None) != key:
            cin, nt, k = self.in_channels, self.node_channel, self.n_edge_type
            w = self.weights.detach().float().view(k, cin + nt, self.out_channels)
            wp = torch.zeros((k, cpad + nt, self.out_channels), dtype=torch.float32, device=w.device)
            wp[:, :cin] = w[:, :cin]
            wp[:, cpad:] = w[:, cin:]
            self._pw_pad = PreparedWeight(k, cpad, nt, self.out_channels)
            self._pw_pad.refresh(wp.view(-1, self.out_channels), 'canon')
            self._pw_pad_src = wp
            self._pw_pad_key = key
        return self._pw_pad

    def run(self, x0, plan, x1=None, **epi):
        if x1 is None and x0.dtype == torch.bfloat16 and self.in_channels % 64 != 0 and self.in_channels < 64:
            xp = torch.zeros((x0.shape[0], 64), dtype=x0.dtype, device=x0.device)
            ops.copy_rows(x0, xp, x0.shape[0], self.in_channels)
            return ops.gather_gemm(xp, self.prepared_padded(64), tap=plan.tap, node_type=plan.node_type,
                                   bias=self.bias if self.use_bias else None, **epi)
        return ops.gather_gemm(x0, self.prepared(), a1=x1, tap=plan.tap, node_type=plan.node_type,
                               bias=self.bias if self.use_bias else None, **epi)

    @torch.no_grad()
    def forward(self, x, doctree, d):
        return self.run(x.contiguous(), doctree.plan[d])

    def extra_repr(self):
        return 'channel_in={}, channel_out={}, n_edge_type={}, avg_degree={}, n_node_type={}'.format(
            self.in_channels, self.out_channels, self.n_edge_type, self.avg_degree, self.n_node_type)


class DualOctreeGroupNorm(nn.Module):
    """reference modules.py:262-330."""

    def __init__(self, in_channels: int, group: int = 32, nempty: bool = False):
        super().__init__()
        self.eps = 1e-5
        self.nempty = nempty
        self.in_channels = in_channels
        self.group = _norm_groups(in_channels, group)
        assert in_channels % self.group == 0
        self.channels_per_group = in_channels // self.group
        self.weights = nn.Parameter(torch.ones(1, in_channels))
        self.bias = nn.Parameter(torch.zeros(1, in_channels))

    def run(self, x0, plan, batch_size, x1=None, act=False):
        return ops.group_norm(x0, self.weights, self.bias, self.group, plan.stat, x1=x1, eps=self.eps,
                              count_eps=self.eps, act=act)

    @torch.no_grad()
    def forward(self, data, doctree, depth):
        return self.run(data.contiguous(), doctree.plan[depth], doctree.batch_size)

    def extra_repr(self):
        return 'in_channels={}, group={}, nempty={}'.format(self.in_channels, self.group, self.nempty)


def graphnormalization(channels):
    return DualOctreeGroupNorm(channels, min(32, channels))


class Conv1x1(nn.Module):
    """reference modules.py:332-339 (nn.Linear, bias-free unless asked)."""

    def __init__(self, channel_in, channel_out, use_bias=False):
        super().__init__()
        self.linear = nn.Linear(channel_in, channel_out, use_bias)
        self._pw = PreparedWeight(1, channel_in, 0, channel_out)

    def prepared(self):
        return self._pw.refresh(self.linear.weight, 'linear')

    def run(self, x0, x1=None, **epi):
        return ops.gather_gemm(x0, self.prepared(), a1=x1, bias=self.linear.bias, **epi)

    @torch.no_grad()
    def forward(self, x):
        return self.run(x.contiguous())


class Downsample(nn.Module):
    """reference modules.py:382-398: x.view(-1, 8C) @ weights.flatten(1).t()."""

    def __init__(self, channels):
        super().__init__()
        self.channels = channels
        self.weights = nn.Parameter(torch.empty(channels, channels, 8))
        nn.init.xavier_uniform_(self.weights)
        self._pw = PreparedWeight(1, 8 * channels, 0, channels)

    def prepared(self):
        return self._pw.refresh(self.weights, 'linear')           # flatten(1) is [N=C, K=8C]

    @torch.no_grad()
    def forward(self, x):
        return ops.gather_gemm(x.contiguous().view(-1, 8 * self.channels), self.prepared())


class Upsample(nn.Module):
    """reference modules.py:430-446: (x @ weights.flatten(1)).view(-1, C)."""

    def __init__(self, channels):
        super().__init__()
        self.channels = channels
        self.weights = nn.Parameter(torch.empty(channels, channels, 8))
        nn.init.xavier_uniform_(self.weights)
        self._pw = PreparedWeight(1, channels, 0, 8 * channels)

    def prepared(self):
        return self._pw.refresh(self.weights, 'canon')            # flatten(1) is [K=C, N=8C]

    @torch.no_grad()
    def forward(self, x):
        return ops.gather_gemm(x.contiguous(), self.prepared()).view(-1, self.channels)


class GraphDownsample(nn.Module):
    """reference modules.py:400-428: depth-d graph features -> depth d-1, then a GraphConv."""

    def __init__(self, channels_in, channels_out, n_edge_type, avg_degree, n_node_type):
        super().__init__()
        self.channels_in, self.channels_out = channels_in, channels_out
        self.downsample = Downsample(channels_in)
        self.conv = GraphConv(channels_in, channels_out, n_edge_type, avg_degree, n_node_type)

    @torch.no_grad()
    def forward(self, x, doctree, d):
        x = x.contiguous()
        pd, pc = doctree.plan[d], doctree.plan[d - 1]
        c = self.channels_in
        mid = torch.empty((pc.rows, c), dtype=x.dtype, device=x.device)
        # leaves (coarser than d) keep their features; they only move to their depth-(d-1) rows
        ops.copy_rows(x, mid, pd.down_copy_rows, c, dst_rows=pd.down_copy_dst)
        # the 8 children of every non-empty depth-(d-1) node are pooled by one [8C -> C] GEMM whose
        # epilogue scatters the result to the parent's row
        xd = x[pd.leaf_base:].view(-1, 8 * c)
        ops.gather_gemm(xd, self.downsample.prepared(), out=mid, out_rows=pd.down_out_rows)
        return self.conv.run(mid, pc, stats=pc.stat)


class GraphUpsample(nn.Module):
    """reference modules.py:449-472: depth-d graph features -> depth d+1, then a GraphConv."""

    def __init__(self, channels_in, channels_out, n_edge_type, avg_degree, n_node_type):
        super().__init__()
        self.channels_in, self.channels_out = channels_in, channels_out
        self.upsample = Upsample(channels_in)
        self.conv = GraphConv(channels_in, channels_out, n_edge_type, avg_degree, n_node_type)

    @torch.no_grad()
    def forward(self, x, doctree, d):
        x = x.contiguous()
        pc, pf = doctree.plan[d], doctree.plan[d + 1]
        c = self.channels_in
        mid = torch.empty((pf.rows, c), dtype=x.dtype, device=x.device)
        ops.copy_rows(x, mid, pc.up_copy_rows, c, src_rows=pc.up_copy_src)
        # every non-leaf depth-d row produces its 8 children rows with one [C -> 8C] GEMM; the [M, 8C]
        # result *is* the [8M, C] block of children rows, written in place
        tail = mid[pc.up_copy_rows:]
        ops.gather_gemm(x, self.upsample.prepared(), in_rows=pc.up_in_rows, out=tail, ldo=8 * c)
        return self.conv.run(mid, pf, stats=pf.stat)


class TimestepBlock(nn.Module):
    pass


class BatchedEmbedding:
    """All `Linear(SiLU(emb))` projections of a network (reference modules.py:709-715 emb_layers, :479-482
    time_mlp) depend only on the timestep embedding, so they are evaluated by ONE launch over the row-wise
    concatenation of their weights; each block then reads its column slice."""

    def __init__(self, linears):
        self.linears = list(linears)
        self._key, self._w, self._b, self._off = None, None, None, None

    def __call__(self, emb):
        key = tuple((l.weight.data_ptr(), l.weight._version, l.bias._version) for l in self.linears)
        if key != self._key:
            self._w = torch.cat([l.weight.detach().float() for l in self.linears], 0).contiguous()
            self._b = torch.cat([l.bias.detach().float() for l in self.linears], 0).contiguous()
            off, self._off = 0, []
            for l in self.linears:
                self._off.append((off, off + l.weight.shape[0]))
                off += l.weight.shape[0]
            self._key = key
        e = ops.linear_small(emb, self._w, self._b, a_silu=True)
        return [e[:, a:b] for a, b in self._off]


def _concat_rows(x0, x1):
    """materialise (x0 | x1) -- only needed where the concatenation itself is the residual."""
    n, c0, c1 = x0.shape[0], x0.shape[1], x1.shape[1]
    cat = torch.empty((n, c0 + c1), dtype=x0.dtype, device=x0.device)
    ops.copy_rows(x0, cat, n, c0)
    ops.copy_rows(x1, cat[:, c0:], n, c1)
    return cat


class GraphResBlockEmbed(TimestepBlock):
    """reference modules.py:661-763.  GN -> SiLU -> conv1 -> + Linear(SiLU(emb))[batch] -> GN -> SiLU ->
    conv2 -> + skip(x).  Fusions: GN-apply+SiLU (+ the channel concat of the skip stack) in one pass,
    the embedding add and the residual / skip add inside the GEMM epilogues."""

    def __init__(self, channels, emb_channels, dropout, out_channels, n_edge_type, avg_degree, n_node_type,
                 use_conv=False, use_scale_shift_norm=False, dims=2, use_checkpoint=False, up=False, down=False):
        super().__init__()
        self.channels, self.emb_channels = channels, emb_channels
        self.out_channels = channels if out_channels is None else out_channels
        self.use_conv, self.use_checkpoint, self.use_scale_shift_norm = use_conv, use_checkpoint, use_scale_shift_norm
        if use_scale_shift_norm or use_conv:
            raise NotImplementedError('the reference never enables use_scale_shift_norm / use_conv (dead branches, '
                                      'modules.py:747-751)')
        self.block1_norm = graphnormalization(self.channels)
        self.silu = nn.SiLU()
        self.conv1 = GraphConv(self.channels, self.out_channels, n_edge_type, avg_degree, n_node_type)
        self.emb_layers = nn.Sequential(nn.SiLU(), nn.Linear(emb_channels, self.out_channels))
        self.block2_norm = graphnormalization(self.out_channels)
        self.dropout = nn.Dropout(p=dropout)
        self.conv2 = zero_module(GraphConv(self.out_channels, self.out_channels, n_edge_type, avg_degree, n_node_type))
        if self.out_channels == channels:
            self.skip_connection = nn.Identity()
        else:
            self.skip_connection = Conv1x1(self.channels, self.out_channels)
        self._pw_emb = PreparedWeight(1, emb_channels, 0, self.out_channels)

    def run(self, x0, emb, plan, batch_size, x1=None, e=None):
        """x = (x0 | x1) virtual concat; emb fp32 [B, emb_channels]; e = Linear(SiLU(emb)) when the caller has
        already computed it for all blocks in one launch (BatchedEmbedding)."""
        h = self.block1_norm.run(x0, plan, batch_size, x1=x1, act=True)
        lin = self.emb_layers[1]
        if e is None:
            e = ops.linear_small(emb, lin.weight, lin.bias, a_silu=True)
        h = self.conv1.run(h, plan, row_add=e, row_add_idx=plan.batch_id, stats=plan.stat)
        h = self.block2_norm.run(h, plan, batch_size, act=True)
        if isinstance(self.skip_connection, Conv1x1):
            skip = self.skip_connection.run(x0, x1)
        elif x1 is None:
            skip = x0
        else:
            skip = _concat_rows(x0, x1)          # identity skip of a concatenated input (e.g. 256+256 -> 512)
        return self.conv2.run(h, plan, resid=skip, stats=plan.stat)      # (the next block's norm consumes it)

    @torch.no_grad()
    def forward(self, x, emb, doctree, depth):
        return self.run(x.contiguous(), emb.float().contiguous(), doctree.plan[depth], doctree.batch_size)


# =================================================================================================
# dense operators of the LR middle U-Net -- Morton-ordered channels-last tensors [B * 8^r, C]
# =================================================================================================
class DenseTables:
    """Neighbour tables of the dense 3^3 convolutions for one (batch, resolution) family, built once by
    of_dense_tap_table; sample ids for the embedding add."""

    def __init__(self, batch: int, device):
        self.batch, self.device = batch, device
        self._tabs, self._sid, self._perm, self._stat = {}, {}, {}, {}

    def conv(self, res_log2):
        return self._get(0, res_log2)

    def down(self, out_res_log2):
        return self._get(1, out_res_log2)

    def up(self, out_res_log2):
        return self._get(2, out_res_log2)

    def _get(self, mode, r):
        k = (mode, r)
        if k not in self._tabs:
            self._tabs[k] = ops.dense_tap_table(mode, r, self.batch, self.device)
        return self._tabs[k]

    def stat_plan(self, res_log2):
        """segment tables of the norm statistics for the [B * 8^r, C] layout (ops.StatPlan)"""
        if res_log2 not in self._stat:
            v = 8 ** res_log2
            self._stat[res_log2] = ops.StatPlan(self.batch * v, self.batch, rows_per_sample=v, device=self.device)
        return self._stat[res_log2]

    def sample_id(self, res_log2):
        if res_log2 not in self._sid:
            v = 8 ** res_log2
            self._sid[res_log2] = (torch.arange(self.batch * v, device=self.device) // v).int()
        return self._sid[res_log2]

    def morton_perm(self, res_log2):
        """index tensor p with x_morton = x_xyz.reshape(B, C, -1)[:, :, p] (API-boundary glue only)."""
        if res_log2 not in self._perm:
            from .octree import key2xyz
            k = torch.arange(8 ** res_log2, device=self.device)
            x, y, z, _ = key2xyz(k, res_log2)
            s = 2 ** res_log2
            self._perm[res_log2] = (x * s + y) * s + z
        return self._perm[res_log2]


def _to_morton(x, tables):
    """[B, C, D, H, W] -> [B*V, C] Morton rows (boundary glue for stand-alone module use)."""
    b, c = x.shape[:2]
    r = int(round(math.log2(x.shape[2])))
    p = tables.morton_perm(r)
    return x.reshape(b, c, -1)[:, :, p].permute(0, 2, 1).reshape(-1, c).contiguous(), r


def _from_morton(y, tables, b, r):
    c = y.shape[1]
    s = 2 ** r
    p = tables.morton_perm(r)
    out = torch.empty((b, s * s * s, c), dtype=y.dtype, device=y.device)
    out[:, p] = y.reshape(b, -1, c)
    return out.permute(0, 2, 1).reshape(b, c, s, s, s).contiguous()


class GroupNorm32(nn.GroupNorm):
    """reference modules.py:26-28 (statistics in fp32; here fp64 accumulators)."""

    def run(self, x0, tables, res_log2, x1=None, act=False):
        return ops.group_norm(x0, self.weight, self.bias, self.num_groups, tables.stat_plan(res_log2), x1=x1,
                              eps=self.eps, count_eps=0.0, act=act)


def convnormalization(channels):
    return GroupNorm32(min(channels, 32), channels)


def activation_function():
    return nn.SiLU()


class our_Identity(nn.Module):
    def forward(self, x, *args, **kwargs):
        return x


class _Conv3dParams(nn.Conv3d):
    """nn.Conv3d as a parameter container (state_dict keys `weight`, `bias`); the convolution itself
    runs as a 27-tap gather GEMM."""

    def prepared(self):
        if not hasattr(self, '_pw'):
            k = self.kernel_size[0] ** 3
            self._pw = PreparedWeight(k, self.in_channels, 0, self.out_channels)
        return self._pw.refresh(self.weight, 'conv3d' if self._pw.taps > 1 else 'linear')

    def run(self, x0, tap, x1=None, **epi):
        return ops.gather_gemm(x0, self.prepared(), a1=x1, tap=tap, bias=self.bias, **epi)

    def forward(self, x):  # pragma: no cover - guarded
        raise RuntimeError('octfusion_b200: dense convolutions run through DenseTables / ResnetBlock.run')


class _Conv1dParams(nn.Conv1d):
    def prepared(self):
        if not hasattr(self, '_pw'):
            self._pw = PreparedWeight(1, self.in_channels, 0, self.out_channels)
        return self._pw.refresh(self.weight, 'linear')

    def run(self, x0, **epi):
        return ops.gather_gemm(x0, self.prepared(), bias=self.bias, **epi)


def conv_nd(dims, *args, **kwargs):
    if dims == 1:
        return _Conv1dParams(*args, **kwargs)
    if dims == 3:
        return _Conv3dParams(*args, **kwargs)
    raise ValueError('octfusion_b200 supports dims 1 and 3 (the OctFusion configs use dims=3)')


class ConvDownsample(nn.Module):
    """reference modules.py:80-95 (3^3, stride 2, padding 1)."""

    def __init__(self, channels, use_conv=True, dims=3):
        super().__init__()
        assert use_conv and dims == 3
        self.channels, self.use_conv, self.dims = channels, use_conv, dims
        self.op = conv_nd(dims, channels, channels, 3, stride=2, padding=1)

    def run(self, x, tables, res_log2):
        return self.op.run(x, tables.down(res_log2 - 1), stats=tables.stat_plan(res_log2 - 1))

    @torch.no_grad()
    def forward(self, x):
        t = DenseTables(x.shape[0], x.device)
        y, r = _to_morton(x, t)
        return _from_morton(self.run(y, t, r), t, x.shape[0], r - 1)


class ConvUpsample(nn.Module):
    """reference modules.py:63-77 (nearest x2 then 3^3 conv; the upsampled tensor is never built)."""

    def __init__(self, channels, use_conv=True, dims=3):
        super().__init__()
        assert use_conv and dims == 3
        self.channels, self.use_conv, self.dims = channels, use_conv, dims
        self.conv = conv_nd(dims, channels, channels, 3, padding=1)

    def run(self, x, tables, res_log2):
        return self.conv.run(x, tables.up(res_log2 + 1), stats=tables.stat_plan(res_log2 + 1))

    @torch.no_grad()
    def forward(self, x):
        t = DenseTables(x.shape[0], x.device)
        y, r = _to_morton(x, t)
        return _from_morton(self.run(y, t, r), t, x.shape[0], r + 1)


class ResnetBlock(nn.Module):
    """reference modules.py:474-513 (use_text_condition=False is the only configuration the U-Net
    builds, graph_unet_lr.py:126-127)."""

    def __init__(self, world_dims: int, dim_in: int, dim_out: int, emb_dim: int, dropout: float = 0.1,
                 use_text_condition: bool = False):
        super().__init__()
        if use_text_condition:
            raise NotImplementedError('text conditioning is not on the OctFusion U-Net path')
        self.world_dims, self.use_text_condition = world_dims, use_text_condition
        self.time_mlp = nn.Sequential(activation_function(), nn.Linear(emb_dim, dim_out))
        self.block1 = nn.Sequential(convnormalization(dim_in), activation_function(),
                                    conv_nd(world_dims, dim_in, dim_out, 3, padding=1))
        self.block2 = nn.Sequential(convnormalization(dim_out), activation_function(), nn.Dropout(dropout),
                                    zero_module(conv_nd(world_dims, dim_out, dim_out, 3, padding=1)))
        self.res_conv = conv_nd(world_dims, dim_in, dim_out, 1) if dim_in != dim_out else nn.Identity()
        self._pw_t = PreparedWeight(1, emb_dim, 0, dim_out)

    def run(self, x0, emb, tables, res_log2, x1=None, e=None):
        tap, sp = tables.conv(res_log2), tables.stat_plan(res_log2)
        h = self.block1[0].run(x0, tables, res_log2, x1=x1, act=True)
        lin = self.time_mlp[1]
        t = e if e is not None else ops.linear_small(emb, lin.weight, lin.bias, a_silu=True)
        h = self.block1[2].run(h, tap, row_add=t, row_add_idx=tables.sample_id(res_log2), stats=sp)
        h = self.block2[0].run(h, tables, res_log2, act=True)
        if isinstance(self.res_conv, nn.Identity):
            skip = x0 if x1 is None else _concat_rows(x0, x1)
        else:
            skip = ops.gather_gemm(x0, self.res_conv.prepared(), a1=x1, bias=self.res_conv.bias)
        return self.block2[3].run(h, tap, resid=skip, stats=sp)

    @torch.no_grad()
    def forward(self, x, time_emb, text_condition=None):
        t = DenseTables(x.shape[0], x.device)
        y, r = _to_morton(x, t)
        return _from_morton(self.run(y, time_emb.float().contiguous(), t, r), t, x.shape[0], r)


class QKVAttention(nn.Module):
    """reference modules.py:538-547; input [b*heads, 3*ch, T] (the reference's layout)."""

    @torch.no_grad()
    def forward(self, qkv):
        bh, c3, t = qkv.shape
        x = qkv.permute(0, 2, 1).reshape(bh * t, c3).contiguous()        # one head per "batch" entry
        out = ops.attention(x, bh, t, 1)
        return out.reshape(bh, t, c3 // 3).permute(0, 2, 1).contiguous()


class AttentionBlock(nn.Module):
    """reference modules.py:515-535."""

    def __init__(self, channels, num_heads=1):
        super().__init__()
        self.channels, self.num_heads = channels, num_heads
        self.norm = convnormalization(channels)
        self.qkv = conv_nd(1, channels, channels * 3, 1)
        self.attention = QKVAttention()
        self.proj_out = zero_module(conv_nd(1, channels, channels, 1))

    def run(self, x, tables, res_log2):
        """x [B*T, C] channels-last Morton rows, T = 8^res_log2."""
        h = self.norm.run(x, tables, res_log2)
        qkv = self.qkv.run(h)
        a = ops.attention(qkv, tables.batch, 8 ** res_log2, self.num_heads)
        return self.proj_out.run(a, resid=x, stats=tables.stat_plan(res_log2))

    @torch.no_grad()
    def forward(self, x):
        b, c = x.shape[:2]
        xf = x.reshape(b, c, -1)
        t = xf.shape[2]
        r = int(round(math.log2(t) / 3))
        assert 8 ** r == t, 'AttentionBlock: token count must be a power of 8 (a cubic grid)'
        y = self.run(xf.permute(0, 2, 1).reshape(b * t, c).contiguous(), DenseTables(b, x.device), r)
        return y.reshape(b, t, c).permute(0, 2, 1).reshape(x.shape).contiguous()


class NormActAttention(nn.Sequential):
    """nn.Sequential(convnormalization, SiLU, AttentionBlock) of reference graph_unet_lr.py:128-132 with
    the same child indices (0, 1, 2) and therefore the same state_dict keys."""

    def __init__(self, channels, num_heads):
        super().__init__(convnormalization(channels), activation_function(), AttentionBlock(channels, num_heads))

    def run(self, x, tables, res_log2):
        return self[2].run(self[0].run(x, tables, res_log2, act=True), tables, res_log2)


class LearnedSinusoidalPosEmb(nn.Module):
    """reference modules.py:550-563."""

    def __init__(self, dim):
        super().__init__()
        assert dim % 2 == 0
        self.weights = nn.Parameter(torch.randn(dim // 2))

    @torch.no_grad()
    def forward(self, x):
        return ops.learned_sinusoidal(x, self.weights)


# =================================================================================================
# input features of the GraphVAE encoder (ocnn.modules.InputFeature, SURVEY.md Appendix B: parity UNPINNED)
# =================================================================================================
def input_feature_nd(octree, leaf_rows: int = 0, dtype=torch.float32):
    """[leaf_rows zero rows | ND feature of every depth-`octree.depth` node] (csrc/points.cu of_input_feature_nd): the
    feature is [normal | sum((frac(point) - 0.5) * normal)] of a non-empty node and zero for an empty one."""
    from ._lib import lib, ptr, stream, check, dt
    D = octree.depth
    points, normals = octree.points[D], octree.normals[D]
    if points is None or normals is None:
        raise RuntimeError('InputFeature ND: the octree has no points / normals at depth %d (build it with '
                           'Octree.build_octree from points with normals)' % D)
    child = octree.children[D].contiguous()
    nnum = int(octree.nnum[D])
    out = torch.empty((leaf_rows + nnum, 4), dtype=dtype, device=child.device)
    check(lib.of_input_feature_nd(ptr(points.contiguous()), ptr(normals.contiguous()), ptr(child), nnum, leaf_rows,
                                  dt(out), ptr(out), 4, stream()), 'of_input_feature_nd')
    return out


class InputFeature:
    """ocnn.modules.InputFeature(feature='ND', nempty=False): [nnum[depth], 4] at the octree's depth, zero rows for the
    empty nodes (octree_pad).  Only the N and D letters are built."""

    def __init__(self, feature: str = 'ND', nempty: bool = False):
        if feature.upper() != 'ND' or nempty:
            raise NotImplementedError("InputFeature: only feature='ND' with nempty=False is built (got %r, nempty=%s)"
                                      % (feature, nempty))
        self.feature, self.nempty = feature, nempty

    def __call__(self, octree):
        return input_feature_nd(octree)
