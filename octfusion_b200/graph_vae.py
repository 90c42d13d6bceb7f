"""GraphVAE decoder (SURVEY.md 8f rank 1): latent code on the depth-6 dual graph -> split logits and MPU
regression values at depths 6..8, growing the octree as it goes.

Drop-in for reference models/networks/dualoctree_networks/graph_vae.py `GraphVAE` as far as `decode_code`
/ `octree_decoder` reach (graph_vae.py:171-223, 300-324): same class name, constructor signature, parameter
names (a reference checkpoint loads with `load_state_dict`), and the same operator classes underneath
(`GraphResBlock(s)`, `Conv1x1Gn*` of reference models/networks/modules.py:343-381, 597-666 and the VAE's own
`GraphUpsample` / `GraphDownsample` of dualoctree_networks/modules.py:39-91).  Every forward runs on the CUDA
kernels of liboctfusion_b200.so; the octree growth (`octree_split` / `octree_grow`) and the dual-graph rebuild per
depth stay on the device.

The encoder runs on the ND input features of an octree built from points (`Octree.build_octree`,
`DualOctree.get_input_feature`, csrc/points.cu) in `extract_code` and `forward` (graph_vae.py:246-298), or on
caller-provided features in `octree_encoder_step` / `encode_moments`.  Inference only: `forward`'s `kl_loss` is a value,
not a training loss.  `decode_code(pos=...)` / `output['neural_mpu']` evaluate the decoded implicit function with
`mpu.NeuralMPU` (csrc/mpu.cu).
"""
from __future__ import annotations
import torch
import torch.nn as nn

from . import ops
from .modules import (GraphConv, DualOctreeGroupNorm, Conv1x1, Upsample, Downsample)
from .dual_octree import DualOctree
from .octree import Octree
from .mpu import NeuralMPU


# =================================================================================================
# operator classes (reference models/networks/modules.py:343-381, 597-666)
# =================================================================================================
class Conv1x1Gn(nn.Module):
    """reference modules.py:343-353: bias-free Linear -> DualOctreeGroupNorm."""
    act = None

    def __init__(self, channel_in, channel_out):
        super().__init__()
        self.conv = Conv1x1(channel_in, channel_out, use_bias=False)
        self.gn = DualOctreeGroupNorm(channel_out)

    def run(self, x, plan, batch_size):
        return self.gn.run(self.conv.run(x), plan, batch_size, act=self.act)

    @torch.no_grad()
    def forward(self, x, doctree, depth):
        return self.run(x.contiguous(), doctree.plan[depth], doctree.batch_size)


class Conv1x1GnGelu(Conv1x1Gn):
    """reference modules.py:355-367: ... -> exact GELU (fused into the norm's apply pass)."""
    act = 'gelu'

    def __init__(self, channel_in, channel_out):
        super().__init__(channel_in, channel_out)
        self.gelu = nn.GELU()


class Conv1x1GnGeluSequential(Conv1x1GnGelu):
    """reference modules.py:369-381: same, called with one `[x, doctree, depth]` argument inside nn.Sequential."""

    @torch.no_grad()
    def forward(self, data):
        x, doctree, depth = data
        return self.run(x.contiguous(), doctree.plan[depth], doctree.batch_size)


class GraphResBlock(nn.Module):
    """reference modules.py:597-648: GN -> swish -> conv1 -> GN -> swish -> dropout -> conv2 (+ Conv1x1Gn skip when the
    channel count changes).  The residual add runs in conv2's GEMM epilogue."""

    def __init__(self, channel_in, channel_out, dropout, n_edge_type=7, avg_degree=7, n_node_type=0,
                 use_checkpoint=False):
        super().__init__()
        self.channel_in, self.channel_out, self.use_checkpoint = channel_in, channel_out, use_checkpoint
        self.norm1 = DualOctreeGroupNorm(channel_in)
        self.conv1 = GraphConv(channel_in, channel_out, n_edge_type, avg_degree, n_node_type)
        self.norm2 = DualOctreeGroupNorm(channel_out)
        self.dropout = nn.Dropout(dropout)
        self.conv2 = GraphConv(channel_out, channel_out, n_edge_type, avg_degree, n_node_type)
        if channel_in != channel_out:
            self.conv1x1c = Conv1x1Gn(channel_in, channel_out)

    def run(self, x, plan, batch_size):
        h = self.norm1.run(x, plan, batch_size, act=True)
        h = self.conv1.run(h, plan)
        h = self.norm2.run(h, plan, batch_size, act=True)
        skip = self.conv1x1c.run(x, plan, batch_size) if self.channel_in != self.channel_out else x
        return self.conv2.run(h, plan, resid=skip)

    @torch.no_grad()
    def forward(self, x, doctree, depth):
        return self.run(x.contiguous(), doctree.plan[depth], doctree.batch_size)


class GraphResBlocks(nn.Module):
    """reference modules.py:651-666."""

    def __init__(self, channel_in, channel_out, dropout, resblk_num, n_edge_type=7, avg_degree=7, n_node_type=0,
                 use_checkpoint=False):
        super().__init__()
        self.resblk_num = resblk_num
        channels = [channel_in] + [channel_out] * resblk_num
        self.resblks = nn.ModuleList([
            GraphResBlock(channels[i], channels[i + 1], dropout, n_edge_type, avg_degree, n_node_type, use_checkpoint)
            for i in range(resblk_num)])

    @torch.no_grad()
    def forward(self, data, doctree, depth):
        x, plan = data.contiguous(), doctree.plan[depth]
        for blk in self.resblks:
            x = blk.run(x, plan, doctree.batch_size)
        return x


class GraphUpsample(nn.Module):
    """The VAE's upsample (reference dualoctree_networks/modules.py:69-95): depth-(d-1) graph -> depth-d graph, no
    graph conv; Conv1x1GnGelu when the channel count changes.  `leaf_mask` / `numd` are accepted for signature
    compatibility; the row maps come from the doctree's plan."""

    def __init__(self, channels_in, channels_out=None):
        super().__init__()
        self.channels_in = channels_in
        self.channels_out = channels_out or channels_in
        self.upsample = Upsample(channels_in)
        if self.channels_in != self.channels_out:
            self.conv1x1 = Conv1x1GnGelu(self.channels_in, self.channels_out)

    @torch.no_grad()
    def forward(self, x, octree, d, leaf_mask=None, numd=None):
        doctree = octree                                    # the reference passes the DualOctree under this name
        x = x.contiguous()
        pc, pf = doctree.plan[d - 1], doctree.plan[d]
        c = self.channels_in
        out = torch.empty((pf.rows, c), dtype=x.dtype, device=x.device)
        ops.copy_rows(x, out, pc.up_copy_rows, c, src_rows=pc.up_copy_src)
        ops.gather_gemm(x, self.upsample.prepared(), in_rows=pc.up_in_rows, out=out[pc.up_copy_rows:], ldo=8 * c)
        if self.channels_in != self.channels_out:
            out = self.conv1x1.run(out, pf, doctree.batch_size)
        return out


class GraphDownsample(nn.Module):
    """The VAE's downsample (reference dualoctree_networks/modules.py:39-66): depth-(d+1) graph -> depth-d graph;
    called with the TARGET depth d (graph_vae.py:155)."""

    def __init__(self, channels_in, channels_out=None):
        super().__init__()
        self.channels_in = channels_in
        self.channels_out = channels_out or channels_in
        self.downsample = Downsample(channels_in)
        if self.channels_in != self.channels_out:
            self.conv1x1 = Conv1x1GnGelu(self.channels_in, self.channels_out)

    @torch.no_grad()
    def forward(self, x, octree, d, leaf_mask=None, numd=None, lnumd=None):
        doctree = octree
        x = x.contiguous()
        pd, pc = doctree.plan[d + 1], doctree.plan[d]
        c = self.channels_in
        out = torch.empty((pc.rows, c), dtype=x.dtype, device=x.device)
        ops.copy_rows(x, out, pd.down_copy_rows, c, dst_rows=pd.down_copy_dst)
        ops.gather_gemm(x[pd.leaf_base:].view(-1, 8 * c), self.downsample.prepared(), out=out, out_rows=pd.down_out_rows)
        if self.channels_in != self.channels_out:
            out = self.conv1x1.run(out, pc, doctree.batch_size)
        return out


class DiagonalGaussianDistribution:
    """reference distributions.py:24-63: mean | logvar halves of the moments, logvar clamped to [-30, 20]; `sample`
    draws its noise from the host default generator (as the reference does) and moves it to the device."""

    def __init__(self, parameters):
        self.parameters = parameters.float()
        self.mean, self.logvar = torch.chunk(self.parameters, 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)
        self.var = torch.exp(self.logvar)

    def sample(self):
        return self.mean + self.std * torch.randn(self.mean.shape).to(device=self.parameters.device)

    def kl(self):
        return 0.5 * (torch.pow(self.mean, 2) + self.var - 1.0 - self.logvar)

    def mode(self):
        return self.mean


# =================================================================================================
# the network
# =================================================================================================
class GraphVAE(nn.Module):
    """reference graph_vae.py:50-131 (constructor), :132-170 (encoder), :171-223 (octree_decoder), :226-244
    (create_*_octree), :246-298 (forward, extract_code), :300-324 (decode_code)."""

    def __init__(self, depth, channel_in, nout, full_depth=2, depth_stop=6, depth_out=8, use_checkpoint=False,
                 resblk_type='bottleneck', bottleneck=4, resblk_num=3, code_channel=3, embed_dim=3):
        super().__init__()
        self.depth, self.channel_in, self.nout = depth, channel_in, nout
        self.full_depth, self.depth_stop, self.depth_out = full_depth, depth_stop, depth_out
        self.use_checkpoint, self.resblk_type, self.bottleneck, self.resblk_num = (use_checkpoint, resblk_type,
                                                                                   bottleneck, resblk_num)
        self.neural_mpu = NeuralMPU(self.full_depth, self.depth_stop, self.depth_out)
        self.resblk_nums = [resblk_num] * 16
        self.channels = [4, 512, 512, 256, 128, 64, 32, 32, 24, 8]          # graph_vae.py:125
        self.dropout = 0.0
        n_edge_type, avg_degree = 7, 7
        ch, rn = self.channels, self.resblk_nums
        # encoder (graph_vae.py:76-88)
        self.conv1 = GraphConv(channel_in, ch[depth], n_edge_type, avg_degree, depth - 1)
        self.encoder = nn.ModuleList([
            GraphResBlocks(ch[d], ch[d], self.dropout, rn[d] - 1, n_edge_type, avg_degree, d - 1, use_checkpoint)
            for d in range(depth, depth_stop - 1, -1)])
        self.downsample = nn.ModuleList([GraphDownsample(ch[d], ch[d - 1]) for d in range(depth, depth_stop, -1)])
        self.encoder_norm_out = DualOctreeGroupNorm(ch[depth_stop])
        self.nonlinearity = nn.GELU()
        # decoder (graph_vae.py:92-105)
        self.decoder = nn.ModuleList([
            GraphResBlocks(ch[d], ch[d], self.dropout, rn[d], n_edge_type, avg_degree, d - 1, use_checkpoint)
            for d in range(depth_stop, depth + 1)])
        self.decoder_mid = nn.Module()
        self.decoder_mid.block_1 = GraphResBlocks(ch[depth_stop], ch[depth_stop], self.dropout, rn[depth_stop],
                                                  n_edge_type, avg_degree, depth_stop - 1, use_checkpoint)
        self.decoder_mid.block_2 = GraphResBlocks(ch[depth_stop], ch[depth_stop], self.dropout, rn[depth_stop],
                                                  n_edge_type, avg_degree, depth_stop - 1, use_checkpoint)
        self.upsample = nn.ModuleList([GraphUpsample(ch[d - 1], ch[d]) for d in range(depth_stop + 1, depth + 1)])
        # heads (graph_vae.py:108-113): split label (2) and MPU value + normal (4) per node
        self.predict = nn.ModuleList([self._make_predict_module(ch[d], 2) for d in range(depth_stop, depth + 1)])
        self.regress = nn.ModuleList([self._make_predict_module(ch[d], 4) for d in range(depth_stop, depth + 1)])
        self.code_channel = code_channel
        self.KL_conv = Conv1x1(ch[depth_stop], 2 * embed_dim, use_bias=True)
        self.post_KL_conv = Conv1x1(embed_dim, ch[depth_stop], use_bias=True)

    def _make_predict_module(self, channel_in, channel_out=2, num_hidden=32):
        return nn.Sequential(Conv1x1GnGeluSequential(channel_in, num_hidden),
                             Conv1x1(num_hidden, channel_out, use_bias=True))

    # ---- octrees (graph_vae.py:226-244) ---------------------------------------------------------
    def create_full_octree(self, octree_in):
        octree = Octree(self.depth, self.full_depth, octree_in.batch_size, octree_in.device)
        for d in range(self.full_depth + 1):
            octree.octree_grow_full(d)
        return octree

    def create_child_octree(self, octree_in):
        octree_out = self.create_full_octree(octree_in)
        octree_out.depth = self.full_depth
        for d in range(self.full_depth, self.depth_stop):
            octree_out.octree_split(octree_in.nempty_mask(d).long(), d)
            octree_out.octree_grow(d + 1)
            octree_out.depth += 1
        return octree_out

    # ---- encoder (graph_vae.py:132-170) -----------------------------------------------------------
    def _get_input_feature(self, doctree, dtype=torch.float32):
        return doctree.get_input_feature(dtype=dtype)

    @torch.no_grad()
    def octree_encoder_step(self, data, doctree):
        convd = data
        for i, d in enumerate(range(self.depth, self.depth_stop - 1, -1)):
            if d == self.depth:
                convd = self.conv1(convd, doctree, d)
            convd = self.encoder[i](convd, doctree, d)
            if d > self.depth_stop:
                convd = self.downsample[i](convd, doctree, d - 1)
        plan = doctree.plan[self.depth_stop]
        return self.encoder_norm_out.run(convd.contiguous(), plan, doctree.batch_size, act='gelu')

    @torch.no_grad()
    def encode_moments(self, data, doctree):
        """mean | logvar of the posterior (`KL_conv`, graph_vae.py:163-168); sampling is the caller's."""
        return self.KL_conv(self.octree_encoder_step(data, doctree))

    @torch.no_grad()
    def octree_encoder(self, octree, doctree, dtype=torch.float32):
        """posterior of the octree built from points (graph_vae.py:158-165)."""
        return DiagonalGaussianDistribution(self.encode_moments(self._get_input_feature(doctree, dtype), doctree))

    @torch.no_grad()
    def extract_code(self, octree_in, dtype=torch.float32):
        """graph_vae.py:291-298: (one posterior sample [rows of the depth_stop graph, embed_dim] fp32, the input's
        DualOctree).  `dtype` is the activation dtype of the encoder (float32 or bfloat16)."""
        doctree_in = DualOctree(octree_in)
        return self.octree_encoder(octree_in, doctree_in, dtype).sample(), doctree_in

    @torch.no_grad()
    def forward(self, octree_in, octree_out=None, pos=None, evaluate=False, dtype=torch.float32):
        """graph_vae.py:246-289 (inference): encode `octree_in`, sample the posterior (twice when `evaluate`, decoding
        with the second sample, as the reference does), decode -- growing the octree from the labels when `octree_out`
        is None.  The `neural_mpu` closure evaluates at depth_stop (:286).  `dtype` is the activation dtype."""
        doctree_in = DualOctree(octree_in)
        update_octree = octree_out is None
        if update_octree:
            octree_out = self.create_child_octree(octree_in)
        doctree_out = DualOctree(octree_out)
        posterior = self.octree_encoder(octree_in, doctree_in, dtype)
        z = posterior.sample()
        if evaluate:
            z = posterior.sample()
        out = self.octree_decoder(z.to(dtype), doctree_out, update_octree)
        output = {'logits': out[0], 'reg_voxs': out[1], 'octree_out': out[2],
                  'kl_loss': posterior.kl().mean(), 'code_max': z.max(), 'code_min': z.min()}
        if pos is not None:
            output['mpus'] = self.neural_mpu(pos, out[1], out[2])

        def _neural_mpu(pos):
            return self.neural_mpu(pos, out[1], out[2])[self.depth_stop][0]
        _neural_mpu.mpu_args = (self.neural_mpu, out[1], out[2], self.depth_stop)
        output['neural_mpu'] = _neural_mpu
        return output

    # ---- decoder ---------------------------------------------------------------------------------
    @torch.no_grad()
    def octree_decoder(self, code, doctree_out, update_octree=False):
        logits, reg_voxs = {}, {}
        ds = self.depth_stop
        h = self.post_KL_conv(code)
        h = self.decoder_mid.block_1(h, doctree_out, ds)
        h = self.decoder_mid.block_2(h, doctree_out, ds)
        for i, d in enumerate(range(ds, self.depth_out + 1)):
            if d > ds:
                h = self.upsample[i - 1](h, doctree_out, d)
            h = self.decoder[i](h, doctree_out, d)
            logit = self.predict[i]([h, doctree_out, d])
            nnum = int(doctree_out.nnum[d])
            logits[d] = logit[logit.shape[0] - nnum:]
            if update_octree:
                label = logits[d].float().argmax(1).to(torch.int32)
                octree_out = doctree_out.octree
                octree_out.octree_split(label, d)
                if d < self.depth_out:
                    octree_out.octree_grow(d + 1)
                    octree_out.depth += 1
                doctree_out = DualOctree(octree_out)
                doctree_out.post_processing_for_docnn()
            reg_vox = self.regress[i]([h, doctree_out, d])
            node_mask = doctree_out.graph[d]['node_mask']
            pad = torch.zeros((node_mask.shape[0], reg_vox.shape[1]), dtype=reg_vox.dtype, device=reg_vox.device)
            pad[node_mask] = reg_vox
            reg_voxs[d] = pad
        return logits, reg_voxs, doctree_out.octree

    @torch.no_grad()
    def decode_code(self, code, doctree_in, update_octree=True, pos=None):
        if update_octree:
            octree_out = self.create_child_octree(doctree_in.octree)
            doctree_out = DualOctree(octree_out)
            doctree_out.post_processing_for_docnn()
        else:
            doctree_out = doctree_in
        out = self.octree_decoder(code, doctree_out, update_octree=update_octree)
        output = {'logits': out[0], 'reg_voxs': out[1], 'octree_out': out[2]}
        if pos is not None:
            output['mpus'] = self.neural_mpu(pos, out[1], out[2])

        def _neural_mpu(pos):                              # graph_vae.py:317-322: SDF at arbitrary points, finest depth
            return self.neural_mpu(pos, out[1], out[2])[self.depth_out][0]
        _neural_mpu.mpu_args = (self.neural_mpu, out[1], out[2])      # lets mpu.calc_sdf generate the grid in-kernel
        output['neural_mpu'] = _neural_mpu
        return output
