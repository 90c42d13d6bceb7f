"""octfusion_b200 -- H100 (sm_90a) kernels behind the OctFusion denoising U-Net hot path.

Importing this package loads liboctfusion_b200.so; it raises if the library is missing (there is no
CPU or library fallback).  Public surface mirrors the reference (octree-nn/octfusion):
  octree.Octree, dual_octree.DualOctree                      (ocnn.octree.Octree subset, dual_octree.py)
  modules.{GraphConv, DualOctreeGroupNorm, GraphResBlockEmbed, GraphDownsample, GraphUpsample, Conv1x1,
           Downsample, Upsample, ResnetBlock, AttentionBlock, QKVAttention, ...}   (models/networks/modules.py)
  graph_unet_{hr,lr,union}.UNet3DModel                        (models/networks/diffusion_networks/*)
  sampler.sample_loop / sample_loop_lr                        (models/octfusion_model_union.py:300-352)
  graph_vae.GraphVAE (extract_code, forward, decode_code)     (models/networks/dualoctree_networks/graph_vae.py)
  octree.Points / merge_points / Octree.build_octree, modules.InputFeature('ND')   (ocnn, SURVEY.md Appendix B)
  octree.split2octree_small / octree2split_small              (utils/util_dualoctree.py:198-250)
"""
from . import _lib  # noqa: F401  (fails loudly when the CUDA library is absent)
from .octree import (Octree, Points, merge_points, octree_from_splits, create_full_octree,  # noqa: F401
                     split2octree_small, octree2split_small)
from .dual_octree import DualOctree  # noqa: F401
from .modules import InputFeature  # noqa: F401

__version__ = '0.1.0'
