"""Shared helpers of the point-cloud encoder tests: octree builds through the oracle (oracle/restate_encode.py, the
ocnn restatement: parity UNPINNED at the ocnn boundary) and through the product, and the oracle's encoder chain."""
from __future__ import annotations
import os
import numpy as np
import torch

from oracle import restate_encode as RE
from tests.util import GOLDEN

FIXTURE = os.path.join(GOLDEN, 'vae_encode_points.npz')
# the case of tests/golden/vae_encode_points.npz (oracle/gen_golden_encode.py)
ENC_BATCH, ENC_POINTS, ENC_SEED = 2, 8000, 5
CODE_SEED, FORWARD_SEED = 11, 12
ROW_STEP = 16


def oracle_build(shapes, depth, full_depth, device='cpu'):
    """batched oracle build of [(xyz, normals)] shapes"""
    pts = RE.merge_points([RE.Points(x.to(device), n.to(device)) for x, n in shapes])
    return RE.Octree(depth, full_depth, len(shapes), device).build_octree(pts)


def product_build(shapes, depth, full_depth, device='cuda'):
    from octfusion_b200 import Octree, Points, merge_points
    pts = merge_points([Points(x.to(device), n.to(device)) for x, n in shapes])
    return Octree(depth, full_depth, len(shapes), device).build_octree(pts)


def assert_same_structure(a, b, depth, full_depth=0):
    assert a.nnum.tolist() == b.nnum.tolist() and a.nnum_nempty.tolist() == b.nnum_nempty.tolist()
    for d in range(full_depth, depth + 1):
        assert torch.equal(a.keys[d].cpu(), b.keys[d].cpu()), d
        assert torch.equal(a.children[d].cpu(), b.children[d].cpu()), d


def fixture():
    return np.load(FIXTURE)


def fixture_shapes():
    from octfusion_b200.synth import synth_shell_points
    return synth_shell_points(ENC_BATCH, ENC_POINTS, ENC_SEED)


def posterior_sample(moments, seed, draws=1):
    """DiagonalGaussianDistribution (reference distributions.py:24-63): `draws` samples after torch.manual_seed(seed),
    noise from the host default generator; returns (last sample, kl)."""
    mean, logvar = torch.chunk(moments.float().cpu(), 2, dim=1)
    logvar = logvar.clamp(-30.0, 20.0)
    torch.manual_seed(seed)
    for _ in range(draws):
        z = mean + torch.exp(0.5 * logvar) * torch.randn(mean.shape)
    return z, 0.5 * (mean ** 2 + torch.exp(logvar) - 1.0 - logvar)


def oracle_feature(octree, doc):
    """DualOctree.get_input_feature (dual_octree.py:343-360) on the oracle: zero rows for the leaves of
    full_depth..D-1, then InputFeature('ND')."""
    data = RE.InputFeature('ND', nempty=False)(octree)
    leaves = int(doc.lnum[octree.full_depth:octree.depth].sum())
    return torch.cat([torch.zeros(leaves, data.shape[1]), data])
