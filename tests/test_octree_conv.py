"""`ocnn.nn.OctreeConv` adapter (BASELINE.json configs[0]: "single OctreeConv 3^3 k=8->8 on one depth-4 synthetic octree").
ocnn is third-party and absent: parity is UNPINNED at that boundary (SURVEY.md section 0, Appendix B).  Anchors used:
  * CPU: the oracle restatement equals torch conv3d (zero padding) on a full octree layer -- a known-answer check that
    does not depend on ocnn;
  * GPU: the CUDA path (of_octree_neigh27 + tap-gather GEMM) equals the oracle on full and adaptive layers, stride 1 / 2,
    nempty, fp32 (CUDA cores) and bf16 (tensor cores)."""
import pytest
import torch
import torch.nn.functional as F

from oracle import restate as R
from tests.util import relerr, oracle_doctree, product_doctree


def _rand(shape, seed, scale=1.0):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)) * scale


def test_oracle_octree_conv_is_conv3d_on_a_full_layer():
    dg, _ = oracle_doctree(2, 0)
    octree = dg.octree
    d, cin, cout, b = 4, 8, 8, 2
    x = _rand((b * 4096, cin), 1)
    w = _rand((27, cin, cout), 2, 0.1)
    y = R.octree_conv(x, octree, d, w)
    xs, ys, zs, bs = octree.xyzb(d)
    vox = torch.zeros(b, 16, 16, 16, cin)
    vox[bs, xs, ys, zs] = x
    wk = w.view(3, 3, 3, cin, cout).permute(4, 3, 0, 1, 2).contiguous()          # [Cout, Cin, dx, dy, dz]
    ref = F.conv3d(vox.permute(0, 4, 1, 2, 3), wk, padding=1).permute(0, 2, 3, 4, 1)[bs, xs, ys, zs]
    assert relerr(y, ref) < 1e-5
    # stride 2: the window of every 8th node = the 3^3 window around the first child of each parent
    y2 = R.octree_conv(x, octree, d, w, stride=2)
    assert y2.shape[0] == x.shape[0] // 8 and torch.equal(y2, y[::8])


def test_oracle_neighbours_are_symmetric_on_adaptive_layers():
    dg, _ = oracle_doctree(1, 0)                                                   # (the restatement is a Python loop per node)
    for d in (5, 6):
        nb = R.octree_neigh27(dg.octree, d)
        n = nb.shape[0]
        assert torch.equal(nb[:, 13], torch.arange(n))                            # centre tap = the node itself
        for t in (0, 5, 12, 22):
            rows = torch.nonzero(nb[:, t] >= 0).squeeze(1)
            assert torch.equal(nb[nb[rows, t], 26 - t], rows)                     # opposite tap points back


@pytest.mark.gpu
@pytest.mark.parametrize('d,cin,cout,dtype,stride,nempty', [
    (4, 8, 8, torch.float32, 1, False),          # configs[0]
    (4, 8, 8, torch.bfloat16, 1, False),
    (5, 64, 128, torch.bfloat16, 1, False),
    (6, 64, 32, torch.float32, 1, False),
    (6, 128, 128, torch.bfloat16, 2, False),
    (5, 16, 24, torch.float32, 1, True),
])
def test_octree_conv_matches_oracle(d, cin, cout, dtype, stride, nempty):
    from octfusion_b200.octree_conv import OctreeConv, octree_neigh
    dg, _ = oracle_doctree(2, 0)
    doc = product_doctree(2, 0)
    octree_o, octree_p = dg.octree, doc.octree
    nb = octree_neigh(octree_p, d, stride, nempty).cpu().long()
    assert torch.equal(nb, R.octree_neigh27(octree_o, d, stride, nempty))
    n_in = int(octree_o.nnum_nempty[d]) if nempty else int(octree_o.nnum[d])
    x = _rand((n_in, cin), 3)
    conv = OctreeConv(cin, cout, [3], stride=stride, nempty=nempty, use_bias=True)
    conv.weights.data.copy_(_rand((27, cin, cout), 4, (27 * cin) ** -0.5))
    conv.bias.data.copy_(_rand((cout,), 5, 0.1))
    xin = x if dtype == torch.float32 else x.to(dtype).float()
    win = conv.weights.data if dtype == torch.float32 else conv.weights.data.to(dtype).float()
    ref = R.octree_conv(xin, octree_o, d, win, stride, nempty, conv.bias.data)
    y = conv.cuda()(x.cuda().to(dtype), octree_p, d).float().cpu()
    assert y.shape == ref.shape
    assert relerr(y, ref) < (1e-4 if dtype == torch.float32 else 8e-3)
