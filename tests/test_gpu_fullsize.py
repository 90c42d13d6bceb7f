"""-m gpu property tests at BASELINE.json's full size (B=32, depth 6: N6 ~ 0.65 M rows), where the CPU
oracle would take minutes: size-independent properties instead of element-wise comparison."""
import pytest
import torch

from tests.util import relerr, product_doctree

pytestmark = pytest.mark.gpu
DEV = 'cuda'
B = 32


@pytest.fixture(scope='module')
def doc():
    return product_doctree(B, 1000)


def test_graph_invariants_full_size(doc):
    """every edge has its mirror (j in nbr(i,dir) <=> i in nbr(j,opp(dir))), every row has its self loop, node
    counts agree with the octree, build is deterministic."""
    opp = torch.tensor([1, 0, 3, 2, 5, 4, 6], device=DEV)
    for d in range(4, 7):
        g = doc.graph[d]
        row, col, edir = g['edge_idx'][0], g['edge_idx'][1], g['edge_dir']
        n = doc.plan[d].rows
        assert n == int(doc.lnum[4:d].sum()) + int(doc.nnum[d])
        fwd = (row * n + col) * 7 + edir
        bwd = (col * n + row) * 7 + opp[edir]
        assert torch.equal(torch.sort(fwd)[0], torch.sort(bwd)[0]), 'edge set is not symmetric at depth %d' % d
        self_loops = (edir == 6)
        assert int(self_loops.sum()) == n and torch.equal(row[self_loops], col[self_loops])
        assert bool((doc.plan[d].rows_of_sample > 0).all()) and int(doc.plan[d].rows_of_sample.sum()) == n
        # same-depth rows see at most one neighbour per direction; coarser rows up to 16
        per_slot = torch.zeros(n * 7, dtype=torch.long, device=DEV).index_add_(0, row * 7 + edir, torch.ones_like(row))
        assert int(per_slot.max()) <= 16
    doc2 = product_doctree(B, 1000)
    for d in range(4, 7):
        assert torch.equal(doc.plan[d].tap.tab, doc2.plan[d].tap.tab)
        assert torch.equal(doc.plan[d].tap.extra, doc2.plan[d].tap.extra)
        assert torch.equal(doc.plan[d].batch_id, doc2.plan[d].batch_id)


def test_graphconv_linearity_and_paths_agree_full_size(doc):
    from octfusion_b200.modules import GraphConv
    from octfusion_b200 import ops
    d, c = 6, 128
    n = doc.plan[d].rows
    g = torch.Generator(device=DEV).manual_seed(0)
    x = torch.randn((n, c), generator=g, device=DEV)
    y = torch.randn((n, c), generator=g, device=DEV)
    conv = GraphConv(c, c, 7, 7, 5).to(DEV)
    xb, yb = x.bfloat16(), y.bfloat16()
    # GraphConv is AFFINE in x (the one-hot node-type columns add a data-independent term), so the
    # combination must have weights that sum to one: conv(x/2 + y/2) = conv(x)/2 + conv(y)/2
    zb = (xb.float() * 0.5 + yb.float() * 0.5)
    fx, fy = conv(xb, doc, d).float(), conv(yb, doc, d).float()
    fz = conv(zb.bfloat16(), doc, d).float()
    assert relerr(fz, 0.5 * fx + 0.5 * fy) < 1e-2          # bf16 rounding of z and of the three outputs
    # tensor-core path == CUDA-core path on the same bf16 operands (differs only by accumulation order + output rounding)
    ops.set_force_simt(True)
    try:
        sx = conv(xb, doc, d).float()
    finally:
        ops.set_force_simt(False)
    assert relerr(fx, sx) < 8e-3
    # fp32 path agrees with bf16 path within the bf16 tolerance
    assert relerr(fx, conv(x, doc, d)) < 2e-2


def test_group_norm_statistics_full_size(doc):
    from octfusion_b200.modules import DualOctreeGroupNorm
    d, c = 6, 128
    n = doc.plan[d].rows
    x = torch.randn((n, c), device=DEV) * 3.0 + 1.5
    gn = DualOctreeGroupNorm(c).to(DEV)
    for dtype, tol in ((torch.float32, 1e-3), (torch.bfloat16, 2e-2)):
        y = gn(x.to(dtype), doc, d).float()
        bid = doc.batch_id(d)
        cnt = torch.bincount(bid, minlength=B).float() * 4
        s = torch.zeros(B, c, device=DEV).index_add_(0, bid, y).view(B, 32, 4).sum(-1) / cnt[:, None]
        q = torch.zeros(B, c, device=DEV).index_add_(0, bid, y * y).view(B, 32, 4).sum(-1) / cnt[:, None]
        assert float(s.abs().max()) < tol * 5 and float((q - 1).abs().max()) < tol * 5


def test_sampler_is_reproducible_full_size(doc):
    """Two runs with the same seed are bit-identical: convolutions, attention, resampling and -- since round 2 -- the
    norm statistics (per-segment partials, fixed summation order, no atomics) are all deterministic."""
    from octfusion_b200 import graph_unet_union
    from octfusion_b200.sampler import sample_loop
    from tests.util import UNCOND
    import bench
    net = bench.randomise_(graph_unet_union.UNet3DModel('hr', **UNCOND), 0).to(DEV).eval()
    for dtype in (torch.float32, torch.bfloat16):
        a = sample_loop(net.unet_hr, net.unet_lr, doc, ddim_steps=2, seed=5, act_dtype=dtype)
        b = sample_loop(net.unet_hr, net.unet_lr, doc, ddim_steps=2, seed=5, act_dtype=dtype)
        assert torch.isfinite(a).all() and float(a.abs().max()) > 0
        assert torch.equal(a, b), str(dtype)
