"""-m gpu parity tests of the individual kernels against the oracle (oracle/restate.py), through the
C ABI (ctypes).  Bit-exact for the integer graph build; fp32 kernels within 1e-4 (accumulation order);
bf16 tensor-core kernels within 2e-2 of the fp32 oracle and within 2e-3 of the oracle fed the same
bf16-rounded operands."""
import math
import pytest
import torch
import torch.nn.functional as F

from oracle import restate as R
from tests.util import relerr, oracle_doctree, product_doctree

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def _rand(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g) * scale


def _bf(x):
    return x.to(torch.bfloat16).float()


# ------------------------------------------------------------------------------------------------
# graph build (integer work: exact)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('batch,seed', [(1, 0), (2, 0), (3, 5)])
def test_graph_build_matches_oracle(batch, seed):
    dg, _ = oracle_doctree(batch, seed)
    doc = product_doctree(batch, seed)
    assert doc.total_num == dg.total_num
    for d in range(4, 7):
        a = R.edge_set({k: v.cpu() for k, v in
                        dict(edge_idx=doc.graph[d]['edge_idx'], edge_dir=doc.graph[d]['edge_dir']).items()})
        b = R.edge_set(dg.graph[d])
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), 'edge set differs at depth %d' % d
        assert torch.equal(doc.graph[d]['node_type'].cpu(), dg.graph[d]['node_type'])
        assert torch.equal(doc.batch_id(d).cpu(), dg.batch_id(d))
        # the reference's sort key (dual_octree.py:332-341): row*7+dir non-decreasing
        key = doc.graph[d]['edge_idx'][0] * 7 + doc.graph[d]['edge_dir']
        assert bool((key[1:] >= key[:-1]).all())


def test_scan_and_histogram():
    from octfusion_b200 import ops
    for n in (0, 1, 5, 2048, 2049, 1000003):
        v = torch.randint(0, 5, (n,), dtype=torch.int32, device=DEV)
        out = ops.exclusive_scan_i32(v).cpu()
        ref = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(v.cpu().long(), 0)])
        assert torch.equal(out.long(), ref), n


# ------------------------------------------------------------------------------------------------
# GraphConv
# ------------------------------------------------------------------------------------------------
def _graphconv_case(batch, d, cin, cout, nt, dtype, seed=0, force_simt=False):
    from octfusion_b200.modules import GraphConv
    from octfusion_b200 import ops
    dg, _ = oracle_doctree(batch, 0)
    doc = product_doctree(batch, 0)
    n = dg.graph[d]['node_type'].shape[0]
    x = _rand((n, cin), seed + 1)
    conv = GraphConv(cin, cout, 7, 7, nt)
    w = _rand(tuple(conv.weights.shape), seed + 2, 1.0 / math.sqrt(conv.weights.shape[0]))
    conv.weights.data.copy_(w)
    conv = conv.to(DEV)
    ops.set_force_simt(force_simt)
    try:
        y = conv(x.to(DEV).to(dtype), doc, d).float().cpu()
    finally:
        ops.set_force_simt(False)
    ref32 = R.graph_conv(x, dg.graph[d], w, nt)
    refbf = R.graph_conv(_bf(x), dg.graph[d], _bf(w), nt)
    return y, ref32, refbf


def test_graphconv_config1_fp32():
    """BASELINE.json configs[0] analogue: 8->8 on the depth-4 full layer of one octree, fp32."""
    y, ref, _ = _graphconv_case(1, 4, 8, 8, 0, torch.float32)
    assert relerr(y, ref) < 1e-5


@pytest.mark.parametrize('d,cin,cout,nt', [(4, 64, 64, 3), (5, 128, 256, 4), (6, 3, 128, 5), (6, 128, 3, 5),
                                           (6, 128, 128, 5)])
def test_graphconv_fp32(d, cin, cout, nt):
    y, ref, _ = _graphconv_case(2, d, cin, cout, nt, torch.float32)
    assert relerr(y, ref) < 1e-4


@pytest.mark.parametrize('d,cin,cout,nt', [(4, 64, 64, 3), (4, 256, 512, 3), (5, 128, 256, 4), (6, 128, 128, 5),
                                           (6, 128, 3, 5), (6, 384, 128, 5), (5, 64, 32, 4)])
def test_graphconv_bf16_tensor_core(d, cin, cout, nt):
    y, ref32, refbf = _graphconv_case(2, d, cin, cout, nt, torch.bfloat16)
    assert relerr(y, refbf) < 8e-3          # output rounding to bf16 (2^-9) dominates
    assert relerr(y, ref32) < 2e-2          # north-star bf16 tolerance


def test_graphconv_bf16_simt_equals_tc():
    y_tc, _, refbf = _graphconv_case(2, 6, 128, 128, 5, torch.bfloat16)
    y_si, _, _ = _graphconv_case(2, 6, 128, 128, 5, torch.bfloat16, force_simt=True)
    assert relerr(y_si, refbf) < 8e-3
    assert relerr(y_tc, y_si) < 8e-3


# ------------------------------------------------------------------------------------------------
# plain GEMMs with the fused epilogues
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('m,k,n', [(1000, 128, 64), (4096, 256, 128), (333, 64, 256), (5000, 512, 512), (77, 64, 16)])
def test_linear_epilogues(dtype, m, k, n):
    from octfusion_b200 import ops
    from octfusion_b200.ops import PreparedWeight
    x, w = _rand((m, k), 1), _rand((n, k), 2, 1 / math.sqrt(k))
    bias, resid = _rand((n,), 3), _rand((m, n), 4)
    emb = _rand((7, n), 5)
    idx = torch.randint(0, 7, (m,), generator=torch.Generator().manual_seed(6)).int()
    pw = PreparedWeight(1, k, 0, n).refresh(w.to(DEV), 'linear')
    y = ops.gather_gemm(x.to(DEV).to(dtype), pw, bias=bias.to(DEV), resid=resid.to(DEV).to(dtype),
                        row_add=emb.to(DEV), row_add_idx=idx.to(DEV)).float().cpu()
    if dtype == torch.float32:
        ref = x @ w.t() + bias + resid + emb[idx.long()]
        assert relerr(y, ref) < 1e-5
    else:
        ref = _bf(x) @ _bf(w).t() + bias + _bf(resid) + emb[idx.long()]
        assert relerr(y, ref) < 8e-3


@pytest.mark.parametrize('m,k,n', [(1000, 2048, 256), (2048, 3456, 128), (300, 1536, 64), (2048, 6912, 32)])
def test_gemm_split_k(m, k, n):
    """small M, long K (the dense 4^3 level of the LR U-Net): of_tc_splitk_plan cuts K into ranges computed by different
    CTAs (fp32 partial slabs), the reduce pass adds them in order with bias / emb / residual and produces the norm
    statistics -- same result as the single-pass kernel up to fp32 summation order, and bit-reproducible"""
    from octfusion_b200 import ops
    from octfusion_b200._lib import lib, GemmArgs
    from octfusion_b200.ops import PreparedWeight
    x, w = _rand((m, k), 1), _rand((n, k), 2, 1 / math.sqrt(k))
    bias, resid = _rand((n,), 3), _rand((m, n), 4)
    emb = _rand((7, n), 5)
    idx = torch.randint(0, 7, (m,), generator=torch.Generator().manual_seed(6)).int()
    pw = PreparedWeight(1, k, 0, n).refresh(w.to(DEV), 'linear')
    plan = ops.StatPlan(m, batch=4, rows_per_sample=(m + 3) // 4, device=DEV) if n % 32 == 0 else None
    run = lambda: ops.gather_gemm(x.to(DEV).bfloat16(), pw, bias=bias.to(DEV), resid=resid.to(DEV).bfloat16(),  # noqa: E731
                                  row_add=emb.to(DEV), row_add_idx=idx.to(DEV), stats=plan)
    keep = ops._SPLIT_K
    y1 = None
    try:
        ops._SPLIT_K = False
        y1 = run()                                           # single pass (also packs the weight image)
        ops._SPLIT_K = True
        launches0 = lib.of_launch_count()
        y = run()
        assert lib.of_launch_count() - launches0 == 2, 'expected the split-K pair of launches'
        y2 = run()
    finally:
        ops._SPLIT_K = keep
    assert torch.equal(y, y2) and torch.equal(y._of_stats.part, y2._of_stats.part)
    ref = _bf(x) @ _bf(w).t() + bias + _bf(resid) + emb[idx.long()]
    assert relerr(y.float().cpu(), ref) < 8e-3
    assert relerr(y.float().cpu(), y1.float().cpu()) < 8e-3          # (max norm: one bf16 ulp at the top of the range)
    assert relerr(y._of_stats.part.cpu(), y1._of_stats.part.cpu()) < 1e-4


def test_gemm_row_maps_and_concat():
    from octfusion_b200 import ops
    from octfusion_b200.ops import PreparedWeight
    m, k0, k1, n = 900, 64, 128, 128
    x0, x1, w = _rand((m, k0), 1), _rand((m, k1), 2), _rand((n, k0 + k1), 3, 0.1)
    g = torch.Generator().manual_seed(4)
    in_rows = torch.randint(0, m, (500,), generator=g).int()
    out_rows = torch.randperm(700, generator=g)[:500].int()
    for dtype, tol in ((torch.float32, 1e-5), (torch.bfloat16, 8e-3)):
        pw = PreparedWeight(1, k0 + k1, 0, n).refresh(w.to(DEV), 'linear')
        out = torch.zeros((700, n), dtype=dtype, device=DEV)
        ops.gather_gemm(x0.to(DEV).to(dtype), pw, a1=x1.to(DEV).to(dtype), in_rows=in_rows.to(DEV),
                        out_rows=out_rows.to(DEV), out=out)
        xx = torch.cat([x0, x1], 1)
        if dtype == torch.bfloat16:
            xx, ww = _bf(xx), _bf(w)
        else:
            ww = w
        ref = torch.zeros(700, n)
        ref[out_rows.long()] = xx[in_rows.long()] @ ww.t()
        assert relerr(out.float().cpu(), ref) < tol


# ------------------------------------------------------------------------------------------------
# group norm
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('d,c0,c1', [(6, 128, 0), (5, 256, 128), (4, 64, 0), (6, 24, 0), (5, 512, 256)])
def test_doctree_group_norm(dtype, d, c0, c1):
    from octfusion_b200.modules import DualOctreeGroupNorm
    dg, _ = oracle_doctree(3, 5)
    doc = product_doctree(3, 5)
    n = dg.batch_id(d).shape[0]
    x = _rand((n, c0 + c1), 1) * 2.0 + 0.7
    gn = DualOctreeGroupNorm(c0 + c1)
    gn.weights.data.copy_(1 + 0.1 * _rand((1, c0 + c1), 2)); gn.bias.data.copy_(0.1 * _rand((1, c0 + c1), 3))
    gam, bet = gn.weights.data.clone(), gn.bias.data.clone()
    gn = gn.to(DEV)
    xin = x if dtype == torch.float32 else _bf(x)
    ref = R.silu(R.doctree_group_norm(xin, dg.batch_id(d), 3, gam, bet))
    xd = x.to(DEV).to(dtype)
    if c1:
        y = gn.run(xd[:, :c0].contiguous(), doc.plan[d], 3, x1=xd[:, c0:].contiguous(), act=True)
    else:
        y = gn.run(xd, doc.plan[d], 3, act=True)
    assert relerr(y.float().cpu(), ref) < (2e-5 if dtype == torch.float32 else 8e-3)


def _nan_parts(monkeypatch):
    """every slot of a partial-statistics buffer must be written by its producer: start them as NaN"""
    from octfusion_b200 import ops
    orig = ops.StatPlan.new_part
    monkeypatch.setattr(ops.StatPlan, 'new_part', lambda self, c, g: orig(self, c, g).fill_(float('nan')))


@pytest.mark.parametrize('d,cin,cout,resid', [(6, 128, 128, True), (5, 128, 256, False), (4, 256, 512, False), (6, 64, 64, False)])
def test_gemm_epilogue_statistics(monkeypatch, d, cin, cout, resid):
    """The tensor-core epilogue's group-norm partials (of_gemm_args.stat_out) against the stand-alone of_gn_stats pass over
    the same output: same slots, sums equal up to the bf16 rounding of the stored tensor; the norm built on either is
    the oracle's norm of the output.  3 ragged samples (chunks that straddle samples take the masked path)."""
    from octfusion_b200 import ops
    from octfusion_b200.modules import GraphConv, DualOctreeGroupNorm
    _nan_parts(monkeypatch)
    dg, _ = oracle_doctree(3, 5)
    doc = product_doctree(3, 5)
    plan = doc.plan[d]
    n = plan.rows
    conv = GraphConv(cin, cout, 7, 7, d - 1).to(DEV)
    x = (_rand((n, cin), 3) * 1.5 + 0.3).to(DEV).bfloat16()
    res = _rand((n, cout), 4).to(DEV).bfloat16() if resid else None
    emb = _rand((3, cout), 5).to(DEV)
    y = conv.run(x, plan, row_add=emb, row_add_idx=plan.batch_id, resid=res, stats=plan.stat)
    st = getattr(y, '_of_stats', None)
    assert st is not None and st.plan is plan.stat and st.part.shape == (plan.stat.n_seg, cout // st.gran * 2)
    fused = st.part.double().cpu()
    assert torch.isfinite(fused).all()
    alone, ga = ops._stats_of(y.clone(), plan.stat, st.gran)
    assert ga == st.gran
    alone = alone.double().cpu()
    assert torch.isfinite(alone).all()
    # per segment the two differ by the bf16 rounding of <= 128 values; per sample (sum over its segments) by much less
    off = plan.stat.sample_seg_off.cpu().tolist()              # a sample's partials are consecutive rows (seg_slot)
    for b in range(3):
        fa, al = fused[off[b]:off[b + 1]].sum(0), alone[off[b]:off[b + 1]].sum(0)
        assert float((fa - al).abs().max() / al.abs().max()) < 2e-3
    gn = DualOctreeGroupNorm(cout).to(DEV)
    a = gn.run(y, plan, 3, act=True).float().cpu()
    ref = R.silu(R.doctree_group_norm(y.float().cpu(), dg.batch_id(d), 3, gn.weights.data.cpu(), gn.bias.data.cpu()))
    assert relerr(a, ref) < 8e-3
    # bit-reproducible: a second launch writes identical partials
    y2 = conv.run(x, plan, row_add=emb, row_add_idx=plan.batch_id, resid=res, stats=plan.stat)
    assert torch.equal(y2._of_stats.part, st.part) and torch.equal(y2, y)


def test_gemm_epilogue_statistics_dense_small_samples(monkeypatch):
    """dense layout with 8 rows per sample (T = 8 tokens of the cond config): four samples per 32-row chunk"""
    from octfusion_b200 import ops
    from octfusion_b200.modules import DenseTables, conv_nd, convnormalization
    _nan_parts(monkeypatch)
    b, c = 5, 128
    t = DenseTables(b, DEV)
    sp = t.stat_plan(1)
    assert sp.n_seg == 5
    lin = conv_nd(1, c, c, 1).to(DEV)
    x = (_rand((b * 8, c), 1) + 0.2).to(DEV).bfloat16()
    y = lin.run(x, stats=sp)
    assert y._of_stats.part.shape == (5, c // 2) and y._of_stats.gran == 4 and torch.isfinite(y._of_stats.part).all()
    norm = convnormalization(c).to(DEV)
    a = norm.run(y, t, 1, act=True).float().cpu()
    yy = y.float().cpu().reshape(b, 8, c).permute(0, 2, 1)                    # [B, C, T]
    ref = R.silu(F.group_norm(yy, 32, norm.weight.data.cpu(), norm.bias.data.cpu(), 1e-5)).permute(0, 2, 1).reshape(b * 8, c)
    assert relerr(a, ref) < 8e-3


# ------------------------------------------------------------------------------------------------
# attention / dense convolutions
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('b,t,heads,ch', [(2, 512, 4, 32), (3, 64, 4, 64), (2, 8, 4, 128), (2, 512, 4, 16)])
def test_attention(dtype, b, t, heads, ch):
    from octfusion_b200 import ops
    c = heads * ch
    qkv = _rand((b, 3 * c, t), 1)                                   # reference layout [b, 3C, T]
    src = qkv if dtype == torch.float32 else _bf(qkv)
    ref = R.qkv_attention(src.reshape(b * heads, 3 * ch, t)).reshape(b, c, t)
    x = qkv.permute(0, 2, 1).reshape(b * t, 3 * c).contiguous().to(DEV).to(dtype)
    y = ops.attention(x, b, t, heads).float().cpu().reshape(b, t, c).permute(0, 2, 1)
    assert relerr(y, ref) < (1e-5 if dtype == torch.float32 else 8e-3)


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('mode,res,cin,cout', [('same', 8, 64, 128), ('down', 16, 64, 64), ('up', 4, 128, 128),
                                               ('same', 16, 64, 64)])
def test_dense_conv3d(dtype, mode, res, cin, cout):
    from octfusion_b200.modules import _Conv3dParams, ConvDownsample, ConvUpsample
    b = 2
    x = _rand((b, cin, res, res, res), 1)
    w = _rand((cout, cin, 3, 3, 3), 2, 1 / math.sqrt(27 * cin))
    bias = _rand((cout,), 3)
    xs, ws = (x, w) if dtype == torch.float32 else (_bf(x), _bf(w))
    if mode == 'same':
        from octfusion_b200.modules import DenseTables, _to_morton, _from_morton
        conv = _Conv3dParams(cin, cout, 3, padding=1)
        conv.weight.data.copy_(w); conv.bias.data.copy_(bias)
        conv = conv.to(DEV)
        t = DenseTables(b, torch.device(DEV))
        xm, r = _to_morton(x.to(DEV).to(dtype), t)
        y = _from_morton(conv.run(xm, t.conv(r)), t, b, r)
        ref = F.conv3d(xs, ws, bias, padding=1)
    elif mode == 'down':
        m = ConvDownsample(cin)
        m.op.weight.data.copy_(w); m.op.bias.data.copy_(bias)
        y = m.to(DEV)(x.to(DEV).to(dtype))
        ref = F.conv3d(xs, ws, bias, stride=2, padding=1)
    else:
        m = ConvUpsample(cin)
        m.conv.weight.data.copy_(w); m.conv.bias.data.copy_(bias)
        y = m.to(DEV)(x.to(DEV).to(dtype))
        ref = F.conv3d(F.interpolate(xs, scale_factor=2, mode='nearest'), ws, bias, padding=1)
    assert y.shape == ref.shape
    assert relerr(y.float().cpu(), ref) < (1e-5 if dtype == torch.float32 else 8e-3)


# ------------------------------------------------------------------------------------------------
# small per-step kernels
# ------------------------------------------------------------------------------------------------
def test_embeddings_and_ddim():
    from octfusion_b200 import ops
    t = torch.tensor([9.2, 1.5, -0.5, -2.3])
    e = ops.timestep_embedding(t.to(DEV), 128).cpu()
    assert relerr(e, R.timestep_embedding(t, 128)) < 1e-5
    w = _rand((32,), 1)
    e = ops.learned_sinusoidal(t.to(DEV), w.to(DEV)).cpu()
    assert relerr(e, R.learned_sinusoidal(t, w)) < 1e-4
    x, eps = _rand((1000, 3), 2), _rand((1000, 3), 3)
    ls, lsn = torch.tensor([1.3]), torch.tensor([2.1])
    ref = R.ddim_eps_update(x, eps, ls, lsn)
    xd = x.to(DEV).clone()
    xa = torch.empty((1000, 3), dtype=torch.bfloat16, device=DEV)
    ops.ddim_eps_update(xd, eps.to(DEV), ls.to(DEV), lsn.to(DEV), xa)
    assert relerr(xd.cpu(), ref) < 1e-5
    assert relerr(xa.float().cpu(), ref) < 8e-3


@pytest.mark.parametrize('b,k,n', [(32, 512, 512), (2, 128, 512), (5, 65, 256), (40, 256, 64)])
def test_linear_small(b, k, n):
    from octfusion_b200 import ops
    x, w, bias = _rand((b, k), 1), _rand((n, k), 2, 1 / math.sqrt(k)), _rand((n,), 3)
    y = ops.linear_small(x.to(DEV), w.to(DEV), bias.to(DEV), a_silu=True).cpu()
    assert relerr(y, F.linear(R.silu(x), w, bias)) < 1e-5


def test_graphconv_small_channel_input_padded_to_tc():
    """the 3- / 8-channel latent of the first conv is zero-padded to 64 channels for the tensor-core path."""
    for cin in (3, 8):
        y, ref32, refbf = _graphconv_case(2, 6, cin, 128, 5, torch.bfloat16)
        assert relerr(y, refbf) < 8e-3 and relerr(y, ref32) < 2e-2


def test_graph_type_block_matches_edge_lists():
    """of_graph_type_block == scatter_mean of one_hot(node_type[col]) over (row, dir) (reference modules.py:199-202)."""
    from tests.util import product_doctree
    doc = product_doctree(2, 7)
    for d in range(4, 7):
        p = doc.plan[d]
        nt = d - 1
        blk = p.tap.type_block(nt, p.node_type).float()
        g = doc.graph[d]
        row, col, edir = g['edge_idx'][0], g['edge_idx'][1], g['edge_dir']
        slot = (row * 7 + edir) * nt + p.node_type.long()[col]
        cnt = torch.zeros(p.rows * 7 * nt, device=DEV).index_add_(0, slot, torch.ones(len(row), device=DEV))
        tot = torch.zeros(p.rows * 7, device=DEV).index_add_(0, row * 7 + edir, torch.ones(len(row), device=DEV))
        want = (cnt.view(p.rows, 7, nt) / tot.clamp(min=1).view(p.rows, 7, 1)).reshape(p.rows, 7 * nt)
        assert blk.shape == (p.rows, 64)
        assert torch.equal(blk[:, :7 * nt], want.bfloat16().float())
        assert float(blk[:, 7 * nt:].abs().max()) == 0.0
