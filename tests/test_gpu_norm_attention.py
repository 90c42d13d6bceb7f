"""Group norm (of_gn_stats / of_gn_finalize / of_gn_apply), attention (of_attention) and of_histogram_i32 on every
dispatch path, against float64 references kept in this file, element by element.

Every comparison has the form |y - ref| <= bound(ref, inputs); each bound is derived in a comment from the kernel's
arithmetic (u = 2^-24, the fp32 unit roundoff).  The C ABI is called directly wherever the functional layer would
choose the path itself (vector width, traversal direction, granules, strides, the number of finalize CTAs).
The unmarked tests check the references against oracle/restate.py and run without a GPU."""
import ctypes
import functools
import math

import numpy as np
import pytest
import torch

from oracle import restate as R

DEV = 'cuda'
U = 2.0 ** -24                      # fp32 unit roundoff
BF_HALF_ULP = 2.0 ** -8             # bf16 unit roundoff: 8 significant bits, half an ulp is up to 2^-8 relative
TINY = 2.0 ** -126                  # smallest normal fp32 / bf16
OF_E_ARG, OF_E_UNSUPPORTED = -1, -2
SLOPE = {0: 1.0, 1: 1.1, 2: 1.13}   # max |f'(v)| of identity, SiLU, erf-GELU


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ------------------------------------------------------------------------------------------------
# float64 references
# ------------------------------------------------------------------------------------------------
def act_ref(v, act):
    """exact activation in float64: 0 none, 1 SiLU = v / (1 + e^-v), 2 GELU = v/2 * erfc(-v / sqrt 2)"""
    v = v.double()
    if act == 1:
        return v / (1.0 + torch.exp(-v))
    if act == 2:
        return 0.5 * v * torch.special.erfc(-v / math.sqrt(2.0))
    return v


def gn_ref(x, sample_id, batch, groups, gamma, beta, eps, count_eps, act, stats_x=None):
    """DualOctreeGroupNorm / GroupNorm32 + activation in float64 with two-pass statistics per (sample, group):
    mean = S / (n + count_eps), var = sum (x - mean)^2 / (n + count_eps), n = rows * channels per group.
    stats_x: the values the statistics are taken over when they differ from the normalised x (a GEMM epilogue sums its
    fp32 accumulators before they are rounded to the stored bf16).
    Returns y, the per-(sample, channel) scale, shift, mean, var of the affine form y = act(x * scale + shift), and the
    group means of |x| and x^2 (absmean, sqmean) that scale the rounding errors of one-pass statistics."""
    x = x.double()
    sx = x if stats_x is None else stats_x.double()
    sid = sample_id.long()
    c = x.shape[1]
    cpg = c // groups
    n = torch.bincount(sid, minlength=batch).double() * cpg
    inv = 1.0 / (n + count_eps)
    s = torch.zeros(batch, c, dtype=torch.float64).index_add_(0, sid, sx)
    mean = (s.reshape(batch, groups, cpg).sum(-1) * inv[:, None]).repeat_interleave(cpg, 1)        # [B, C]
    xc = sx - mean[sid]
    q = torch.zeros(batch, c, dtype=torch.float64).index_add_(0, sid, xc * xc)
    var = (q.reshape(batch, groups, cpg).sum(-1) * inv[:, None]).repeat_interleave(cpg, 1)
    rstd = 1.0 / torch.sqrt(var + eps)
    scale = rstd * gamma.double().reshape(1, c)
    shift = beta.double().reshape(1, c) - mean * scale
    y = act_ref((x - mean[sid]) * scale[sid] + beta.double().reshape(1, c), act)
    grp = lambda t: (torch.zeros(batch, c, dtype=torch.float64).index_add_(0, sid, t).reshape(batch, groups, cpg).sum(-1)  # noqa: E731
                     * inv[:, None]).repeat_interleave(cpg, 1)
    return dict(y=y, scale=scale, shift=shift, mean=mean, var=var, eps=eps, absmean=grp(sx.abs()), sqmean=grp(sx * sx))


def attn_ref(qkv, b, t, heads):
    """QKVAttention over channels-last qkv [b*t, 3C] with the legacy head-major split (head h owns columns
    [3h ch, 3(h+1) ch) = q | k | v), float64.  Returns out [b*t, C], sum_s p_s |v_s| [b*t, C] (the scale of the
    rounding errors of P V) and, per output row, the largest |q|.|k| sum behind one score (the scale of the rounding
    errors of Q K^T)."""
    x = qkv.double().reshape(b, t, heads, 3, -1)
    ch = x.shape[-1]
    q, k, v = x[..., 0, :], x[..., 1, :], x[..., 2, :]
    s = torch.einsum('bthc,bshc->bhts', q, k) / math.sqrt(ch)
    p = torch.softmax(s, -1)
    out = torch.einsum('bhts,bshc->bthc', p, v).reshape(b * t, heads * ch)
    pv = torch.einsum('bhts,bshc->bthc', p, v.abs()).reshape(b * t, heads * ch)
    qk = torch.einsum('bthc,bshc->bhts', q.abs(), k.abs()).amax(-1) / math.sqrt(ch)               # [b, h, t]
    qk = qk.permute(0, 2, 1).repeat_interleave(ch, 2).reshape(b * t, heads * ch)
    return out, pv, qk


# ------------------------------------------------------------------------------------------------
# error bounds
# ------------------------------------------------------------------------------------------------
def act_rel_fp32(v, act):
    """relative error of the fp32 activation of gn_apply_kernel at (exact) input v.
    SiLU = v / (1 + __expf(-v)): __expf is good to 2 + floor(1.173 |v|) ulp (CUDA C Programming Guide), an ulp is at
    most 2^-23 relative, and 1 + E and the division add one rounding each.
    GELU = 0.5 v erfcf(-v / sqrt 2): erfcf is good to 4 ulp; the argument carries 2 roundings (constant, product), which
    d ln erfc(x)/dx amplifies by at most 2x + 1.5 for x >= 0 (v <= 0) and not at all for v > 0 (|x erfc'/erfc| <= 0.5);
    two more roundings in the products."""
    v = v.double()
    if act == 1:
        return (3.0 + 1.173 * v.abs()) * 2.0 * U
    if act == 2:
        x = v.abs() / math.sqrt(2.0)
        sens = torch.where(v < 0, 2.0 * x * x + 1.5 * x, torch.full_like(x, 0.5))
        return (4.0 * 2.0 + 2.0 * sens + 2.0 + 1.0) * U
    return torch.zeros_like(v)


def act_cond(v, act):
    """|v f'(v) / f(v)|: how much a relative error of the pre-activation v grows through f (1 for the identity;
    SiLU 1 + v (1 - sigmoid v), GELU 1 + v phi(v) / Phi(v): below 1.3 for v >= 0, below 1 + |v| (|v| + 2) for v < 0)"""
    if act == 0:
        return torch.ones_like(v, dtype=torch.float64)
    a = v.double().abs().clamp(max=1e6)
    return torch.where(v < 0, 1.0 + a * (a + 2.0), torch.full_like(a, 1.3))


def gn_pre_err(xs, g, b_of, k_terms=128):
    """error bound of the pre-activation x * scale + shift the kernel forms from one-pass statistics.
    The partials are sequential fp32 sums of at most k_terms = 32 rows x 4 channels values (sum) and fma'd squares (sum
    of squares), added in fp64: the group sum S carries <= k_terms u sum |x| and Q <= k_terms u sum x^2.  So the mean
    is off by dm <= k_terms u E|x|, the variance Q/n - m^2 by dvar <= k_terms u E[x^2] + 2 |m| dm, and rstd by
    dvar / (2 (var + eps)) relative.  scale = rstd gamma and shift = beta - m rstd gamma share these errors, so in
    x * scale + shift they combine to (x - m) scale drstd - scale dm.  The fp32 rounding of scale and shift and the fma
    add u |x scale| + u |shift| + u |v| <= 2 u (|x scale| + |shift|)."""
    sc, sh, m = g['scale'][b_of], g['shift'][b_of], g['mean'][b_of]
    dm = k_terms * U * g['absmean'][b_of]
    dvar = k_terms * U * g['sqmean'][b_of] + 2.0 * m.abs() * dm
    drstd = dvar / (2.0 * (g['var'][b_of] + g['eps']))
    return 2.0 * U * ((xs * sc).abs() + sh.abs()) + ((xs - m) * sc).abs() * drstd + sc.abs() * dm


def gn_bound(xs, g, b_of, act, out_dtype, extra=0.0):
    """|y - ref| <= output rounding + activation error + slope * (pre-activation error + extra), per element;
    + |v| 2^-126 where the activation's fp32 factor (sigmoid, erfc) may flush to zero."""
    ref = g['y']
    pre = xs * g['scale'][b_of] + g['shift'][b_of]
    out_rel = BF_HALF_ULP if out_dtype == torch.bfloat16 else U
    rel = out_rel + act_rel_fp32(pre, act)
    return rel * ref.abs() + SLOPE[act] * (gn_pre_err(xs, g, b_of) + extra) * (1.0 + out_rel) + TINY * pre.abs().clamp(min=1.0)


def attn_bound(ref, pv, qk, t, ch, tc, out_dtype):
    """A score error d (natural-log units) changes the normalised output by at most 2 d sum p|v|.  The scores are fp32
    sums of ch exact products (bf16 x bf16) or of ch fma terms (fp32), scaled once: d <= (ch + 2) u |q|.|k| / sqrt(ch)
    (`qk`), which also covers the subtraction of the running maximum.
    tensor-core path: P is rounded to bf16 before P V (2^-9 relative per p) while the denominator sums the unrounded p;
    P V accumulates in fp32: together <= 2^-8 sum p|v|.
    CUDA-core path: fp32 throughout; __expf is good to 2 + 1.173 |s - max| ulp (<= 2^-16 relative for every p that does
    not underflow), the sum of T values and the P V fma chain add T u each.
    Output rounding: half an ulp of the output type."""
    d = (ch + 2) * U * qk
    if tc:
        e = (2.0 ** -8 + 2.0 * d) * pv
    else:
        e = ((2.0 * t + 8.0) * U + 2.0 ** -16 + 2.0 * d) * pv
    out_rel = BF_HALF_ULP if out_dtype == torch.bfloat16 else U
    return out_rel * ref.abs() + (1.0 + out_rel) * e


def _assert_within(y, ref, bound, what):
    y, ref = y.double().cpu(), ref.double().cpu()
    err = (y - ref).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        i = int(torch.nonzero(bad.reshape(-1))[0])
        raise AssertionError('%s: %d elements out of bound; first at flat %d: y=%r ref=%r bound=%r (max err/bound %.3g)' % (
            what, int(bad.sum()), i, float(y.reshape(-1)[i]), float(ref.reshape(-1)[i]), float(bound.reshape(-1)[i]),
            float((err / bound.clamp(min=1e-300)).max())))
    return float((err / bound.clamp(min=1e-300)).max())


# ------------------------------------------------------------------------------------------------
# CPU: the references against oracle/restate.py
# ------------------------------------------------------------------------------------------------
def test_gn_ref_matches_restate_doctree_group_norm():
    g = _gen(0)
    batch, c = 3, 96
    sid = torch.sort(torch.randint(0, batch, (500,), generator=g)).values
    x = torch.randn(500, c, generator=g, dtype=torch.float64) * 1.7 + 0.4
    gam, bet = 1 + 0.1 * torch.randn(c, generator=g, dtype=torch.float64), torch.randn(c, generator=g, dtype=torch.float64)
    want = R.doctree_group_norm(x, sid, batch, gam, bet)
    got = gn_ref(x, sid, batch, R.group_count(c), gam, bet, 1e-5, 1e-5, 0)
    assert torch.allclose(got['y'], want, rtol=0, atol=1e-12)
    for act, f in ((1, R.silu), (2, torch.nn.functional.gelu)):
        got = gn_ref(x, sid, batch, R.group_count(c), gam, bet, 1e-5, 1e-5, act)
        assert torch.allclose(got['y'], f(want), rtol=0, atol=1e-12)
    # the affine form reproduces y
    assert torch.allclose(x * got['scale'][sid] + got['shift'][sid], (x - got['mean'][sid]) * got['scale'][sid] + bet,
                          atol=1e-12)


def test_gn_ref_matches_restate_group_norm32():
    g = _gen(1)
    b, t, c = 4, 64, 128
    x = torch.randn(b, c, t, generator=g, dtype=torch.float64) + 3.0
    gam, bet = torch.randn(c, generator=g, dtype=torch.float64), torch.randn(c, generator=g, dtype=torch.float64)
    want = R.group_norm32(x, gam, bet).permute(0, 2, 1).reshape(b * t, c)
    sid = torch.arange(b * t) // t
    got = gn_ref(x.permute(0, 2, 1).reshape(b * t, c), sid, b, 32, gam, bet, 1e-5, 0.0, 0)['y']
    assert torch.allclose(got, want, rtol=0, atol=1e-11)


def test_attn_ref_matches_restate_qkv_attention():
    g = _gen(2)
    b, t, heads, ch = 2, 37, 4, 16
    c = heads * ch
    qkv = torch.randn(b, 3 * c, t, generator=g, dtype=torch.float64)
    want = R.qkv_attention(qkv.reshape(b * heads, 3 * ch, t)).reshape(b, c, t).permute(0, 2, 1).reshape(b * t, c)
    out, pv, qk = attn_ref(qkv.permute(0, 2, 1).reshape(b * t, 3 * c), b, t, heads)
    # restate's softmax runs in fp32: |p - p64| <= ~2^-22 p, so the outputs agree to 2^-20 sum p|v|
    assert bool(((out - want).abs() <= 2.0 ** -20 * pv).all())
    assert bool((pv >= out.abs() - 1e-12).all()) and bool((qk > 0).all())


def test_act_ref_values():
    v = torch.tensor([-1e30, -20.0, -3.0, -0.0, 0.0, 1e-40, 2.0, 1e30], dtype=torch.float64)
    s = act_ref(v, 1)
    assert float(s[0]) == 0.0 and float(s[-1]) == 1e30 and torch.isfinite(s).all()
    assert torch.allclose(s[1:-1], v[1:-1] * torch.sigmoid(v[1:-1]), rtol=1e-15, atol=0)
    ge = act_ref(v, 2)
    assert torch.allclose(ge[2:-1], torch.nn.functional.gelu(v[2:-1]), rtol=1e-12, atol=0)
    # erfc keeps the far negative tail that 1 + erf loses to cancellation
    assert -1e-80 < float(ge[1]) < 0 and float(torch.nn.functional.gelu(v[1:2])) == 0.0
    assert float(ge[0]) == 0.0 and float(ge[-1]) == 1e30


def test_host_side_rejections():
    """argument checks that return before any launch.  Every pointer is a real zeroed buffer (device memory when there is
    a device) large enough for the launch the call describes, so no check can send a kernel to an invalid address."""
    from octfusion_b200._lib import lib, last_error
    dev = 'cuda' if torch.cuda.is_available() else 'cpu'
    keep = []

    def buf(nbytes):
        t = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
        keep.append(t)
        return ctypes.c_void_p(t.data_ptr())
    qkv, out = buf(8 * 48 * 4), buf(8 * 16 * 4)
    assert lib.of_attention(qkv, 30, out, 10, 1, 8, 1, 10, 1, None) == OF_E_ARG       # ch % 4 != 0
    assert 'multiple of 4' in last_error()
    assert lib.of_attention(qkv, 48, out, 16, 1, 8, 1, 16, 7, None) == OF_E_ARG       # bad dtype
    assert 'dtype' in last_error()
    assert lib.of_attention(qkv, 48, out, 16, 1, 0, 1, 16, 1, None) == OF_E_ARG       # no tokens
    x, idx, part = buf(64 * 64 * 4), buf(64 * 4), buf(64 * 64 * 4)
    assert lib.of_gn_stats(x, 64, 64, None, 0, 0, idx, idx, None, 8, 64, 1, 3, part, None) == OF_E_ARG   # granule 3
    assert 'gran' in last_error()
    tab = buf(4096 * 4)
    assert lib.of_gn_apply(x, 64, 64, None, 0, 0, None, 8, 64, tab, tab, 1, 5, part, 64, 0, None) == OF_E_ARG  # dtype
    xw, yw = buf(64 * 4096 * 4), buf(64 * 4096 * 4)
    assert lib.of_gn_apply(xw, 4096, 4096, None, 0, 0, None, 64, 64, tab, tab, 1, 0, yw, 4096, 0, None) == OF_E_ARG
    assert 'too wide' in last_error()                                                  # C / V = 1024 > 256 threads
    assert lib.of_gn_finalize(part, 96, 4, None, 0, 0, idx, 1, None, 8, tab, tab, 1, 32, 1e-5, 0.0, tab, tab, None,
                              None, None) == OF_E_ARG                                  # 3 channels per group, granule 4
    vals, hist = buf(10 * 4), buf(8193 * 4)
    assert lib.of_histogram_i32(vals, 10, 8193, hist, None) == OF_E_ARG
    assert lib.of_histogram_i32(vals, 10, 0, hist, None) == OF_E_ARG


# ------------------------------------------------------------------------------------------------
# GPU helpers
# ------------------------------------------------------------------------------------------------
def _L():
    from octfusion_b200 import _lib
    return _lib


def _call(name, *args):
    L = _L()
    rc = getattr(L.lib, name)(*args, L.stream())
    assert rc == 0, '%s failed (rc=%d): %s' % (name, rc, L.last_error())


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _dt(dtype):
    return 0 if dtype == torch.float32 else 1


def _apply(x0, scale, shift, act, y, *, x1=None, sample_id=None, rows_per_sample=0, reverse=0, dtype=None):
    dtype = dtype or x0.dtype
    c1 = 0 if x1 is None else x1.shape[1]
    _call('of_gn_apply', _p(x0), x0.stride(0), x0.shape[1], _p(x1), x1.stride(0) if x1 is not None else 0, c1,
          _p(sample_id), rows_per_sample, x0.shape[0], _p(scale), _p(shift), act, _dt(dtype), _p(y), y.stride(0), reverse)


def _padded(rows, c, dtype, extra_cols, offset, fill=0.0):
    """[rows, c] view into a [rows, c + extra_cols] buffer starting `offset` elements into each row"""
    buf = torch.full((rows, c + extra_cols), fill, dtype=dtype, device=DEV)
    return buf[:, offset:offset + c]


@functools.lru_cache(maxsize=None)
def _doctree():
    from tests.util import product_doctree
    return product_doctree(3, 5)


def _bf_bits_ordered(t):
    """bf16 values -> integers ordered like the values (+0 and -0 both 0); neighbours differ by 1"""
    b = t.contiguous().view(torch.int16).cpu().numpy().astype(np.int32) & 0xFFFF
    mag = b & 0x7FFF
    return np.where(b & 0x8000, -mag, mag)


def _bf16_round(x64):
    return x64.to(torch.float32).to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------
# of_gn_apply: the activations over every finite bf16 value and a dense fp32 grid
# ------------------------------------------------------------------------------------------------
def _all_finite_bf16():
    bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16)
    v = bits.view(torch.bfloat16)
    return v[torch.isfinite(v.float())]


def _fp32_grid():
    dense = torch.linspace(-30.0, 30.0, (1 << 20) + 1, dtype=torch.float64).float()
    tail = torch.linspace(-100.0, -80.0, 4097, dtype=torch.float64).float()          # where e^-v leaves fp32
    special = torch.tensor([0.0, -0.0, 1e-45, -1e-45, 1e-40, -1e-40, 2.0 ** -127, -2.0 ** -127, 2.0 ** -126, 1e30, -1e30,
                            3e38, -3e38], dtype=torch.float32)
    return torch.cat([dense, tail, special])


def _sweep_layout(v, c=256):
    n = v.numel()
    rows = (n + c - 1) // c
    x = torch.zeros(rows * c, dtype=v.dtype)
    x[:n] = v
    return x.reshape(rows, c), n


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float32])
@pytest.mark.parametrize('vector', [True, False])
@pytest.mark.parametrize('tables', ['identity', 'random'])
@pytest.mark.parametrize('act', [0, 1, 2])
def test_gn_apply_activation_sweep(dtype, vector, tables, act):
    """act 0 / 1 / 2 of of_gn_apply on every finite bf16 value (bf16) or on [-30, 30] plus the far tails, zeros,
    subnormals and +-1e30 (fp32), through the vector path (16-byte rows) and the scalar path (an odd, unaligned row
    pitch).  With scale 1 and shift -0 (the exact additive identity of the fma) act 0 returns the input bit for bit."""
    v = _all_finite_bf16() if dtype == torch.bfloat16 else _fp32_grid()
    xh, n = _sweep_layout(v)
    rows, c = xh.shape
    g = _gen(11)
    if tables == 'identity':
        sc, sh = torch.ones(1, c), torch.full((1, c), -0.0)
    else:
        sc = (0.25 + 0.75 * torch.rand(1, c, generator=g)) * torch.where(torch.rand(1, c, generator=g) < 0.5, -1.0, 1.0)
        sh = torch.randn(1, c, generator=g)
    if vector:
        x = xh.to(DEV)
    else:
        x = _padded(rows, c, dtype, 3, 1)                    # element offset 1, pitch c + 3: V = 1
        x.copy_(xh.to(DEV))
    pre = (xh.double() * sc.double() + sh.double()).reshape(-1)[:n]
    y = torch.full((rows, c), float('nan'), dtype=dtype, device=DEV)
    _apply(x, sc.to(DEV), sh.to(DEV), act, y, rows_per_sample=rows)
    y = y.cpu().reshape(-1)[:n]
    if act == 0 and tables == 'identity':
        assert torch.equal(y.view(torch.int16 if dtype == torch.bfloat16 else torch.int32),
                           xh.reshape(-1)[:n].view(torch.int16 if dtype == torch.bfloat16 else torch.int32))
        return
    ref = act_ref(pre, act)
    # the fp32 factor sigmoid / erfc may flush below 2^-126 (e^-v overflows fp32 beyond v = -88.7): |v| 2^-126
    floor = TINY * pre.abs().clamp(min=1.0)
    if dtype == torch.bfloat16:
        # within one bf16 ulp of the exact value rounded to bf16 (the fma adds u |v|, which act_cond amplifies by
        # at most 1 + |v|(|v| + 2) relative -- far below 2^-9 wherever e^v has not underflowed)
        d = np.abs(_bf_bits_ordered(y) - _bf_bits_ordered(_bf16_round(ref)))
        ok = (d <= 1) | ((y.double() - ref).abs() <= floor).numpy()
        if not ok.all():
            i = int(np.nonzero(~ok)[0][0])
            raise AssertionError('act %d: %d values off by more than one bf16 ulp (max %d ulp); first v=%r y=%r ref=%r' % (
                act, int((~ok).sum()), int(d[~ok].max()), float(pre[i]), float(y[i]), float(ref[i])))
        print('\nbf16 act %d (%s tables): max %d ulp from the rounded exact value, %d values not correctly rounded' % (
            act, tables, int(d[(y.double() - ref).abs().numpy() > floor.numpy()].max(initial=0)), int((d == 1).sum())))
    else:
        bound = (act_rel_fp32(pre, act) + act_cond(pre, act) * U) * ref.abs() + floor
        _assert_within(y, ref, bound, 'fp32 act %d' % act)


# ------------------------------------------------------------------------------------------------
# of_gn_apply: traversal direction, uniform vs general chunks, layouts, strides
# ------------------------------------------------------------------------------------------------
def _apply_case(layout):
    """(rows, batch, sample_id or None, rows_per_sample)"""
    if layout.startswith('doctree'):
        plan = _doctree().plan[int(layout[-1])]
        return plan.rows, 3, plan.batch_id, 0
    rps = int(layout.split('_')[1])
    return 5 * rps, 5, None, rps


@pytest.mark.gpu
@pytest.mark.parametrize('dtype,vector', [(torch.bfloat16, True), (torch.bfloat16, False), (torch.float32, True),
                                          (torch.float32, False)])
@pytest.mark.parametrize('layout', ['doctree4', 'doctree5', 'doctree6', 'dense_512', 'dense_337'])
def test_gn_apply_direction_and_chunk_invariance(dtype, vector, layout):
    """reverse in {0, 1, 2, 3} (bit 0: CTA order, bit 1: general per-row path for every chunk) gives bit-identical
    outputs, and each equals act(x * scale + shift) of the sample's table row (SiLU and GELU).  x = x0 | x1 concat."""
    rows, batch, sid, rps = _apply_case(layout)
    c0, c1 = 64, 32
    g = _gen(12)
    xh = torch.randn(rows, c0 + c1, generator=g) * 2.0
    sc, sh = torch.randn(batch, c0 + c1, generator=g), torch.randn(batch, c0 + c1, generator=g)
    if vector:
        x0, x1 = xh[:, :c0].to(DEV).to(dtype), xh[:, c0:].contiguous().to(DEV).to(dtype)
        x0 = x0.contiguous()
    else:
        x0, x1 = _padded(rows, c0, dtype, 1, 0), _padded(rows, c1, dtype, 5, 0)       # odd pitches: V = 1
        x0.copy_(xh[:, :c0].to(dtype)); x1.copy_(xh[:, c0:].to(dtype))
    xs = torch.cat([x0.double().cpu(), x1.double().cpu()], 1)
    b_of = (sid.long().cpu() if sid is not None else torch.arange(rows) // rps)
    pre = xs * sc.double()[b_of] + sh.double()[b_of]
    bits = torch.int16 if dtype == torch.bfloat16 else torch.int32
    for act in (1, 2):
        outs = []
        for rev in (0, 1, 2, 3):
            y = torch.full((rows, c0 + c1), float('nan'), dtype=dtype, device=DEV)
            _apply(x0, sc.to(DEV), sh.to(DEV), act, y, x1=x1, sample_id=sid, rows_per_sample=rps, reverse=rev)
            outs.append(y)
        for rev in (1, 2, 3):
            assert torch.equal(outs[rev].view(bits), outs[0].view(bits)), 'act=%d reverse=%d' % (act, rev)
        ref = act_ref(pre, act)
        out_rel = BF_HALF_ULP if dtype == torch.bfloat16 else U
        # one fma rounding (u |v|, times the slope), the activation's own error, the output rounding
        bound = (out_rel + act_rel_fp32(pre, act)) * ref.abs() + SLOPE[act] * U * pre.abs() * 1.01 + TINY
        _assert_within(outs[0], ref, bound, 'gn_apply act %d %s' % (act, layout))


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float32])
@pytest.mark.parametrize('pitch_extra', [24, 3])
@pytest.mark.parametrize('reverse', [0, 3])
def test_gn_apply_writes_nothing_outside_the_output(dtype, pitch_extra, reverse):
    """y is a [rows, C] window (pitch C + 24: vector path; C + 3: scalar path) at the top-left of a NaN-filled buffer
    with 7 extra rows: the sentinel columns and rows stay NaN, every output element is written."""
    rows, batch, sid, _ = _apply_case('doctree5')
    c = 128
    g = _gen(13)
    x = (torch.randn(rows, c, generator=g)).to(DEV).to(dtype)
    sc, sh = torch.randn(batch, c, generator=g).to(DEV), torch.randn(batch, c, generator=g).to(DEV)
    big = torch.full((rows + 7, c + pitch_extra), float('nan'), dtype=dtype, device=DEV)
    y = big[:rows, :c]
    _apply(x, sc, sh, 2, y, sample_id=sid, reverse=reverse)
    big = big.float().cpu()
    assert torch.isnan(big[:, c:]).all() and torch.isnan(big[rows:]).all()
    yy = big[:rows, :c]
    assert torch.isfinite(yy).all()
    pre = x.double().cpu() * sc.double().cpu()[sid.long().cpu()] + sh.double().cpu()[sid.long().cpu()]
    ref = act_ref(pre, 2)
    out_rel = BF_HALF_ULP if dtype == torch.bfloat16 else U
    bound = (out_rel + act_rel_fp32(pre, 2)) * ref.abs() + SLOPE[2] * U * pre.abs() * 1.01 + TINY
    _assert_within(yy, ref, bound, 'gn_apply strided')


# ------------------------------------------------------------------------------------------------
# of_gn_stats: the partials of every segment against float64 sums of the same rows
# ------------------------------------------------------------------------------------------------
def _segments(rows, b_of):
    """segment of each row: a new one at every 32-row chunk start and at every change of sample (ops.StatPlan)"""
    r = torch.arange(rows)
    new = torch.ones(rows, dtype=torch.bool)
    new[1:] = (b_of[1:] != b_of[:-1]) | ((r[1:] % 32) == 0)
    return torch.cumsum(new.long(), 0) - 1


def _stat_plan(layout):
    from octfusion_b200 import ops
    if layout == 'doctree':
        p = _doctree().plan[5]
        return p.stat, p.batch_id.long().cpu()
    rows, rps = 4 * 300, 300
    return ops.StatPlan(rows, 4, rows_per_sample=rps, device=DEV), torch.arange(rows) // rps


def _ref_partials(x64, b_of, seg_slot, gran, n_seg):
    rows, c = x64.shape
    slot = seg_slot.long().cpu()[_segments(rows, b_of)]
    xg = x64.reshape(rows, c // gran, gran)
    out = torch.zeros(n_seg, c // gran, 2, dtype=torch.float64)
    absum = torch.zeros(n_seg, c // gran, dtype=torch.float64)
    out[:, :, 0].index_add_(0, slot, xg.sum(-1))
    out[:, :, 1].index_add_(0, slot, (xg * xg).sum(-1))
    absum.index_add_(0, slot, xg.abs().sum(-1))
    return out.reshape(n_seg, -1), absum


@pytest.mark.gpu
@pytest.mark.parametrize('path', ['f32_v4', 'bf16_v8', 'bf16_v4'])
@pytest.mark.parametrize('gran', [2, 4])
@pytest.mark.parametrize('layout', ['doctree', 'dense'])
@pytest.mark.parametrize('concat', [False, True])
def test_gn_stats_partials(path, gran, layout, concat):
    """(sum, sum of squares) per (segment, granule) in the NaN-prefilled slot of the segment.  Each is a sequential fp32
    sum of at most 32 rows x gran values: error <= 32 gran u of the sum of magnitudes (+ u per square for the fma)."""
    plan, b_of = _stat_plan(layout)
    rows = plan.rows
    c0, c1 = (64, 64) if concat else (128, 0)
    dtype = torch.float32 if path.startswith('f32') else torch.bfloat16
    g = _gen(14)
    xh = (torch.randn(rows, c0 + c1, generator=g) * 1.5 + 0.5).to(dtype)
    off = 4 if path == 'bf16_v4' else 0                     # 8 bytes into the row: only 8-byte aligned -> V = 4
    x0 = _padded(rows, c0, dtype, 8, off)
    x0.copy_(xh[:, :c0].to(DEV))
    x1 = None
    if concat:
        x1 = _padded(rows, c1, dtype, 8, off)
        x1.copy_(xh[:, c0:].to(DEV))
    part = plan.new_part(c0 + c1, gran).fill_(float('nan'))
    _call('of_gn_stats', _p(x0), x0.stride(0), c0, _p(x1), x1.stride(0) if x1 is not None else 0, c1,
          _p(plan.chunk_seg), _p(plan.seg_slot), _p(plan.sample_id), plan.rows_per_sample, rows, _dt(dtype), gran,
          _p(part))
    part = part.cpu().double()
    assert torch.isfinite(part).all(), 'slots left unwritten'
    ref, absum = _ref_partials(xh.double(), b_of, plan.seg_slot, gran, plan.n_seg)
    k = 32 * gran
    bound = torch.stack([k * U * absum, (k + 1) * U * ref[:, 1::2]], -1).reshape(ref.shape)
    _assert_within(part, ref, bound, 'partials')


# ------------------------------------------------------------------------------------------------
# of_gn_finalize: split over CTAs, tickets, end to end against gn_ref
# ------------------------------------------------------------------------------------------------
def _finalize(part, c0, g0, plan, gamma, beta, groups, eps, count_eps, *, part1=None, c1=0, g1=0, split=True):
    batch, c = plan.batch, c0 + c1
    scale = torch.full((batch, c), float('nan'), device=DEV)
    shift = torch.full((batch, c), float('nan'), device=DEV)
    scratch = torch.full((batch * 8 * c,), float('nan'), dtype=torch.float64, device=DEV) if split else None
    ticket = torch.zeros(batch, dtype=torch.int32, device=DEV) if split else None
    _call('of_gn_finalize', _p(part), c0, g0, _p(part1), c1, g1, _p(plan.sample_seg_off), plan.n_seg,
          _p(plan.rows_of_sample), plan.rows_per_sample, _p(gamma), _p(beta), batch, groups, ctypes.c_float(eps),
          ctypes.c_float(count_eps), _p(scale), _p(shift), _p(scratch), _p(ticket))
    return scale, shift, ticket


def _f32_ulps(a, b):
    a = a.contiguous().view(torch.int32).cpu().long()
    b = b.contiguous().view(torch.int32).cpu().long()
    a = torch.where(a < 0, -(a & 0x7FFFFFFF), a)
    b = torch.where(b < 0, -(b & 0x7FFFFFFF), b)
    return (a - b).abs()


def _finalize_layout(layout):
    """16384 rows per sample (512 segments: S = 4 CTAs per sample); 'empty': sample 1 of 3 has no rows"""
    from octfusion_b200 import ops
    if layout == 'dense':
        rps, batch = 16384, 3
        plan = ops.StatPlan(rps * batch, batch, rows_per_sample=rps, device=DEV)
        return plan, torch.arange(rps * batch) // rps
    b_of = torch.cat([torch.zeros(20000, dtype=torch.long), torch.full((13000,), 2, dtype=torch.long)])
    sid = b_of.int().to(DEV)
    hist = torch.zeros(3, dtype=torch.int32, device=DEV)
    _call('of_histogram_i32', _p(sid), sid.numel(), 3, _p(hist))
    return ops.StatPlan(sid.numel(), 3, sample_id=sid, rows_of_sample=hist), b_of


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('ratio', [0, 8, 64])
@pytest.mark.parametrize('count_eps', [0.0, 1e-5])
@pytest.mark.parametrize('layout', ['dense', 'empty'])
def test_gn_finalize_split_and_end_to_end(dtype, ratio, count_eps, layout):
    """S > 1 CTAs per sample against S = 1 (scratch = ticket = NULL): scale and shift within one fp32 ulp; the tickets
    are zero after every call; two calls are bit-identical.  Then stats -> finalize -> apply (SiLU) against gn_ref with
    inputs whose mean is `ratio` standard deviations (the conditioning of the one-pass variance grows with it)."""
    plan, b_of = _finalize_layout(layout)
    rows, batch, c, groups = plan.rows, plan.batch, 128, 32
    g = _gen(15 + ratio)
    sigma = 0.75
    xh = (torch.randn(rows, c, generator=g) * sigma + ratio * sigma).to(dtype)
    gam, bet = 1 + 0.2 * torch.randn(c, generator=g), 0.3 * torch.randn(c, generator=g)
    x = xh.to(DEV)
    part = plan.new_part(c, 4).fill_(float('nan'))
    _call('of_gn_stats', _p(x), c, c, None, 0, 0, _p(plan.chunk_seg), _p(plan.seg_slot), _p(plan.sample_id),
          plan.rows_per_sample, rows, _dt(dtype), 4, _p(part))
    gd, bd = gam.to(DEV), bet.to(DEV)
    s1, h1, _ = _finalize(part, c, 4, plan, gd, bd, groups, 1e-5, count_eps, split=False)
    s2, h2, t2 = _finalize(part, c, 4, plan, gd, bd, groups, 1e-5, count_eps)
    assert int(t2.abs().sum()) == 0, 'tickets not reset'
    s3, h3, t3 = _finalize(part, c, 4, plan, gd, bd, groups, 1e-5, count_eps)
    assert int(t3.abs().sum()) == 0
    # bitwise: with count_eps = 0 the table rows of the empty sample are NaN (0 / 0) -- and never read
    assert torch.equal(s2.view(torch.int32), s3.view(torch.int32)) and torch.equal(h2.view(torch.int32), h3.view(torch.int32))
    live = [b for b in range(batch) if int((b_of == b).sum()) > 0]
    assert int(_f32_ulps(s1[live], s2[live]).max()) <= 1 and int(_f32_ulps(h1[live], h2[live]).max()) <= 1
    y = torch.full((rows, c), float('nan'), dtype=dtype, device=DEV)
    _apply(x, s2, h2, 1, y, sample_id=plan.sample_id, rows_per_sample=plan.rows_per_sample, reverse=1)
    assert torch.isfinite(y).all()
    ref = gn_ref(xh, b_of, batch, groups, gam, bet, 1e-5, count_eps, 1)
    bound = gn_bound(xh.double(), ref, b_of, 1, dtype)
    worst = _assert_within(y, ref['y'], bound, 'group norm ratio %d' % ratio)
    err = float((y.double().cpu() - ref['y']).abs().max())
    print('\ngroup norm %s ratio %d count_eps %g %s: max |err| %.3e (%.3e of max |y|), max err/bound %.3f' % (
        dtype, ratio, count_eps, layout, err, err / float(ref['y'].abs().max()), worst))


@pytest.mark.gpu
@pytest.mark.parametrize('split', [False, True])
def test_gn_mixed_granules_fused_gemm_statistics(monkeypatch, split):
    """x0 = a 64-wide tensor-core GEMM output whose epilogue wrote granule-2 partials, concatenated with a stand-alone
    granule-4 x1: C = 128, 4 channels per group, so every group spans one granule pair of x0 or one granule of x1 (the
    64-channel decoder level of the LR U-Net).  The reference statistics are taken over the exact fp64 product (the
    epilogue sums its fp32 accumulators before rounding); their 64-term fp32 accumulation adds d <= 64 u |a|.|w| per
    element, i.e. <= mean(d) to the mean and <= 2 mean(|x - m| d) + mean(d)^2 to the variance of each group."""
    from octfusion_b200 import ops
    from octfusion_b200.ops import PreparedWeight
    from tests.test_gpu_kernels import _nan_parts
    _nan_parts(monkeypatch)
    plan = _doctree().plan[6]
    sp, b_of = plan.stat, plan.batch_id.long().cpu()
    rows, k, n = plan.rows, 64, 64
    g = _gen(16)
    a = torch.randn(rows, k, generator=g).bfloat16()
    w = (torch.randn(n, k, generator=g) / 8).bfloat16()
    x1h = (torch.randn(rows, 64, generator=g) * 0.8 + 0.3).bfloat16()
    pw = PreparedWeight(1, k, 0, n).refresh(w.float().to(DEV), 'linear')
    x0 = ops.gather_gemm(a.to(DEV), pw, stats=sp)
    st = x0._of_stats
    assert st.gran == 2 and torch.isfinite(st.part).all()
    x1 = x1h.to(DEV)
    p1 = sp.new_part(64, 4)
    _call('of_gn_stats', _p(x1), 64, 64, None, 0, 0, _p(sp.chunk_seg), _p(sp.seg_slot), _p(sp.sample_id), 0, rows, 1, 4,
          _p(p1))
    assert torch.isfinite(p1).all()
    gam, bet = 1 + 0.2 * torch.randn(128, generator=g), 0.3 * torch.randn(128, generator=g)
    scale, shift, ticket = _finalize(st.part, 64, 2, sp, gam.to(DEV), bet.to(DEV), 32, 1e-5, 1e-5, part1=p1, c1=64, g1=4,
                                     split=split)
    if split:
        assert int(ticket.abs().sum()) == 0
    y = torch.full((rows, 128), float('nan'), dtype=torch.bfloat16, device=DEV)
    _apply(x0, scale, shift, 1, y, x1=x1, sample_id=sp.sample_id)
    xs = torch.cat([x0.double().cpu(), x1h.double()], 1)
    exact = a.double() @ w.double().t()
    ref = gn_ref(xs, b_of, 3, 32, gam, bet, 1e-5, 1e-5, 1, stats_x=torch.cat([exact, x1h.double()], 1))
    d = torch.cat([64 * U * (a.double().abs() @ w.double().abs().t()), torch.zeros(rows, 64, dtype=torch.float64)], 1)
    cnt = torch.bincount(b_of, minlength=3).double()[:, None]
    dm = torch.zeros(3, 128, dtype=torch.float64).index_add_(0, b_of, d) / cnt
    dm = dm.reshape(3, 32, 4).mean(-1).repeat_interleave(4, 1)
    dev_ = (torch.cat([exact, x1h.double()], 1) - ref['mean'][b_of]).abs() * d
    dv = torch.zeros(3, 128, dtype=torch.float64).index_add_(0, b_of, dev_) / cnt
    dv = 2 * dv.reshape(3, 32, 4).mean(-1).repeat_interleave(4, 1) + dm ** 2
    sc = ref['scale'][b_of].abs()
    extra = sc * (dm[b_of] + (xs - ref['mean'][b_of]).abs() * dv[b_of] / (2 * ref['var'][b_of]))
    bound = gn_bound(xs, ref, b_of, 1, torch.bfloat16, extra=extra)
    _assert_within(y, ref['y'], bound, 'mixed granules')


# ------------------------------------------------------------------------------------------------
# of_histogram_i32
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('n,bins', [(0, 3), (1, 1), (1, 3), (1000, 3), (100_000, 8192), (1_000_000, 7), (1_000_000, 8192)])
def test_histogram_i32(n, bins):
    """hist[v] += 1 for 0 <= v < bins; other values (negative, >= bins) are ignored; hist is accumulated into"""
    g = _gen(17 + n)
    v = torch.randint(-3, bins + 3, (n,), generator=g, dtype=torch.int32)
    if n:
        v[0] = bins - 1
    vd = v.to(DEV)
    hist = torch.full((bins,), 5, dtype=torch.int32, device=DEV)
    _call('of_histogram_i32', _p(vd if n else torch.zeros(1, dtype=torch.int32, device=DEV)), n, bins, _p(hist))
    keep = v[(v >= 0) & (v < bins)].long()
    want = torch.bincount(keep, minlength=bins) + 5
    assert torch.equal(hist.cpu().long(), want)


# ------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------
def _attention(qkv, out, b, t, heads, ch, dtype):
    L = _L()
    return L.lib.of_attention(_p(qkv), qkv.stride(0), _p(out), out.stride(0), b, t, heads, ch, _dt(dtype), L.stream())


def _check_attention(qkv_h, b, t, heads, dtype, *, tc, qkv_pitch_extra=0, qkv_offset=0, what=''):
    """run of_attention on qkv_h (CPU, exactly representable in `dtype`) laid into a buffer of pitch 3C + extra,
    output into a NaN-prefilled [b t + 5, C + 16] buffer at column 8; check the sentinels and the bound"""
    c3 = qkv_h.shape[1]
    c = c3 // 3
    ch = c // heads
    rows = b * t
    qkv = _padded(rows, c3, dtype, qkv_pitch_extra, qkv_offset)
    qkv.copy_(qkv_h.to(DEV).to(dtype))
    big = torch.full((rows + 5, c + 16), float('nan'), dtype=dtype, device=DEV)
    out = big[:rows, 8:8 + c]
    # which kernel ran, from the CUDA activity record; the profiler now and then drops a record, so an empty record is
    # retried (the call is idempotent) -- a wrong kernel name fails at once
    ran = []
    for _ in range(3):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            rc = _attention(qkv, out, b, t, heads, ch, dtype)
            torch.cuda.synchronize()
        assert rc == 0, 'of_attention rc=%d: %s' % (rc, _L().last_error())
        ran = [e.name for e in prof.events() if 'attention' in e.name]
        if ran:
            break
    want = 'attention_tc_kernel' if tc else 'attention_kernel<'
    assert len(ran) == 1 and want in ran[0], 'expected %s, ran %s' % (want, ran)
    big = big.float().cpu()
    assert torch.isnan(big[:, :8]).all() and torch.isnan(big[:, 8 + c:]).all() and torch.isnan(big[rows:]).all()
    y = big[:rows, 8:8 + c]
    assert torch.isfinite(y).all()
    ref, pv, qk = attn_ref(qkv_h, b, t, heads)
    return _assert_within(y, ref, attn_bound(ref, pv, qk, t, ch, tc, dtype), what)


def _tc_smem(t, ch):
    tpad = (t + 63) // 64 * 64
    return (2 * tpad + 64) * (2 * ch + 16)


def _simt_smem(t, ch):
    return (2 * t * (ch + 4) + 8 * t * 4 + 8 * 4 * ch) * 4


def _qkv(b, t, heads, ch, seed, dtype=torch.bfloat16):
    return torch.randn(b * t, 3 * heads * ch, generator=_gen(seed)).to(dtype).double()


_TS = [1, 8, 63, 64, 65, 100, 129, 512]


@pytest.mark.gpu
@pytest.mark.parametrize('t', _TS)
@pytest.mark.parametrize('ch', [16, 32, 64, 128])
@pytest.mark.parametrize('heads', [1, 4])
def test_attention_tensor_core(t, ch, heads):
    """bf16, 16-byte aligned rows: the tensor-core kernel (64-query tiles, 64-key blocks, online softmax); T not a
    multiple of 64 leaves both a partial query tile and a partial key block.  Shapes over its shared-memory budget fall
    to the CUDA-core kernel and, over that one's too, return OF_E_UNSUPPORTED."""
    b = 32 if t <= 8 else (2 if t >= 512 else 3)
    if _tc_smem(t, ch) > 200 * 1024:
        assert _simt_smem(t, ch) > 220 * 1024
        qkv = torch.zeros(b * t, 3 * heads * ch, dtype=torch.bfloat16, device=DEV)
        out = torch.zeros(b * t, heads * ch, dtype=torch.bfloat16, device=DEV)
        assert _attention(qkv, out, b, t, heads, ch, torch.bfloat16) == OF_E_UNSUPPORTED
        assert 'shared memory' in _L().last_error()
        return
    _check_attention(_qkv(b, t, heads, ch, t * 7 + ch), b, t, heads, torch.bfloat16, tc=True, qkv_pitch_extra=8,
                     what='tc T=%d ch=%d h=%d' % (t, ch, heads))


@pytest.mark.gpu
@pytest.mark.parametrize('t,ch', [(1, 8), (100, 8), (512, 8), (1, 24), (129, 24), (512, 24), (65, 48), (300, 48)])
def test_attention_simt_bf16_odd_head_width(t, ch):
    """head widths outside {16, 32, 64, 128}: the bf16 CUDA-core kernel"""
    assert _simt_smem(t, ch) <= 220 * 1024
    b, heads = 3, 2
    _check_attention(_qkv(b, t, heads, ch, t + ch, ), b, t, heads, torch.bfloat16, tc=False,
                     what='simt bf16 T=%d ch=%d' % (t, ch))


@pytest.mark.gpu
@pytest.mark.parametrize('t,ch', [(100, 64), (65, 16), (129, 128), (512, 32)])
def test_attention_tc_and_simt_on_one_input(t, ch):
    """the same bf16 input through the tensor-core kernel (pitch 3C + 8) and, by a pitch that is not a multiple of 8
    elements, through the CUDA-core kernel: each within its own bound of attn_ref"""
    b, heads = 2, 2
    qkv = _qkv(b, t, heads, ch, 99 + t)
    _check_attention(qkv, b, t, heads, torch.bfloat16, tc=True, qkv_pitch_extra=8, what='tc')
    _check_attention(qkv, b, t, heads, torch.bfloat16, tc=False, qkv_pitch_extra=3, qkv_offset=1, what='simt misaligned')


@pytest.mark.gpu
@pytest.mark.parametrize('t', _TS)
@pytest.mark.parametrize('ch', [16, 32, 64, 128])
def test_attention_fp32(t, ch):
    """fp32 activations: the CUDA-core kernel with fp32 softmax; shapes over 220 KB of shared memory (T = 512 with
    ch = 64 or 128) return OF_E_UNSUPPORTED"""
    b, heads = (4 if t <= 64 else 2), 2
    if _simt_smem(t, ch) > 220 * 1024:
        qkv = torch.zeros(b * t, 3 * heads * ch, device=DEV)
        out = torch.zeros(b * t, heads * ch, device=DEV)
        assert _attention(qkv, out, b, t, heads, ch, torch.float32) == OF_E_UNSUPPORTED
        assert 'shared memory' in _L().last_error()
        return
    _check_attention(_qkv(b, t, heads, ch, 5 * t + ch, torch.float32), b, t, heads, torch.float32, tc=False,
                     qkv_pitch_extra=4, what='fp32 T=%d ch=%d' % (t, ch))


def _structured(kind, b, t, heads, ch):
    g = _gen(21)
    x = torch.randn(b, t, heads, 3, ch, generator=g).bfloat16().double()
    q, k = x[:, :, :, 0], x[:, :, :, 1]
    if kind == 'uniform':                   # q = 0: every score 0, the output is the mean of v
        q.zero_()
    elif kind == 'peaked':                  # the last key scores 20 * 20 / sqrt(64) = 50 (72 log2 units) above the rest
        q.zero_(); k.zero_()
        q[..., 0] = 20.0
        k[:, -1, :, 0] = 20.0
    else:                                   # monotone: score_s = 16 * 5 s / T / 8 = 10 s / T, every block raises the max
        q.zero_(); k.zero_()
        q[..., 0] = 16.0
        k[..., 0] = (5.0 * torch.arange(t, dtype=torch.float64) / t).bfloat16().double()[None, :, None]
    return x.reshape(b * t, heads * 3 * ch)


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['uniform', 'peaked', 'monotone'])
@pytest.mark.parametrize('t', [200, 320])
@pytest.mark.parametrize('path', ['tc', 'simt'])
def test_attention_structured(kind, t, path):
    """q = 0 (uniform softmax: the mean of v); one key in the last block 72 log2 units above every earlier score (the
    online-softmax correction of the earlier blocks falls to 2^-72); scores increasing across the blocks.
    (T <= 323 keeps ch = 64 within the CUDA-core kernel's shared memory.)"""
    b, heads, ch = 2, 2, 64
    qkv = _structured(kind, b, t, heads, ch)
    extra, off = (8, 0) if path == 'tc' else (3, 1)
    _check_attention(qkv, b, t, heads, torch.bfloat16, tc=path == 'tc', qkv_pitch_extra=extra, qkv_offset=off,
                     what='%s %s' % (kind, path))
    if kind == 'uniform':
        ref, _, _ = attn_ref(qkv, b, t, heads)
        v = qkv.reshape(b, t, heads, 3, ch)[:, :, :, 2].mean(1, keepdim=True).expand(b, t, heads, ch)
        assert torch.allclose(ref, v.reshape(b * t, heads * ch), rtol=0, atol=1e-12)
