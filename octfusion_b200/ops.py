"""Functional layer over the C ABI: torch tensors in, torch tensors out, every arithmetic
operation executed by a kernel of liboctfusion_b200.so on the current CUDA stream.

torch is used for device memory (torch.empty / zeros), streams and nothing else.
"""
from __future__ import annotations
import ctypes as C
import torch

from . import _lib
from ._lib import lib, ptr, stream, check, dt, GemmArgs

_FORCE_SIMT = False
_PROFILE = None        # when a list: (kind, meta, start_event, end_event) per GEMM launch (bench.py roofline leg)


def set_profile(sink):
    """sink: a list to append per-launch CUDA-event pairs to, or None to switch profiling off."""
    global _PROFILE
    _PROFILE = sink


_TRACE = None          # debug: list receiving (op, shape, checksum) for every op output


def set_trace(sink):
    global _TRACE
    _TRACE = sink


_TRACE_KEEP = False


def _trace(op, t):
    if _TRACE is not None:
        _TRACE.append((op, tuple(t.shape), float(t.float().abs().sum()), t.clone() if _TRACE_KEEP else None))


def set_force_simt(flag: bool):
    """Debug switch: route every GEMM through the CUDA-core kernel."""
    global _FORCE_SIMT
    _FORCE_SIMT = bool(flag)


class TapTable:
    """Neighbour table of the tap-gather GEMM (see include/octfusion_b200.h): tab [rows, taps] and the CSR lists `extra`
    of its n_multi multi-neighbour slots (None when there is none)."""
    __slots__ = ('tab', 'extra', 'taps', 'rows', 'n_multi', '_type_blocks')

    def __init__(self, tab: torch.Tensor, extra, taps: int, n_multi: int = 0):
        assert tab.dtype == torch.int32 and tab.is_contiguous()
        self.tab, self.extra, self.taps, self.n_multi = tab, extra, taps, n_multi
        self.rows = tab.numel() // taps
        self._type_blocks = {}

    def type_block(self, ntype, node_type):
        """bf16 [rows, 64] node-type K block of the tensor-core GEMM (graph constant, built once per ntype)."""
        if ntype not in self._type_blocks:
            out = torch.empty((self.rows, 64), dtype=torch.bfloat16, device=self.tab.device)
            check(lib.of_graph_type_block(ptr(self.tab), ptr(self.extra), ptr(node_type), self.rows, self.taps, ntype,
                                          ptr(out), stream()), 'of_graph_type_block')
            self._type_blocks[ntype] = out
        return self._type_blocks[ntype]


class StatPlan:
    """Segment tables of the deterministic group-norm statistics for one row layout (include/octfusion_b200.h,
    of_gemm_args.stat_out): rows are cut into 32-row chunks, a chunk into segments at every change of sample id.
      chunk_seg      int32 [n_chunks + 1]  exclusive prefix sum of segments per chunk
      sample_seg_off int32 [B + 1], sample_seg_idx int32 [n_seg]: the segments of each sample, in row order
      seg_slot       int32 [n_seg]  row of the partial buffers that segment s owns = its rank in sample_seg_idx, so a
                     sample's partials are contiguous rows [sample_seg_off[b], sample_seg_off[b+1])
    Built once per graph depth (sample ids from DualOctree.batch_id) or per dense resolution (rows_per_sample).
    The segment count is data dependent: `pending_count()` exposes it as a device scalar so that a caller building
    several plans (DualOctree: one per depth) can fetch all counts with ONE host synchronisation and then `finish`."""
    __slots__ = ('rows', 'batch', 'n_seg', 'chunk_seg', 'sample_seg_off', 'sample_seg_idx', 'seg_slot', 'sample_id',
                 'rows_per_sample', 'rows_of_sample', '_pending')

    def __init__(self, rows: int, batch: int, *, sample_id=None, rows_per_sample=0, rows_of_sample=None, device=None,
                 defer=False):
        assert (sample_id is None) != (rows_per_sample == 0)
        dev = sample_id.device if sample_id is not None else torch.device(device)
        self.rows, self.batch = rows, batch
        self.sample_id, self.rows_per_sample, self.rows_of_sample = sample_id, rows_per_sample, rows_of_sample
        self.n_seg, self._pending = None, None
        if sample_id is None:
            # dense layout: pure index arithmetic -> build on the host, no device synchronisation at all
            r = torch.arange(rows)
            self._build(r // rows_per_sample, r, torch.device('cpu'))
            self.finish(int(self._pending[0]))
            for name in ('chunk_seg', 'sample_seg_off', 'sample_seg_idx', 'seg_slot'):
                setattr(self, name, getattr(self, name).to(dev))
        else:
            self._build(sample_id.long(), torch.arange(rows, device=dev), dev)
            if not defer:
                self.finish(int(self._pending[0].item()))

    def _build(self, bid, r, dev):
        rows, batch = self.rows, self.batch
        new = torch.ones(rows, dtype=torch.bool, device=dev)
        if rows > 1:
            new[1:] = (bid[1:] != bid[:-1]) | ((r[1:] & 31) == 0)
        seg_of_row = torch.cumsum(new.int(), 0) - 1
        n_chunks = (rows + 31) // 32
        count = (seg_of_row[-1:] + 1) if rows > 0 else torch.zeros(1, dtype=torch.int32, device=dev)
        cs = torch.empty(n_chunks + 1, dtype=torch.int32, device=dev)
        cs[:n_chunks] = seg_of_row[::32].int()
        cs[n_chunks:] = count.int()
        self.chunk_seg = cs
        # segments of each sample in row order: stable sort of the per-row sample ids restricted to segment starts.
        # Sized by rows (an upper bound of n_seg) so that no count is needed here: non-starts sort to the end.
        key = torch.where(new, bid, torch.full_like(bid, batch))
        order = torch.sort(key, stable=True).indices                      # row indices, segment starts first, by sample
        self.sample_seg_idx = seg_of_row[order].int()                     # -> segment index of each start (prefix valid)
        cnt = torch.bincount(key, minlength=batch + 1)[:batch]
        off = torch.zeros(batch + 1, dtype=torch.int32, device=dev)
        off[1:] = torch.cumsum(cnt, 0).int()
        self.sample_seg_off = off
        self._pending = count

    def pending_count(self):
        return self._pending

    def finish(self, n_seg: int):
        self.n_seg = int(n_seg)
        self.sample_seg_idx = self.sample_seg_idx[: max(self.n_seg, 1)].contiguous()
        self.seg_slot = torch.zeros(max(self.n_seg, 1), dtype=torch.int32, device=self.sample_seg_idx.device)
        if self.n_seg > 0:
            self.seg_slot[self.sample_seg_idx.long()] = torch.arange(self.n_seg, dtype=torch.int32,
                                                                     device=self.sample_seg_idx.device)
        self._pending = None
        return self

    def new_part(self, channels: int, gran: int):
        """partial buffer [n_seg, channels/gran, 2] fp32 (every slot is overwritten by its producer: no zeroing)"""
        return torch.empty((max(self.n_seg, 1), channels // gran * 2), dtype=torch.float32, device=self.chunk_seg.device)


def tc_stat_gran(n: int) -> int:
    """granule width of the statistics the tensor-core epilogue writes for an N-column output (gemm_tc.cu: 4 for the
    128/256-wide tiles, 2 below -- a 64-channel GroupNorm32 has 2 channels per group)"""
    return 4 if n % 128 == 0 else 2


class Stats:
    """partial statistics of one tensor: (buffer, StatPlan, granule); attached to GEMM outputs as `t._of_stats`."""
    __slots__ = ('part', 'plan', 'channels', 'gran')

    def __init__(self, part, plan, channels, gran):
        self.part, self.plan, self.channels, self.gran = part, plan, channels, gran


class PreparedWeight:
    """A GEMM weight in the two layouts the kernels read:
    canonical fp32 [taps*(c+ntype), N] (CUDA-core path) and the bf16 swizzled tile image (tensor-core
    path, built lazily by of_pack_weight_tc).  Rebuilt when the source parameter changes."""

    def __init__(self, taps: int, c: int, ntype: int, n: int):
        self.taps, self.c, self.ntype, self.n = taps, c, ntype, n
        self.canon = None
        self._packed = None
        self._src_key = None

    def refresh(self, param: torch.Tensor, layout: str):
        """layout: 'canon' ([K,N], GraphConv.weights / Upsample flat view), 'linear' ([N,K]: nn.Linear,
        Conv1d k=1, Downsample flat view), 'conv3d' ([N,C,3,3,3])."""
        key = (param.data_ptr(), param._version, str(param.device))
        if key == self._src_key and self.canon is not None:
            return self
        _lib.require_cuda(param)
        src = param.detach().to(torch.float32).contiguous()
        k = self.taps * (self.c + self.ntype)
        if layout == 'canon':
            assert src.numel() == k * self.n, (src.shape, k, self.n)
            self.canon = src.reshape(k, self.n)
        else:
            dst = torch.empty((k, self.n), dtype=torch.float32, device=src.device)
            if layout == 'linear':
                assert self.taps == 1 and self.ntype == 0 and src.numel() == k * self.n
                args = (1, 1, k)
            elif layout == 'conv3d':
                assert self.ntype == 0 and src.numel() == k * self.n
                args = (1, self.taps, self.taps * self.c)
            else:
                raise ValueError(layout)
            check(lib.of_repack_weight(ptr(src), args[0], args[1], args[2], self.taps, self.c, self.n,
                                       ptr(dst), stream()), 'of_repack_weight')
            self.canon = dst
        self._packed = None
        self._src_key = key
        return self

    def tc_ok(self) -> bool:
        return self.c % 64 == 0 and self.taps * self.ntype <= 64 and self.ntype <= 8 and self.taps <= 27

    def packed(self):
        if self._packed is None:
            nbytes = lib.of_pack_weight_tc_bytes(self.taps, self.c, self.ntype, self.n)
            if nbytes <= 0:
                raise RuntimeError('weight shape not packable for the tensor-core path')
            buf = torch.empty(nbytes, dtype=torch.uint8, device=self.canon.device)
            check(lib.of_pack_weight_tc(ptr(self.canon), self.taps, self.c, self.ntype, self.n, ptr(buf), stream()),
                  'of_pack_weight_tc')
            self._packed = buf
        return self._packed


def gather_gemm(a0, w: PreparedWeight, *, a1=None, tap: TapTable = None, in_rows=None, node_type=None,
                bias=None, row_add=None, row_add_idx=None, resid=None, out_rows=None,
                out=None, ldo=None, out_f32=False, stats: StatPlan = None):
    """out[m,:] = sum_tap mean_nbr [a0|a1|onehot] . W[tap] + bias + row_add[row_add_idx[m]] + resid[m].
    stats: the StatPlan of the output rows when a group norm consumes the output next -- the tensor-core epilogue then
    writes the norm's partial statistics (attached to the result as `_of_stats`), and ops.group_norm skips its
    statistics pass."""
    _lib.require_cuda(a0, a1, bias, row_add, resid, out)
    assert a0.dim() == 2 and a0.stride(1) == 1
    c0 = a0.shape[1]
    c1 = 0 if a1 is None else a1.shape[1]
    assert c0 + c1 == w.c, 'channel mismatch: %d + %d vs %d' % (c0, c1, w.c)
    if a1 is not None:
        assert a1.dtype == a0.dtype and a1.stride(1) == 1
    taps = 1 if tap is None else tap.taps
    assert taps == w.taps
    m = tap.rows if tap is not None else (in_rows.numel() if in_rows is not None else a0.shape[0])
    n = w.n
    act_dtype = a0.dtype
    if out is None:
        out = torch.empty((m, n), dtype=torch.float32 if out_f32 else act_dtype, device=a0.device)
    if ldo is None:
        ldo = out.stride(0)
    if resid is not None:
        assert resid.dtype == act_dtype and resid.stride(1) == 1
    if w.ntype > 0:
        assert node_type is not None and node_type.dtype == torch.uint8
    use_tc = (not _FORCE_SIMT and act_dtype == torch.bfloat16 and w.tc_ok() and c0 % 64 == 0 and c1 % 64 == 0
              and m >= 1)
    g = GemmArgs()
    g.a0, g.lda0, g.c0 = a0.data_ptr(), a0.stride(0), c0
    g.a1, g.lda1, g.c1 = (a1.data_ptr(), a1.stride(0), c1) if a1 is not None else (None, 0, 0)
    g.a_multi, g.ld_multi = None, 0
    g.nt_block = None
    g.reverse = _next_direction() if use_tc else 0
    if use_tc and w.ntype > 0 and tap is not None:
        g.nt_block = tap.type_block(w.ntype, node_type).data_ptr()
    if use_tc and tap is not None and tap.n_multi > 0:
        # slots with several (4..16) finer neighbours: their mean rows are built once per input tensor
        aux = torch.empty((tap.n_multi, c0 + c1), dtype=act_dtype, device=a0.device)
        check(lib.of_gather_mean_rows(a0.data_ptr(), a0.stride(0), c0, a1.data_ptr() if a1 is not None else None,
                                      a1.stride(0) if a1 is not None else 0, c1, ptr(tap.extra), tap.n_multi, dt(a0),
                                      ptr(aux), aux.stride(0), stream()), 'of_gather_mean_rows')
        g.a_multi, g.ld_multi = aux.data_ptr(), aux.stride(0)
    g.tap_tab = tap.tab.data_ptr() if tap is not None else None
    g.tap_extra = tap.extra.data_ptr() if (tap is not None and tap.extra is not None) else None
    g.in_rows = in_rows.data_ptr() if in_rows is not None else None
    g.taps = taps
    g.node_type = node_type.data_ptr() if (node_type is not None and w.ntype > 0) else None
    g.ntype = w.ntype
    g.w = (w.packed() if use_tc else w.canon).data_ptr()
    g.bias = bias.data_ptr() if bias is not None else None
    if row_add is not None:
        assert row_add.dtype == torch.float32 and row_add_idx is not None and row_add_idx.dtype == torch.int32
        g.row_add, g.ld_row_add, g.row_add_idx = row_add.data_ptr(), row_add.stride(0), row_add_idx.data_ptr()
    else:
        g.row_add, g.ld_row_add, g.row_add_idx = None, 0, None
    g.resid, g.ld_resid = (resid.data_ptr(), resid.stride(0)) if resid is not None else (None, 0)
    g.out_rows = out_rows.data_ptr() if out_rows is not None else None
    g.out, g.ldo = out.data_ptr(), ldo
    g.out_f32 = 1 if (out_f32 or (out.dtype == torch.float32 and act_dtype != torch.float32)) else 0
    g.M, g.N = m, n
    g.dtype = dt(a0)
    st_obj = None
    g.stat_out, g.stat_chunk_seg, g.stat_seg_slot, g.stat_sample, g.stat_rows_per_sample = None, None, None, None, 0
    if (stats is not None and use_tc and n % 32 == 0 and out_rows is None and stats.rows == m
            and not g.out_f32):
        st_obj = Stats(stats.new_part(n, tc_stat_gran(n)), stats, n, tc_stat_gran(n))
        g.stat_out, g.stat_chunk_seg = st_obj.part.data_ptr(), stats.chunk_seg.data_ptr()
        g.stat_seg_slot = stats.seg_slot.data_ptr()
        g.stat_sample = stats.sample_id.data_ptr() if stats.sample_id is not None else None
        g.stat_rows_per_sample = stats.rows_per_sample
    prof = _PROFILE
    if prof is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    if use_tc:
        check(lib.of_gather_gemm_tc(C.byref(g), stream()), 'of_gather_gemm_tc')
    else:
        check(lib.of_gather_gemm_simt(C.byref(g), stream()), 'of_gather_gemm_simt')
    if prof is not None:
        e1.record()
        es = 2 if act_dtype == torch.bfloat16 else 4
        k = taps * (c0 + c1 + w.ntype)
        nnz = 0 if tap is None else tap.rows * taps          # table entries read (4 B each)
        prof.append(dict(kind='tc' if use_tc else 'simt', M=m, N=n, K=k, taps=taps, c=c0 + c1, ntype=w.ntype,
                         flops=2.0 * m * k * n,
                         bytes=float(m * (c0 + c1) * es + m * n * (4 if g.out_f32 else es) + nnz * 4 + k * n * es
                                     + (m * n * es if resid is not None else 0)),
                         start=e0, end=e1))
    _trace('gemm_tc' if use_tc else 'gemm_simt', out)
    if st_obj is not None:
        out._of_stats = st_obj
    return out


def linear_small(x, weight, bias=None, a_silu=False):
    """out = act(x) @ weight.T + bias for a few rows of fp32 (timestep-embedding MLPs); weight is [N, K]."""
    _lib.require_cuda(x, weight, bias)
    assert x.dtype == torch.float32 and x.stride(1) == 1 and weight.dtype == torch.float32 and weight.is_contiguous()
    b, k = x.shape
    n = weight.shape[0]
    out = torch.empty((b, n), dtype=torch.float32, device=x.device)
    check(lib.of_linear_small(ptr(x), x.stride(0), ptr(weight), ptr(bias) if bias is not None else None, b, k, n,
                              1 if a_silu else 0, ptr(out), out.stride(0), stream()), 'of_linear_small')
    _trace('linear_small', out)
    return out


_sweep = [0]          # traversal direction of the next streaming kernel (see include/octfusion_b200.h: `reverse`)


def _next_direction() -> int:
    """Alternate the row traversal direction from one big kernel to the next, so that each kernel starts on the rows
    its producer wrote (or read) last -- the part of the tensor that is still resident in L2."""
    _sweep[0] ^= 1
    return _sweep[0]


_ACT = {False: 0, None: 0, True: 1, 'silu': 1, 'gelu': 2}


GN_FINALIZE_SPLIT = 8          # OF_GN_FINALIZE_SPLIT of include/octfusion_b200.h
_TICKETS = {}


def _gn_ticket(dev, batch):
    """per-device ticket counters of of_gn_finalize (zero-initialised once; the kernel leaves them zero)"""
    t = _TICKETS.get(dev)
    if t is None or t.numel() < batch:
        t = torch.zeros(max(batch, 64), dtype=torch.int32, device=dev)
        _TICKETS[dev] = t
    return t


def _stats_of(x, plan: StatPlan, cpg: int):
    """(partials, granule) of x under `plan`: those its producing GEMM attached when their granule divides the
    channels-per-group `cpg`, else one stand-alone statistics pass"""
    st = getattr(x, '_of_stats', None)
    if st is not None and st.plan is plan and st.channels == x.shape[1] and cpg % st.gran == 0:
        return st.part, st.gran
    gran = 4 if cpg % 4 == 0 else 2
    part = plan.new_part(x.shape[1], gran)
    check(lib.of_gn_stats(ptr(x), x.stride(0), x.shape[1], None, 0, 0, ptr(plan.chunk_seg), ptr(plan.seg_slot), ptr(plan.sample_id),
                          plan.rows_per_sample, x.shape[0], dt(x), gran, ptr(part), stream()), 'of_gn_stats')
    return part, gran


def group_norm(x0, gamma, beta, groups: int, plan: StatPlan, *, x1=None, eps=1e-5, count_eps=0.0, act=False, out=None):
    """(x0|x1) -> act(groupnorm) with per-sample statistics over the row layout `plan` describes.  Statistics:
    deterministic fp32 partials per (32-row segment, 4 channels) -- written by the producing tensor-core GEMM's epilogue
    when it was asked to (`gather_gemm(stats=plan)`), else by of_gn_stats -- summed in fixed order in fp64."""
    _lib.require_cuda(x0, x1, gamma, beta, out)
    rows = x0.shape[0]
    assert rows == plan.rows, (rows, plan.rows)
    c0 = x0.shape[1]
    c1 = 0 if x1 is None else x1.shape[1]
    c = c0 + c1
    cpg = c // groups
    if cpg % 2 != 0 or c0 % 4 != 0 or c1 % 4 != 0:
        raise NotImplementedError('group_norm: channels per group (%d) must be even and the concat split (%d | %d) '
                                  'multiples of 4' % (cpg, c0, c1))
    dev = x0.device
    batch = plan.batch
    p0, g0 = _stats_of(x0, plan, cpg)
    p1, g1 = _stats_of(x1, plan, cpg) if x1 is not None else (None, g0)
    scale = torch.empty((batch, c), dtype=torch.float32, device=dev)
    shift = torch.empty((batch, c), dtype=torch.float32, device=dev)
    scratch = torch.empty(batch * GN_FINALIZE_SPLIT * c, dtype=torch.float64, device=dev)
    check(lib.of_gn_finalize(ptr(p0), c0, g0, ptr(p1), c1, g1, ptr(plan.sample_seg_off), plan.n_seg,
                             ptr(plan.rows_of_sample), plan.rows_per_sample, ptr(gamma), ptr(beta), batch, groups,
                             float(eps), float(count_eps), ptr(scale), ptr(shift), ptr(scratch), ptr(_gn_ticket(dev, batch)),
                             stream()), 'of_gn_finalize')
    if out is None:
        out = torch.empty((rows, c), dtype=x0.dtype, device=dev)
    a1 = (ptr(x1), x1.stride(0), c1) if x1 is not None else (None, 0, 0)
    check(lib.of_gn_apply(ptr(x0), x0.stride(0), c0, a1[0], a1[1], a1[2], ptr(plan.sample_id), plan.rows_per_sample, rows,
                          ptr(scale), ptr(shift), _ACT[act], dt(x0), ptr(out), out.stride(0),
                          _next_direction(), stream()), 'of_gn_apply')
    if _PROFILE is not None:
        es = 2 if x0.dtype == torch.bfloat16 else 4
        _PROFILE.append(dict(kind='gn', M=rows, N=c, bytes=float(2 * rows * c * es), flops=0.0))
    _trace('group_norm', out)
    return out


def attention(qkv, batch: int, tokens: int, heads: int, out=None):
    _lib.require_cuda(qkv)
    c = qkv.shape[1] // 3
    ch = c // heads
    if out is None:
        out = torch.empty((batch * tokens, c), dtype=qkv.dtype, device=qkv.device)
    check(lib.of_attention(ptr(qkv), qkv.stride(0), ptr(out), out.stride(0), batch, tokens, heads, ch, dt(qkv),
                           stream()), 'of_attention')
    _trace('attention', out)
    return out


def timestep_embedding(t, dim: int, max_period: float = 10000.0):
    _lib.require_cuda(t)
    t = t.to(torch.float32).contiguous()
    out = torch.empty((t.shape[0], dim), dtype=torch.float32, device=t.device)
    check(lib.of_timestep_embedding(ptr(t), t.shape[0], dim, float(max_period), ptr(out), stream()),
          'of_timestep_embedding')
    return out


def learned_sinusoidal(t, w):
    _lib.require_cuda(t, w)
    t = t.to(torch.float32).contiguous()
    half = w.numel()
    out = torch.empty((t.shape[0], 2 * half + 1), dtype=torch.float32, device=t.device)
    check(lib.of_learned_sinusoidal(ptr(t), ptr(w), t.shape[0], half, ptr(out), stream()), 'of_learned_sinusoidal')
    return out


def embedding_add(out, table, label):
    check(lib.of_embedding_add(ptr(table), ptr(label), out.shape[0], out.shape[1], ptr(out), stream()),
          'of_embedding_add')
    return out


def copy_rows(src, dst, rows: int, c: int, *, src_rows=None, dst_rows=None):
    check(lib.of_copy_rows(ptr(src), src.stride(0), dt(src), ptr(src_rows) if src_rows is not None else None,
                           ptr(dst), dst.stride(0), dt(dst), ptr(dst_rows) if dst_rows is not None else None,
                           rows, c, stream()), 'of_copy_rows')
    return dst


def ddim_eps_update(x, eps, log_snr, log_snr_next, x_act=None):
    """x (fp32, in place) <- eps-DDIM step; log_snr / log_snr_next are 0-dim or 1-element device tensors."""
    assert x.dtype == torch.float32 and eps.dtype == torch.float32 and x.is_contiguous() and eps.is_contiguous()
    check(lib.of_ddim_eps_update(ptr(x), ptr(eps), ptr(log_snr), ptr(log_snr_next), x.numel(),
                                 ptr(x_act) if x_act is not None else None,
                                 dt(x_act) if x_act is not None else 0, stream()), 'of_ddim_eps_update')
    return x


def ddpm_x0_update(x, pred, log_snr, log_snr_next, noise=None, do_sign=False):
    """x (fp32, in place) <- ancestral x0-parameterised step; pred is sign()-ed in place when do_sign."""
    assert x.dtype == torch.float32 and pred.dtype == torch.float32 and x.is_contiguous() and pred.is_contiguous()
    check(lib.of_ddpm_x0_update(ptr(x), ptr(pred), ptr(noise) if noise is not None else None, ptr(log_snr),
                                ptr(log_snr_next), x.numel(), 1 if do_sign else 0, stream()), 'of_ddpm_x0_update')
    return x


def exclusive_scan_i32(values, out=None):
    """returns int32 [n+1]: out[i] = sum(values[:i]), out[n] = total."""
    n = values.numel()
    if n == 0:
        return torch.zeros(1, dtype=torch.int32, device=values.device)
    if out is None:
        out = torch.empty(n + 1, dtype=torch.int32, device=values.device)
    scratch = torch.empty(max(int(lib.of_scan_scratch_bytes(n)), 8), dtype=torch.uint8, device=values.device)
    check(lib.of_exclusive_scan_i32(ptr(values), ptr(out), n, None, ptr(scratch), stream()), 'of_exclusive_scan_i32')
    return out


def dense_tap_table(mode: int, out_res_log2: int, batch: int, device):
    rows = batch * 8 ** out_res_log2
    tab = torch.empty((rows, 27), dtype=torch.int32, device=device)
    check(lib.of_dense_tap_table(mode, out_res_log2, batch, ptr(tab), stream()), 'of_dense_tap_table')
    return TapTable(tab, None, 27)
