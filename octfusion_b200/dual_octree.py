"""DualOctree: the per-depth dual graph of an octree, built by CUDA kernels (csrc/graph.cu).

Drop-in for reference models/networks/dualoctree_networks/dual_octree.py `DualOctree` +
`post_processing_for_docnn()` as far as the U-Net reads it (SURVEY.md 8b): `.graph[d]['edge_idx' |
'edge_dir' | 'node_type']`, `.batch_id(d)`, `.batch_size`, `.nnum`, `.lnum`, `.node_child(d)`,
`.octree`, `.total_num`, and `.get_input_feature()` for octrees built from points.  Internally the graph is a *tap table* (one int32 per (row, direction)
slot, see include/octfusion_b200.h) which is what the tap-gather GEMM consumes; the reference-format
sorted edge lists are materialised lazily, only if somebody asks for them.
"""
from __future__ import annotations
import ctypes as C
import torch

from . import _lib, ops
from ._lib import lib, ptr, stream, check, OctreeLevels

N_DIR = 7


class GraphPlan:
    """Device-resident description of the depth-d dual graph."""
    __slots__ = ('depth', 'rows', 'tap', 'node_type', 'batch_id', 'rows_of_sample', 'leaf_base', 'stat',
                 'down_copy_dst', 'down_copy_rows', 'down_out_rows', 'up_copy_src', 'up_copy_rows', 'up_in_rows')

    def __init__(self):
        for s in self.__slots__:
            setattr(self, s, None)


class _LazyGraph(dict):
    """graph[d]: dict with the reference's keys, edge lists expanded on first access."""

    def __init__(self, owner, d):
        super().__init__()
        self._owner, self._d = owner, d

    def __missing__(self, key):
        if key in ('edge_idx', 'edge_dir'):
            self._owner._expand_edges(self._d, self)
            return dict.__getitem__(self, key)
        if key == 'node_mask':                           # dual_octree.py:391-398: over all octree nodes of depths fd..d
            o = self._owner
            oc = o.octree
            parts = [oc.children[k] < 0 for k in range(o.full_depth, self._d)]
            parts.append(torch.ones(int(o.nnum[self._d]), dtype=torch.bool, device=o.device))
            v = torch.cat(parts)
            self[key] = v
            return v
        if key == 'node_type':
            v = self._owner.plan[self._d].node_type.long()
            self[key] = v
            return v
        raise KeyError(key)

    def get(self, key, default=None):
        try:
            return self[key]
        except KeyError:
            return default


class DualOctree:
    def __init__(self, octree):
        self.octree = octree
        self.device = octree.device
        if self.device.type != 'cuda':
            raise RuntimeError('octfusion_b200.DualOctree builds the graph with CUDA kernels: the octree must '
                               'live on a CUDA device (there is no CPU path)')
        self.depth, self.full_depth, self.batch_size = octree.depth, octree.full_depth, octree.batch_size
        self.nnum = octree.nnum.clone()
        self.nenum = octree.nnum_nempty.clone()
        self.lnum = self.nnum - self.nenum
        fd, dep = self.full_depth, self.depth
        dev = self.device
        # ---- per-level helpers: leaf rank, leaf / non-empty index lists ----
        lv = OctreeLevels()
        lv.full_depth, lv.depth, lv.batch = fd, dep, self.batch_size
        self._keep = []                                   # tensors referenced by raw pointers below
        self.leaf_idx, self.nonempty_idx = {}, {}
        for d in range(fd, dep + 1):
            keys = octree.keys[d].contiguous()
            child = octree.children[d].contiguous()
            assert keys.dtype == torch.int64 and child.dtype == torch.int32
            n = int(self.nnum[d])
            rank = torch.empty(n + 1, dtype=torch.int32, device=dev)
            scratch = torch.empty(max(int(lib.of_scan_scratch_bytes(n)), 8), dtype=torch.uint8, device=dev)
            check(lib.of_leaf_rank(ptr(child), n, ptr(rank), None, ptr(scratch), stream()), 'of_leaf_rank')
            nleaf = int(self.lnum[d]) if d < dep else 0
            nne = int(self.nenum[d])
            if d < dep:
                li = torch.empty(max(nleaf, 1), dtype=torch.int32, device=dev)
                ni = torch.empty(max(nne, 1), dtype=torch.int32, device=dev)
                check(lib.of_compact_idx(ptr(child), ptr(rank), n, ptr(li), ptr(ni), stream()), 'of_compact_idx')
                self.leaf_idx[d], self.nonempty_idx[d] = li[:nleaf], ni[:nne]
            lv.keys[d], lv.children[d], lv.leaf_rank[d] = keys.data_ptr(), child.data_ptr(), rank.data_ptr()
            lv.nnum[d] = n
            self._keep += [keys, child, rank, scratch]
        self._levels = lv
        # ---- one tap table per graph depth ----
        # Two phases so that the data-dependent sizes of ALL depths are fetched with two host synchronisations per
        # octree (not ~3 per depth): (A) count + scans, sync 1 = neighbour words and multi-slot counts; (B) fill,
        # statistics segments, sync 2 = segment counts.
        self.plan = {}
        self.graph = [dict() for _ in range(dep + 1)]
        depths = list(range(fd, dep + 1))
        scans, rows_of = {}, {}
        for D in depths:
            rows = int(lib.of_graph_rows(C.byref(lv), D))
            if rows < 0:
                raise RuntimeError('of_graph_rows: ' + _lib.last_error())
            need = torch.empty(rows * N_DIR, dtype=torch.int32, device=dev)
            multi = torch.empty(rows * N_DIR, dtype=torch.int32, device=dev)
            check(lib.of_graph_count(C.byref(lv), D, ptr(need), ptr(multi), stream()), 'of_graph_count')
            scans[D], rows_of[D] = (ops.exclusive_scan_i32(need), ops.exclusive_scan_i32(multi)), rows
        totals = torch.cat([s[-1:] for D in depths for s in scans[D]]).tolist()   # sync 1
        pending = []
        for i, D in enumerate(depths):
            rows, (need_off, multi_ord) = rows_of[D], scans[D]
            words, n_multi = totals[2 * i], totals[2 * i + 1]
            tab = torch.empty((rows, N_DIR), dtype=torch.int32, device=dev)
            extra = torch.empty(n_multi + 1 + words, dtype=torch.int32, device=dev)
            ntype = torch.empty(rows, dtype=torch.uint8, device=dev)
            bid = torch.empty(rows, dtype=torch.int32, device=dev)
            check(lib.of_graph_fill(C.byref(lv), D, ptr(need_off), ptr(multi_ord), n_multi, ptr(tab), ptr(extra),
                                    ptr(ntype), ptr(bid), stream()), 'of_graph_fill')
            hist = torch.zeros(self.batch_size, dtype=torch.int32, device=dev)
            check(lib.of_histogram_i32(ptr(bid), rows, self.batch_size, ptr(hist), stream()), 'of_histogram_i32')
            p = GraphPlan()
            p.depth, p.rows = D, rows
            p.tap = ops.TapTable(tab, extra, N_DIR, n_multi)
            p.node_type, p.batch_id, p.rows_of_sample = ntype, bid, hist
            p.stat = ops.StatPlan(rows, self.batch_size, sample_id=bid, rows_of_sample=hist, defer=True)
            pending.append(p.stat.pending_count().long())
            p.leaf_base = int(self.lnum[fd:D].sum())          # rows of leaves coarser than D
            self.plan[D] = p
            self.graph[D] = _LazyGraph(self, D)
        counts = torch.cat(pending).tolist()                                      # sync 2
        for D, n_seg in zip(depths, counts):
            self.plan[D].stat.finish(n_seg)
        # ---- row maps of GraphDownsample / GraphUpsample (reference modules.py:409-428, 458-472) ----
        ar = lambda n: torch.arange(n, dtype=torch.int32, device=dev)  # noqa: E731
        for D in range(fd + 1, dep + 1):
            pd, pc = self.plan[D], self.plan[D - 1]
            base = pc.leaf_base                                # leaves coarser than D-1: same rows in both graphs
            # depth-D graph rows [0, base+lnum[D-1]) are leaves -> scatter them into the depth-(D-1) graph
            pd.down_copy_dst = torch.cat([ar(base), base + self.leaf_idx[D - 1]])
            pd.down_copy_rows = base + int(self.lnum[D - 1])
            pd.down_out_rows = (base + self.nonempty_idx[D - 1]).contiguous()   # pooled 8->1 rows
            # depth-(D-1) graph -> depth-D graph
            pc.up_copy_src = torch.cat([ar(base), base + self.leaf_idx[D - 1]])
            pc.up_copy_rows = base + int(self.lnum[D - 1])
            pc.up_in_rows = (base + self.nonempty_idx[D - 1]).contiguous()      # rows that get 8 children
        self.total_num = self.plan[dep].rows
        self._bid64 = {}

    # ---- reference-compatible accessors ---------------------------------------------------------
    def post_processing_for_docnn(self):
        """The reference needs this second call (dual_octree.py:400-409); here the constructor has
        already produced the post-processed graph, so this is a no-op kept for drop-in use."""
        return self

    def batch_id(self, depth, nempty=False):
        if depth not in self._bid64:
            self._bid64[depth] = self.plan[depth].batch_id.long()
        return self._bid64[depth]

    def node_child(self, depth):
        return self.octree.children[depth]

    def get_input_feature(self, all_leaf_nodes=True, dtype=torch.float32):
        """reference dual_octree.py:343-360: the ND input feature of the octree's depth-D nodes (InputFeature('ND')),
        preceded by zero rows for the leaves of full_depth..D-1 when `all_leaf_nodes` -- i.e. one row per row of the
        depth-D graph, written by one kernel in `dtype` (float32 or bfloat16)."""
        from .modules import input_feature_nd
        leaf_rows = int(self.lnum[self.full_depth:self.depth].sum()) if all_leaf_nodes else 0
        return input_feature_nd(self.octree, leaf_rows, dtype)

    def _expand_edges(self, d, g):
        p = self.plan[d]
        slots = p.rows * N_DIR
        per = torch.empty(slots, dtype=torch.int32, device=self.device)
        check(lib.of_graph_edge_count(ptr(p.tap.tab), ptr(p.tap.extra), slots, ptr(per), stream()),
              'of_graph_edge_count')
        off = ops.exclusive_scan_i32(per)
        e = int(off[-1].item())
        idx = torch.empty((2, max(e, 1)), dtype=torch.int64, device=self.device)
        edir = torch.empty(max(e, 1), dtype=torch.int64, device=self.device)
        check(lib.of_graph_edges(ptr(p.tap.tab), ptr(p.tap.extra), slots, N_DIR, ptr(off), ptr(idx[0]), ptr(idx[1]),
                                 ptr(edir), stream()), 'of_graph_edges')
        dict.__setitem__(g, 'edge_idx', idx[:, :e])
        dict.__setitem__(g, 'edge_dir', edir[:e])
