// Dual-octree graph build on the GPU (integer / index work, HBM- and latency-bound).
//
// Replaces DualOctree.__init__ + post_processing_for_docnn (reference
// models/networks/dualoctree_networks/dual_octree.py:19-63, 119-239, 241-271, 332-341, 381-409):
// ~150 small int64 torch ops, an argsort and a unique per depth.  The reference discovers
// neighbours hierarchically (keep leaf-leaf edges of the parent level :207, re-wire edges of
// subdivided nodes to their 4 facing children via dir_table :90-94,:214, add the 24 fixed
// intra-sibling edges :101-112).  The edge set it ends with is exactly "two graph nodes are
// joined in direction d when their cells share a face in direction d", so the kernel walks the
// octree instead: locate the cell that contains the face neighbour (top-down through
// `children`), and when that cell is subdivided enumerate its descendants that touch the face.
// No hashing, no sort: rows come out in graph order and each (row, dir) slot is written once.
//
// Output is the tap table consumed by the tap-gather GEMM (include/octfusion_b200.h):
// tab[row, 7] int32 with -1 / single row / -(offset+2) into tap_extra for 4..16 finer neighbours.
#include "common.cuh"

namespace of {

// ---------------------------------------------------------------------------------------------
// exclusive scan (int32): local scan per 2048-item block, scan of the block sums, add back
// ---------------------------------------------------------------------------------------------
constexpr int SCAN_T = 256, SCAN_I = 8, SCAN_B = SCAN_T * SCAN_I;

template <int MODE>  // 0: raw values, 1: flag (value < 0)
__global__ void __launch_bounds__(SCAN_T) scan_local_kernel(const int32_t* __restrict__ in, int32_t* __restrict__ out,
                                                            int64_t n, int32_t* __restrict__ block_sums) {
  __shared__ int32_t warp_tot[SCAN_T / 32];
  const int64_t base = (int64_t)blockIdx.x * SCAN_B + (int64_t)threadIdx.x * SCAN_I;
  int32_t v[SCAN_I];
  int32_t local = 0;
#pragma unroll
  for (int j = 0; j < SCAN_I; ++j) {
    int32_t x = 0;
    if (base + j < n) {
      x = in[base + j];
      if (MODE == 1) x = x < 0 ? 1 : 0;
    }
    v[j] = local;
    local += x;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int32_t incl = local;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int32_t t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) warp_tot[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    int32_t w = lane < SCAN_T / 32 ? warp_tot[lane] : 0;
    int32_t wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int32_t t = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) wi += t;
    }
    if (lane < SCAN_T / 32) warp_tot[lane] = wi - w;       // exclusive warp offsets
    if (lane == SCAN_T / 32 - 1) block_sums[blockIdx.x] = wi;
  }
  __syncthreads();
  const int32_t off = warp_tot[warp] + (incl - local);
#pragma unroll
  for (int j = 0; j < SCAN_I; ++j)
    if (base + j < n) out[base + j] = off + v[j];
}

__global__ void __launch_bounds__(1024) scan_sums_kernel(int32_t* __restrict__ sums, int nb, int32_t* __restrict__ total_out,
                                                         int32_t* __restrict__ out_tail) {
  __shared__ int32_t warp_tot[32];
  __shared__ int32_t carry_s;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int c0 = 0; c0 < nb; c0 += 1024) {
    const int i = c0 + threadIdx.x;
    const int32_t x = i < nb ? sums[i] : 0;
    int32_t incl = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int32_t t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int32_t w = warp_tot[lane];
      int32_t wi = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        int32_t t = __shfl_up_sync(0xffffffffu, wi, o);
        if (lane >= o) wi += t;
      }
      warp_tot[lane] = wi - w;
    }
    __syncthreads();
    const int32_t carry = carry_s;
    const int32_t excl = carry + warp_tot[warp] + incl - x;
    if (i < nb) sums[i] = excl;
    __syncthreads();
    if (threadIdx.x == 1023) carry_s = excl + x;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    if (total_out) *total_out = carry_s;
    if (out_tail) *out_tail = carry_s;                    // out[n] = total (scan has n+1 entries)
  }
}

__global__ void __launch_bounds__(SCAN_T) scan_add_kernel(int32_t* __restrict__ out, int64_t n,
                                                          const int32_t* __restrict__ sums) {
  const int64_t base = (int64_t)blockIdx.x * SCAN_B + (int64_t)threadIdx.x * SCAN_I;
  const int32_t off = sums[blockIdx.x];
#pragma unroll
  for (int j = 0; j < SCAN_I; ++j)
    if (base + j < n) out[base + j] += off;
}

template <int MODE>
static int run_scan(const int32_t* in, int32_t* out, int64_t n, int32_t* total_out, void* scratch,
                    cudaStream_t st, const char* who) {
  OF_REQUIRE(in && out && scratch && n >= 0, "%s: bad arguments", who);
  const int nb = (int)((n + SCAN_B - 1) / SCAN_B);
  int32_t* sums = reinterpret_cast<int32_t*>(scratch);
  if (nb > 0) scan_local_kernel<MODE><<<nb, SCAN_T, 0, st>>>(in, out, n, sums);
  scan_sums_kernel<<<1, 1024, 0, st>>>(sums, nb, total_out, out + n);
  if (nb > 0) scan_add_kernel<<<nb, SCAN_T, 0, st>>>(out, n, sums);
  if (nb > 0) add_launches(2);
  OF_LAUNCH_CHECK(who);
  return OF_OK;
}

__global__ void compact_idx_kernel(const int32_t* __restrict__ children, const int32_t* __restrict__ leaf_rank, int n,
                                   int32_t* __restrict__ leaf_idx, int32_t* __restrict__ nonempty_idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = children[i];
  if (c < 0) { if (leaf_idx) leaf_idx[leaf_rank[i]] = i; }
  else if (nonempty_idx) nonempty_idx[c] = i;
}

// ---------------------------------------------------------------------------------------------
// graph build
// ---------------------------------------------------------------------------------------------
struct GraphCtx {
  const int64_t* keys[16];
  const int32_t* children[16];
  const int32_t* leaf_rank[16];
  int32_t nnum[16];
  int32_t row_base[16];
  int32_t fd, depth, D, batch;
};

__device__ __forceinline__ void key_decode(int64_t key, int bits, int& x, int& y, int& z, int& b) {
  b = (int)(key >> 48);
  const uint64_t k = (uint64_t)key & ((1ull << 48) - 1);
  x = y = z = 0;
  for (int i = 0; i < bits; ++i) {
    x |= (int)((k >> (3 * i + 2)) & 1ull) << i;
    y |= (int)((k >> (3 * i + 1)) & 1ull) << i;
    z |= (int)((k >> (3 * i)) & 1ull) << i;
  }
}
__device__ __forceinline__ int64_t morton3(int x, int y, int z, int bits) {
  int64_t k = 0;
  for (int i = 0; i < bits; ++i)
    k |= ((int64_t)((x >> i) & 1) << (3 * i + 2)) | ((int64_t)((y >> i) & 1) << (3 * i + 1)) |
         ((int64_t)((z >> i) & 1) << (3 * i));
  return k;
}

__device__ __forceinline__ bool is_graph_node(const GraphCtx& g, int d, int i) {
  return d == g.D || g.children[d][i] < 0;
}
__device__ __forceinline__ int graph_row(const GraphCtx& g, int d, int i) {
  return d == g.D ? g.row_base[d] + i : g.row_base[d] + g.leaf_rank[d][i];
}

// dual_octree.py:85-89  (dir 0..5 = +z,-z,+y,-y,+x,-x on (x,y,z))
__device__ __forceinline__ void dir_delta(int dir, int& dx, int& dy, int& dz) {
  dx = dir == 4 ? 1 : dir == 5 ? -1 : 0;
  dy = dir == 2 ? 1 : dir == 3 ? -1 : 0;
  dz = dir == 0 ? 1 : dir == 1 ? -1 : 0;
}

// Calls f(row) for every graph node that shares the `dir` face of node (d, i).
template <typename F>
__device__ __forceinline__ void for_each_face_neighbour(const GraphCtx& g, int d, int x, int y, int z, int b, int dir,
                                                        F f) {
  int dx, dy, dz;
  dir_delta(dir, dx, dy, dz);
  const int nx = x + dx, ny = y + dy, nz = z + dz;
  const int lim = 1 << d;
  if (nx < 0 || ny < 0 || nz < 0 || nx >= lim || ny >= lim || nz >= lim) return;   // domain boundary
  // locate the existing cell containing (nx,ny,nz): the full layer is indexed by its key
  int cd = g.fd;
  int ci = (int)(((int64_t)b << (3 * g.fd)) + morton3(nx >> (d - g.fd), ny >> (d - g.fd), nz >> (d - g.fd), g.fd));
  while (cd < d) {
    const int c = g.children[cd][ci];
    if (c < 0) break;
    const int sh = d - cd - 1;
    ci = 8 * c + ((((nx >> sh) & 1) << 2) | (((ny >> sh) & 1) << 1) | ((nz >> sh) & 1));
    ++cd;
  }
  if (is_graph_node(g, cd, ci)) { f(graph_row(g, cd, ci)); return; }
  // subdivided same-size neighbour: enumerate descendants touching the shared face.  The face of
  // the neighbour that looks back at us is the opposite direction (remap table dual_octree.py:98-100);
  // its octants (4x+2y+z) are the 4 with the axis bit equal to `want` (dir_table :90-94).
  const int axis = dir < 2 ? 0 : dir < 4 ? 1 : 2;         // bit of the octant index: z=0, y=1, x=2
  const int want = (dir & 1) ? 1 : 0;                     // we look in +axis -> neighbour's low side (bit 0)
  int st_d[24], st_i[24];
  int sp = 0;
  st_d[0] = cd; st_i[0] = ci; sp = 1;
  while (sp > 0) {
    --sp;
    const int nd = st_d[sp], ni = st_i[sp];
    if (is_graph_node(g, nd, ni)) { f(graph_row(g, nd, ni)); continue; }
    const int c8 = 8 * g.children[nd][ni];
    for (int o = 7; o >= 0; --o) {
      if (((o >> axis) & 1) != want) continue;
      if (sp < 24) { st_d[sp] = nd + 1; st_i[sp] = c8 + o; ++sp; }
    }
  }
}

__global__ void graph_count_kernel(GraphCtx g, int d, int32_t* __restrict__ need) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int i = (int)(idx / 6), dir = (int)(idx % 6);
  if (i >= g.nnum[d]) return;
  if (!is_graph_node(g, d, i)) return;
  int x, y, z, b;
  key_decode(g.keys[d][i], d, x, y, z, b);
  int n = 0;
  for_each_face_neighbour(g, d, x, y, z, b, dir, [&](int) { ++n; });
  const int64_t row = graph_row(g, d, i);
  need[row * 7 + dir] = n > 1 ? n + 1 : 0;
  if (dir == 0) need[row * 7 + 6] = 0;
}

__global__ void graph_fill_kernel(GraphCtx g, int d, const int32_t* __restrict__ need_off, int32_t* __restrict__ tab,
                                  int32_t* __restrict__ extra, uint8_t* __restrict__ node_type,
                                  int32_t* __restrict__ batch_id) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int i = (int)(idx / 6), dir = (int)(idx % 6);
  if (i >= g.nnum[d]) return;
  if (!is_graph_node(g, d, i)) return;
  int x, y, z, b;
  key_decode(g.keys[d][i], d, x, y, z, b);
  const int64_t row = graph_row(g, d, i);
  const int64_t slot = row * 7 + dir;
  const int32_t off = need_off[slot];
  const int32_t cap = need_off[slot + 1] - off;
  if (cap == 0) {
    int32_t v = -1;
    for_each_face_neighbour(g, d, x, y, z, b, dir, [&](int r) { v = r; });
    tab[slot] = v;
  } else {
    int n = 0;
    for_each_face_neighbour(g, d, x, y, z, b, dir, [&](int r) {
      if (n + 1 < cap) extra[off + 1 + n] = r;
      ++n;
    });
    extra[off] = n;
    tab[slot] = -(off + 2);
  }
  if (dir == 0) {
    tab[row * 7 + 6] = (int32_t)row;                       // self loop, dual_octree.py:241-249
    if (node_type) node_type[row] = (uint8_t)(d - g.fd);   // dual_octree.py:381-389
    if (batch_id) batch_id[row] = b;                       // dual_octree.py:65-79
  }
}

static int make_ctx(const of_octree_levels* oct, int D, GraphCtx& g, const char* who) {
  OF_REQUIRE(oct != nullptr, "%s: null octree", who);
  OF_REQUIRE(oct->full_depth >= 1 && oct->depth < 16 && oct->full_depth <= oct->depth, "%s: bad depths", who);
  OF_REQUIRE(D >= oct->full_depth && D <= oct->depth, "%s: graph depth %d outside [%d, %d]", who, D,
             oct->full_depth, oct->depth);
  OF_REQUIRE(D - oct->full_depth <= 6, "%s: more than 6 adaptive levels are not supported", who);
  g.fd = oct->full_depth; g.depth = oct->depth; g.D = D; g.batch = oct->batch;
  int64_t base = 0;
  for (int d = 0; d < 16; ++d) {
    g.keys[d] = oct->keys[d]; g.children[d] = oct->children[d]; g.leaf_rank[d] = oct->leaf_rank[d];
    g.nnum[d] = oct->nnum[d]; g.row_base[d] = 0;
  }
  for (int d = g.fd; d <= D; ++d) {
    OF_REQUIRE(oct->keys[d] && oct->children[d] && oct->nnum[d] >= 0, "%s: level %d missing", who, d);
    OF_REQUIRE(d == D || oct->leaf_rank[d], "%s: leaf_rank[%d] missing", who, d);
    g.row_base[d] = (int32_t)base;
    if (d < D) {
      OF_REQUIRE(oct->nnum[d + 1] % 8 == 0, "%s: nnum[%d] is not a multiple of 8", who, d + 1);
      base += oct->nnum[d] - oct->nnum[d + 1] / 8;          // leaves of depth d
    } else {
      base += oct->nnum[d];
    }
  }
  OF_REQUIRE(base * 7 < (1ll << 31), "%s: graph too large for int32 slots", who);
  return OF_OK;
}

__global__ void edge_count_kernel(const int32_t* __restrict__ tab, const int32_t* __restrict__ extra, int64_t slots,
                                  int32_t* __restrict__ per_slot) {
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= slots) return;
  const int t = tab[s];
  per_slot[s] = t == -1 ? 0 : t >= 0 ? 1 : extra[-(t + 2)];
}

__global__ void edge_fill_kernel(const int32_t* __restrict__ tab, const int32_t* __restrict__ extra, int64_t slots,
                                 int taps, const int32_t* __restrict__ slot_off, int64_t* __restrict__ er,
                                 int64_t* __restrict__ ec, int64_t* __restrict__ ed) {
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= slots) return;
  const int t = tab[s];
  if (t == -1) return;
  const int64_t row = s / taps, dir = s % taps;
  int64_t o = slot_off[s];
  if (t >= 0) { er[o] = row; ec[o] = t; ed[o] = dir; return; }
  const int32_t* e = extra + (-(t + 2));
  const int n = e[0];
  for (int j = 1; j <= n; ++j, ++o) { er[o] = row; ec[o] = e[j]; ed[o] = dir; }
}

__global__ void multi_flags_kernel(const int32_t* __restrict__ tab, int64_t slots, int32_t* __restrict__ flags) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < slots) flags[i] = tab[i] <= -2 ? 1 : 0;
}

__global__ void multi_index_kernel(const int32_t* __restrict__ tab, const int32_t* __restrict__ extra,
                                   const uint8_t* __restrict__ node_type, int64_t slots,
                                   const int32_t* __restrict__ scan, int32_t* __restrict__ tab_ord,
                                   int32_t* __restrict__ multi_off, unsigned long long* __restrict__ multi_types) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= slots) return;
  const int32_t v = tab[i];
  if (v > -2) { tab_ord[i] = v; return; }
  const int32_t ord = scan[i];
  const int32_t o = -(v + 2);
  tab_ord[i] = -(ord + 2);
  multi_off[ord] = o;
  const int n = extra[o];
  unsigned long long packed = 0ull;
  for (int k = 1; k <= n; ++k) packed += 1ull << (8 * (node_type ? node_type[extra[o + k]] : 0));
  multi_types[ord] = packed;
}

// Node-type K block of the tensor-core GEMM, precomputed once per graph: row m, column tap*ntype + type holds
// (#neighbours of that type in slot (m, tap)) / (#neighbours) = the mean of the one-hot columns the reference
// appends to the features (modules.py:199-202) -- a graph constant, so the GEMM streams it like any other A tile
// instead of chasing tap table -> node_type for every tile.
__global__ void type_block_kernel(const int32_t* __restrict__ tab, const int32_t* __restrict__ extra,
                                  const uint8_t* __restrict__ node_type, int64_t rows, int taps, int ntype,
                                  __nv_bfloat16* __restrict__ out) {
  const int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= rows) return;
  __nv_bfloat16* o = out + m * 64;
  const uint4 z = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
  for (int c = 0; c < 8; ++c) reinterpret_cast<uint4*>(o)[c] = z;
  for (int tap = 0; tap < taps; ++tap) {
    const int32_t tv = tab[m * taps + tap];
    if (tv == -1) continue;
    int cnt[8] = {0, 0, 0, 0, 0, 0, 0, 0};                 // a coarse leaf can face up to 4^k finer cells: plain ints
    int n = 1;
    if (tv >= 0) {
      cnt[node_type[tv] & 7] = 1;
    } else {
      const int32_t* e = extra + (-(tv + 2));
      n = e[0];
      for (int k = 1; k <= n; ++k) ++cnt[node_type[e[k]] & 7];
    }
#pragma unroll
    for (int ty = 0; ty < 8; ++ty)
      if (ty < ntype && cnt[ty]) o[tap * ntype + ty] = __float2bfloat16_rn((float)cnt[ty] / (float)n);
  }
}

// one thread per (slot, 16-byte chunk): mean over the slot's neighbours, fp32 accumulate
template <typename T, int V>
__global__ void gather_mean_rows_kernel(const T* __restrict__ a0, int64_t lda0, int c0, const T* __restrict__ a1,
                                        int64_t lda1, int c1, const int32_t* __restrict__ extra,
                                        const int32_t* __restrict__ multi_off, int count, T* __restrict__ out,
                                        int64_t ldo) {
  const int cpr = (c0 + c1) / V;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)count * cpr) return;
  const int ord = (int)(idx / cpr);
  const int c = (int)(idx - (int64_t)ord * cpr) * V;
  const int32_t* e = extra + multi_off[ord];
  const int n = e[0];
  const T* base = c < c0 ? a0 + c : a1 + (c - c0);
  const int64_t ld = c < c0 ? lda0 : lda1;
  float acc[V];
#pragma unroll
  for (int j = 0; j < V; ++j) acc[j] = 0.0f;
  for (int k = 1; k <= n; ++k) {
    const T* src = base + (int64_t)e[k] * ld;
    if (V == 8) {
      float f[8];
      bf16x8_to_f32(*reinterpret_cast<const uint4*>(src), f);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j % V] += f[j];
    } else {
#pragma unroll
      for (int j = 0; j < V; ++j) acc[j] += Elem<T>::ld(src + j);
    }
  }
  const float dn = (float)n;
  T* o = out + (int64_t)ord * ldo + c;
  if (V == 8) {
    float f[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = acc[j % V] / dn;
    *reinterpret_cast<uint4*>(o) = f32_to_bf16x8(f);
  } else {
#pragma unroll
    for (int j = 0; j < V; ++j) Elem<T>::st(o + j, acc[j] / dn);
  }
}

}  // namespace of

using namespace of;

extern "C" int of_graph_multi_flags(const int32_t* tap_tab, int64_t slots, int32_t* flags, void* stream) {
  OF_REQUIRE(tap_tab && flags && slots >= 0, "of_graph_multi_flags: bad arguments");
  if (slots == 0) return OF_OK;
  multi_flags_kernel<<<(unsigned)((slots + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(tap_tab, slots,
                                                                                                        flags);
  OF_LAUNCH_CHECK("of_graph_multi_flags");
  return OF_OK;
}

extern "C" int of_graph_multi_index(const int32_t* tap_tab, const int32_t* tap_extra, const uint8_t* node_type,
                                    int64_t slots, const int32_t* flag_scan, int32_t* tap_tab_ord, int32_t* multi_off,
                                    uint64_t* multi_types, void* stream) {
  OF_REQUIRE(tap_tab && tap_extra && flag_scan && tap_tab_ord && multi_off && multi_types && slots >= 0,
             "of_graph_multi_index: bad arguments");
  if (slots == 0) return OF_OK;
  multi_index_kernel<<<(unsigned)((slots + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      tap_tab, tap_extra, node_type, slots, flag_scan, tap_tab_ord, multi_off,
      reinterpret_cast<unsigned long long*>(multi_types));
  OF_LAUNCH_CHECK("of_graph_multi_index");
  return OF_OK;
}

extern "C" int of_graph_type_block(const int32_t* tap_tab, const int32_t* tap_extra, const uint8_t* node_type, int64_t rows,
                                   int32_t taps, int32_t ntype, void* out_bf16, void* stream) {
  OF_REQUIRE(tap_tab && node_type && out_bf16 && rows >= 0 && taps > 0 && ntype > 0 && taps * ntype <= 64 && ntype <= 8,
             "of_graph_type_block: bad arguments");
  if (rows == 0) return OF_OK;
  type_block_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      tap_tab, tap_extra, node_type, rows, taps, ntype, reinterpret_cast<__nv_bfloat16*>(out_bf16));
  OF_LAUNCH_CHECK("of_graph_type_block");
  return OF_OK;
}

extern "C" int of_gather_mean_rows(const void* a0, int64_t lda0, int32_t c0, const void* a1, int64_t lda1, int32_t c1,
                                   const int32_t* tap_extra, const int32_t* multi_off, int32_t count, int32_t dtype,
                                   void* out, int64_t ldo, void* stream) {
  OF_REQUIRE(a0 && c0 > 0 && ((a1 == nullptr) == (c1 == 0)) && tap_extra && multi_off && out && count >= 0,
             "of_gather_mean_rows: bad arguments");
  OF_REQUIRE(dtype == OF_F32 || dtype == OF_BF16, "of_gather_mean_rows: bad dtype");
  if (count == 0) return OF_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int C = c0 + c1;
  if (dtype == OF_BF16 && c0 % 8 == 0 && c1 % 8 == 0 && lda0 % 8 == 0 && lda1 % 8 == 0 && ldo % 8 == 0) {
    const int64_t n = (int64_t)count * (C / 8);
    gather_mean_rows_kernel<__nv_bfloat16, 8><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(
        (const __nv_bfloat16*)a0, lda0, c0, (const __nv_bfloat16*)a1, lda1, c1, tap_extra, multi_off, count,
        (__nv_bfloat16*)out, ldo);
  } else if (dtype == OF_BF16) {
    const int64_t n = (int64_t)count * C;
    gather_mean_rows_kernel<__nv_bfloat16, 1><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(
        (const __nv_bfloat16*)a0, lda0, c0, (const __nv_bfloat16*)a1, lda1, c1, tap_extra, multi_off, count,
        (__nv_bfloat16*)out, ldo);
  } else {
    const int64_t n = (int64_t)count * C;
    gather_mean_rows_kernel<float, 1><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(
        (const float*)a0, lda0, c0, (const float*)a1, lda1, c1, tap_extra, multi_off, count, (float*)out, ldo);
  }
  OF_LAUNCH_CHECK("of_gather_mean_rows");
  return OF_OK;
}

extern "C" int64_t of_scan_scratch_bytes(int64_t n) {
  return ((n + SCAN_B - 1) / SCAN_B + 1) * (int64_t)sizeof(int32_t);
}

extern "C" int of_leaf_rank(const int32_t* children, int32_t n, int32_t* rank_out, int32_t* total_out, void* scratch,
                            void* stream) {
  return run_scan<1>(children, rank_out, n, total_out, scratch, reinterpret_cast<cudaStream_t>(stream), "of_leaf_rank");
}

extern "C" int of_exclusive_scan_i32(const int32_t* in, int32_t* out, int64_t n, int32_t* total_out, void* scratch,
                                     void* stream) {
  return run_scan<0>(in, out, n, total_out, scratch, reinterpret_cast<cudaStream_t>(stream), "of_exclusive_scan_i32");
}

extern "C" int of_compact_idx(const int32_t* children, const int32_t* leaf_rank, int32_t n, int32_t* leaf_idx,
                              int32_t* nonempty_idx, void* stream) {
  OF_REQUIRE(children && leaf_rank && n >= 0, "of_compact_idx: bad arguments");
  if (n == 0) return OF_OK;
  compact_idx_kernel<<<(n + 255) / 256, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(children, leaf_rank, n,
                                                                                         leaf_idx, nonempty_idx);
  OF_LAUNCH_CHECK("of_compact_idx");
  return OF_OK;
}

extern "C" int64_t of_graph_rows(const of_octree_levels* oct, int32_t D) {
  GraphCtx g;
  if (make_ctx(oct, D, g, "of_graph_rows")) return -1;
  return (int64_t)g.row_base[D] + oct->nnum[D];
}

extern "C" int of_graph_count(const of_octree_levels* oct, int32_t D, int32_t* need, void* stream) {
  GraphCtx g;
  int rc = make_ctx(oct, D, g, "of_graph_count");
  if (rc) return rc;
  OF_REQUIRE(need != nullptr, "of_graph_count: null output");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  for (int d = g.fd; d <= D; ++d) {
    const int64_t n = (int64_t)g.nnum[d] * 6;
    if (n == 0) continue;
    graph_count_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(g, d, need);
    if (d > g.fd) add_launches(1);
  }
  OF_LAUNCH_CHECK("of_graph_count");
  return OF_OK;
}

extern "C" int of_graph_fill(const of_octree_levels* oct, int32_t D, const int32_t* need_off, int32_t* tap_tab,
                             int32_t* tap_extra, uint8_t* node_type, int32_t* batch_id, void* stream) {
  GraphCtx g;
  int rc = make_ctx(oct, D, g, "of_graph_fill");
  if (rc) return rc;
  OF_REQUIRE(need_off && tap_tab && tap_extra, "of_graph_fill: null pointer");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  for (int d = g.fd; d <= D; ++d) {
    const int64_t n = (int64_t)g.nnum[d] * 6;
    if (n == 0) continue;
    graph_fill_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(g, d, need_off, tap_tab, tap_extra, node_type,
                                                                  batch_id);
    if (d > g.fd) add_launches(1);
  }
  OF_LAUNCH_CHECK("of_graph_fill");
  return OF_OK;
}

// ---------------------------------------------------------------------------------------------
// 3^3 neighbour table of ocnn.nn.OctreeConv (`octree.get_neigh(depth, '333')`; BASELINE.json configs[0]): for every
// octree node of `depth` the index (within that depth) of the node at (x+dx, y+dy, z+dz), tap = (dx+1)*9 + (dy+1)*3 +
// (dz+1), or -1 when that cell is outside the volume or does not exist (its parent is empty).  One warp per node,
// one lane per tap: the cell is located top-down through `children` from the full layer (no key hashing / search).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) octree_neigh27_kernel(GraphCtx g, int d, int32_t* __restrict__ out) {
  const int64_t node = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int tap = threadIdx.x & 31;
  if (node >= g.nnum[d] || tap >= 27) return;
  int x, y, z, b;
  key_decode(g.keys[d][node], d, x, y, z, b);
  const int nx = x + tap / 9 - 1, ny = y + (tap / 3) % 3 - 1, nz = z + tap % 3 - 1;
  const int lim = 1 << d;
  int res = -1;
  if (nx >= 0 && ny >= 0 && nz >= 0 && nx < lim && ny < lim && nz < lim) {
    int cd = g.fd;
    int ci = (int)(((int64_t)b << (3 * g.fd)) + morton3(nx >> (d - g.fd), ny >> (d - g.fd), nz >> (d - g.fd), g.fd));
    while (cd < d) {
      const int c = g.children[cd][ci];
      if (c < 0) break;
      const int sh = d - cd - 1;
      ci = 8 * c + ((((nx >> sh) & 1) << 2) | (((ny >> sh) & 1) << 1) | ((nz >> sh) & 1));
      ++cd;
    }
    if (cd == d) res = ci;
  }
  out[node * 27 + tap] = res;
}

extern "C" int of_octree_neigh27(const of_octree_levels* oct, int32_t depth, int32_t* neigh, void* stream) {
  using namespace of;
  OF_REQUIRE(oct != nullptr && neigh != nullptr, "of_octree_neigh27: null pointer");
  OF_REQUIRE(oct->full_depth >= 1 && depth >= oct->full_depth && depth <= oct->depth && depth < 16,
             "of_octree_neigh27: depth %d outside [full_depth %d, depth %d]", depth, oct->full_depth, oct->depth);
  GraphCtx g;
  for (int d = 0; d < 16; ++d) {
    g.keys[d] = oct->keys[d]; g.children[d] = oct->children[d]; g.leaf_rank[d] = nullptr;
    g.nnum[d] = oct->nnum[d]; g.row_base[d] = 0;
  }
  g.fd = oct->full_depth; g.depth = oct->depth; g.D = depth; g.batch = oct->batch;
  for (int d = g.fd; d <= depth; ++d)
    OF_REQUIRE(oct->keys[d] && oct->children[d] && oct->nnum[d] >= 0, "of_octree_neigh27: level %d missing", d);
  const int64_t n = oct->nnum[depth];
  if (n == 0) return OF_OK;
  const int64_t threads = n * 32;
  octree_neigh27_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(g, depth, neigh);
  OF_LAUNCH_CHECK("of_octree_neigh27");
  return OF_OK;
}

extern "C" int of_graph_edge_count(const int32_t* tap_tab, const int32_t* tap_extra, int64_t slots, int32_t* per_slot,
                                   void* stream) {
  OF_REQUIRE(tap_tab && per_slot && slots >= 0, "of_graph_edge_count: bad arguments");
  if (slots == 0) return OF_OK;
  edge_count_kernel<<<(unsigned)((slots + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      tap_tab, tap_extra, slots, per_slot);
  OF_LAUNCH_CHECK("of_graph_edge_count");
  return OF_OK;
}

extern "C" int of_graph_edges(const int32_t* tap_tab, const int32_t* tap_extra, int64_t slots, int32_t taps,
                              const int32_t* slot_off, int64_t* edge_row, int64_t* edge_col, int64_t* edge_dir,
                              void* stream) {
  OF_REQUIRE(tap_tab && slot_off && edge_row && edge_col && edge_dir && taps > 0, "of_graph_edges: bad arguments");
  if (slots == 0) return OF_OK;
  edge_fill_kernel<<<(unsigned)((slots + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      tap_tab, tap_extra, slots, taps, slot_off, edge_row, edge_col, edge_dir);
  OF_LAUNCH_CHECK("of_graph_edges");
  return OF_OK;
}
