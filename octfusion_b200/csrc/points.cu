// Octree build from point clouds and the ND input feature of the GraphVAE encoder.
//
// The build restates ocnn.octree.Octree.build_octree (ocnn-pytorch 2.2.x, SURVEY.md Appendix B; parity UNPINNED at the
// ocnn boundary): a batched, deterministic construction from one sorted array of point keys.
//   keys      one thread per point: p' = (p + 1) * 2^(depth-1) in fp32, truncated, masked to depth bits, Morton
//             interleaved; the SORT key is the compact (shape << 3*depth) | morton
//   sort      stable LSD radix sort of (key, point index), 8-bit digits, over the 3*depth + ceil(log2 batch)
//             significant bits only.  One warp ranks a 2048-element chunk with __match_any_sync, so the rank of an
//             element among equal digits follows input order: points of a node stay in input order.
//   levels    at every depth d in full_depth..depth the node of sorted element i is key >> 3(depth - d); a run head
//             (first element of a node) gets flag 1, an exclusive scan of the flags gives the node ranks and, in its
//             total, the number of non-empty nodes.  No second sort, no hashing.
//   fill      keys[d] = the 8 children of every non-empty depth-(d-1) node, children[d][8 parent + child] = rank.
//   signal    one thread per non-empty depth-`depth` node sums its points and normals in sorted (= input) order, fp32.
// The ND feature kernel writes [normal | sum((frac(point) - 0.5) * normal)] straight into depth-D graph rows.
#include "common.cuh"

namespace of {

constexpr int PT_T = 256;                     // threads per block
constexpr int PT_WARPS = PT_T / 32;
constexpr int PT_CHUNK = 32 * 64;             // elements per warp chunk of a radix pass

static inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

// scratch layout of one build, a pure function of (npts, batch, depth, full_depth)
struct BuildLayout {
  int64_t n, nchunks, nhist;
  int bits, passes, levels;
  size_t keys[2], idx[2], hist, hist_scan, scan_tmp, flags, rank, total;
};

static BuildLayout make_layout(int64_t n, int batch, int depth, int full_depth) {
  BuildLayout L;
  int bb = 0;
  while ((1 << bb) < batch) ++bb;
  L.n = n;
  L.bits = 3 * depth + bb;
  L.passes = (L.bits + 7) / 8;
  L.levels = depth - full_depth + 1;
  L.nchunks = (n + PT_CHUNK - 1) / PT_CHUNK;
  L.nhist = 256 * L.nchunks;
  const int64_t scan_n = n > L.nhist ? n : L.nhist;
  size_t off = 0;
  for (int k = 0; k < 2; ++k) { L.keys[k] = off; off += align256((size_t)n * 8); }
  for (int k = 0; k < 2; ++k) { L.idx[k] = off; off += align256((size_t)n * 4); }
  L.hist = off; off += align256((size_t)L.nhist * 4);
  L.hist_scan = off; off += align256((size_t)(L.nhist + 1) * 4);
  L.scan_tmp = off; off += align256((size_t)of_scan_scratch_bytes(scan_n));
  L.flags = off; off += align256((size_t)n * 4);
  L.rank = off; off += align256((size_t)L.levels * (n + 1) * 4);
  L.total = off;
  return L;
}

// rank array of depth d: exclusive scan of the run-head flags, n + 1 entries (the last one = node count)
static inline size_t rank_off(const BuildLayout& L, int d, int full_depth) {
  return L.rank + (size_t)(d - full_depth) * (L.n + 1) * 4;
}

__device__ __forceinline__ float scaled_coord(float p, float s) { return __fmul_rn(__fadd_rn(p, 1.0f), s); }

__global__ void check_offsets_kernel(const int64_t* __restrict__ off, int batch, int64_t n, int32_t* __restrict__ status) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  int bad = off[0] != 0 || off[batch] != n;
  for (int b = 0; b < batch; ++b) bad |= off[b + 1] < off[b];
  *status = bad;
}

__global__ void point_keys_kernel(const float* __restrict__ xyz, const int64_t* __restrict__ off, int batch, int64_t n,
                                  int depth, uint64_t* __restrict__ key, uint32_t* __restrict__ idx) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int lo = 0, hi = batch - 1;                 // shape of point i: the last b with off[b] <= i
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (off[mid] <= i) lo = mid; else hi = mid - 1;
  }
  const float s = (float)(1 << (depth - 1));
  const uint64_t mask = (1ull << depth) - 1;
  uint64_t c[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) c[a] = (uint64_t)__float2ll_rz(scaled_coord(xyz[3 * i + a], s)) & mask;
  uint64_t m = 0;
  for (int k = 0; k < depth; ++k)
    m |= (((c[0] >> k) & 1) << (3 * k + 2)) | (((c[1] >> k) & 1) << (3 * k + 1)) | (((c[2] >> k) & 1) << (3 * k));
  key[i] = ((uint64_t)lo << (3 * depth)) | m;
  idx[i] = (uint32_t)i;
}

// per (digit, chunk) counts, digit-major so that one exclusive scan gives every chunk's output offset per digit
__global__ void __launch_bounds__(PT_T) radix_hist_kernel(const uint64_t* __restrict__ key, int64_t n, int shift,
                                                          int64_t nchunks, int32_t* __restrict__ hist) {
  __shared__ int32_t cnt[PT_WARPS][256];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t chunk = (int64_t)blockIdx.x * PT_WARPS + w;
  if (chunk >= nchunks) return;
  for (int j = lane; j < 256; j += 32) cnt[w][j] = 0;
  __syncwarp();
  const int64_t base = chunk * PT_CHUNK;
  const int64_t end = base + PT_CHUNK < n ? base + PT_CHUNK : n;
  for (int64_t i = base + lane; i < end; i += 32) atomicAdd(&cnt[w][(unsigned)(key[i] >> shift) & 255u], 1);
  __syncwarp();
  for (int j = lane; j < 256; j += 32) hist[(int64_t)j * nchunks + chunk] = cnt[w][j];
}

// stable scatter: element i of a chunk goes to offset[digit] + (elements of its chunk before it with that digit)
__global__ void __launch_bounds__(PT_T) radix_scatter_kernel(const uint64_t* __restrict__ key_in,
                                                             const uint32_t* __restrict__ idx_in, int64_t n, int shift,
                                                             int64_t nchunks, const int32_t* __restrict__ hist_scan,
                                                             uint64_t* __restrict__ key_out,
                                                             uint32_t* __restrict__ idx_out) {
  __shared__ int32_t next[PT_WARPS][256];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t chunk = (int64_t)blockIdx.x * PT_WARPS + w;
  if (chunk >= nchunks) return;
  for (int j = lane; j < 256; j += 32) next[w][j] = hist_scan[(int64_t)j * nchunks + chunk];
  __syncwarp();
  const int64_t base = chunk * PT_CHUNK;
  const int64_t end = base + PT_CHUNK < n ? base + PT_CHUNK : n;
  const unsigned below = (1u << lane) - 1u;
  for (int64_t r = base; r < end; r += 32) {
    const int64_t i = r + lane;
    const bool ok = i < end;
    const uint64_t k = ok ? key_in[i] : 0;
    const unsigned dg = ok ? ((unsigned)(k >> shift) & 255u) : 256u;
    const unsigned peers = __match_any_sync(0xffffffffu, dg);
    const int leader = __ffs(peers) - 1;
    int b = (ok && lane == leader) ? next[w][dg] : 0;
    b = __shfl_sync(0xffffffffu, b, leader);
    if (ok) {
      const int64_t dst = (int64_t)b + __popc(peers & below);
      key_out[dst] = k;
      idx_out[dst] = idx_in[i];
    }
    __syncwarp();
    if (ok && lane == leader) next[w][dg] = b + __popc(peers);
    __syncwarp();
  }
}

__global__ void head_flags_kernel(const uint64_t* __restrict__ key, int64_t n, int shift, int32_t* __restrict__ flags) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  flags[i] = i == 0 || (key[i] >> shift) != (key[i - 1] >> shift);
}

// children of the full layer: slot = shape * 8^fd + morton = the compact depth-fd key
__global__ void fill_full_kernel(const uint64_t* __restrict__ key, int64_t n, int shift, const int32_t* __restrict__ rank,
                                 int32_t* __restrict__ children) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t k = key[i] >> shift;
  if (i == 0 || (key[i - 1] >> shift) != k) children[k] = rank[i];
}

// depth d > full_depth: parent run heads write the 8 child keys, child run heads their rank
__global__ void fill_level_kernel(const uint64_t* __restrict__ key, int64_t n, int depth, int d,
                                  const int32_t* __restrict__ rank_p, const int32_t* __restrict__ rank_d,
                                  int64_t* __restrict__ keys_d, int32_t* __restrict__ children_d) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int sp = 3 * (depth - d + 1), sd = 3 * (depth - d);
  const uint64_t kp = key[i] >> sp, kd = key[i] >> sd;
  const int64_t pr = rank_p[i + 1] - 1;       // rank of the parent node of element i
  if (i == 0 || (key[i - 1] >> sp) != kp) {
    const int pbits = 3 * (d - 1);
    const uint64_t b = kp >> pbits, m = kp & ((1ull << pbits) - 1);
    const uint64_t head = (b << 48) | (m << 3);
#pragma unroll
    for (int c = 0; c < 8; ++c) keys_d[8 * pr + c] = (int64_t)(head | (uint64_t)c);
  }
  if (i == 0 || (key[i - 1] >> sd) != kd) children_d[8 * pr + (int64_t)(kd & 7)] = rank_d[i];
}

__global__ void node_signal_kernel(const uint64_t* __restrict__ key, const uint32_t* __restrict__ idx, int64_t n,
                                   int depth, const int32_t* __restrict__ rank, const float* __restrict__ xyz,
                                   const float* __restrict__ nrm, float* __restrict__ points,
                                   float* __restrict__ normals) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t k = key[i];
  if (i > 0 && key[i - 1] == k) return;
  const float s = (float)(1 << (depth - 1));
  float p[3] = {0.f, 0.f, 0.f}, q[3] = {0.f, 0.f, 0.f};
  int64_t j = i;
  for (; j < n && key[j] == k; ++j) {
    const int64_t src = idx[j];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      p[a] = __fadd_rn(p[a], scaled_coord(xyz[3 * src + a], s));
      if (nrm) q[a] = __fadd_rn(q[a], nrm[3 * src + a]);
    }
  }
  const int64_t r = rank[i];
  const float cnt = (float)(j - i);
#pragma unroll
  for (int a = 0; a < 3; ++a) points[3 * r + a] = __fdiv_rn(p[a], cnt);
  if (nrm) {
    float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(q[0], q[0]), __fmul_rn(q[1], q[1])), __fmul_rn(q[2], q[2])));
    len = fmaxf(len, 1e-12f);
#pragma unroll
    for (int a = 0; a < 3; ++a) normals[3 * r + a] = __fdiv_rn(q[a], len);
  }
}

template <typename T>
__global__ void input_feature_nd_kernel(const float* __restrict__ points, const float* __restrict__ normals,
                                        const int32_t* __restrict__ children, int64_t nnum, int64_t leaf_rows,
                                        T* __restrict__ out, int64_t ldo) {
  const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= leaf_rows + nnum) return;
  float f[4] = {0.f, 0.f, 0.f, 0.f};
  const int64_t r = row < leaf_rows ? -1 : (int64_t)children[row - leaf_rows];
  if (r >= 0) {
    float dsum = 0.f;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const float pa = points[3 * r + a], na = normals[3 * r + a];
      f[a] = na;
      const float t = __fmul_rn(__fsub_rn(__fsub_rn(pa, truncf(pa)), 0.5f), na);
      dsum = a == 0 ? t : __fadd_rn(dsum, t);
    }
    f[3] = dsum;
  }
  T* o = out + row * ldo;
#pragma unroll
  for (int a = 0; a < 4; ++a) Elem<T>::st(o + a, f[a]);
}

static int check_build_args(int64_t npts, int32_t batch, int32_t depth, int32_t full_depth, const char* who) {
  OF_REQUIRE(depth <= 16 && full_depth >= 0 && full_depth < depth, "%s: need 0 <= full_depth < depth <= 16 (got %d, %d)",
             who, full_depth, depth);
  OF_REQUIRE(batch >= 1 && batch < 1024, "%s: need 1 <= batch < 1024 (got %d)", who, batch);
  OF_REQUIRE(npts >= 0 && npts < ((int64_t)1 << 31), "%s: need 0 <= npts < 2^31 (got %lld)", who, (long long)npts);
  OF_REQUIRE((int64_t)batch << (3 * full_depth) < ((int64_t)1 << 31), "%s: batch * 8^full_depth must be below 2^31",
             who);
  return OF_OK;
}

static inline unsigned blocks_of(int64_t n) { return (unsigned)((n + PT_T - 1) / PT_T); }

}  // namespace of

using namespace of;

extern "C" int64_t of_octree_build_bytes(int64_t npts, int32_t batch, int32_t depth, int32_t full_depth) {
  if (check_build_args(npts, batch, depth, full_depth, "of_octree_build_bytes")) return OF_E_ARG;
  return (int64_t)make_layout(npts, batch, depth, full_depth).total;
}

extern "C" int of_octree_build_levels(const float* xyz, const int64_t* shape_offsets, int64_t npts, int32_t batch,
                                      int32_t depth, int32_t full_depth, void* scratch, int32_t* level_counts,
                                      void* stream) {
  const char* who = "of_octree_build_levels";
  if (int rc = check_build_args(npts, batch, depth, full_depth, who)) return rc;
  OF_REQUIRE(shape_offsets && scratch && level_counts && (xyz || npts == 0), "%s: null pointer", who);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const BuildLayout L = make_layout(npts, batch, depth, full_depth);
  char* base = static_cast<char*>(scratch);
  if (cudaMemsetAsync(level_counts, 0, (size_t)(depth + 2) * sizeof(int32_t), st) != cudaSuccess) {
    set_error("%s: cudaMemsetAsync failed", who);
    return OF_E_CUDA;
  }
  check_offsets_kernel<<<1, 32, 0, st>>>(shape_offsets, batch, npts, level_counts + depth + 1);
  OF_LAUNCH_CHECK(who);
  if (npts == 0) return OF_OK;
  uint64_t* keys[2] = {reinterpret_cast<uint64_t*>(base + L.keys[0]), reinterpret_cast<uint64_t*>(base + L.keys[1])};
  uint32_t* idx[2] = {reinterpret_cast<uint32_t*>(base + L.idx[0]), reinterpret_cast<uint32_t*>(base + L.idx[1])};
  int32_t* hist = reinterpret_cast<int32_t*>(base + L.hist);
  int32_t* hist_scan = reinterpret_cast<int32_t*>(base + L.hist_scan);
  void* scan_tmp = base + L.scan_tmp;
  int32_t* flags = reinterpret_cast<int32_t*>(base + L.flags);
  point_keys_kernel<<<blocks_of(npts), PT_T, 0, st>>>(xyz, shape_offsets, batch, npts, depth, keys[0], idx[0]);
  OF_LAUNCH_CHECK(who);
  const unsigned chunk_blocks = (unsigned)((L.nchunks + PT_WARPS - 1) / PT_WARPS);
  for (int p = 0; p < L.passes; ++p) {
    const int src = p & 1, dst = src ^ 1;
    radix_hist_kernel<<<chunk_blocks, PT_T, 0, st>>>(keys[src], npts, 8 * p, L.nchunks, hist);
    OF_LAUNCH_CHECK(who);
    if (int rc = of_exclusive_scan_i32(hist, hist_scan, L.nhist, nullptr, scan_tmp, stream)) return rc;
    radix_scatter_kernel<<<chunk_blocks, PT_T, 0, st>>>(keys[src], idx[src], npts, 8 * p, L.nchunks, hist_scan,
                                                        keys[dst], idx[dst]);
    OF_LAUNCH_CHECK(who);
  }
  const uint64_t* sorted = keys[L.passes & 1];
  for (int d = full_depth; d <= depth; ++d) {
    head_flags_kernel<<<blocks_of(npts), PT_T, 0, st>>>(sorted, npts, 3 * (depth - d), flags);
    OF_LAUNCH_CHECK(who);
    int32_t* rank = reinterpret_cast<int32_t*>(base + rank_off(L, d, full_depth));
    if (int rc = of_exclusive_scan_i32(flags, rank, npts, level_counts + d, scan_tmp, stream)) return rc;
  }
  return OF_OK;
}

extern "C" int of_octree_build_fill(const void* scratch, int64_t npts, int32_t batch, int32_t depth, int32_t full_depth,
                                    int32_t d, int64_t nnum_d, int64_t* keys_d, int32_t* children_d, void* stream) {
  const char* who = "of_octree_build_fill";
  if (int rc = check_build_args(npts, batch, depth, full_depth, who)) return rc;
  OF_REQUIRE(d >= full_depth && d <= depth, "%s: depth %d outside full_depth..depth", who, d);
  OF_REQUIRE(scratch && children_d && (keys_d || d == full_depth) && nnum_d >= 0, "%s: bad arguments", who);
  OF_REQUIRE(d > full_depth || nnum_d == ((int64_t)batch << (3 * full_depth)), "%s: full layer needs batch * 8^%d nodes",
             who, full_depth);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (nnum_d == 0) return OF_OK;
  if (cudaMemsetAsync(children_d, 0xff, (size_t)nnum_d * sizeof(int32_t), st) != cudaSuccess) {
    set_error("%s: cudaMemsetAsync failed", who);
    return OF_E_CUDA;
  }
  if (npts == 0) return OF_OK;
  const BuildLayout L = make_layout(npts, batch, depth, full_depth);
  const char* base = static_cast<const char*>(scratch);
  const uint64_t* sorted = reinterpret_cast<const uint64_t*>(base + L.keys[L.passes & 1]);
  const int32_t* rank_d = reinterpret_cast<const int32_t*>(base + rank_off(L, d, full_depth));
  if (d == full_depth) {
    fill_full_kernel<<<blocks_of(npts), PT_T, 0, st>>>(sorted, npts, 3 * (depth - d), rank_d, children_d);
  } else {
    const int32_t* rank_p = reinterpret_cast<const int32_t*>(base + rank_off(L, d - 1, full_depth));
    fill_level_kernel<<<blocks_of(npts), PT_T, 0, st>>>(sorted, npts, depth, d, rank_p, rank_d, keys_d, children_d);
  }
  OF_LAUNCH_CHECK(who);
  return OF_OK;
}

extern "C" int of_octree_build_signal(const void* scratch, int64_t npts, int32_t batch, int32_t depth,
                                      int32_t full_depth, const float* xyz, const float* normals_in, float* points,
                                      float* normals, void* stream) {
  const char* who = "of_octree_build_signal";
  if (int rc = check_build_args(npts, batch, depth, full_depth, who)) return rc;
  OF_REQUIRE(scratch && (npts == 0 || (xyz && points)) && ((normals_in == nullptr) == (normals == nullptr)),
             "%s: bad arguments", who);
  if (npts == 0) return OF_OK;
  const BuildLayout L = make_layout(npts, batch, depth, full_depth);
  const char* base = static_cast<const char*>(scratch);
  node_signal_kernel<<<blocks_of(npts), PT_T, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const uint64_t*>(base + L.keys[L.passes & 1]),
      reinterpret_cast<const uint32_t*>(base + L.idx[L.passes & 1]), npts, depth,
      reinterpret_cast<const int32_t*>(base + rank_off(L, depth, full_depth)), xyz, normals_in, points, normals);
  OF_LAUNCH_CHECK(who);
  return OF_OK;
}

extern "C" int of_input_feature_nd(const float* points, const float* normals, const int32_t* children, int64_t nnum,
                                   int64_t leaf_rows, int32_t dtype, void* out, int64_t ldo, void* stream) {
  const char* who = "of_input_feature_nd";
  OF_REQUIRE(out && nnum >= 0 && leaf_rows >= 0 && ldo >= 4 && (nnum == 0 || (points && normals && children)),
             "%s: bad arguments", who);
  OF_REQUIRE(dtype == OF_F32 || dtype == OF_BF16, "%s: bad dtype %d", who, dtype);
  const int64_t rows = leaf_rows + nnum;
  if (rows == 0) return OF_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == OF_F32)
    input_feature_nd_kernel<float><<<blocks_of(rows), PT_T, 0, st>>>(points, normals, children, nnum, leaf_rows,
                                                                      static_cast<float*>(out), ldo);
  else
    input_feature_nd_kernel<__nv_bfloat16><<<blocks_of(rows), PT_T, 0, st>>>(
        points, normals, children, nnum, leaf_rows, static_cast<__nv_bfloat16*>(out), ldo);
  OF_LAUNCH_CHECK(who);
  return OF_OK;
}
