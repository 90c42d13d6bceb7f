// Group normalisation over ragged per-sample node sets, fused with SiLU and the channel concat.
//
// Replaces DualOctreeGroupNorm.forward (reference models/networks/modules.py:291-326: three
// scatter_add passes, two index_select passes and six elementwise passes = ~12 HBM round trips)
// and the dense GroupNorm32 (modules.py:26-28) by
//   of_gn_stats     one read  of x            -> per (32-row segment, 4-channel granule) sum / sum of squares in fp32,
//                   no atomics (bit-reproducible); skipped when the producing tensor-core GEMM wrote the partials itself
//   of_gn_finalize  partials summed in fixed order in fp64 -> [B, C] scale / shift table (fp32 result)
//   of_gn_apply     one read + one write      -> y = SiLU(x * scale + shift), concat fused
// HBM-bound kernels: 16-byte vector accesses, grid sized in multiples of the SM count.
#include "common.cuh"

namespace of {

template <typename T> struct Vec;
template <> struct Vec<float> { static constexpr int N = 4; };
template <> struct Vec<__nv_bfloat16> { static constexpr int N = 8; };

template <typename T, int V>
__device__ __forceinline__ void load_vec(const T* p, float* f);
template <>
__device__ __forceinline__ void load_vec<float, 4>(const float* p, float* f) {
  float4 q = *reinterpret_cast<const float4*>(p);
  f[0] = q.x; f[1] = q.y; f[2] = q.z; f[3] = q.w;
}
template <>
__device__ __forceinline__ void load_vec<float, 1>(const float* p, float* f) { f[0] = *p; }
template <>
__device__ __forceinline__ void load_vec<__nv_bfloat16, 8>(const __nv_bfloat16* p, float* f) {
  uint4 q = *reinterpret_cast<const uint4*>(p);
  bf16x8_to_f32(q, f);
}
template <>
__device__ __forceinline__ void load_vec<__nv_bfloat16, 4>(const __nv_bfloat16* p, float* f) {
  const uint2 q = *reinterpret_cast<const uint2*>(p);
  const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&q.x));
  const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&q.y));
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y;
}
template <>
__device__ __forceinline__ void load_vec<__nv_bfloat16, 1>(const __nv_bfloat16* p, float* f) {
  f[0] = __bfloat162float(*p);
}
template <typename T, int V>
__device__ __forceinline__ void store_vec(T* p, const float* f);
template <>
__device__ __forceinline__ void store_vec<float, 4>(float* p, const float* f) {
  *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
}
template <>
__device__ __forceinline__ void store_vec<float, 1>(float* p, const float* f) { *p = f[0]; }
template <>
__device__ __forceinline__ void store_vec<__nv_bfloat16, 8>(__nv_bfloat16* p, const float* f) {
  *reinterpret_cast<uint4*>(p) = f32_to_bf16x8(f);
}
template <>
__device__ __forceinline__ void store_vec<__nv_bfloat16, 1>(__nv_bfloat16* p, const float* f) {
  *p = __float2bfloat16_rn(f[0]);
}

struct GnSrc {
  const void* x0; int64_t ld0; int c0;
  const void* x1; int64_t ld1; int c1;
  const int32_t* sample_id; int rows_per_sample;
  int64_t rows;
};

template <typename T, int V>
__device__ __forceinline__ const T* src_ptr(const GnSrc& s, int64_t r, int c) {
  return c < s.c0 ? reinterpret_cast<const T*>(s.x0) + r * s.ld0 + c
                  : reinterpret_cast<const T*>(s.x1) + r * s.ld1 + (c - s.c0);
}

constexpr int GN_UNROLL = 4;                               // independent 16-byte loads in flight per thread

// true when all rows [r0, r1) of this CTA belong to one sample (the common case: rows are grouped by sample inside
// each depth segment of the graph, so only a handful of the 256-row chunks straddle a boundary)
__device__ __forceinline__ bool chunk_is_uniform(const GnSrc& s, int64_t r0, int64_t r1, int& b0) {
  if (s.sample_id) {
    b0 = s.sample_id[r0];
    bool same = true;
    for (int64_t r = r0 + threadIdx.x; r < r1; r += blockDim.x) same = same && (s.sample_id[r] == b0);
    return __syncthreads_and(same) != 0;
  }
  b0 = (int)(r0 / s.rows_per_sample);
  return (int)((r1 - 1) / s.rows_per_sample) == b0;
}

// Deterministic partial statistics: one thread per (32-row chunk, channel vector) adds its rows in order and writes
// (sum, sum of squares) per 4-channel granule into the slot of the chunk's segment -- the layout the tensor-core GEMM
// epilogue produces (of_gemm_args.stat_out), so of_gn_finalize serves both.  A new segment starts at every change
// of sample id inside the chunk.
template <typename T, int V, int GRAN>
__global__ void __launch_bounds__(256) gn_stats_kernel(GnSrc s, const int32_t* __restrict__ chunk_seg,
                                                       const int32_t* __restrict__ seg_slot, float* __restrict__ part) {
  const int C = s.c0 + s.c1;
  const int tpr = C / V;                                   // threads per chunk
  const int64_t gidx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t chunk = gidx / tpr;
  const int cv = (int)(gidx - chunk * tpr) * V;
  const int64_t r0 = chunk * 32;
  if (r0 >= s.rows) return;
  const int64_t r1 = min(r0 + 32, s.rows);
  const T* base = cv < s.c0 ? reinterpret_cast<const T*>(s.x0) + cv : reinterpret_cast<const T*>(s.x1) + (cv - s.c0);
  const int64_t ld = cv < s.c0 ? s.ld0 : s.ld1;
  constexpr int G = V / GRAN;                              // granules per thread (V = 4 or 8, GRAN = 2 or 4)
  float sum[G], sq[G];
#pragma unroll
  for (int i = 0; i < G; ++i) { sum[i] = 0.0f; sq[i] = 0.0f; }
  int seg = chunk_seg[chunk];
  const int half = C / GRAN * 2;                           // floats per segment slot
  auto sample_of = [&](int64_t r) { return s.sample_id ? s.sample_id[r] : (int)(r / s.rows_per_sample); };
  int cur = sample_of(r0);
  auto flush = [&]() {
#pragma unroll
    for (int i = 0; i < G; ++i) {
      *reinterpret_cast<float2*>(part + (int64_t)seg_slot[seg] * half + (cv / GRAN + i) * 2) = make_float2(sum[i], sq[i]);
      sum[i] = 0.0f; sq[i] = 0.0f;
    }
  };
  for (int64_t r = r0; r < r1; r += 8) {
    float f[8][V];
#pragma unroll
    for (int u = 0; u < 8; ++u)
      if (r + u < r1) load_vec<T, V>(base + (r + u) * ld, f[u]);
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      if (r + u >= r1) break;
      const int b = sample_of(r + u);
      if (b != cur) { flush(); ++seg; cur = b; }
#pragma unroll
      for (int i = 0; i < V; ++i) { sum[i / GRAN] += f[u][i]; sq[i / GRAN] = fmaf(f[u][i], f[u][i], sq[i / GRAN]); }
    }
  }
  flush();
}

// Partial slots of a sample are summed in slot order (fixed order, fp64), then the group statistics and the [C] scale /
// shift rows of the sample are formed.  grid = (batch, S): the S CTAs of a sample each reduce a contiguous range of
// its slots into a fp64 scratch row; the CTA that finishes last (a ticket per sample, self-resetting) adds the S rows in
// index order -- the ticket only decides WHO does the last step, never the order of the additions, so the result is
// bit-reproducible -- and writes scale / shift.
//   smem: double red[slices][nval] | double tot[nval]
__global__ void __launch_bounds__(1024) gn_finalize_kernel(const float* __restrict__ part0, int c0, int gran0,
                                                            const float* __restrict__ part1, int c1, int gran1,
                                                            const int32_t* __restrict__ seg_off,
                                                            const int32_t* __restrict__ rows_of_sample, int rows_per_sample,
                                                            const float* __restrict__ gamma, const float* __restrict__ beta,
                                                            int groups, float eps, float count_eps, float* __restrict__ scale,
                                                            float* __restrict__ shift, double* __restrict__ scratch,
                                                            int* __restrict__ ticket) {
  extern __shared__ double gn_sm[];
  __shared__ int is_last;
  const int b = blockIdx.x, sb = blockIdx.y, S = gridDim.y;
  const int C = c0 + c1;
  const int h0 = c0 / gran0 * 2, h1 = c1 > 0 ? c1 / gran1 * 2 : 0;   // floats per segment slot of the two buffers
  const int nval = h0 + h1;
  const int slices = blockDim.x / nval;                    // >= 1 (checked on host)
  double* red = gn_sm;
  double* tot = gn_sm + (size_t)slices * nval;
  const int j = threadIdx.x % nval, sl = threadIdx.x / nval;
  const int k0 = seg_off[b], k1 = seg_off[b + 1];
  const int per_blk = (k1 - k0 + S - 1) / S;
  const int a0 = k0 + sb * per_blk, e0 = min(a0 + per_blk, k1);
  if (sl < slices) {
    // contiguous sub-range of this CTA's slots for this slice; eight independent loads in flight, four interleaved
    // accumulators, fixed order
    const int n = max(e0 - a0, 0);
    const int per = (n + slices - 1) / slices;
    const int a = a0 + sl * per, e = min(a + per, e0);
    const float* src = j < h0 ? part0 + j : part1 + (j - h0);
    const int64_t stride = j < h0 ? h0 : h1;
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    int k = a;
    for (; k + 7 < e; k += 8) {
      float v8[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) v8[u] = src[(int64_t)(k + u) * stride];
#pragma unroll
      for (int u = 0; u < 8; ++u) acc[u & 3] += (double)v8[u];
    }
    for (int u = 0; k < e; ++k, ++u) acc[u & 3] += (double)src[(int64_t)k * stride];
    red[(size_t)sl * nval + j] = (acc[0] + acc[1]) + (acc[2] + acc[3]);
  }
  __syncthreads();
  if ((int)threadIdx.x < nval) {
    double t = 0.0;
    for (int q = 0; q < slices; ++q) t += red[(size_t)q * nval + threadIdx.x];
    tot[threadIdx.x] = t;
    if (S > 1) scratch[((size_t)b * S + sb) * nval + threadIdx.x] = t;
  }
  if (S > 1) {
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) is_last = (atomicAdd(&ticket[b], 1) == S - 1) ? 1 : 0;
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    if ((int)threadIdx.x < nval) {
      double t = 0.0;
      for (int q = 0; q < S; ++q) t += __ldcg(&scratch[((size_t)b * S + q) * nval + threadIdx.x]);
      tot[threadIdx.x] = t;
    }
    if (threadIdx.x == 0) ticket[b] = 0;                   // ready for the next launch
  }
  __syncthreads();
  const int cpg = C / groups;
  const double n = (double)(rows_of_sample ? rows_of_sample[b] : rows_per_sample) * (double)cpg;
  const double inv = 1.0 / (n + (double)count_eps);      // modules.py:302: eps joins the COUNT
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int g = c / cpg;
    const int lo = g * cpg, hi = lo + cpg;                 // the group's channels: granules of x0 then of x1
    double S_ = 0.0, Q = 0.0;
    for (int ch = lo; ch < min(hi, c0); ch += gran0) { S_ += tot[ch / gran0 * 2]; Q += tot[ch / gran0 * 2 + 1]; }
    for (int ch = max(lo, c0); ch < hi; ch += gran1) { S_ += tot[h0 + (ch - c0) / gran1 * 2]; Q += tot[h0 + (ch - c0) / gran1 * 2 + 1]; }
    const double m = S_ * inv;                             // modules.py:304
    double var = (Q - 2.0 * m * S_ + n * m * m) * inv;     // sum (x-m)^2 * inv_count, modules.py:308
    if (var < 0.0) var = 0.0;
    const double rstd = 1.0 / sqrt(var + (double)eps);     // modules.py:310
    const double ga = gamma[c];
    scale[(int64_t)b * C + c] = (float)(rstd * ga);
    shift[(int64_t)b * C + c] = (float)((double)beta[c] - m * rstd * ga);
  }
}

template <typename T> struct FastAct;
template <> struct FastAct<float> { static __device__ __forceinline__ float silu(float v) { return silu_f(v); } };
template <> struct FastAct<__nv_bfloat16> { static __device__ __forceinline__ float silu(float v) { return silu_fast(v); } };

// Each thread owns one channel vector and walks down the rows of its CTA's 256-row chunk; the per-(sample,
// channel) scale/shift pair stays in registers until the sample id changes.  Chunks that lie inside one sample
// (nearly all) take the unrolled path: GN_UNROLL loads in flight, no per-row sample lookup.
template <typename T, int V>
__global__ void __launch_bounds__(256, 5) gn_apply_kernel(GnSrc s, const float* __restrict__ scale,
                                                          const float* __restrict__ shift, int act, int chunk, int reverse,
                                                          T* y, int64_t ldy) {
  const int C = s.c0 + s.c1;
  const int tpr = C / V;
  const int rp = blockDim.x / tpr;
  const int cv = (threadIdx.x % tpr) * V;
  const int64_t r0 = (int64_t)((reverse & 1) ? gridDim.x - 1 - blockIdx.x : blockIdx.x) * chunk;
  const int64_t r1 = min(r0 + (int64_t)chunk, s.rows);
  int b0;
  const bool uniform = chunk_is_uniform(s, r0, r1, b0) && !(reverse & 2);
  if ((int)threadIdx.x >= rp * tpr) return;
  const T* base = cv < s.c0 ? reinterpret_cast<const T*>(s.x0) + cv : reinterpret_cast<const T*>(s.x1) + (cv - s.c0);
  const int64_t ld = cv < s.c0 ? s.ld0 : s.ld1;
  T* yb = y + cv;
  float sc[V], sh[V];
  auto norm_act = [&](float* f) {
    if (act == 1) {
#pragma unroll
      for (int i = 0; i < V; ++i) f[i] = FastAct<T>::silu(fmaf(f[i], sc[i], sh[i]));
    } else if (act == 2) {                                 // exact (erf) GELU = torch.nn.GELU() of the VAE heads
#pragma unroll
      for (int i = 0; i < V; ++i) {
        const float v = fmaf(f[i], sc[i], sh[i]);
        f[i] = 0.5f * v * (1.0f + erff(v * 0.70710678118654752f));
      }
    } else {
#pragma unroll
      for (int i = 0; i < V; ++i) f[i] = fmaf(f[i], sc[i], sh[i]);
    }
  };
  int64_t r = r0 + threadIdx.x / tpr;
  if (uniform) {
#pragma unroll
    for (int i = 0; i < V; ++i) { sc[i] = scale[(int64_t)b0 * C + cv + i]; sh[i] = shift[(int64_t)b0 * C + cv + i]; }
    for (; r + (GN_UNROLL - 1) * rp < r1; r += GN_UNROLL * rp) {
      float f[GN_UNROLL][V];
#pragma unroll
      for (int u = 0; u < GN_UNROLL; ++u) load_vec<T, V>(base + (r + u * rp) * ld, f[u]);
#pragma unroll
      for (int u = 0; u < GN_UNROLL; ++u) {
        norm_act(f[u]);
        store_vec<T, V>(yb + (r + u * rp) * ldy, f[u]);
      }
    }
    for (; r < r1; r += rp) {
      float f[V];
      load_vec<T, V>(base + r * ld, f);
      norm_act(f);
      store_vec<T, V>(yb + r * ldy, f);
    }
    return;
  }
  int cur_b = -1;
  for (; r < r1; r += rp) {
    const int b = s.sample_id ? s.sample_id[r] : (int)(r / s.rows_per_sample);
    if (b != cur_b) {
      cur_b = b;
#pragma unroll
      for (int i = 0; i < V; ++i) { sc[i] = scale[(int64_t)b * C + cv + i]; sh[i] = shift[(int64_t)b * C + cv + i]; }
    }
    float f[V];
    load_vec<T, V>(base + r * ld, f);
    norm_act(f);
    store_vec<T, V>(yb + r * ldy, f);
  }
}

static bool vec_ok(const void* p, int64_t ld, int c, int v, int esz) {
  if (p == nullptr) return true;
  return (c % v == 0) && (ld % v == 0) && ((reinterpret_cast<uintptr_t>(p) % (v * esz)) == 0);
}

// rows per CTA: a fixed number of BYTES per CTA (so that every thread streams enough rows to amortise the
// prologue/epilogue latency chain), at least 256 rows.  OCTFUSION_GN_CHUNK_KB overrides (experiments).
static int gn_chunk_rows(int C, int esz) {
  static int kb = -1;
  if (kb < 0) { const char* e = getenv("OCTFUSION_GN_CHUNK_KB"); kb = e ? atoi(e) : 64; }
  int64_t rows = ((int64_t)kb * 1024) / ((int64_t)C * esz);
  rows = (rows / 256) * 256;
  return (int)(rows < 256 ? 256 : rows);
}

static int check_src(const GnSrc& s, const char* who) {
  OF_REQUIRE(s.x0 != nullptr && s.c0 > 0, "%s: x0/c0 missing", who);
  OF_REQUIRE((s.x1 == nullptr) == (s.c1 == 0), "%s: x1/c1 inconsistent", who);
  OF_REQUIRE(s.sample_id != nullptr || s.rows_per_sample > 0, "%s: need sample_id or rows_per_sample", who);
  OF_REQUIRE(s.rows >= 0, "%s: negative rows", who);
  return OF_OK;
}

}  // namespace of

extern "C" int of_gn_stats(const void* x0, int64_t ld0, int32_t c0, const void* x1, int64_t ld1, int32_t c1,
                           const int32_t* chunk_seg, const int32_t* seg_slot, const int32_t* sample_id,
                           int32_t rows_per_sample, int64_t rows, int32_t dtype, int32_t gran, float* part, void* stream) {
  using namespace of;
  GnSrc s{x0, ld0, c0, x1, ld1, c1, sample_id, rows_per_sample, rows};
  int rc = check_src(s, "of_gn_stats");
  if (rc) return rc;
  const int C = c0 + c1;
  OF_REQUIRE(chunk_seg != nullptr && seg_slot != nullptr && part != nullptr, "of_gn_stats: null chunk_seg/seg_slot/part");
  OF_REQUIRE(dtype == OF_F32 || dtype == OF_BF16, "of_gn_stats: bad dtype");
  OF_REQUIRE(gran == 2 || gran == 4, "of_gn_stats: gran must be 2 or 4");
  const int esz = dtype == OF_F32 ? 4 : 2;
  int V = dtype == OF_F32 ? 4 : 8;
  if (V == 8 && !(C % 8 == 0 && vec_ok(x0, ld0, c0, 8, 2) && vec_ok(x1, ld1, c1, 8, 2))) V = 4;
  OF_REQUIRE(C % V == 0 && c0 % V == 0, "of_gn_stats: channel counts must be multiples of %d (C=%d c0=%d)", V, C, c0);
  OF_REQUIRE(vec_ok(x0, ld0, c0, V, esz) && vec_ok(x1, ld1, c1, V, esz),
             "of_gn_stats: x0/x1 must be %d-byte aligned with ld %% %d == 0", V * esz, V);
  if (rows == 0) return OF_OK;
  const int64_t chunks = (rows + 31) / 32;
  const int64_t threads = chunks * (C / V);
  const int grid = (int)((threads + 255) / 256);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
#define OF_GN_STATS(T, VV)                                                                     \
  do {                                                                                         \
    if (gran == 4) gn_stats_kernel<T, VV, 4><<<grid, 256, 0, st>>>(s, chunk_seg, seg_slot, part);        \
    else gn_stats_kernel<T, VV, 2><<<grid, 256, 0, st>>>(s, chunk_seg, seg_slot, part);                  \
  } while (0)
  if (dtype == OF_F32) OF_GN_STATS(float, 4);
  else if (V == 8) OF_GN_STATS(__nv_bfloat16, 8);
  else OF_GN_STATS(__nv_bfloat16, 4);
#undef OF_GN_STATS
  OF_LAUNCH_CHECK("of_gn_stats");
  return OF_OK;
}

extern "C" int of_gn_finalize(const float* part0, int32_t c0, int32_t gran0, const float* part1, int32_t c1,
                              int32_t gran1, const int32_t* sample_seg_off, int32_t n_segments,
                              const int32_t* rows_of_sample, int32_t rows_per_sample, const float* gamma,
                              const float* beta, int32_t batch, int32_t groups, float eps, float count_eps,
                              float* scale, float* shift, double* scratch, int32_t* ticket, void* stream) {
  using namespace of;
  OF_REQUIRE(part0 && gamma && beta && scale && shift && sample_seg_off, "of_gn_finalize: null pointer");
  OF_REQUIRE((part1 == nullptr) == (c1 == 0), "of_gn_finalize: part1/c1 inconsistent");
  OF_REQUIRE((gran0 == 2 || gran0 == 4) && (c1 == 0 || gran1 == 2 || gran1 == 4), "of_gn_finalize: granules must be 2 or 4");
  if (c1 == 0) gran1 = gran0;
  const int C = c0 + c1;
  OF_REQUIRE(groups > 0 && C % groups == 0, "of_gn_finalize: C=%d not divisible by groups=%d", C, groups);
  const int cpg = C / groups;
  OF_REQUIRE(cpg % gran0 == 0 && c0 % gran0 == 0 && (c1 == 0 || (cpg % gran1 == 0 && c1 % gran1 == 0 && c0 % gran1 == 0)),
             "of_gn_finalize: C=%d groups=%d c0=%d: channels per group and c0 must be multiples of the granules (%d, %d)",
             C, groups, c0, gran0, gran1);
  OF_REQUIRE(rows_of_sample != nullptr || rows_per_sample > 0, "of_gn_finalize: need a row count");
  OF_REQUIRE(batch > 0 && n_segments >= 0, "of_gn_finalize: bad batch / n_segments");
  const int nval = c0 / gran0 * 2 + (c1 > 0 ? c1 / gran1 * 2 : 0);
  OF_REQUIRE(nval <= 1024, "of_gn_finalize: C=%d too wide", C);
  const int slices = 1024 / nval;
  const int threads = slices * nval;
  // CTAs per sample: ~128 slots each, at most OF_GN_FINALIZE_SPLIT; more than one needs the scratch rows and tickets
  int S = (n_segments / batch + 127) / 128;
  S = S < 1 ? 1 : (S > OF_GN_FINALIZE_SPLIT ? OF_GN_FINALIZE_SPLIT : S);
  if (scratch == nullptr || ticket == nullptr) S = 1;
  const size_t smem = ((size_t)slices * nval + nval) * sizeof(double);
  gn_finalize_kernel<<<dim3(batch, S), threads, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
      part0, c0, gran0, part1, c1, gran1, sample_seg_off, rows_of_sample, rows_per_sample, gamma, beta, groups, eps,
      count_eps, scale, shift, scratch, ticket);
  OF_LAUNCH_CHECK("of_gn_finalize");
  return OF_OK;
}

extern "C" int of_gn_apply(const void* x0, int64_t ld0, int32_t c0, const void* x1, int64_t ld1, int32_t c1,
                           const int32_t* sample_id, int32_t rows_per_sample, int64_t rows, const float* scale,
                           const float* shift, int32_t act, int32_t dtype, void* y, int64_t ldy, int32_t reverse,
                           void* stream) {
  using namespace of;
  GnSrc s{x0, ld0, c0, x1, ld1, c1, sample_id, rows_per_sample, rows};
  int rc = check_src(s, "of_gn_apply");
  if (rc) return rc;
  OF_REQUIRE(scale && shift && y, "of_gn_apply: null pointer");
  OF_REQUIRE(dtype == OF_F32 || dtype == OF_BF16, "of_gn_apply: bad dtype");
  if (rows == 0) return OF_OK;
  const int C = c0 + c1;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
#define OF_GN_APPLY_LAUNCH(T, V)                                                              \
  do {                                                                                        \
    OF_REQUIRE(C / V <= 256, "of_gn_apply: C=%d too wide", C);                                \
    int chunk = gn_chunk_rows(C, (int)sizeof(T));                                             \
    {                                                                                         \
      /* small tensors (the dense 4^3 / 8^3 levels: 2048 / 16384 rows): rather 4 CTAs per SM with one or two     \
         passes each than a handful of CTAs walking 256 rows -- those launches were latency-bound at 30 us */   \
      const int rp = 256 / (C / V);                                                           \
      int64_t want = (rows + 4 * num_sms() - 1) / (4 * num_sms());                            \
      want = (want + rp - 1) / rp * rp;                                                       \
      if (want < chunk) chunk = (int)want;                                                    \
    }                                                                                         \
    const int grid = (int)((rows + chunk - 1) / chunk);                                       \
    gn_apply_kernel<T, V><<<grid, 256, 0, st>>>(s, scale, shift, act, chunk, reverse, reinterpret_cast<T*>(y), ldy); \
  } while (0)
  if (dtype == OF_F32) {
    if (vec_ok(x0, ld0, c0, 4, 4) && vec_ok(x1, ld1, c1, 4, 4) && vec_ok(y, ldy, C, 4, 4)) OF_GN_APPLY_LAUNCH(float, 4);
    else OF_GN_APPLY_LAUNCH(float, 1);
  } else {
    if (vec_ok(x0, ld0, c0, 8, 2) && vec_ok(x1, ld1, c1, 8, 2) && vec_ok(y, ldy, C, 8, 2)) OF_GN_APPLY_LAUNCH(__nv_bfloat16, 8);
    else OF_GN_APPLY_LAUNCH(__nv_bfloat16, 1);
  }
#undef OF_GN_APPLY_LAUNCH
  OF_LAUNCH_CHECK("of_gn_apply");
  return OF_OK;
}
