// Point-cloud shape metrics: nearest-neighbour (Chamfer) distances and the approximate EMD of the OctFusion
// evaluation (reference metrics/evaluation_metrics.py, backed by metrics/pytorch_structural_losses/src/
// nndistance.cu and approxmatch.cu).
//
// Everything is fp32 on the CUDA cores plus ex2 / sqrt on the SFU.  No tensor cores: the |x|^2 + |y|^2 - 2 x.y
// expansion cancels exactly on the small nearest-neighbour distances the metrics are made of.  The squared distance
// is the reference's expression on (b - a) differences with the same FMA contraction (see sqdist), so per-point
// minima are bit-identical to nndistance.  No float atomics: the only atomics are integer minima of non-negative
// float bit patterns, which do not depend on order; every sum has a fixed order.
//
// chamfer_kernel   one CTA per cloud pair; 16 x 16 threads, each owning 8 rows (points of a) x 8 columns (points of
//                  b) of a 128 x 128 distance tile.  Row minima stay in registers over all column tiles and are
//                  reduced across the 16 column threads by shuffles; column minima are reduced by one shuffle and
//                  an integer atomicMin per tile into shared memory (all-pairs mode) or into dist2 (paired mode).
// emd_cd_kernel    one CTA per cloud pair on a persistent grid.  Both clouds, remainL / remainR / ratioL / ratioR
//                  are resident in shared memory; the 9 levels x 3 passes of approxmatch run inside the CTA.  The
//                  cost sum_level sum_kl w_kl * sqrt(d_kl) is accumulated on the fly (the reference's cost is linear
//                  in its match matrix), so no match matrix exists.  The CD of the pair is folded into the row pass
//                  (dist1) and the column pass (dist2) of the first level, which already compute every distance.
#include "common.cuh"

namespace of {

constexpr unsigned kInfBits = 0x7f800000u;

// |b - a|^2 exactly as nvcc contracts the reference's dx*dx+dy*dy+dz*dz (NmDistanceKernel, approxmatchkernel):
// fma(dz, dz, fma(dx, dx, dy * dy))
__device__ __forceinline__ float sqdist(float ax, float ay, float az, float bx, float by, float bz) {
  const float dx = __fsub_rn(bx, ax), dy = __fsub_rn(by, ay), dz = __fsub_rn(bz, az);
  return __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
}

// exp(level * d) as ex2(d * (level * log2 e)).  level is a power of 4, so d * (level * log2 e) rounds exactly like the
// reference's (level * d) * log2 e inside __expf.  Unlike __expf this flushes results below 2^-126 to zero: such a
// term is below the last bit of every sum it enters (sums start at 1e-9 or add to a remainder up to 1).
__device__ __forceinline__ float exp2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ float sqrt_approx(float x) {
  float y;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// fixed-order block sum of one value per thread (warp shuffles, then the warps in order); result in every thread
template <int THREADS>
__device__ __forceinline__ float block_sum(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.0f;
#pragma unroll
  for (int w = 0; w < THREADS / 32; ++w) s += red[w];
  __syncthreads();
  return s;
}

// pair p -> (cloud of a, cloud of b): paired mode (a_p, b_p) or all pairs (a_{p / nb}, b_{p % nb})
__device__ __forceinline__ void pair_clouds(int64_t p, int64_t nb, bool paired, int64_t& ia, int64_t& ib) {
  ia = paired ? p : p / nb;
  ib = paired ? p : p % nb;
}

// ------------------------------------------------------------------------------------------------------------------
// Chamfer / nearest-neighbour distances
// ------------------------------------------------------------------------------------------------------------------
constexpr int CD_THREADS = 256, CD_T = 8, CD_TILE = 16 * CD_T;      // 128 x 128 tile, 8 x 8 per thread

template <bool PAIRED>
__global__ void __launch_bounds__(CD_THREADS) chamfer_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                             int64_t pairs, int64_t nb, int P, int Q,
                                                             float* __restrict__ dist1, float* __restrict__ dist2,
                                                             float* __restrict__ cd) {
  extern __shared__ unsigned cd_mins[];             // all-pairs mode: row minima [P], column minima [Q]
  __shared__ float4 tb[CD_TILE];
  __shared__ float red[CD_THREADS / 32];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4, lane = tid & 31;
  const float inf = __int_as_float(kInfBits);
  for (int64_t p = blockIdx.x; p < pairs; p += gridDim.x) {
    int64_t ia, ib;
    pair_clouds(p, nb, PAIRED, ia, ib);
    const float* pa = a + ia * P * 3;
    const float* pb = b + ib * Q * 3;
    unsigned* rmin = PAIRED ? reinterpret_cast<unsigned*>(dist1 + p * P) : cd_mins;
    unsigned* cmin = PAIRED ? reinterpret_cast<unsigned*>(dist2 + p * Q) : cd_mins + P;
    for (int l = tid; l < Q; l += CD_THREADS) cmin[l] = kInfBits;
    for (int a0 = 0; a0 < P; a0 += CD_TILE) {
      // padding points sit at +inf: their distance to any real point is +inf (or NaN between two padding points,
      // which fminf ignores), so they never lower a real minimum
      float ax[CD_T], ay[CD_T], az[CD_T], rm[CD_T];
#pragma unroll
      for (int r = 0; r < CD_T; ++r) {
        const int k = a0 + r * 16 + ty;
        ax[r] = k < P ? pa[3 * k + 0] : inf;
        ay[r] = k < P ? pa[3 * k + 1] : inf;
        az[r] = k < P ? pa[3 * k + 2] : inf;
        rm[r] = inf;
      }
      for (int b0 = 0; b0 < Q; b0 += CD_TILE) {
        __syncthreads();                                   // previous tile consumed, cmin initialised
        if (tid < CD_TILE) {
          const int l = b0 + tid;
          tb[tid] = l < Q ? make_float4(pb[3 * l + 0], pb[3 * l + 1], pb[3 * l + 2], 0.0f) : make_float4(inf, inf, inf, 0.0f);
        }
        __syncthreads();
        float cm[CD_T];
#pragma unroll
        for (int c = 0; c < CD_T; ++c) {
          const float4 q = tb[c * 16 + tx];
          cm[c] = inf;
#pragma unroll
          for (int r = 0; r < CD_T; ++r) {
            const float d = sqdist(ax[r], ay[r], az[r], q.x, q.y, q.z);
            rm[r] = fminf(rm[r], d);
            cm[c] = fminf(cm[c], d);
          }
        }
        // a warp holds rows ty = 2w, 2w+1 of the same 16 columns: one shuffle, then one atomic per column and warp
#pragma unroll
        for (int c = 0; c < CD_T; ++c) {
          const float o = __shfl_xor_sync(0xffffffffu, cm[c], 16);
          const int l = b0 + c * 16 + tx;
          if (lane < 16 && l < Q) atomicMin(&cmin[l], __float_as_uint(fminf(cm[c], o)));
        }
      }
#pragma unroll
      for (int r = 0; r < CD_T; ++r) {
        float v = rm[r];
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
        const int k = a0 + r * 16 + ty;
        if (tx == 0 && k < P) rmin[k] = __float_as_uint(v);
      }
    }
    __syncthreads();
    if (cd != nullptr) {
      float s1 = 0.0f, s2 = 0.0f;
      for (int k = tid; k < P; k += CD_THREADS) s1 += __uint_as_float(rmin[k]);
      for (int l = tid; l < Q; l += CD_THREADS) s2 += __uint_as_float(cmin[l]);
      s1 = block_sum<CD_THREADS>(s1, red);
      s2 = block_sum<CD_THREADS>(s2, red);
      if (tid == 0) cd[p] = s1 / (float)P + s2 / (float)Q;
    }
    __syncthreads();                                       // minima read before the next pair resets them
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Approximate EMD (approxmatch + matchcost) fused with the CD of the same pair
// ------------------------------------------------------------------------------------------------------------------
constexpr int EMD_THREADS = 512, EMD_R = 4, EMD_SPAN = EMD_THREADS * EMD_R;   // points owned per thread per sweep

struct EmdSmem {
  float4* sa;       // [n] a: x, y, z, ratioL
  float4* sb;       // [n] b: x, y, z, remainR
  float* remL;      // [n]
  float* ratR;      // [n]
};

__host__ __device__ constexpr size_t emd_smem_bytes(int n) { return (size_t)n * (2 * sizeof(float4) + 2 * sizeof(float)); }

// pass 1: ratioL[k] = remainL[k] / (1e-9 + sum_l exp(level d_kl) remainR[l])   (+ dist1 on the first level)
// pass 2: per column l: sumr = remainR[l] * sum_k exp(level d_kl) ratioL[k], then ratioR / remainR   (+ dist2)
// pass 3: w_kl = exp(level d_kl) ratioL[k] ratioR[l]; remainL[k] -= sum_l w_kl; cost += w_kl sqrt(d_kl)
//         (ratioL[k] is factored out of both row sums)
// Each thread sums over the other cloud in index order, like the reference's per-thread loops.
template <int PASS, bool CD>
__device__ __forceinline__ void emd_pass(const EmdSmem& s, int n, float level, float& cost, float& cdsum) {
  const float c = level * 1.44269504f;
  const int tid = threadIdx.x;
  const float4* own = PASS == 2 ? s.sb : s.sa;
  const float4* other = PASS == 2 ? s.sa : s.sb;
  for (int base = 0; base < n; base += EMD_SPAN) {
    if (base + (tid & ~31) >= n) break;                   // whole warp past the end (no barrier inside)
    float px[EMD_R], py[EMD_R], pz[EMD_R], acc[EMD_R], mn[EMD_R], rl[EMD_R], cst[EMD_R];
#pragma unroll
    for (int r = 0; r < EMD_R; ++r) {
      const int i = min(base + r * EMD_THREADS + tid, n - 1);
      const float4 q = own[i];
      px[r] = q.x; py[r] = q.y; pz[r] = q.z;
      rl[r] = q.w;
      acc[r] = PASS == 1 ? 1e-9f : 0.0f;
      mn[r] = __int_as_float(kInfBits);
      cst[r] = 0.0f;
    }
#pragma unroll 2
    for (int l = 0; l < n; ++l) {
      const float4 q = other[l];
      const float wq = PASS == 3 ? s.ratR[l] : q.w;
#pragma unroll
      for (int r = 0; r < EMD_R; ++r) {
        const float d = PASS == 2 ? sqdist(q.x, q.y, q.z, px[r], py[r], pz[r]) : sqdist(px[r], py[r], pz[r], q.x, q.y, q.z);
        if (CD) mn[r] = fminf(mn[r], d);
        const float w = exp2_approx(d * c) * wq;
        acc[r] += w;
        if (PASS == 3) cst[r] = fmaf(w, sqrt_approx(d), cst[r]);
      }
    }
#pragma unroll
    for (int r = 0; r < EMD_R; ++r) {
      const int i = base + r * EMD_THREADS + tid;
      if (i >= n) continue;
      if (PASS == 3) cost += cst[r] * rl[r];               // per (row, level) partial: short fp32 sum chains
      if (CD) cdsum += mn[r];
      if (PASS == 1) {
        s.sa[i].w = s.remL[i] / acc[r];
      } else if (PASS == 2) {
        const float remR = rl[r];
        const float sumr = acc[r] * remR;
        const float consumption = fminf(remR / (sumr + 1e-9f), 1.0f);
        s.ratR[i] = consumption * remR;
        s.sb[i].w = fmaxf(0.0f, remR - sumr);
      } else {
        s.remL[i] = fmaxf(0.0f, s.remL[i] - acc[r] * rl[r]);
      }
    }
  }
}

__global__ void __launch_bounds__(EMD_THREADS, 2) emd_cd_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                                int64_t pairs, int64_t nb, int paired, int n,
                                                                float* __restrict__ cost_out, float* __restrict__ cd_out) {
  extern __shared__ float4 emd_smem[];
  __shared__ float red[EMD_THREADS / 32];
  EmdSmem s;
  s.sa = emd_smem;
  s.sb = s.sa + n;
  s.remL = reinterpret_cast<float*>(s.sb + n);
  s.ratR = s.remL + n;
  const int tid = threadIdx.x;
  for (int64_t p = blockIdx.x; p < pairs; p += gridDim.x) {
    int64_t ia, ib;
    pair_clouds(p, nb, paired != 0, ia, ib);
    const float* pa = a + ia * n * 3;
    const float* pb = b + ib * n * 3;
    for (int k = tid; k < n; k += EMD_THREADS) {          // n == m: multiL = multiR = 1
      s.sa[k] = make_float4(pa[3 * k + 0], pa[3 * k + 1], pa[3 * k + 2], 0.0f);
      s.sb[k] = make_float4(pb[3 * k + 0], pb[3 * k + 1], pb[3 * k + 2], 1.0f);
      s.remL[k] = 1.0f;
    }
    __syncthreads();
    float cost = 0.0f, cd1 = 0.0f, cd2 = 0.0f;
    // levels -4^7 ... -4^-1 (the reference's loop j = 7 .. -1; powers of 4 are exact)
    emd_pass<1, true>(s, n, -16384.0f, cost, cd1);
    __syncthreads();
    emd_pass<2, true>(s, n, -16384.0f, cost, cd2);
    __syncthreads();
    emd_pass<3, false>(s, n, -16384.0f, cost, cd1);
    __syncthreads();
    for (int j = 6; j >= -1; --j) {
      const float level = -ldexpf(1.0f, 2 * j);
      emd_pass<1, false>(s, n, level, cost, cd1);
      __syncthreads();
      emd_pass<2, false>(s, n, level, cost, cd2);
      __syncthreads();
      emd_pass<3, false>(s, n, level, cost, cd1);
      __syncthreads();
    }
    cost = block_sum<EMD_THREADS>(cost, red);
    cd1 = block_sum<EMD_THREADS>(cd1, red);
    cd2 = block_sum<EMD_THREADS>(cd2, red);
    if (tid == 0) {
      cost_out[p] = cost;
      if (cd_out != nullptr) cd_out[p] = cd1 / (float)n + cd2 / (float)n;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------------
static int persistent_grid(const void* kernel, int threads, size_t smem, int64_t pairs) {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
  const int64_t slots = (int64_t)per_sm * num_sms();
  return (int)(pairs < slots ? pairs : slots);
}

static int launch_chamfer(const float* a, const float* b, int64_t pairs, int64_t nb, bool paired, int P, int Q,
                          float* dist1, float* dist2, float* cd, void* stream, const char* who) {
  const size_t smem = paired ? 0 : (size_t)(P + Q) * sizeof(unsigned);
  const void* k = paired ? (const void*)chamfer_kernel<true> : (const void*)chamfer_kernel<false>;
  if (smem > 48 * 1024 && cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
    set_error("%s: cannot reserve %zu bytes of shared memory", who, smem);
    return OF_E_CUDA;
  }
  const int grid = persistent_grid(k, CD_THREADS, smem, pairs);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (paired) chamfer_kernel<true><<<grid, CD_THREADS, smem, st>>>(a, b, pairs, nb, P, Q, dist1, dist2, cd);
  else chamfer_kernel<false><<<grid, CD_THREADS, smem, st>>>(a, b, pairs, nb, P, Q, dist1, dist2, cd);
  OF_LAUNCH_CHECK(who);
  return OF_OK;
}

static int launch_emd(const float* a, const float* b, int64_t pairs, int64_t nb, bool paired, int n, float* cost,
                      float* cd, void* stream, const char* who) {
  const size_t smem = emd_smem_bytes(n);
  if (cudaFuncSetAttribute(emd_cd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
    set_error("%s: cannot reserve %zu bytes of shared memory", who, smem);
    return OF_E_CUDA;
  }
  const int grid = persistent_grid((const void*)emd_cd_kernel, EMD_THREADS, smem, pairs);
  emd_cd_kernel<<<grid, EMD_THREADS, smem, reinterpret_cast<cudaStream_t>(stream)>>>(a, b, pairs, nb, paired ? 1 : 0, n,
                                                                                   cost, cd);
  OF_LAUNCH_CHECK(who);
  return OF_OK;
}

static_assert(emd_smem_bytes(OF_EMD_MAX_POINTS) <= 227 * 1024, "EMD working set must fit one SM's shared memory");
static_assert((size_t)OF_CD_PAIRWISE_MAX_POINTS * sizeof(unsigned) + CD_TILE * sizeof(float4) + 64 <= 227 * 1024,
              "pairwise Chamfer minima must fit one SM's shared memory");

}  // namespace of

extern "C" int of_nn_distance(const float* a, const float* b, int32_t batch, int32_t P, int32_t Q, float* dist1,
                              float* dist2, float* cd, void* stream) {
  using namespace of;
  OF_REQUIRE(a && b && dist1 && dist2, "of_nn_distance: null pointer");
  OF_REQUIRE(batch >= 0 && P >= 1 && Q >= 1, "of_nn_distance: need batch >= 0, P >= 1, Q >= 1 (got %d, %d, %d)", batch, P, Q);
  if (batch == 0) return OF_OK;
  return launch_chamfer(a, b, batch, 1, true, P, Q, dist1, dist2, cd, stream, "of_nn_distance");
}

extern "C" int of_chamfer_pairwise(const float* a, int32_t na, int32_t P, const float* b, int32_t nb, int32_t Q, float* cd,
                                   void* stream) {
  using namespace of;
  OF_REQUIRE(a && b && cd, "of_chamfer_pairwise: null pointer");
  OF_REQUIRE(na >= 0 && nb >= 0 && P >= 1 && Q >= 1, "of_chamfer_pairwise: need na, nb >= 0 and P, Q >= 1");
  OF_REQUIRE((int64_t)P + Q <= OF_CD_PAIRWISE_MAX_POINTS, "of_chamfer_pairwise: P + Q = %lld exceeds %d",
             (long long)P + Q, OF_CD_PAIRWISE_MAX_POINTS);
  if ((int64_t)na * nb == 0) return OF_OK;
  return launch_chamfer(a, b, (int64_t)na * nb, nb, false, P, Q, nullptr, nullptr, cd, stream, "of_chamfer_pairwise");
}

extern "C" int of_match_cost(const float* a, const float* b, int32_t batch, int32_t n, float* cost, float* cd,
                             void* stream) {
  using namespace of;
  OF_REQUIRE(a && b && cost, "of_match_cost: null pointer");
  OF_REQUIRE(batch >= 0 && n >= 1 && n <= OF_EMD_MAX_POINTS, "of_match_cost: need batch >= 0 and 1 <= n <= %d (got %d, %d)",
             OF_EMD_MAX_POINTS, batch, n);
  if (batch == 0) return OF_OK;
  return launch_emd(a, b, batch, 1, true, n, cost, cd, stream, "of_match_cost");
}

extern "C" int of_emd_cd_pairwise(const float* a, int32_t na, const float* b, int32_t nb, int32_t n, float* cost, float* cd,
                                  void* stream) {
  using namespace of;
  OF_REQUIRE(a && b && cost && cd, "of_emd_cd_pairwise: null pointer");
  OF_REQUIRE(na >= 0 && nb >= 0 && n >= 1 && n <= OF_EMD_MAX_POINTS,
             "of_emd_cd_pairwise: need na, nb >= 0 and 1 <= n <= %d (got n = %d)", OF_EMD_MAX_POINTS, n);
  if ((int64_t)na * nb == 0) return OF_OK;
  return launch_emd(a, b, (int64_t)na * nb, nb, false, n, cost, cd, stream, "of_emd_cd_pairwise");
}
