// Tap-gather GEMM on the CUDA cores (FFMA): the any-shape, fp32-accumulate path.
//
//   out[m,:] = sum_tap mean_{j in nbr(m,tap)} [A[j,:] | onehot(type_j)] . W[tap]  (+bias +row_add +resid)
//
// Replaces, for shapes the tensor-core kernel does not take (fp32 activations, Cin = 3, Cout = 3,
// the [B,512] embedding MLPs) the reference op sequence  x[col] -> scatter_mean -> view @ W
// (reference models/networks/modules.py:194-220, diffusion_networks/utils/scatter.py:42-66),
// nn.Linear / Conv1x1 (modules.py:332-339) and dense Conv3d (modules.py:493-502) in fp32 mode.
//
// Tiling: 64x64 output tile per CTA, K step 16, 256 threads, 4x4 register tile per thread.
// The A tile is *built* (gathered + averaged) straight into shared memory, so the
// [7N, C] im2col buffer the reference materialises (47 % of its run time) never exists.
#include "common.cuh"

namespace of {

template <typename T>
__device__ __forceinline__ float load_feat(const of_gemm_args& p, int src, int c) {
  float v;
  if (c < p.c0) {
    v = Elem<T>::ld(reinterpret_cast<const T*>(p.a0) + (int64_t)src * p.lda0 + c);
  } else if (c < p.c0 + p.c1) {
    v = Elem<T>::ld(reinterpret_cast<const T*>(p.a1) + (int64_t)src * p.lda1 + (c - p.c0));
  } else {
    return p.node_type[src] == (uint8_t)(c - p.c0 - p.c1) ? 1.0f : 0.0f;
  }
  return p.a_silu ? silu_f(v) : v;
}

template <typename T>
__device__ __forceinline__ float load_a(const of_gemm_args& p, int m, int tap, int c) {
  if (p.tap_tab == nullptr) {
    int src = p.in_rows ? p.in_rows[m] : m;
    return src < 0 ? 0.0f : load_feat<T>(p, src, c);
  }
  int t = p.tap_tab[(int64_t)m * p.taps + tap];
  if (t == -1) return 0.0f;
  if (t >= 0) return load_feat<T>(p, t, c);
  const int32_t* e = p.tap_extra + (-(t + 2));
  int n = e[0];
  float s = 0.0f;
  for (int i = 1; i <= n; ++i) s += load_feat<T>(p, e[i], c);
  return s / (float)n;
}

constexpr int SBM = 64, SBN = 64, SBK = 16;

template <typename T>
__global__ void __launch_bounds__(256) gather_gemm_simt_kernel(const of_gemm_args p) {
  __shared__ float As[SBK][SBM + 4];
  __shared__ float Bs[SBK][SBN + 4];
  const int tid = threadIdx.x;
  const int tile_m = blockIdx.x * SBM, tile_n = blockIdx.y * SBN;
  const int ty = tid >> 4, tx = tid & 15;
  const int cp = p.c0 + p.c1 + p.ntype;
  const int K = p.taps * cp;
  const float* __restrict__ W = reinterpret_cast<const float*>(p.w);
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;

  const int ar = tid >> 2, akq = (tid & 3) * 4;       // A build: row, first k of 4
  const int bk = tid >> 4, bn = (tid & 15) * 4;       // B load: k row, first n of 4
  for (int k0 = 0; k0 < K; k0 += SBK) {
    {
      const int m = tile_m + ar;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int k = k0 + akq + j;
        float v = 0.0f;
        if (m < p.M && k < K) {
          const int tap = k / cp;
          v = load_a<T>(p, m, tap, k - tap * cp);
        }
        As[akq + j][ar] = v;
      }
    }
    {
      const int k = k0 + bk;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int n = tile_n + bn + j;
        Bs[bk][bn + j] = (k < K && n < p.N) ? W[(int64_t)k * p.N + n] : 0.0f;
      }
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < SBK; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }

#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = tile_m + ty * 4 + i;
    if (m >= p.M) continue;
    const int64_t orow = p.out_rows ? p.out_rows[m] : m;
    const float* radd = p.row_add ? p.row_add + (int64_t)p.row_add_idx[m] * p.ld_row_add : nullptr;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = tile_n + tx * 4 + j;
      if (n >= p.N) continue;
      float v = acc[i][j];
      if (p.bias) v += p.bias[n];
      if (radd) v += radd[n];
      if (p.resid) v += Elem<T>::ld(reinterpret_cast<const T*>(p.resid) + (int64_t)m * p.ld_resid + n);
      if (p.out_f32) reinterpret_cast<float*>(p.out)[orow * p.ldo + n] = v;
      else Elem<T>::st(reinterpret_cast<T*>(p.out) + orow * p.ldo + n, v);
    }
  }
}

int check_gemm_args(const of_gemm_args* a, const char* who) {
  OF_REQUIRE(a != nullptr, "%s: null args", who);
  OF_REQUIRE(a->M >= 0 && a->N > 0, "%s: bad M/N (%d, %d)", who, a->M, a->N);
  OF_REQUIRE(a->a0 != nullptr && a->c0 > 0, "%s: a0/c0 missing", who);
  OF_REQUIRE((a->a1 == nullptr) == (a->c1 == 0), "%s: a1/c1 inconsistent", who);
  OF_REQUIRE(a->taps >= 1, "%s: taps must be >= 1", who);
  OF_REQUIRE(a->tap_tab != nullptr || a->taps == 1, "%s: identity mode needs taps == 1", who);
  OF_REQUIRE(a->tap_tab == nullptr || a->in_rows == nullptr, "%s: in_rows only in identity mode", who);
  OF_REQUIRE((a->ntype == 0) || (a->node_type != nullptr), "%s: ntype > 0 needs node_type", who);
  OF_REQUIRE(a->w != nullptr && a->out != nullptr, "%s: w/out missing", who);
  OF_REQUIRE((a->row_add == nullptr) == (a->row_add_idx == nullptr), "%s: row_add needs row_add_idx", who);
  OF_REQUIRE(a->dtype == OF_F32 || a->dtype == OF_BF16, "%s: bad dtype %d", who, a->dtype);
  return OF_OK;
}

}  // namespace of

extern "C" int of_gather_gemm_simt(const of_gemm_args* args, void* stream) {
  int rc = of::check_gemm_args(args, "of_gather_gemm_simt");
  if (rc) return rc;
  if (args->stat_out != nullptr) {
    of::set_error("of_gather_gemm_simt: stat_out is a tensor-core-path feature (run of_gn_stats on the output instead)");
    return OF_E_UNSUPPORTED;
  }
  if (args->M == 0) return OF_OK;
  dim3 grid((args->M + of::SBM - 1) / of::SBM, (args->N + of::SBN - 1) / of::SBN);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (args->dtype == OF_F32)
    of::gather_gemm_simt_kernel<float><<<grid, 256, 0, s>>>(*args);
  else
    of::gather_gemm_simt_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(*args);
  OF_LAUNCH_CHECK("of_gather_gemm_simt");
  return OF_OK;
}
