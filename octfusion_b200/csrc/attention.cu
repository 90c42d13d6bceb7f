// QKVAttention.forward (reference models/networks/modules.py:538-547) over the dense voxel
// tokens of the LR middle U-Net: T in {512, 64, 8} tokens per shape, ch in {16, 32, 64, 128}.
// The reference materialises the [b*h, T, T] fp32 score tensor (134 MB at B=32); here one CTA
// keeps K and V of one (shape, head) in shared memory and streams the queries through it --
// scores never leave the SM.  <0.2 % of the step FLOPs (SURVEY.md section 0).  Two kernels: a flash-style
// tensor-core kernel for bf16 activations (attention_tc_kernel below) and the CUDA-core fp32 kernel (fp32 activations,
// odd head widths) with fp32 softmax exactly as the reference (modules.py:546).
//
// qkv is channels-last [B*T, 3C] with the reference's legacy head-major split: head h owns
// columns [h*3ch, (h+1)*3ch) = q | k | v (modules.py:531,540-541).
#include "common.cuh"

namespace of {

constexpr int ATT_WARPS = 8;
constexpr int ATT_QTILE = 128;
constexpr int ATT_QB = 4;                 // queries processed together by one warp (register blocking)

template <typename T>
__global__ void __launch_bounds__(ATT_WARPS * 32) attention_kernel(const T* __restrict__ qkv, int64_t ld_qkv,
                                                                   T* __restrict__ out, int64_t ld_out, int tokens,
                                                                   int heads, int ch) {
  extern __shared__ __align__(16) float sm[];
  const int kst = ch + 4;                               // 16-byte aligned rows, conflict-free float4 column reads
  float* Ks = sm;                                       // [T][ch+4]
  float* Vs = Ks + (size_t)tokens * kst;                // [T][ch+4]
  float* Ps = Vs + (size_t)tokens * kst;                // [warps][T][QB]
  float* Qs = Ps + (size_t)ATT_WARPS * tokens * ATT_QB; // [warps][QB][ch]
  const int bh = blockIdx.x;
  const int b = bh / heads, h = bh - b * heads;
  const int64_t row0 = (int64_t)b * tokens;
  const int colq = h * 3 * ch, colk = colq + ch, colv = colq + 2 * ch;
  for (int i = threadIdx.x; i < tokens * ch; i += blockDim.x) {
    const int s = i / ch, c = i - s * ch;
    const T* r = qkv + (row0 + s) * ld_qkv;
    Ks[s * kst + c] = Elem<T>::ld(r + colk + c);
    Vs[s * kst + c] = Elem<T>::ld(r + colv + c);
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* P = Ps + (size_t)warp * tokens * ATT_QB;       // P[s][q]
  float* Q = Qs + (size_t)warp * ATT_QB * ch;           // Q[q][c]
  const float scale = rsqrtf((float)ch);                // (ch^-1/4)^2, modules.py:542-545
  const int q_end = min(tokens, (int)(blockIdx.y + 1) * ATT_QTILE);
  for (int t0 = blockIdx.y * ATT_QTILE + warp * ATT_QB; t0 < q_end; t0 += ATT_WARPS * ATT_QB) {
    const int nq = min(ATT_QB, q_end - t0);
    for (int i = lane; i < ATT_QB * ch; i += 32) {
      const int qi = i / ch, c = i - qi * ch;
      Q[i] = qi < nq ? Elem<T>::ld(qkv + (row0 + t0 + qi) * ld_qkv + colq + c) * scale : 0.0f;
    }
    __syncwarp();
    float mx[ATT_QB];
#pragma unroll
    for (int qi = 0; qi < ATT_QB; ++qi) mx[qi] = -INFINITY;
    for (int s = lane; s < tokens; s += 32) {
      const float4* kr = reinterpret_cast<const float4*>(Ks + s * kst);
      float d[ATT_QB];
#pragma unroll
      for (int qi = 0; qi < ATT_QB; ++qi) d[qi] = 0.0f;
      for (int c4 = 0; c4 < ch / 4; ++c4) {
        const float4 kv = kr[c4];
#pragma unroll
        for (int qi = 0; qi < ATT_QB; ++qi) {
          const float4 qv = reinterpret_cast<const float4*>(Q + qi * ch)[c4];
          d[qi] = fmaf(qv.x, kv.x, fmaf(qv.y, kv.y, fmaf(qv.z, kv.z, fmaf(qv.w, kv.w, d[qi]))));
        }
      }
      *reinterpret_cast<float4*>(P + s * ATT_QB) = make_float4(d[0], d[1], d[2], d[3]);
#pragma unroll
      for (int qi = 0; qi < ATT_QB; ++qi) mx[qi] = fmaxf(mx[qi], d[qi]);
    }
    float sum[ATT_QB];
#pragma unroll
    for (int qi = 0; qi < ATT_QB; ++qi) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx[qi] = fmaxf(mx[qi], __shfl_xor_sync(0xffffffffu, mx[qi], o));
      sum[qi] = 0.0f;
    }
    for (int s = lane; s < tokens; s += 32) {
      float4 pv = *reinterpret_cast<float4*>(P + s * ATT_QB);
      pv.x = __expf(pv.x - mx[0]); pv.y = __expf(pv.y - mx[1]); pv.z = __expf(pv.z - mx[2]); pv.w = __expf(pv.w - mx[3]);
      *reinterpret_cast<float4*>(P + s * ATT_QB) = pv;
      sum[0] += pv.x; sum[1] += pv.y; sum[2] += pv.z; sum[3] += pv.w;
    }
#pragma unroll
    for (int qi = 0; qi < ATT_QB; ++qi) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sum[qi] += __shfl_xor_sync(0xffffffffu, sum[qi], o);
    }
    __syncwarp();
    for (int c = lane; c < ch; c += 32) {
      float a[ATT_QB];
#pragma unroll
      for (int qi = 0; qi < ATT_QB; ++qi) a[qi] = 0.0f;
      for (int s = 0; s < tokens; ++s) {
        const float v = Vs[s * kst + c];
        const float4 pv = *reinterpret_cast<const float4*>(P + s * ATT_QB);
        a[0] = fmaf(pv.x, v, a[0]); a[1] = fmaf(pv.y, v, a[1]); a[2] = fmaf(pv.z, v, a[2]); a[3] = fmaf(pv.w, v, a[3]);
      }
#pragma unroll
      for (int qi = 0; qi < ATT_QB; ++qi)
        if (qi < nq) Elem<T>::st(out + (row0 + t0 + qi) * ld_out + h * ch + c, a[qi] / sum[qi]);
    }
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------
// bf16 tensor-core path (ch in {16, 32, 64, 128}): flash-style, one CTA per (shape, head, 64 queries).
// K and V of the (shape, head) are staged once in shared memory by 16-byte cp.async (rows padded by 16 B: the
// ldmatrix row addresses of an 8x8 tile then fall into 8 different 16-byte bank groups); each of the 4 warps owns
// 16 query rows: S = Q K^T per 64-key block with mma.sync.m16n8k16 (bf16 x bf16 -> fp32), online softmax in fp32
// (exp2 with the ch^-1/2 scale folded into the exponent, modules.py:542-546), P re-used from the accumulator
// registers as the A operand of P V (V fragments by ldmatrix.trans), O rescaled per block.  Scores never leave
// the registers.  ~9 GFLOP per denoising step in total, so the legacy warp-level MMA is ample: the whole
// attention of a step takes tens of microseconds (the CUDA-core version took 0.8 ms).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x2(uint32_t addr, uint32_t& r0, uint32_t& r1) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0,%1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}

constexpr int ATC_QB = 64;                 // queries per CTA (4 warps x 16)
constexpr int ATC_KB = 64;                 // keys per softmax block

template <int CH>
__global__ void __launch_bounds__(128) attention_tc_kernel(const __nv_bfloat16* __restrict__ qkv, int64_t ld_qkv,
                                                           __nv_bfloat16* __restrict__ out, int64_t ld_out, int tokens,
                                                           int heads, float scale_log2) {
  constexpr int RS = CH * 2 + 16;           // shared-memory row stride in bytes
  constexpr int CPR = CH / 8;               // 16-byte chunks per row
  extern __shared__ __align__(16) uint8_t smraw[];
  const int tpad = (tokens + ATC_KB - 1) / ATC_KB * ATC_KB;
  const uint32_t sK = (uint32_t)__cvta_generic_to_shared(smraw);
  const uint32_t sV = sK + (uint32_t)tpad * RS;
  const uint32_t sQ = sV + (uint32_t)tpad * RS;
  const int bh = blockIdx.y;
  const int b = bh / heads, h = bh - b * heads;
  const int64_t row0 = (int64_t)b * tokens;
  const int q0 = blockIdx.x * ATC_QB;
  const __nv_bfloat16* base = qkv + row0 * ld_qkv + h * 3 * CH;
  // ---- stage K, V (all keys) and this CTA's 64 queries; rows beyond `tokens` are zero ----
  for (int i = threadIdx.x; i < tpad * CPR; i += 128) {
    const int r = i / CPR, c = i - r * CPR;
    const uint32_t off = (uint32_t)r * RS + c * 16;
    if (r < tokens) {
      cp_async16(sK + off, base + (int64_t)r * ld_qkv + CH + c * 8);
      cp_async16(sV + off, base + (int64_t)r * ld_qkv + 2 * CH + c * 8);
    } else {
      *reinterpret_cast<uint4*>(smraw + (size_t)off) = make_uint4(0, 0, 0, 0);
      *reinterpret_cast<uint4*>(smraw + (size_t)tpad * RS + off) = make_uint4(0, 0, 0, 0);
    }
  }
  for (int i = threadIdx.x; i < ATC_QB * CPR; i += 128) {
    const int r = i / CPR, c = i - r * CPR;
    const uint32_t off = (uint32_t)r * RS + c * 16;
    if (q0 + r < tokens) cp_async16(sQ + off, base + (int64_t)(q0 + r) * ld_qkv + c * 8);
    else *reinterpret_cast<uint4*>(smraw + (size_t)2 * tpad * RS + off) = make_uint4(0, 0, 0, 0);
  }
  asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t4 = lane & 3;
  if (q0 + warp * 16 >= tokens) return;                    // (no later block-wide barrier)
  // ---- Q fragments of the warp's 16 rows ----
  uint32_t qf[CH / 16][4];
  {
    const uint32_t a = sQ + (uint32_t)(warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * RS + ((lane >> 4) * 8) * 2;
#pragma unroll
    for (int ks = 0; ks < CH / 16; ++ks) ldsm_x4(a + ks * 32, qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3]);
  }
  float o[CH / 8][4];
#pragma unroll
  for (int i = 0; i < CH / 8; ++i) { o[i][0] = 0.f; o[i][1] = 0.f; o[i][2] = 0.f; o[i][3] = 0.f; }
  float mrow[2] = {-INFINITY, -INFINITY}, lrow[2] = {0.f, 0.f};
  for (int k0 = 0; k0 < tokens; k0 += ATC_KB) {
    // ---- S = Q K^T for 64 keys: 8 n-tiles of 8 keys ----
    float sc[ATC_KB / 8][4];
#pragma unroll
    for (int nt = 0; nt < ATC_KB / 8; ++nt) {
      sc[nt][0] = 0.f; sc[nt][1] = 0.f; sc[nt][2] = 0.f; sc[nt][3] = 0.f;
      // one ldmatrix.x4 = the (b0, b1) fragments of two 16-channel steps of this key tile
      const uint32_t a = sK + (uint32_t)(k0 + nt * 8 + (lane & 7)) * RS + ((lane >> 3) * 8) * 2;
      if constexpr (CH == 16) {                            // one 16-channel step: ldmatrix.x2 (lanes 0-15 give the rows)
        uint32_t b0, b1;
        ldsm_x2(sK + (uint32_t)(k0 + nt * 8 + (lane & 7)) * RS + (((lane >> 3) & 1) * 8) * 2, b0, b1);
        mma_bf16_16816(sc[nt], qf[0], b0, b1);
      } else {
#pragma unroll
        for (int kp = 0; kp < CH / 32; ++kp) {
          uint32_t b0, b1, b2, b3;
          ldsm_x4(a + kp * 64, b0, b1, b2, b3);
          mma_bf16_16816(sc[nt], qf[2 * kp], b0, b1);
          mma_bf16_16816(sc[nt], qf[2 * kp + 1], b2, b3);
        }
      }
    }
    // ---- online softmax (rows g and g+8 of the warp tile; a row lives in the 4 lanes of a quad) ----
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nt = 0; nt < ATC_KB / 8; ++nt) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int key = k0 + nt * 8 + 2 * t4 + (j & 1);
        const float v = key < tokens ? sc[nt][j] * scale_log2 : -INFINITY;
        sc[nt][j] = v;
        mx[j >> 1] = fmaxf(mx[j >> 1], v);
      }
    }
    float corr[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float mnew = fmaxf(mrow[r], mx[r]);             // finite: every block holds at least one valid key
      corr[r] = exp2f(mrow[r] - mnew);
      mrow[r] = mnew;
      lrow[r] *= corr[r];
    }
    float ps[2] = {0.f, 0.f};
    uint32_t pf[ATC_KB / 16][4];                            // P as A fragments of the P V product
#pragma unroll
    for (int nt = 0; nt < ATC_KB / 8; ++nt) {
      const float p0 = exp2f(sc[nt][0] - mrow[0]), p1 = exp2f(sc[nt][1] - mrow[0]);
      const float p2 = exp2f(sc[nt][2] - mrow[1]), p3 = exp2f(sc[nt][3] - mrow[1]);
      ps[0] += p0 + p1; ps[1] += p2 + p3;
      pf[nt >> 1][(nt & 1) * 2] = pack_bf16x2(p0, p1);
      pf[nt >> 1][(nt & 1) * 2 + 1] = pack_bf16x2(p2, p3);
    }
    lrow[0] += ps[0]; lrow[1] += ps[1];                     // (quad-partial sums; reduced once at the end)
#pragma unroll
    for (int i = 0; i < CH / 8; ++i) { o[i][0] *= corr[0]; o[i][1] *= corr[0]; o[i][2] *= corr[1]; o[i][3] *= corr[1]; }
    // ---- O += P V: 4 steps of 16 keys, CH/8 channel tiles ----
#pragma unroll
    for (int kk = 0; kk < ATC_KB / 16; ++kk) {
      const uint32_t a = sV + (uint32_t)(k0 + kk * 16 + ((lane >> 3) & 1) * 8 + (lane & 7)) * RS + ((lane >> 4) * 8) * 2;
#pragma unroll
      for (int cp = 0; cp < CH / 16; ++cp) {
        uint32_t b0, b1, b2, b3;
        ldsm_x4_t(a + cp * 32, b0, b1, b2, b3);
        mma_bf16_16816(o[2 * cp], pf[kk], b0, b1);
        mma_bf16_16816(o[2 * cp + 1], pf[kk], b2, b3);
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    lrow[r] += __shfl_xor_sync(0xffffffffu, lrow[r], 1);
    lrow[r] += __shfl_xor_sync(0xffffffffu, lrow[r], 2);
  }
  const float inv0 = 1.0f / lrow[0], inv1 = 1.0f / lrow[1];
  const int r0 = q0 + warp * 16 + g, r1 = r0 + 8;
#pragma unroll
  for (int i = 0; i < CH / 8; ++i) {
    const int c = h * CH + i * 8 + 2 * t4;
    if (r0 < tokens) *reinterpret_cast<uint32_t*>(out + (row0 + r0) * ld_out + c) = pack_bf16x2(o[i][0] * inv0, o[i][1] * inv0);
    if (r1 < tokens) *reinterpret_cast<uint32_t*>(out + (row0 + r1) * ld_out + c) = pack_bf16x2(o[i][2] * inv1, o[i][3] * inv1);
  }
}

template <int CH>
static int launch_attention_tc(const void* qkv, int64_t ld_qkv, void* out, int64_t ld_out, int batch, int tokens,
                               int heads, cudaStream_t st) {
  const int tpad = (tokens + ATC_KB - 1) / ATC_KB * ATC_KB;
  const size_t smem = (size_t)(2 * tpad + ATC_QB) * (CH * 2 + 16);
  if (smem > 200 * 1024) return OF_E_UNSUPPORTED;
  static bool configured[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !configured[dev]) {
    cudaFuncSetAttribute(attention_tc_kernel<CH>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (dev >= 0 && dev < 64) configured[dev] = true;
  }
  dim3 grid((tokens + ATC_QB - 1) / ATC_QB, batch * heads);
  const float scale_log2 = rsqrtf((float)CH) * 1.4426950408889634f;     // (ch^-1/4)^2 * log2(e)
  attention_tc_kernel<CH><<<grid, 128, smem, st>>>((const __nv_bfloat16*)qkv, ld_qkv, (__nv_bfloat16*)out, ld_out, tokens,
                                                   heads, scale_log2);
  return OF_OK;
}

}  // namespace of

extern "C" int of_attention(const void* qkv, int64_t ld_qkv, void* out, int64_t ld_out, int32_t batch,
                            int32_t tokens, int32_t heads, int32_t ch, int32_t dtype, void* stream) {
  using namespace of;
  OF_REQUIRE(qkv && out && batch > 0 && tokens > 0 && heads > 0 && ch > 0, "of_attention: bad arguments");
  OF_REQUIRE(dtype == OF_F32 || dtype == OF_BF16, "of_attention: bad dtype");
  OF_REQUIRE(ch % 4 == 0, "of_attention: ch must be a multiple of 4");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // tensor-core path: bf16, 16-byte aligned rows
  if (dtype == OF_BF16 && (ch == 16 || ch == 32 || ch == 64 || ch == 128) && ld_qkv % 8 == 0 && ld_out % 2 == 0 &&
      reinterpret_cast<uintptr_t>(qkv) % 16 == 0 && reinterpret_cast<uintptr_t>(out) % 4 == 0) {
    int rc = ch == 16 ? launch_attention_tc<16>(qkv, ld_qkv, out, ld_out, batch, tokens, heads, st)
           : ch == 32 ? launch_attention_tc<32>(qkv, ld_qkv, out, ld_out, batch, tokens, heads, st)
           : ch == 64 ? launch_attention_tc<64>(qkv, ld_qkv, out, ld_out, batch, tokens, heads, st)
                      : launch_attention_tc<128>(qkv, ld_qkv, out, ld_out, batch, tokens, heads, st);
    if (rc == OF_OK) {
      OF_LAUNCH_CHECK("of_attention(tc)");
      return OF_OK;
    }
  }
  const size_t smem = ((size_t)2 * tokens * (ch + 4) + (size_t)ATT_WARPS * tokens * ATT_QB + (size_t)ATT_WARPS * ATT_QB * ch) * 4;
  if (smem > 220 * 1024) {
    set_error("of_attention: T=%d ch=%d needs %zu B of shared memory (> 220 KB)", tokens, ch, smem);
    return OF_E_UNSUPPORTED;
  }
  dim3 grid(batch * heads, (tokens + ATT_QTILE - 1) / ATT_QTILE);
  if (dtype == OF_F32) {
    static size_t cfg_f32 = 48 * 1024;
    if (smem > cfg_f32) {
      cudaFuncSetAttribute(attention_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
      cfg_f32 = 220 * 1024;
    }
    attention_kernel<float><<<grid, ATT_WARPS * 32, smem, st>>>((const float*)qkv, ld_qkv, (float*)out, ld_out, tokens,
                                                                heads, ch);
  } else {
    static size_t cfg_bf16 = 48 * 1024;
    if (smem > cfg_bf16) {
      cudaFuncSetAttribute(attention_kernel<__nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
      cfg_bf16 = 220 * 1024;
    }
    attention_kernel<__nv_bfloat16><<<grid, ATT_WARPS * 32, smem, st>>>((const __nv_bfloat16*)qkv, ld_qkv,
                                                                        (__nv_bfloat16*)out, ld_out, tokens, heads, ch);
  }
  OF_LAUNCH_CHECK("of_attention");
  return OF_OK;
}
