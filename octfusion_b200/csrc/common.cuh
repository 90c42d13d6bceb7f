// Shared helpers for the octfusion_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include "../../include/octfusion_b200.h"

namespace of {

void set_error(const char* fmt, ...);

#define OF_REQUIRE(cond, ...)                         \
  do {                                                \
    if (!(cond)) {                                    \
      ::of::set_error(__VA_ARGS__);                   \
      return OF_E_ARG;                                \
    }                                                 \
  } while (0)

#define OF_LAUNCH_CHECK(name)                                                   \
  do {                                                                          \
    cudaError_t e__ = cudaGetLastError();                                       \
    if (e__ != cudaSuccess) {                                                   \
      ::of::set_error("%s: launch failed: %s", name, cudaGetErrorString(e__));  \
      return OF_E_CUDA;                                                         \
    }                                                                           \
    ::of::add_launches(1);                                                      \
  } while (0)

int num_sms();
void add_launches(int n);   // kernel-launch counter behind of_launch_count()

template <typename T> struct Elem;
template <> struct Elem<float> {
  static __device__ __forceinline__ float ld(const float* p) { return *p; }
  static __device__ __forceinline__ void st(float* p, float v) { *p = v; }
};
template <> struct Elem<__nv_bfloat16> {
  static __device__ __forceinline__ float ld(const __nv_bfloat16* p) { return __bfloat162float(*p); }
  static __device__ __forceinline__ void st(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }
};

__device__ __forceinline__ float silu_f(float v) { return v / (1.0f + __expf(-v)); }
// one MUFU op instead of two: x*sigmoid(x) = 0.5x(1 + tanh(x/2)); tanh.approx is good to ~2^-11, i.e. below
// the bf16 rounding of the stored result (used for bf16 outputs only)
__device__ __forceinline__ float silu_fast(float v) {
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.5f * v));
  return 0.5f * v * (1.0f + t);
}

// 8 bf16 <-> 8 floats through one 16-byte register quad
__device__ __forceinline__ void bf16x8_to_f32(const uint4& q, float* f) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&q);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t = __bfloat1622float2(h[i]);
    f[2 * i] = t.x; f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 f32_to_bf16x8(const float* f) {
  uint4 q;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&q);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return q;
}

}  // namespace of
