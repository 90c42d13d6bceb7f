// TEST INFRASTRUCTURE.  Plain C entry points around the reference's own structural-loss kernels
// (metrics/pytorch_structural_losses/src/{approxmatch,nndistance}.cu), which oracle/build_ref.py compiles in place
// from the reference tree and links with this file into oracle/_ref/libref_structural.so.  The reference launchers
// throw C++ exceptions on a launch error; ctypes cannot see those, so they become a nonzero return here.
#include <cuda_runtime.h>
#include "approxmatch.cuh"
#include "nndistance.cuh"

extern "C" {

// match [b, m, n] fp32 (written), temp [b, 2 * (n + m)] fp32 scratch
int ref_approxmatch(int b, int n, int m, const float* xyz1, const float* xyz2, float* match, float* temp, void* stream) {
  try {
    approxmatch(b, n, m, xyz1, xyz2, match, temp, reinterpret_cast<cudaStream_t>(stream));
  } catch (...) {
    return -1;
  }
  return 0;
}

// out [b]: sum_kl match[b, l, k] * |xyz2_l - xyz1_k|
int ref_matchcost(int b, int n, int m, const float* xyz1, const float* xyz2, float* match, float* out, void* stream) {
  try {
    matchcost(b, n, m, xyz1, xyz2, match, out, reinterpret_cast<cudaStream_t>(stream));
  } catch (...) {
    return -1;
  }
  return 0;
}

// dist1 [b, n], idx1 [b, n], dist2 [b, m], idx2 [b, m]
int ref_nndistance(int b, int n, const float* xyz1, int m, const float* xyz2, float* dist1, int* idx1, float* dist2,
                   int* idx2, void* stream) {
  nndistance(b, n, xyz1, m, xyz2, dist1, idx1, dist2, idx2, reinterpret_cast<cudaStream_t>(stream));
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

}  // extern "C"
