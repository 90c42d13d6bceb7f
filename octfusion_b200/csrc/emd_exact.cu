// Exact EMD of equal-size point clouds: the optimal assignment cost that reference metrics/evaluation_metrics.py
// `emd_approx` (:35-52) computes with scipy.optimize.linear_sum_assignment on the fp32 distance matrix, solved on the
// GPU by Bertsekas' auction algorithm with epsilon scaling on integer costs.  Contract in include/octfusion_b200.h.
//
// Costs.  d_ij = sqrt((dx^2 + dy^2) + dz^2) of dx = x_i - y_j, ... in fp32 with every operation rounded on its own (no
// FMA contraction), so d(x_i, y_j) and d(y_j, x_i) are the same bits.  s = 2^k is the smallest power of two >= the
// diagonal of the pair's joint bounding box (k clamped below at -100, so that identical points are an ordinary case),
// q = s 2^-24 and c_ij = rint(d_ij / q): an integer <= 2^24 (plus rounding slack), exact in fp32 because d_ij / q is a
// scaling by a power of two.  The auction runs on C_ij = c_ij (n + 1).
//
// Auction (minimisation form).  Objects j (points of y) carry int64 prices p_j; an unassigned person i (point of x)
// finds the best value w1 = min_j C_ij + p_j at j1 and the second best w2 and bids p_j1 + (w2 - w1) + eps for j1.
// All unassigned persons bid in one Jacobi round, one warp per bidder; an object takes the largest bid through a
// 64-bit shared-memory atomicMax on (price << 12 | bidder), which does not depend on the order of the atomics, and
// its previous owner becomes unassigned.  Every assignment made keeps eps-complementary slackness
//   C_i,sigma(i) + p_sigma(i) <= min_j (C_ij + p_j) + eps.
// Phases run at eps_0 = ceil(Cmax / 8), then eps / 8 ... down to eps = 1, each restarting from no assignment with the
// prices of the one before.  At eps = 1 the total slack is below n < n + 1, the cost unit of C: the assignment is
// optimal for c.  Every step is deterministic, so prices, round counts and the gap repeat bit for bit.
//
// Round cap.  Let sigma' be the previous phase's final assignment, eps'-CS with the phase's start prices p0
// (phase 0: p0 = 0 and eps' = Cmax, which any assignment satisfies).  For a winning bid of person i on j with
// j != sigma'(i), the path i -> sigma'(i) -> current owner -> its sigma' object -> ... ends at an object no one has bid
// for in this phase (the path cannot close, i being unassigned); adding the eps-CS of each owner on the path to the
// eps'-CS of sigma' gives p_j - p0_j <= n (eps + eps') after the bid.  Bids of sigma'^-1(j) on j alternate with bids
// of others, so j wins at most 2 n (eps + eps') / eps + 1 bids, and every round has a winner:
//   rounds per phase <= n (2 n (eps + eps') / eps + 1).
// A pair that reaches the cap stops with status 1 (a bug, never an input): no trap, the caller reads the status.
//
// Certificate.  After the last phase, P = sum_i C_i,sigma(i) and the dual D = sum_i min_j (C_ij + p_j) - sum_j p_j
// (u_i = min_j (C_ij + p_j), v_j = -p_j is dual feasible: u_i + v_j <= C_ij), so P - D >= 0 bounds the distance to the
// optimum; eps-CS at eps = 1 gives P - D <= n.
//
// Prices stay below 2^51 (each phase raises a price by at most Cmax + eps above the previous maximum, Cmax < 2^37,
// at most 13 phases), so a bid packs into 64 bits with the bidder in the low 12.
#include <float.h>
#include "common.cuh"

namespace of {

constexpr int EX_THREADS = 512, EX_WARPS = EX_THREADS / 32;
constexpr int64_t EX_ALPHA = 8;                                 // eps reduction per phase
constexpr int EX_BIDDER_BITS = 12;                              // 2^12 = OF_EMD_MAX_POINTS persons
constexpr int EX_K_MIN = -100, EX_K_MAX = 62;                   // s = 2^k; above 2^62 squares may overflow fp32
constexpr int64_t EX_C_BOUND = (1 << 24) + 1024;                // >= every c_ij (d_ij <= s up to fp32 rounding)

static_assert(OF_EMD_MAX_POINTS <= (1 << EX_BIDDER_BITS), "bidder ids must fit the low bits of a bid");

__host__ __device__ constexpr size_t emd_exact_smem_bytes(int n) {
  return (size_t)n * (6 * sizeof(float) + sizeof(int64_t) + sizeof(unsigned long long) + 2 * sizeof(int32_t));
}
static_assert(emd_exact_smem_bytes(OF_EMD_MAX_POINTS) <= 227 * 1024, "exact-EMD working set must fit one SM");

__device__ __forceinline__ float pair_dist(float ax, float ay, float az, float bx, float by, float bz) {
  const float dx = __fsub_rn(ax, bx), dy = __fsub_rn(ay, by), dz = __fsub_rn(az, bz);
  return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
}

// c = rint(d 2^24 / s); scale = 2^(24 - k) is a normal fp32 for k in [EX_K_MIN, EX_K_MAX], so the product is exact
__device__ __forceinline__ int int_cost(float d, float scale) { return __float2int_rn(__fmul_rn(d, scale)); }

struct ExSmem {
  float *ax, *ay, *az, *bx, *by, *bz;
  int64_t* price;               // [n] object prices
  unsigned long long* bid;      // [n] best bid of the round, 0 = none
  int32_t* owner;               // [n] object -> person, -1 = free
  int32_t* assign;              // [n] person -> object, -1 = unassigned
};

// best (w1 at j1) and second best (w2) value min_j C_ij + p_j of person i, identical in every lane; ties -> lower j
__device__ __forceinline__ void best_two(const ExSmem& s, int n, int64_t np1, float scale, int i, int64_t& w1, int& j1,
                                         int64_t& w2) {
  const int lane = threadIdx.x & 31;
  const float px = s.ax[i], py = s.ay[i], pz = s.az[i];
  w1 = INT64_MAX; w2 = INT64_MAX; j1 = n;
  for (int j = lane; j < n; j += 32) {
    const int64_t v = (int64_t)int_cost(pair_dist(px, py, pz, s.bx[j], s.by[j], s.bz[j]), scale) * np1 + s.price[j];
    if (v < w1) { w2 = w1; w1 = v; j1 = j; }
    else if (v < w2) w2 = v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const int64_t ow1 = __shfl_xor_sync(0xffffffffu, w1, o), ow2 = __shfl_xor_sync(0xffffffffu, w2, o);
    const int oj1 = __shfl_xor_sync(0xffffffffu, j1, o);
    if (ow1 < w1 || (ow1 == w1 && oj1 < j1)) { w2 = min(w1, ow2); w1 = ow1; j1 = oj1; }
    else w2 = min(w2, ow1);
  }
}

__device__ __forceinline__ int64_t block_sum_i64(int64_t v, unsigned long long* acc) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(acc, (unsigned long long)v);     // integer: order-independent
  __syncthreads();
  const int64_t r = (int64_t)*acc;
  __syncthreads();
  return r;
}

// status word: bits 0-3 code, 4-7 phases run, 8-31 bidding rounds over all phases (saturating)
__device__ __forceinline__ int32_t status_word(int code, int phases, int64_t rounds) {
  const int64_t r = rounds < 0xffffff ? rounds : 0xffffff;
  return code | (phases << 4) | (int32_t)(r << 8);
}

// pair p -> (ia, ib): paired (p, p), all pairs (p / nb, p % nb), symmetric p-th (i < j) in row order of an [nb, nb]
__device__ __forceinline__ void exact_pair(int64_t p, int64_t nb, int mode, int64_t& ia, int64_t& ib) {
  if (mode == 0) { ia = ib = p; return; }
  if (mode == 1) { ia = p / nb; ib = p % nb; return; }
  // row i starts at i (2 nb - i - 1) / 2
  const double t = (double)(2 * nb - 1);
  int64_t i = (int64_t)((t - sqrt(t * t - 8.0 * (double)p)) * 0.5);
  i = max((int64_t)0, min(i, nb - 2));
  while (i > 0 && i * (2 * nb - i - 1) / 2 > p) --i;
  while ((i + 1) * (2 * nb - i - 2) / 2 <= p) ++i;
  ia = i;
  ib = i + 1 + (p - i * (2 * nb - i - 1) / 2);
}

__global__ void __launch_bounds__(EX_THREADS, 2) emd_exact_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                                  int64_t nb, int mode, int64_t pairs, int n,
                                                                  float* __restrict__ out, int64_t* __restrict__ gap,
                                                                  int32_t* __restrict__ status) {
  extern __shared__ __align__(16) unsigned char ex_raw[];
  __shared__ float red[EX_WARPS][6];
  __shared__ int s_k, s_unassigned;
  __shared__ unsigned long long s_acc;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t p = blockIdx.x;

  if (p == pairs) {                                         // symmetric mode: one extra CTA writes the diagonal
    for (int64_t i = tid; i < nb; i += EX_THREADS) {
      out[i * nb + i] = 0.0f;
      if (gap) gap[i * nb + i] = 0;
      status[i * nb + i] = 0;
    }
    return;
  }
  int64_t ia, ib;
  exact_pair(p, nb, mode, ia, ib);
  const int64_t o1 = mode == 0 ? p : ia * nb + ib, o2 = ib * nb + ia;

  ExSmem s;
  s.price = reinterpret_cast<int64_t*>(ex_raw);
  s.bid = reinterpret_cast<unsigned long long*>(s.price + n);
  s.ax = reinterpret_cast<float*>(s.bid + n);
  s.ay = s.ax + n; s.az = s.ay + n; s.bx = s.az + n; s.by = s.bx + n; s.bz = s.by + n;
  s.owner = reinterpret_cast<int32_t*>(s.bz + n);
  s.assign = s.owner + n;

  const float* pa = a + ia * n * 3;
  const float* pb = b + ib * n * 3;
  float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  bool finite = true;
  for (int k = tid; k < n; k += EX_THREADS) {
    const float x0 = pa[3 * k], x1 = pa[3 * k + 1], x2 = pa[3 * k + 2];
    const float y0 = pb[3 * k], y1 = pb[3 * k + 1], y2 = pb[3 * k + 2];
    s.ax[k] = x0; s.ay[k] = x1; s.az[k] = x2;
    s.bx[k] = y0; s.by[k] = y1; s.bz[k] = y2;
    finite = finite && isfinite(x0) && isfinite(x1) && isfinite(x2) && isfinite(y0) && isfinite(y1) && isfinite(y2);
    lo[0] = fminf(lo[0], fminf(x0, y0)); hi[0] = fmaxf(hi[0], fmaxf(x0, y0));
    lo[1] = fminf(lo[1], fminf(x1, y1)); hi[1] = fmaxf(hi[1], fmaxf(x1, y1));
    lo[2] = fminf(lo[2], fminf(x2, y2)); hi[2] = fmaxf(hi[2], fmaxf(x2, y2));
    s.price[k] = 0;
    s.bid[k] = 0ull;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      lo[c] = fminf(lo[c], __shfl_xor_sync(0xffffffffu, lo[c], o));
      hi[c] = fmaxf(hi[c], __shfl_xor_sync(0xffffffffu, hi[c], o));
    }
  }
  if (lane == 0) {
#pragma unroll
    for (int c = 0; c < 3; ++c) { red[warp][c] = lo[c]; red[warp][3 + c] = hi[c]; }
  }
  const bool bad = __syncthreads_or(!finite);
  if (bad) {
    if (tid == 0) {
      out[o1] = __int_as_float(0x7fc00000);
      if (gap) gap[o1] = -1;
      status[o1] = status_word(2, 0, 0);
      if (mode == 2) { out[o2] = out[o1]; if (gap) gap[o2] = -1; status[o2] = status[o1]; }
    }
    return;
  }
  if (tid == 0) {
    // squared diagonal in fp64 from the exact fp32 extremes, each operation rounded on its own
    double d2 = 0.0;
    for (int c = 0; c < 3; ++c) {
      float l = red[0][c], h = red[0][3 + c];
      for (int w = 1; w < EX_WARPS; ++w) { l = fminf(l, red[w][c]); h = fmaxf(h, red[w][3 + c]); }
      const double e = __dsub_rn((double)h, (double)l);
      d2 = __dadd_rn(d2, __dmul_rn(e, e));
    }
    // smallest k with 4^k >= d2: with d2 = m 2^e, m in [0.5, 1), the smallest t with 2^t >= d2 is e (e - 1 if m = 0.5)
    int k = EX_K_MIN;
    if (d2 > 0.0) {
      int e;
      const double m = frexp(d2, &e);
      const int t = m == 0.5 ? e - 1 : e;
      k = max(EX_K_MIN, t >= 0 ? (t + 1) / 2 : -((-t) / 2));
    }
    s_k = k;
  }
  __syncthreads();
  const int k = s_k;
  if (k > EX_K_MAX) {
    if (tid == 0) {
      out[o1] = __int_as_float(0x7fc00000);
      if (gap) gap[o1] = -1;
      status[o1] = status_word(3, 0, 0);
      if (mode == 2) { out[o2] = out[o1]; if (gap) gap[o2] = -1; status[o2] = status[o1]; }
    }
    return;
  }
  const float scale = __int_as_float((127 + 24 - k) << 23);
  const int64_t np1 = n + 1;
  const int64_t cmax = EX_C_BOUND * np1;

  int phases = 0, code = 0;
  int64_t rounds = 0;
  if (n == 1) {
    if (tid == 0) { s.assign[0] = 0; s.owner[0] = 0; }
  } else {
    int64_t eps_prev = cmax, eps = (cmax + EX_ALPHA - 1) / EX_ALPHA;
    for (;;) {
      for (int j = tid; j < n; j += EX_THREADS) { s.owner[j] = -1; s.assign[j] = -1; }
      if (tid == 0) s_unassigned = n;
      __syncthreads();
      ++phases;
      const int64_t cap = (int64_t)n * (2 * (int64_t)n * ((eps + eps_prev) / eps + 1) + 1);
      int64_t phase_rounds = 0;
      for (;;) {
        // every unassigned person bids, one warp per bidder
        for (int base = warp * 32; base < n; base += EX_THREADS) {
          const int i0 = base + lane;
          unsigned m = __ballot_sync(0xffffffffu, i0 < n && s.assign[i0] < 0);
          while (m) {
            const int i = base + __ffs(m) - 1;
            m &= m - 1;
            int64_t w1, w2;
            int j1;
            best_two(s, n, np1, scale, i, w1, j1, w2);
            if (lane == 0) {
              const int64_t bid_price = s.price[j1] + (w2 - w1) + eps;
              atomicMax(&s.bid[j1], ((unsigned long long)bid_price << EX_BIDDER_BITS) | (unsigned long long)i);
            }
          }
        }
        __syncthreads();
        // each object with a bid goes to its best bidder; the previous owner becomes unassigned
        int taken = 0;
        for (int j = tid; j < n; j += EX_THREADS) {
          const unsigned long long w = s.bid[j];
          if (w == 0ull) continue;
          s.bid[j] = 0ull;
          const int ni = (int)(w & ((1ull << EX_BIDDER_BITS) - 1));
          const int old = s.owner[j];
          if (old >= 0) s.assign[old] = -1;
          else ++taken;
          s.owner[j] = ni;
          s.assign[ni] = j;
          s.price[j] = (int64_t)(w >> EX_BIDDER_BITS);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) taken += __shfl_xor_sync(0xffffffffu, taken, o);
        if (lane == 0 && taken) atomicSub(&s_unassigned, taken);
        __syncthreads();
        ++phase_rounds;
        if (s_unassigned == 0) break;
        if (phase_rounds >= cap) { code = 1; break; }
      }
      rounds += phase_rounds;
      if (code != 0 || eps == 1) break;
      eps_prev = eps;
      eps = max((int64_t)1, eps / EX_ALPHA);
      __syncthreads();                                       // s_unassigned read by all before the reset
    }
  }
  if (code != 0) {
    if (tid == 0) {
      out[o1] = __int_as_float(0x7fc00000);
      if (gap) gap[o1] = -1;
      status[o1] = status_word(code, phases, rounds);
      if (mode == 2) { out[o2] = out[o1]; if (gap) gap[o2] = -1; status[o2] = status[o1]; }
    }
    return;
  }
  __syncthreads();

  // certificate: primal P = sum_i C_i,sigma(i), dual D = sum_i min_j (C_ij + p_j) - sum_j p_j
  int64_t primal = 0, prices = 0, minima = 0;
  for (int i = tid; i < n; i += EX_THREADS) {
    const int j = s.assign[i];
    primal += (int64_t)int_cost(pair_dist(s.ax[i], s.ay[i], s.az[i], s.bx[j], s.by[j], s.bz[j]), scale) * np1;
    prices += s.price[i];
  }
  for (int i = warp; i < n; i += EX_WARPS) {
    int64_t w1, w2;
    int j1;
    best_two(s, n, np1, scale, i, w1, j1, w2);
    if (lane == 0) minima += w1;
  }
  if (tid == 0) s_acc = 0ull;
  __syncthreads();
  primal = block_sum_i64(primal, &s_acc);
  if (tid == 0) s_acc = 0ull;
  __syncthreads();
  const int64_t dual = block_sum_i64(minima - prices, &s_acc);
  if (tid == 0) {
    const int64_t cstar = primal / np1;
    const float emd = (float)(ldexp((double)cstar, k - 24) / (double)n);
    out[o1] = emd;
    if (gap) gap[o1] = primal - dual;
    status[o1] = status_word(0, phases, rounds);
    if (mode == 2) { out[o2] = emd; if (gap) gap[o2] = primal - dual; status[o2] = status[o1]; }
  }
}

static int launch_emd_exact(const float* a, const float* b, int64_t nb, int mode, int64_t pairs, int n, float* out,
                            int64_t* gap, int32_t* status, void* stream, const char* who) {
  const size_t smem = emd_exact_smem_bytes(n);
  if (cudaFuncSetAttribute(emd_exact_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
    set_error("%s: cannot reserve %zu bytes of shared memory", who, smem);
    return OF_E_CUDA;
  }
  const int64_t grid = pairs + (mode == 2 ? 1 : 0);
  emd_exact_kernel<<<(unsigned)grid, EX_THREADS, smem, reinterpret_cast<cudaStream_t>(stream)>>>(a, b, nb, mode, pairs, n,
                                                                                             out, gap, status);
  OF_LAUNCH_CHECK(who);
  return OF_OK;
}

}  // namespace of

extern "C" int of_emd_exact(const float* x, const float* y, int32_t batch, int32_t n, float* emd, int64_t* gap,
                            int32_t* status, void* stream) {
  using namespace of;
  OF_REQUIRE(x && y && emd && status, "of_emd_exact: null pointer");
  OF_REQUIRE(batch >= 0 && n >= 1 && n <= OF_EMD_MAX_POINTS, "of_emd_exact: need batch >= 0 and 1 <= n <= %d (got %d, %d)",
             OF_EMD_MAX_POINTS, batch, n);
  if (batch == 0) return OF_OK;
  return launch_emd_exact(x, y, 1, 0, batch, n, emd, gap, status, stream, "of_emd_exact");
}

extern "C" int of_emd_exact_pairwise(const float* a, int32_t na, const float* b, int32_t nb, int32_t n, int32_t symmetric,
                                     float* out, int64_t* gap, int32_t* status, void* stream) {
  using namespace of;
  OF_REQUIRE(a && b && out && status, "of_emd_exact_pairwise: null pointer");
  OF_REQUIRE(na >= 0 && nb >= 0 && n >= 1 && n <= OF_EMD_MAX_POINTS,
             "of_emd_exact_pairwise: need na, nb >= 0 and 1 <= n <= %d (got n = %d)", OF_EMD_MAX_POINTS, n);
  OF_REQUIRE(!symmetric || (a == b && na == nb), "of_emd_exact_pairwise: symmetric mode needs a == b and na == nb");
  const int64_t pairs = symmetric ? (int64_t)na * (na - 1) / 2 : (int64_t)na * nb;
  OF_REQUIRE(pairs < INT32_MAX, "of_emd_exact_pairwise: %lld pairs exceed one launch", (long long)pairs);
  if ((int64_t)na * nb == 0) return OF_OK;
  return launch_emd_exact(a, b, nb, symmetric ? 2 : 1, pairs, n, out, gap, status, stream, "of_emd_exact_pairwise");
}
