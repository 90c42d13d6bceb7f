// Tap-gather GEMM on the Hopper tensor cores (wgmma.mma_async, fp32 accumulators in registers).
//
//   out[m,:] = sum_tap mean_{j in nbr(m,tap)} [A[j,:] | onehot(type_j)] . W[tap]  (+bias +row_add +resid)
//
// This replaces the reference's GraphConv op sequence
//   x[col] (aten::index) -> scatter_mean into a [7N, C] buffer -> view(N, 7C) @ W
// (reference models/networks/modules.py:194-220, diffusion_networks/utils/scatter.py:42-66) and of
// its dense Conv3d / Conv1x1 / Down/Upsample GEMMs (modules.py:332-339, 392-395, 440-443, 493-502).
// The im2col buffer is never written to HBM: producer warps build each [128 x 64] bf16 A tile
// directly in shared memory, in the 128-byte-swizzled K-major layout wgmma reads.
//
// One persistent CTA per SM, 384 threads = three warpgroups:
//   warpgroup 0    producers: each warp fills every PW-th stage of the shared-memory ring (PW = 4, or the ring depth
//                  when it is shallower).  Tap table -> thirty-two 16-byte cp.async (LDGSTS) per lane straight into the
//                  swizzled A stage, completion by cp.async.mbarrier.arrive.noinc; lane 0 also streams the stage's
//                  pre-swizzled [BN x 64] weight tile with cp.async.bulk (1-D TMA) onto the same full barrier.  The
//                  table entries of the warp's next stage are fetched before it waits for the current one to be freed.
//   warpgroups 1-2 consumers, 64 rows of the 128-row tile each: wgmma 64 x BN x 16 from shared memory into register
//                  accumulators, one stage in flight; then the epilogue: accumulators -> shared-memory staging (64
//                  columns at a time) -> +bias/+emb[batch]/+residual, store; optionally the group-norm partial statistics
//                  of the tile (warp-shuffle reduction, one write per 32-row chunk -- no atomics, bit-reproducible): the
//                  statistics pass of the following DualOctreeGroupNorm (modules.py:291-326) never reads the tensor again.
// While the consumers drain a tile the producers already fill the ring with the next tile's stages.
//
// K is consumed as 64-wide blocks ordered (channel block outer, tap inner): the 7 (or 27) taps
// of one 64-channel slab touch the same few hundred source rows, which then sit in L2.
// The one-hot node-type columns (modules.py:199-202) are one extra K block of per-slot type fractions, read
// from a per-graph precomputed tensor (of_graph_type_block); slots with several finer neighbours read a
// pre-averaged row (of_gather_mean_rows); the weights are re-laid once by of_pack_weight_tc.
#include "common.cuh"
#include <stdlib.h>
#include <string.h>
#include <type_traits>

namespace of {

constexpr int TC_BM = 128;
constexpr int TC_BK = 64;                 // bf16 elements = 128 bytes = one swizzle row
constexpr int TC_THREADS = 3 * 128;
constexpr int TC_MAX_TAPS = 27;
constexpr int TC_SMEM_MAX = 227 * 1024;   // opt-in dynamic shared memory per block on H100
// setmaxnreg only moves registers inside the allocation made at launch (384 threads x 168): 128 * 96 + 256 * 200 <= 384 * 168
constexpr int TC_PROD_REGS = 96, TC_CONS_REGS = 200;

// ------------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug becomes a trap (an error the host sees), never a hung GPU.  (No printf here: a function
// call inside the consumers' MMA loop would make ptxas serialise the wgmma pipeline.)
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000ll) __trap();
  }
}
// register budget of a warpgroup (the producers give theirs to the accumulators of the consumers)
template <int R> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// the stage was written by cp.async (generic proxy) and is read by wgmma (async proxy)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
__device__ __forceinline__ uint4 ldg_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
// 16-byte asynchronous global->shared copy (LDGSTS); src_bytes = 0 zero-fills the destination
__device__ __forceinline__ void cp_async_16(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_mbar_arrive_noinc(uint32_t bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}

// K-major, SWIZZLE_128B wgmma operand descriptor: start>>4 in [0,14), LBO>>4 in [16,30) (unused for swizzled K-major: 1),
// SBO>>4 in [32,46) = 1024 B between 8-row groups, layout type SWIZZLE_128B = 1 in [62,64).  One 16-element K step is
// +32 bytes = +2 in the start field (the tile bases are 1024-byte aligned).
__device__ __forceinline__ uint64_t make_desc_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
__device__ __forceinline__ void fence_operand(float& r) { asm volatile("" : "+f"(r)::"memory"); }

// D[64 x N] (+)= A[64 x 16] * B[16 x N], both operands K-major in shared memory, bf16 x bf16 -> fp32.  Accumulator
// fragment of thread t of the warpgroup: d[i] holds row 16*(t/32) + (t%32)/4 + 8*((i/2)%2), column 8*(i/4) + 2*(t%4) + i%2.
template <int N> struct Wgmma;
template <> struct Wgmma<16> {
  static __device__ __forceinline__ void mma(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(da), "l"(db), "r"(acc));
  }
};
template <> struct Wgmma<32> {
  static __device__ __forceinline__ void mma(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(acc));
  }
};
template <> struct Wgmma<64> {
  static __device__ __forceinline__ void mma(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(acc));
  }
};
template <> struct Wgmma<128> {
  static __device__ __forceinline__ void mma(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(acc));
  }
};
template <> struct Wgmma<256> {
  static __device__ __forceinline__ void mma(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db), "r"(acc));
  }
};
// ------------------------------------------------------------------------------------------------
// shared-memory plan
// ------------------------------------------------------------------------------------------------
// BN: output columns per tile (the wgmma N).  A stage holds one 64-wide K block of the 128-row A tile and of the weight
// tile; the ring takes what is left of the 227 KB beside the epilogue staging and the barriers.
template <int BN>
struct TcCfg {
  static constexpr int A_BYTES = TC_BM * 128;
  static constexpr int B_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int EPI_COLS = BN < 64 ? BN : 64;                // columns per epilogue round
  static constexpr int EPI_LD = EPI_COLS + 4;                       // staging row stride in floats (conflict-free float4 rows)
  static constexpr int EPI_BYTES = 2 * 64 * EPI_LD * 4;             // one 64-row block per consumer warpgroup
  static constexpr int AUX_BYTES = 1024 + 8 * 1024;                 // mbarriers | per-consumer-warp row of (bias + emb)
  static constexpr int FIT = (TC_SMEM_MAX - 1024 - EPI_BYTES - AUX_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = FIT > 16 ? 16 : FIT;
  // producer warps.  A warp that waits for the release of its slot must know that the slot's previous use has been
  // released as well (the mbarrier parity tells two phases apart, not three): PW <= STAGES guarantees it.
  static constexpr int PW = STAGES < 4 ? STAGES : 4;
  static constexpr int SMEM_BYTES = 1024 /*align slack*/ + STAGES * STAGE_BYTES + EPI_BYTES + AUX_BYTES;
  static_assert(STAGES >= 2 && SMEM_BYTES <= TC_SMEM_MAX, "ring depth");
};

struct TcParams {
  of_gemm_args g;
  int num_kb;        // K blocks per (virtual) tile = all K blocks / ksplit
  int ksplit;        // split-K: every output tile is computed as ksplit virtual tiles over consecutive K ranges, each
                     // writing fp32 partial sums to its own [M, N] slab of the workspace (of_gather_gemm_tc_splitk)
  int cblocks;       // (c0+c1)/64
  int npad;          // N rounded up to 16 (rows per K block in the packed weight image)
  int m_tiles, n_tiles;
};

// Sum of a[0..NV-1] (NV = 16 or 32) over the 32 lanes of the warp by recursive halving: NV = 16: 8+4+2+1+1 = 16 shuffles,
// afterwards a[0] of lane L holds the warp total of the ORIGINAL a[(L >> 1) & 15]; NV = 32: 16+8+4+2+1 = 31 shuffles,
// a[0] of lane L holds the total of the original a[L] (a plain butterfly needs 5 * NV).  The order of the additions
// is fixed, so the result is bit-reproducible.
template <int NV>
__device__ __forceinline__ void warp_reduce_vals(float (&a)[NV], int lane) {
#pragma unroll
  for (int half = NV / 2, bit = 16; half >= 1; half >>= 1, bit >>= 1) {
    const bool up = (lane & bit) != 0;
#pragma unroll
    for (int i = 0; i < half; ++i) {
      const float send = up ? a[i] : a[i + half];
      const float keep = up ? a[i + half] : a[i];
      a[i] = keep + __shfl_xor_sync(0xffffffffu, send, bit);
    }
  }
  if (NV == 16) a[0] += __shfl_xor_sync(0xffffffffu, a[0], 1);
}

// ------------------------------------------------------------------------------------------------
// the kernel
// ------------------------------------------------------------------------------------------------
template <int BN>
__global__ void __launch_bounds__(TC_THREADS, 1) gather_gemm_tc_kernel(const __grid_constant__ TcParams p) {
  using Cfg = TcCfg<BN>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t epi = smem_base + Cfg::STAGES * Cfg::STAGE_BYTES;
  const uint32_t aux = epi + Cfg::EPI_BYTES;
  const uint32_t bar_full = aux, bar_empty = aux + 128;             // one pair per ring slot

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int warp = t >> 5, lane = t & 31;
  const of_gemm_args& g = p.g;
  const int taps = g.taps;
  const int ksplit = p.ksplit;
  const int total_tiles = p.m_tiles * p.n_tiles * ksplit;   // virtual tile v: output tile v / ksplit, K range v % ksplit

  if (threadIdx.x == 0) {
    for (int s = 0; s < Cfg::STAGES; ++s) {
      mbar_init(bar_full + 8 * s, 32 + 1);                  // the producer warp's lanes + the weight copy's expect_tx
      mbar_init(bar_empty + 8 * s, 2);                      // the two consumer warpgroups
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    // =========================== producers ===========================
    setmaxnreg_dec<TC_PROD_REGS>();
    if (warp < Cfg::PW) {
      const int q = lane & 7;                              // 16-byte chunk of the 128-byte row
      const int rbase = lane >> 3;                         // rows rbase + 4 i
      const __nv_bfloat16* a0 = reinterpret_cast<const __nv_bfloat16*>(g.a0);
      const __nv_bfloat16* a1 = reinterpret_cast<const __nv_bfloat16*>(g.a1);
      const int32_t* __restrict__ tab = g.tap_tab;
      const uint8_t* wp = reinterpret_cast<const uint8_t*>(g.w);
      const int my_tiles = (total_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
      const int total_stages = my_tiles * p.num_kb;
      struct Pos { int m0, n0, kabs; };
      // stage s of this CTA -> rows, columns and ABSOLUTE K block (split-K: the K range's offset included)
      auto pos_of = [&](int s) {
        const int ti = s / p.num_kb, kb = s - ti * p.num_kb;
        const int tile = (int)blockIdx.x + ti * (int)gridDim.x;
        const int vtile = g.reverse ? total_tiles - 1 - tile : tile;
        const int ptile = vtile / ksplit;
        return Pos{(ptile / p.n_tiles) * TC_BM, (ptile % p.n_tiles) * BN, (vtile - ptile * ksplit) * p.num_kb + kb};
      };
      auto fetch_taps = [&](const Pos& c, int32_t (&tv)[32]) {
        const int cb = c.kabs / taps;
        if (cb >= p.cblocks) return;                        // the node-type block
        const int tap = c.kabs - cb * taps;
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const int m = c.m0 + rbase + 4 * i;
          tv[i] = -1;
          if (m < g.M)
            tv[i] = tab != nullptr ? __ldg(tab + ((uint32_t)m * (uint32_t)taps + (uint32_t)tap))   // < 2^31 (checked on host)
                                   : (g.in_rows != nullptr ? __ldg(g.in_rows + m) : m);
        }
      };
      int32_t tnext[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) tnext[i] = -1;
      if (warp < total_stages) fetch_taps(pos_of(warp), tnext);
      for (int s = warp; s < total_stages; s += Cfg::PW) {
        const Pos c = pos_of(s);
        int32_t tv[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) tv[i] = tnext[i];
        if (s + Cfg::PW < total_stages) fetch_taps(pos_of(s + Cfg::PW), tnext);
        const int stage = s % Cfg::STAGES;
        const uint32_t phase = (uint32_t)(s / Cfg::STAGES) & 1u;
        mbar_wait(bar_empty + 8 * stage, phase ^ 1);
        const uint32_t a_addr = smem_base + stage * Cfg::STAGE_BYTES;
        const uint32_t full = bar_full + 8 * stage;
        if (lane == 0) {
          mbar_arrive_expect_tx(full, (uint32_t)Cfg::B_BYTES);
          bulk_g2s(a_addr + Cfg::A_BYTES, wp + ((int64_t)c.kabs * p.npad + c.n0) * 128, Cfg::B_BYTES, full);
        }
        const int cb = c.kabs / taps;
        if (cb < p.cblocks) {
          const int ch = cb * TC_BK;
          const __nv_bfloat16* src;
          int64_t ld;
          if (ch < g.c0) { src = a0 + ch; ld = g.lda0; } else { src = a1 + (ch - g.c0); ld = g.lda1; }
          src += q * 8;
          const __nv_bfloat16* msrc = reinterpret_cast<const __nv_bfloat16*>(g.a_multi) + ch + q * 8;
          // one neighbour -> its row; none -> zero fill; several -> the pre-averaged row of a_multi
          const uint64_t sbase = reinterpret_cast<uint64_t>(src), mbase = reinterpret_cast<uint64_t>(msrc);
          const uint32_t ldb = (uint32_t)ld * 2u, ldmb = (uint32_t)g.ld_multi * 2u;   // row strides in bytes
          int32_t lo = tv[0];
#pragma unroll
          for (int i = 1; i < 32; ++i) lo = min(lo, tv[i]);
          if (!__any_sync(0xffffffffu, lo < -1)) {
#pragma unroll
            for (int i = 0; i < 32; ++i) {
              const int row = rbase + 4 * i;
              const int32_t v = tv[i];
              const uint64_t addr = sbase + (uint64_t)(uint32_t)max(v, 0) * (uint64_t)ldb;
              cp_async_16(a_addr + row * 128 + ((q ^ (row & 7)) << 4), reinterpret_cast<const void*>(addr), v == -1 ? 0u : 16u);
            }
          } else {
#pragma unroll
            for (int i = 0; i < 32; ++i) {
              const int row = rbase + 4 * i;
              const int32_t v = tv[i];
              const bool multi = v < -1;
              const uint32_t idx = multi ? (uint32_t)(-2 - v) : (uint32_t)(v < 0 ? 0 : v);
              const uint64_t addr = (multi ? mbase : sbase) + (uint64_t)idx * (uint64_t)(multi ? ldmb : ldb);
              cp_async_16(a_addr + row * 128 + ((q ^ (row & 7)) << 4), reinterpret_cast<const void*>(addr), v == -1 ? 0u : 16u);
            }
          }
        } else {
          // node-type block, precomputed per graph (of_graph_type_block): a plain coalesced copy of rows m0..m0+127
          const __nv_bfloat16* nb = reinterpret_cast<const __nv_bfloat16*>(g.nt_block) + q * 8;
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            const int row = rbase + 4 * i;
            const int m = c.m0 + row;
            cp_async_16(a_addr + row * 128 + ((q ^ (row & 7)) << 4), m < g.M ? (const void*)(nb + (int64_t)m * 64) : (const void*)nb,
                        m < g.M ? 16u : 0u);
          }
        }
        // one counted arrival per lane: it fires when this lane's cp.asyncs have landed
        cp_async_mbar_arrive_noinc(full);
      }
    }
  } else {
    // =========================== consumers: MMA + epilogue ===========================
    setmaxnreg_inc<TC_CONS_REGS>();
    const int cw = wg - 1;                                 // rows 64 cw .. 64 cw + 63 of the tile
    float acc[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int vtile = g.reverse ? total_tiles - 1 - tile : tile;
      const int ptile = vtile / ksplit;
      const int64_t split_row0 = (int64_t)(vtile - ptile * ksplit) * g.M;        // this K range's slab of the workspace
      const int m0 = (ptile / p.n_tiles) * TC_BM, n0 = (ptile % p.n_tiles) * BN;
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) fence_operand(acc[i]);
      int prev = 0;
      for (int kb = 0; kb < p.num_kb; ++kb) {
        mbar_wait(bar_full + 8 * stage, phase);
        fence_proxy_async_smem();
        const uint32_t a_addr = smem_base + stage * Cfg::STAGE_BYTES;
        const uint64_t da = make_desc_sw128(a_addr + cw * 64 * 128), db = make_desc_sw128(a_addr + Cfg::A_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < TC_BK / 16; ++k) Wgmma<BN>::mma(acc, da + 2 * k, db + 2 * k, (kb > 0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();                                   // the previous stage's MMAs have read their operands
        if (kb > 0 && t == 0) mbar_arrive(bar_empty + 8 * prev);
        prev = stage;
        if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) fence_operand(acc[i]);
      if (t == 0) mbar_arrive(bar_empty + 8 * prev);

      // ---- epilogue: warp (w & 1) owns rows 32 (w & 1) .. +31 of the warpgroup's 64, column half (w >> 1) of each
      // staged 64-column block; lane = row ----
      constexpr int CH = BN >= 32 ? 32 : 16;
      const int rl = (warp & 1) * 32 + lane;
      const int cc = (warp >> 1) * 32;
      const bool active = cc < Cfg::EPI_COLS;             // (warp-uniform)
      const uint32_t stg = epi + (uint32_t)cw * 64 * Cfg::EPI_LD * 4;
      const int m = m0 + cw * 64 + rl;
      const bool row_ok = m < g.M;
      const int64_t orow = row_ok ? (g.out_rows ? (int64_t)g.out_rows[m] : (int64_t)m + split_row0) : 0;
      const float* radd = (row_ok && g.row_add) ? g.row_add + (int64_t)g.row_add_idx[m] * g.ld_row_add : nullptr;
      const __nv_bfloat16* res =
          (row_ok && g.resid) ? reinterpret_cast<const __nv_bfloat16*>(g.resid) + (int64_t)m * g.ld_resid : nullptr;
      // ---- group-norm partial statistics of this 32-row chunk (see of_gemm_args.stat_out) ----
      int nseg = 0, my_seg = 0, my_slot = 0;
      if (active && g.stat_out != nullptr) {
        const int chunk = (m0 + cw * 64 + (warp & 1) * 32) / 32;
        if (chunk * 32 < g.M) {
          const int seg0 = __ldg(g.stat_chunk_seg + chunk);
          nseg = __ldg(g.stat_chunk_seg + chunk + 1) - seg0;
          if (lane < nseg) my_slot = __ldg(g.stat_seg_slot + seg0 + lane);   // lane s: slot of the chunk's segment s
          if (nseg > 1) {                                  // rows of several samples in this chunk: rank of my sample run
            const int b = row_ok ? (g.stat_sample ? __ldg(g.stat_sample + m) : m / g.stat_rows_per_sample) : -1;
            const int bp = __shfl_up_sync(0xffffffffu, b, 1);
            const unsigned chg = __ballot_sync(0xffffffffu, lane > 0 && row_ok && b != bp);
            my_seg = __popc(chg & (0xffffffffu >> (31 - lane)));
          }
        }
      }
      // ---- per-column addends (bias + emb[batch]): when the 32 rows of this warp share one sample -- nearly always --
      // the BN-wide row is staged ONCE per tile in the warp's shared-memory slot and read back as broadcast ld.shared.v4
      bool staged = false;
      const uint32_t my_stage = aux + 1024 + (uint32_t)(cw * 4 + warp) * 1024;
      if (active && (g.bias != nullptr || g.row_add != nullptr) && n0 + BN <= g.N && (g.N % 4 == 0) &&
          (g.row_add == nullptr || (g.ld_row_add % 4 == 0 && reinterpret_cast<uintptr_t>(g.row_add) % 16 == 0)) &&
          (g.bias == nullptr || reinterpret_cast<uintptr_t>(g.bias) % 16 == 0)) {
        const int bsel = (row_ok && g.row_add) ? g.row_add_idx[m] : -1;
        const int b0 = __shfl_sync(0xffffffffu, bsel, 0);
        if (__all_sync(0xffffffffu, !row_ok || bsel == b0) && (g.row_add == nullptr || b0 >= 0)) {
          staged = true;
          __syncwarp();                                   // the previous tile's reads of the slot are done
#pragma unroll
          for (int i = lane * 4; i < BN; i += 128) {
            float4 tb = make_float4(0.f, 0.f, 0.f, 0.f);
            if (g.bias) tb = __ldg(reinterpret_cast<const float4*>(g.bias + n0 + i));
            if (g.row_add) {
              const float4 e = __ldg(reinterpret_cast<const float4*>(g.row_add + (int64_t)b0 * g.ld_row_add + n0 + i));
              tb.x += e.x; tb.y += e.y; tb.z += e.z; tb.w += e.w;
            }
            asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(my_stage + i * 4), "f"(tb.x), "f"(tb.y), "f"(tb.z), "f"(tb.w) : "memory");
          }
          __syncwarp();
        }
      }
      // one CH-column chunk of my row: (+bias, +emb, +residual) -> store (+ norm statistics)
      auto process = [&](float (&v)[32], int c0) {
        const int nb = n0 + c0;
        const bool full = (nb + CH <= g.N);
        if (staged) {
#pragma unroll
          for (int q = 0; q < CH / 4; ++q) {
            float4 tb;
            asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(tb.x), "=f"(tb.y), "=f"(tb.z), "=f"(tb.w) : "r"(my_stage + (c0 + 4 * q) * 4));
            v[4 * q] += tb.x; v[4 * q + 1] += tb.y; v[4 * q + 2] += tb.z; v[4 * q + 3] += tb.w;
          }
        }
        if (row_ok) {
          if (g.bias && !staged) {
            if (full && (reinterpret_cast<uintptr_t>(g.bias) % 16 == 0)) {
#pragma unroll
              for (int q = 0; q < CH / 4; ++q) {
                const float4 tb = __ldg(reinterpret_cast<const float4*>(g.bias + nb) + q);
                v[4 * q] += tb.x; v[4 * q + 1] += tb.y; v[4 * q + 2] += tb.z; v[4 * q + 3] += tb.w;
              }
            } else {
#pragma unroll
              for (int j = 0; j < CH; ++j) if (full || nb + j < g.N) v[j] += g.bias[nb + j];
            }
          }
          if (radd && !staged) {
            if (full && (g.ld_row_add % 4 == 0) && (reinterpret_cast<uintptr_t>(g.row_add) % 16 == 0)) {
#pragma unroll
              for (int q = 0; q < CH / 4; ++q) {
                const float4 tb = __ldg(reinterpret_cast<const float4*>(radd + nb) + q);
                v[4 * q] += tb.x; v[4 * q + 1] += tb.y; v[4 * q + 2] += tb.z; v[4 * q + 3] += tb.w;
              }
            } else {
#pragma unroll
              for (int j = 0; j < CH; ++j) if (full || nb + j < g.N) v[j] += radd[nb + j];
            }
          }
          if (res) {
            if (full && (g.ld_resid % 8 == 0)) {
#pragma unroll
              for (int q = 0; q < CH / 8; ++q) {
                float f[8];
                bf16x8_to_f32(ldg_nc_v4(res + nb + q * 8), f);
#pragma unroll
                for (int j = 0; j < 8; ++j) v[q * 8 + j] += f[j];
              }
            } else {
#pragma unroll
              for (int j = 0; j < CH; ++j) if (nb + j < g.N) v[j] += __bfloat162float(res[nb + j]);
            }
          }
          if (g.out_f32) {
            float* o = reinterpret_cast<float*>(g.out) + orow * g.ldo + nb;
            if (full && (g.ldo % 4 == 0)) {
#pragma unroll
              for (int q = 0; q < CH / 4; ++q)
                *reinterpret_cast<float4*>(o + q * 4) = make_float4(v[q * 4], v[q * 4 + 1], v[q * 4 + 2], v[q * 4 + 3]);
            } else {
#pragma unroll
              for (int j = 0; j < CH; ++j) if (nb + j < g.N) o[j] = v[j];
            }
          } else {
            __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(g.out) + orow * g.ldo + nb;
            if (full && (g.ldo % 8 == 0)) {
#pragma unroll
              for (int q = 0; q < CH / 8; ++q) *reinterpret_cast<uint4*>(o + q * 8) = f32_to_bf16x8(v + q * 8);
            } else {
#pragma unroll
              for (int j = 0; j < CH; ++j) if (nb + j < g.N) o[j] = __float2bfloat16_rn(v[j]);
            }
          }
        }
        if constexpr (CH == 32) {
          if (nseg > 0 && full) {
            // (sum, sum of squares) of every GRAN-channel granule of my row; rows beyond M contribute zero.
            // GRAN = 4 when N is a multiple of 128, else 2 (a 64-channel norm has 2 channels per group) -- a property of
            // the layer, not of the tile shape, so that the small-M dispatch may run a wide layer on narrow tiles.
            auto stats = [&](auto gran_c) {
              constexpr int GRAN = decltype(gran_c)::value;
              constexpr int NV = 2 * 32 / GRAN;
              float a[NV];
#pragma unroll
              for (int q = 0; q < 32 / GRAN; ++q) {
                float sv = 0.0f, qv = 0.0f;
#pragma unroll
                for (int e = 0; e < GRAN; ++e) { const float x = v[GRAN * q + e]; sv += x; qv = fmaf(x, x, qv); }
                a[2 * q] = row_ok ? sv : 0.0f;
                a[2 * q + 1] = row_ok ? qv : 0.0f;
              }
              const int nval = g.N / GRAN * 2;             // floats per segment slot
              float* dst = g.stat_out + nb / GRAN * 2 + (NV == 16 ? (lane >> 1) : lane);
              const bool writer = NV == 32 || (lane & 1) == 0;
              if (nseg == 1) {
                const int slot = __shfl_sync(0xffffffffu, my_slot, 0);
                warp_reduce_vals<NV>(a, lane);
                if (writer) dst[(int64_t)slot * nval] = a[0];
              } else {
#pragma unroll 1
                for (int s = 0; s < nseg; ++s) {
                  const int slot = __shfl_sync(0xffffffffu, my_slot, s);
                  float tt[NV];
#pragma unroll
                  for (int j = 0; j < NV; ++j) tt[j] = (my_seg == s) ? a[j] : 0.0f;
                  warp_reduce_vals<NV>(tt, lane);
                  if (writer) dst[(int64_t)slot * nval] = tt[0];
                }
              }
            };
            if constexpr (BN >= 128) stats(std::integral_constant<int, 4>{});
            else if (g.N % 128 == 0) stats(std::integral_constant<int, 4>{});
            else stats(std::integral_constant<int, 2>{});
          }
        }
      };
#pragma unroll
      for (int blk = 0; blk < BN / Cfg::EPI_COLS; ++blk) {
        named_bar_sync(1 + cw, 128);                       // the previous block's reads of the staging are done
#pragma unroll
        for (int j = 0; j < Cfg::EPI_COLS / 8; ++j) {
          const int i = blk * (Cfg::EPI_COLS / 2) + 4 * j;
          const int col = 8 * j + 2 * (lane & 3);
          const int r0 = warp * 16 + (lane >> 2);
          asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(stg + (uint32_t)(r0 * Cfg::EPI_LD + col) * 4), "f"(acc[i]), "f"(acc[i + 1]) : "memory");
          asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(stg + (uint32_t)((r0 + 8) * Cfg::EPI_LD + col) * 4), "f"(acc[i + 2]), "f"(acc[i + 3]) : "memory");
        }
        named_bar_sync(1 + cw, 128);
        if (active) {
          float v[32];
#pragma unroll
          for (int q = 0; q < CH / 4; ++q)
            asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v[4 * q]), "=f"(v[4 * q + 1]), "=f"(v[4 * q + 2]), "=f"(v[4 * q + 3])
                         : "r"(stg + (uint32_t)(rl * Cfg::EPI_LD + cc + 4 * q) * 4));
          process(v, blk * Cfg::EPI_COLS + cc);
        }
      }
    }
  }
  __syncthreads();                                         // no CTA exits while its copies are in flight
}

// ------------------------------------------------------------------------------------------------
// weight packing: canonical fp32 [taps*(c+ntype), N] -> bf16 image [num_kb][npad rows][64], each
// 8-row group 128B-swizzled exactly as the MMA expects it, so a [BN x 64] tile is one contiguous
// cp.async.bulk.  K-block order = (channel block outer, tap inner), then the node-type block.
// ------------------------------------------------------------------------------------------------
__global__ void pack_weight_tc_kernel(const float* __restrict__ w, int taps, int c, int ntype, int N, int npad,
                                      int num_kb, __nv_bfloat16* __restrict__ out) {
  const int64_t total = (int64_t)num_kb * npad * 64;
  const int cblocks = c / 64;
  const int cp = c + ntype;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int j = (int)(i & 63);                       // logical k within the block
    const int64_t rn = i >> 6;
    const int n = (int)(rn % npad);
    const int kb = (int)(rn / npad);
    float v = 0.0f;
    if (n < N) {
      if (kb < cblocks * taps) {
        const int cb = kb / taps, tap = kb - cb * taps;
        v = w[((int64_t)tap * cp + cb * 64 + j) * N + n];
      } else if (j < taps * ntype) {
        const int tap = j / ntype, ty = j - tap * ntype;
        v = w[((int64_t)tap * cp + c + ty) * N + n];
      }
    }
    const int64_t dst = ((int64_t)kb * npad + n) * 64 + ((((j >> 3) ^ (n & 7)) << 3) | (j & 7));
    out[dst] = __float2bfloat16_rn(v);
  }
}

template <int BN>
static int launch_tc(TcParams& p, cudaStream_t st) {
  using Cfg = TcCfg<BN>;
  // the opt-in to > 48 KB of dynamic shared memory is a per-device attribute of the function
  static bool configured[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !configured[dev]) {
    cudaError_t e = cudaFuncSetAttribute(gather_gemm_tc_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
    if (e != cudaSuccess) {
      set_error("of_gather_gemm_tc: cudaFuncSetAttribute(%d B): %s", Cfg::SMEM_BYTES, cudaGetErrorString(e));
      return OF_E_CUDA;
    }
    if (dev >= 0 && dev < 64) configured[dev] = true;
  }
  p.m_tiles = (p.g.M + TC_BM - 1) / TC_BM;
  p.n_tiles = p.npad / BN;
  const int total = p.m_tiles * p.n_tiles * p.ksplit;
  const int grid = total < num_sms() ? total : num_sms();
  gather_gemm_tc_kernel<BN><<<grid, TC_THREADS, Cfg::SMEM_BYTES, st>>>(p);
  OF_LAUNCH_CHECK("of_gather_gemm_tc");
  return OF_OK;
}

static int launch_tc_bn(int bn, TcParams& p, cudaStream_t st) {
  switch (bn) {
    case 256: return launch_tc<256>(p, st);
    case 128: return launch_tc<128>(p, st);
    case 64: return launch_tc<64>(p, st);
    case 32: return launch_tc<32>(p, st);
    default: return launch_tc<16>(p, st);
  }
}

int check_gemm_args(const of_gemm_args* a, const char* who);

}  // namespace of

using namespace of;

extern "C" int64_t of_pack_weight_tc_bytes(int32_t taps, int32_t c, int32_t ntype, int32_t N) {
  if (taps <= 0 || c <= 0 || c % 64 != 0 || N <= 0 || ntype < 0 || taps * ntype > 64) return -1;
  const int64_t num_kb = (int64_t)taps * (c / 64) + (ntype > 0 ? 1 : 0);
  const int64_t npad = (N + 15) / 16 * 16;
  return num_kb * npad * 64 * 2;
}

extern "C" int of_pack_weight_tc(const float* w_canonical, int32_t taps, int32_t c, int32_t ntype, int32_t N,
                                 void* out, void* stream) {
  OF_REQUIRE(w_canonical && out, "of_pack_weight_tc: null pointer");
  OF_REQUIRE(of_pack_weight_tc_bytes(taps, c, ntype, N) > 0, "of_pack_weight_tc: unsupported shape taps=%d c=%d nt=%d N=%d",
             taps, c, ntype, N);
  const int num_kb = taps * (c / 64) + (ntype > 0 ? 1 : 0);
  const int npad = (N + 15) / 16 * 16;
  const int64_t total = (int64_t)num_kb * npad * 64;
  int64_t want = (total + 255) / 256;
  const int64_t cap = (int64_t)num_sms() * 32;
  const int grid = (int)(want < cap ? want : cap);
  pack_weight_tc_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      w_canonical, taps, c, ntype, N, npad, num_kb, reinterpret_cast<__nv_bfloat16*>(out));
  OF_LAUNCH_CHECK("of_pack_weight_tc");
  return OF_OK;
}

// ksplit > 1 (of_gather_gemm_tc_splitk): K is cut into ksplit equal ranges of whole K blocks, the virtual tile (output
// tile, range) writes its fp32 partial sums into slab `range` of args->out ([ksplit][M][N] fp32, no epilogue extras)
static int run_tc(const of_gemm_args* args, int ksplit, void* stream) {
  int rc = check_gemm_args(args, "of_gather_gemm_tc");
  if (rc) return rc;
  const of_gemm_args& a = *args;
  if (a.dtype != OF_BF16 || a.c0 % 64 != 0 || a.c1 % 64 != 0 || a.taps > TC_MAX_TAPS || a.taps * a.ntype > 64 ||
      a.ntype > 8 || a.a_silu) {
    set_error("of_gather_gemm_tc: unsupported (dtype=%d c0=%d c1=%d taps=%d ntype=%d a_silu=%d)", a.dtype, a.c0, a.c1,
              a.taps, a.ntype, a.a_silu);
    return OF_E_UNSUPPORTED;
  }
  if (a.ntype > 0 && a.nt_block == nullptr) {
    set_error("of_gather_gemm_tc: ntype > 0 needs the precomputed node-type block (of_graph_type_block)");
    return OF_E_UNSUPPORTED;
  }
  OF_REQUIRE(a.lda0 % 8 == 0 && (a.c1 == 0 || a.lda1 % 8 == 0), "of_gather_gemm_tc: lda must be a multiple of 8");
  OF_REQUIRE(reinterpret_cast<uintptr_t>(a.a0) % 16 == 0 && reinterpret_cast<uintptr_t>(a.a1) % 16 == 0 &&
                 reinterpret_cast<uintptr_t>(a.w) % 16 == 0,
             "of_gather_gemm_tc: a0/a1/w must be 16-byte aligned");
  if (a.stat_out != nullptr) {
    OF_REQUIRE(a.N % 32 == 0 && a.out_rows == nullptr && a.stat_chunk_seg != nullptr && a.stat_seg_slot != nullptr &&
                   (a.stat_sample != nullptr || a.stat_rows_per_sample > 0),
               "of_gather_gemm_tc: stat_out needs N %% 32 == 0, no out_rows, stat_chunk_seg, stat_seg_slot and a sample map");
  }
  if (a.M == 0) return OF_OK;
  TcParams p;
  p.g = a;
  p.cblocks = (a.c0 + a.c1) / 64;
  p.num_kb = p.cblocks * a.taps + (a.ntype > 0 ? 1 : 0);
  p.ksplit = 1;
  p.npad = (a.N + 15) / 16 * 16;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (ksplit > 1) {
    OF_REQUIRE(p.num_kb % ksplit == 0 && p.npad % 32 == 0 && a.N == p.npad && a.out_rows == nullptr && a.out_f32 == 1 &&
                   a.bias == nullptr && a.row_add == nullptr && a.resid == nullptr && a.stat_out == nullptr,
               "of_gather_gemm_tc_splitk: internal argument error");
    p.ksplit = ksplit;
    p.num_kb /= ksplit;
    return launch_tc_bn(p.npad % 256 == 0 ? 256 : p.npad % 128 == 0 ? 128 : p.npad % 64 == 0 ? 64 : 32, p, st);
  }
  if (p.npad % 32 != 0) return launch_tc<16>(p, st);
  // Small M (the dense 4^3 / 8^3 levels: 2048 / 16384 rows): the widest tile would leave most SMs idle (16 row tiles of 128
  // rows for 132 SMs) with every CTA walking the whole K loop alone.  Take the widest tile shape whose tile count still
  // fills 3/4 of the SMs, else the shape with the most tiles: narrower column tiles re-gather the (L2-resident) rows but
  // split the weight stream and the MMAs over more SMs.  (The statistics granule follows N, not the tile shape.)
  static const int widths[] = {256, 128, 64, 32};
  const int64_t row_tiles = (a.M + TC_BM - 1) / TC_BM;
  const int64_t enough = (int64_t)num_sms() * 3 / 4;
  int bn = 0;
  int64_t best_tiles = -1;
  for (int w : widths) {
    if (p.npad % w != 0) continue;
    const int64_t t = row_tiles * (p.npad / w);
    if (bn == 0) { bn = w; best_tiles = t; }              // the default: the widest shape that divides N
    if (best_tiles >= enough) break;
    if (t > best_tiles) { bn = w; best_tiles = t; }
    if (t >= enough) break;
  }
  return launch_tc_bn(bn, p, st);
}

extern "C" int of_gather_gemm_tc(const of_gemm_args* args, void* stream) { return run_tc(args, 1, stream); }

namespace of {

// Second pass of a split-K GEMM: out[m, :] = sum over the K ranges (in range order: bit-reproducible) of the fp32 partial
// slabs + bias + emb[sample] + residual, stored in the activation dtype, and -- like the single-pass epilogue -- the
// group-norm partial statistics of the fp32 values before rounding.  One CTA per (32-row chunk, 128 columns): warp w owns
// row w of the chunk, lane l its columns 4l..4l+3 (coalesced 16-byte loads of every slab); the per-row (sum, sum of
// squares) of each granule go through shared memory and warp 0 adds the chunk's rows in row order, starting a new
// statistics segment at every change of sample id (the scheme of gn_stats_kernel, csrc/norm.cu).
template <int GRAN>
__global__ void __launch_bounds__(1024) splitk_reduce_kernel(of_gemm_args g, const float* __restrict__ ws, int splits) {
  constexpr int G = 4 / GRAN;                               // granules per thread
  __shared__ float part[32][32][G][2];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t chunk = blockIdx.x;
  const int64_t r = chunk * 32 + w;
  const int cv = blockIdx.y * 128 + lane * 4;
  const bool col_ok = cv < g.N;
  const bool st = g.stat_out != nullptr;
  float sum[G], sq[G];
#pragma unroll
  for (int i = 0; i < G; ++i) { sum[i] = 0.0f; sq[i] = 0.0f; }
  if (r < g.M && col_ok) {
    const int64_t slab = (int64_t)g.M * g.N;
    const float* src = ws + r * g.N + cv;
    float4 v = *reinterpret_cast<const float4*>(src);
    for (int sidx = 1; sidx < splits; ++sidx) {
      const float4 t = *reinterpret_cast<const float4*>(src + sidx * slab);
      v.x += t.x; v.y += t.y; v.z += t.z; v.w += t.w;
    }
    if (g.bias != nullptr) { v.x += g.bias[cv]; v.y += g.bias[cv + 1]; v.z += g.bias[cv + 2]; v.w += g.bias[cv + 3]; }
    if (g.row_add != nullptr) {
      const float* e = g.row_add + (int64_t)g.row_add_idx[r] * g.ld_row_add + cv;
      v.x += e[0]; v.y += e[1]; v.z += e[2]; v.w += e[3];
    }
    if (g.resid != nullptr) {
      const __nv_bfloat16* q = reinterpret_cast<const __nv_bfloat16*>(g.resid) + r * g.ld_resid + cv;
      v.x += __bfloat162float(q[0]); v.y += __bfloat162float(q[1]); v.z += __bfloat162float(q[2]); v.w += __bfloat162float(q[3]);
    }
    if (g.out_f32) {
      float* o = reinterpret_cast<float*>(g.out) + r * g.ldo + cv;
      o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
    } else {
      __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(g.out) + r * g.ldo + cv;
      o[0] = __float2bfloat16_rn(v.x); o[1] = __float2bfloat16_rn(v.y); o[2] = __float2bfloat16_rn(v.z); o[3] = __float2bfloat16_rn(v.w);
    }
    const float f[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) { sum[i / GRAN] += f[i]; sq[i / GRAN] = fmaf(f[i], f[i], sq[i / GRAN]); }
  }
  if (!st) return;
#pragma unroll
  for (int i = 0; i < G; ++i) { part[w][lane][i][0] = sum[i]; part[w][lane][i][1] = sq[i]; }
  __syncthreads();
  if (w != 0 || !col_ok) return;
  const int64_t r0 = chunk * 32;
  const int64_t r1 = r0 + 32 < g.M ? r0 + 32 : (int64_t)g.M;
  const int half = g.N / GRAN * 2;
  auto sample_of = [&](int64_t row) { return g.stat_sample ? g.stat_sample[row] : (int)(row / g.stat_rows_per_sample); };
  int seg = g.stat_chunk_seg[chunk];
  int cur = sample_of(r0);
  float ts[G], tq[G];
#pragma unroll
  for (int i = 0; i < G; ++i) { ts[i] = 0.0f; tq[i] = 0.0f; }
  auto flush = [&]() {
#pragma unroll
    for (int i = 0; i < G; ++i) {
      *reinterpret_cast<float2*>(g.stat_out + (int64_t)g.stat_seg_slot[seg] * half + (cv / GRAN + i) * 2) = make_float2(ts[i], tq[i]);
      ts[i] = 0.0f; tq[i] = 0.0f;
    }
  };
  for (int64_t row = r0; row < r1; ++row) {
    const int b = sample_of(row);
    if (b != cur) { flush(); ++seg; cur = b; }
#pragma unroll
    for (int i = 0; i < G; ++i) { ts[i] += part[row - r0][lane][i][0]; tq[i] += part[row - r0][lane][i][1]; }
  }
  flush();
}

// How many K ranges of_gather_gemm_tc_splitk should use for this launch (1 = do not split): only for launches whose
// 128-row tiles cannot fill half of the SMs, whole K blocks per range, at least 4 per range, at most one wave of CTAs.
static int splitk_plan(const of_gemm_args& a) {
  if (a.dtype != OF_BF16 || a.c0 % 64 != 0 || a.c1 % 64 != 0 || a.N % 32 != 0 || a.out_rows != nullptr || a.M <= 0 ||
      a.a_silu || (a.ntype > 0 && a.nt_block == nullptr))
    return 1;
  const int num_kb = (a.c0 + a.c1) / 64 * a.taps + (a.ntype > 0 ? 1 : 0);
  const int bn = a.N % 256 == 0 ? 256 : a.N % 128 == 0 ? 128 : a.N % 64 == 0 ? 64 : 32;
  const int64_t tiles = (int64_t)((a.M + 127) / 128) * (a.N / bn);
  const int sms = num_sms();
  if (tiles * 2 > sms) return 1;
  int best = 1;
  for (int d = 2; d <= num_kb / 4 && tiles * d <= sms; ++d)
    if (num_kb % d == 0) best = d;
  return best;
}

}  // namespace of

extern "C" int of_tc_splitk_plan(const of_gemm_args* args) {
  if (args == nullptr) return 1;
  return of::splitk_plan(*args);
}

extern "C" int of_gather_gemm_tc_splitk(const of_gemm_args* args, int32_t splits, float* workspace, void* stream) {
  OF_REQUIRE(args != nullptr && workspace != nullptr && splits >= 2, "of_gather_gemm_tc_splitk: bad arguments");
  OF_REQUIRE(splits == of::splitk_plan(*args), "of_gather_gemm_tc_splitk: splits=%d is not the plan for this launch", splits);
  const of_gemm_args& a = *args;
  if (a.stat_out != nullptr) {
    OF_REQUIRE(a.stat_chunk_seg != nullptr && a.stat_seg_slot != nullptr && (a.stat_sample != nullptr || a.stat_rows_per_sample > 0),
               "of_gather_gemm_tc_splitk: stat_out needs stat_chunk_seg, stat_seg_slot and a sample map");
  }
  OF_REQUIRE((a.row_add == nullptr) == (a.row_add_idx == nullptr), "of_gather_gemm_tc_splitk: row_add and row_add_idx go together");
  of_gemm_args part = a;                                   // pass 1: plain fp32 partial sums into the workspace slabs
  part.out = workspace; part.ldo = a.N; part.out_f32 = 1;
  part.bias = nullptr; part.row_add = nullptr; part.row_add_idx = nullptr; part.resid = nullptr; part.stat_out = nullptr;
  int rc = run_tc(&part, splits, stream);
  if (rc) return rc;
  const dim3 grid((unsigned)((a.M + 31) / 32), (unsigned)((a.N + 127) / 128));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (a.N % 128 == 0) of::splitk_reduce_kernel<4><<<grid, 1024, 0, st>>>(a, workspace, splits);
  else of::splitk_reduce_kernel<2><<<grid, 1024, 0, st>>>(a, workspace, splits);
  OF_LAUNCH_CHECK("of_gather_gemm_tc_splitk (reduce)");
  return OF_OK;
}
