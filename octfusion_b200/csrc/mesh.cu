// Meshes and metric point clouds: marching cubes over the calc_sdf grid (reference models/octfusion_model_union.py:
// 435-468, skimage.measure.marching_cubes) and area-weighted surface sampling (metrics/generate_pointclouds.py:14-37,
// trimesh sample_surface).
//
// Marching cubes over one [R, R, R] fp32 grid, sdf[i, j, k] with i (x) slowest.  Grid point p owns the up to three
// edges p -> p + e_axis inside the grid; a crossing edge (one end f < level, the other not) carries one vertex.  Cells
// are the (R-1)^3 cubes, indexed by their lowest corner.  The triangle table comes from the face rule of
// mc_table.py (generated csrc/mc_table.inc).
//
// mc_count_kernel   per grid point: vertex count (crossing edges it owns, 0..3) and triangle count of the cell it
//                   is the lowest corner of (0..5).  Exclusive scans of both (of_exclusive_scan_i32) give every
//                   point its first vertex id and its cell's first face.
// mc_emit_kernel    per grid point: writes its vertices at vertex_scan[p] + rank of the axis among its crossing
//                   edges, then its cell's triangles at tri_scan[p] + table order, each face vertex id read from the
//                   neighbouring point's scan.  No hash, no atomics: the output order is (point, axis) for vertices
//                   and (cell, table order) for faces whatever the launch configuration, so results are
//                   bit-reproducible.
// mesh_bbox_kernel  one CTA per shape: min / max of its vertices.
// area_scan_kernel  one CTA per shape: inclusive fp64 prefix sum of its face areas, in a fixed order.
// sample_kernel     one thread per sample: face by searchsorted(side='left') of u * total area, then a uniform point
//                   of that triangle.  Uniforms come from Philox keyed by (seed, shape, sample).
#include "common.cuh"
#include <curand_kernel.h>

namespace of {

#include "mc_table.inc"

constexpr int MC_THREADS = 256;

__device__ __forceinline__ unsigned is_in(const float* __restrict__ f, int64_t p, float level) {
  return __ldg(f + p) < level ? 1u : 0u;                  // NaN and f == level are outside
}

// lowest corner (x + 2y + 4z) of edge e = 4 * axis + k: k with a 0 bit inserted at position `axis`
__device__ __forceinline__ int edge_corner(int e) {
  const int a = e >> 2, k = e & 3;
  return ((k >> a) << (a + 1)) | (k & ((1 << a) - 1));
}

// bits 0..7: inside-ness of the cell corners that exist inside the grid (x + 2y + 4z), for the point (i, j, k)
__device__ __forceinline__ unsigned corner_mask(const float* __restrict__ f, int R, int i, int j, int k, int64_t p,
                                                float level) {
  const int64_t RR = (int64_t)R * R;
  const bool hx = i + 1 < R, hy = j + 1 < R, hz = k + 1 < R;
  unsigned m = is_in(f, p, level);
  if (hx) m |= is_in(f, p + RR, level) << 1;
  if (hy) m |= is_in(f, p + R, level) << 2;
  if (hz) m |= is_in(f, p + 1, level) << 4;
  if (hx && hy && hz) {
    m |= is_in(f, p + RR + R, level) << 3;
    m |= is_in(f, p + RR + 1, level) << 5;
    m |= is_in(f, p + R + 1, level) << 6;
    m |= is_in(f, p + RR + R + 1, level) << 7;
  }
  return m;
}

// crossing-edge bits (x, y, z) of the point with corner mask m
__device__ __forceinline__ unsigned edge_bits(unsigned m, int R, int i, int j, int k) {
  return ((i + 1 < R) & ((m ^ (m >> 1)) & 1u)) | (((j + 1 < R) & ((m ^ (m >> 2)) & 1u)) << 1) |
         (((k + 1 < R) & ((m ^ (m >> 4)) & 1u)) << 2);
}

__global__ void __launch_bounds__(MC_THREADS) mc_count_kernel(const float* __restrict__ f, int R, float level,
                                                              int32_t* __restrict__ vcount, int32_t* __restrict__ tcount) {
  const int64_t n = (int64_t)R * R * R;
  const int64_t p = (int64_t)blockIdx.x * MC_THREADS + threadIdx.x;
  if (p >= n) return;
  const int k = (int)(p % R), j = (int)((p / R) % R), i = (int)(p / ((int64_t)R * R));
  const unsigned m = corner_mask(f, R, i, j, k, p, level);
  vcount[p] = __popc(edge_bits(m, R, i, j, k));
  tcount[p] = (i + 1 < R && j + 1 < R && k + 1 < R) ? __ldg(kMcTriCount + m) : 0;
}

// vertex id of edge `axis` of point (i, j, k): its first id plus the crossing edges it owns on lower axes
__device__ __forceinline__ int32_t vertex_id(const float* __restrict__ f, const int32_t* __restrict__ vscan, int R,
                                             float level, int i, int j, int k, int axis) {
  const int64_t p = ((int64_t)i * R + j) * R + k;
  int32_t id = __ldg(vscan + p);
  if (axis > 0) {
    const unsigned in = is_in(f, p, level);
    if (i + 1 < R) id += (int32_t)(in ^ is_in(f, p + (int64_t)R * R, level));
    if (axis > 1 && j + 1 < R) id += (int32_t)(in ^ is_in(f, p + R, level));
  }
  return id;
}

__global__ void __launch_bounds__(MC_THREADS) mc_emit_kernel(const float* __restrict__ f, int R, float level,
                                                             const int32_t* __restrict__ vscan,
                                                             const int32_t* __restrict__ tscan,
                                                             float* __restrict__ verts, int32_t* __restrict__ faces) {
  const int64_t RR = (int64_t)R * R, n = RR * R;
  const int64_t p = (int64_t)blockIdx.x * MC_THREADS + threadIdx.x;
  if (p >= n) return;
  const int k = (int)(p % R), j = (int)((p / R) % R), i = (int)(p / RR);
  const unsigned m = corner_mask(f, R, i, j, k, p, level);
  const unsigned eb = edge_bits(m, R, i, j, k);
  if (eb) {
    const float fa = __ldg(f + p);
    int32_t v = __ldg(vscan + p);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (!(eb >> a & 1u)) continue;
      const float fb = __ldg(f + p + (a == 0 ? RR : a == 1 ? (int64_t)R : 1));
      // a is the lower-index end, so the two cells sharing the edge see one value
      const float t = __fdiv_rn(__fsub_rn(level, fa), __fsub_rn(fb, fa));
      float* o = verts + (int64_t)v * 3;
      o[0] = a == 0 ? __fadd_rn((float)i, t) : (float)i;
      o[1] = a == 1 ? __fadd_rn((float)j, t) : (float)j;
      o[2] = a == 2 ? __fadd_rn((float)k, t) : (float)k;
      ++v;
    }
  }
  if (i + 1 >= R || j + 1 >= R || k + 1 >= R) return;
  const int nt = __ldg(kMcTriCount + m);
  if (nt == 0) return;
  int32_t* o = faces + (int64_t)__ldg(tscan + p) * 3;
  const signed char* te = &kMcTriEdges[m][0][0];
  for (int t = 0; t < nt * 3; ++t) {
    const int e = __ldg(te + t), c = edge_corner(e);
    o[t] = vertex_id(f, vscan, R, level, i + (c & 1), j + (c >> 1 & 1), k + (c >> 2), e >> 2);
  }
}

constexpr int MESH_THREADS = 256;

__global__ void __launch_bounds__(MESH_THREADS) mesh_bbox_kernel(const float* __restrict__ verts,
                                                                 const int64_t* __restrict__ voff,
                                                                 float* __restrict__ bbox) {
  __shared__ float red[6][MESH_THREADS / 32];
  const int b = blockIdx.x;
  const int64_t v0 = voff[b], v1 = voff[b + 1];
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int64_t v = v0 + threadIdx.x; v < v1; v += MESH_THREADS)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float x = verts[v * 3 + c];
      lo[c] = fminf(lo[c], x);
      hi[c] = fmaxf(hi[c], x);
    }
#pragma unroll
  for (int c = 0; c < 3; ++c)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lo[c] = fminf(lo[c], __shfl_xor_sync(0xffffffffu, lo[c], o));
      hi[c] = fmaxf(hi[c], __shfl_xor_sync(0xffffffffu, hi[c], o));
    }
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      red[c][threadIdx.x >> 5] = lo[c];
      red[3 + c][threadIdx.x >> 5] = hi[c];
    }
  __syncthreads();
  if (threadIdx.x < 6) {
    const int c = threadIdx.x;
    float r = red[c][0];
    for (int w = 1; w < MESH_THREADS / 32; ++w) r = c < 3 ? fminf(r, red[c][w]) : fmaxf(r, red[c][w]);
    bbox[b * 6 + c] = r;
  }
}

constexpr int AREA_ITEMS = 8;

__device__ __forceinline__ double face_area(const float* __restrict__ v, const int32_t* __restrict__ tri) {
  const int32_t a = tri[0], b = tri[1], c = tri[2];
  const double ax = v[a * 3], ay = v[a * 3 + 1], az = v[a * 3 + 2];
  const double ux = v[b * 3] - ax, uy = v[b * 3 + 1] - ay, uz = v[b * 3 + 2] - az;
  const double wx = v[c * 3] - ax, wy = v[c * 3 + 1] - ay, wz = v[c * 3 + 2] - az;
  const double cx = uy * wz - uz * wy, cy = uz * wx - ux * wz, cz = ux * wy - uy * wx;
  return 0.5 * sqrt(cx * cx + cy * cy + cz * cz);
}

// inclusive prefix sum of the face areas of shape blockIdx.x: each thread sums AREA_ITEMS consecutive faces in order,
// the per-thread totals are scanned across the block (shuffles, then the warps in order) and carried between chunks
__global__ void __launch_bounds__(MESH_THREADS) area_scan_kernel(const float* __restrict__ verts,
                                                                 const int64_t* __restrict__ voff,
                                                                 const int32_t* __restrict__ faces,
                                                                 const int64_t* __restrict__ foff,
                                                                 double* __restrict__ cum) {
  __shared__ double warp_tot[MESH_THREADS / 32];
  __shared__ double carry_s;
  const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* v = verts + voff[b] * 3;
  const int64_t f0 = foff[b], nf = foff[b + 1] - f0;
  double carry = 0.0;
  for (int64_t c0 = 0; c0 < nf; c0 += (int64_t)MESH_THREADS * AREA_ITEMS) {
    const int64_t base = c0 + (int64_t)threadIdx.x * AREA_ITEMS;
    double run[AREA_ITEMS];
    double s = 0.0;
#pragma unroll
    for (int t = 0; t < AREA_ITEMS; ++t) {
      if (base + t < nf) s += face_area(v, faces + (f0 + base + t) * 3);
      run[t] = s;
    }
    double incl = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double u = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += u;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    if (threadIdx.x == 0) {
      double acc = carry;
      for (int w = 0; w < MESH_THREADS / 32; ++w) {
        const double t = warp_tot[w];
        warp_tot[w] = acc;
        acc += t;
      }
      carry_s = acc;
    }
    __syncthreads();
    const double off = warp_tot[warp] + (incl - s);
#pragma unroll
    for (int t = 0; t < AREA_ITEMS; ++t)
      if (base + t < nf) cum[f0 + base + t] = off + run[t];
    carry = carry_s;
    __syncthreads();
  }
}

__global__ void __launch_bounds__(MESH_THREADS) sample_kernel(const float* __restrict__ verts,
                                                              const int64_t* __restrict__ voff,
                                                              const int32_t* __restrict__ faces,
                                                              const int64_t* __restrict__ foff,
                                                              const double* __restrict__ cum, int batch, int count,
                                                              unsigned long long seed, float* __restrict__ points,
                                                              int32_t* __restrict__ face_index) {
  const int64_t g = (int64_t)blockIdx.x * MESH_THREADS + threadIdx.x;
  if (g >= (int64_t)batch * count) return;
  const int b = (int)(g / count), s = (int)(g % count);
  const int64_t f0 = foff[b], nf = foff[b + 1] - f0;
  float* o = points + g * 3;
  if (nf == 0) {
    o[0] = o[1] = o[2] = __int_as_float(0x7fc00000);
    face_index[g] = -1;
    return;
  }
  curandStatePhilox4_32_10_t st;
  curand_init(seed, ((unsigned long long)b << 32) | (unsigned)s, 0, &st);
  const uint4 r = curand4(&st);
  const double u = _curand_uniform_double_hq(r.x, r.y);          // (0, 1]
  float r1 = _curand_uniform(r.z), r2 = _curand_uniform(r.w);
  const double* c = cum + f0;
  const double x = u * c[nf - 1];
  int64_t lo = 0, hi = nf - 1;                                   // first face with cum >= x (x <= cum[nf - 1])
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (c[mid] < x) lo = mid + 1;
    else hi = mid;
  }
  if (r1 + r2 > 1.0f) {
    r1 = fabsf(r1 - 1.0f);
    r2 = fabsf(r2 - 1.0f);
  }
  const int32_t* tri = faces + (f0 + lo) * 3;
  const float* v = verts + voff[b] * 3;
  const float* a = v + (int64_t)tri[0] * 3;
  const float* p = v + (int64_t)tri[1] * 3;
  const float* q = v + (int64_t)tri[2] * 3;
#pragma unroll
  for (int d = 0; d < 3; ++d) o[d] = a[d] + r1 * (p[d] - a[d]) + r2 * (q[d] - a[d]);
  face_index[g] = (int32_t)lo;
}

}  // namespace of

extern "C" int of_mc_count(const float* sdf, int32_t size, float level, int32_t* vert_count, int32_t* tri_count,
                           void* stream) {
  using namespace of;
  OF_REQUIRE(sdf && vert_count && tri_count, "of_mc_count: null pointer");
  OF_REQUIRE(size >= 2 && size <= OF_MC_MAX_SIZE, "of_mc_count: need 2 <= size <= %d (got %d)", OF_MC_MAX_SIZE, size);
  const int64_t n = (int64_t)size * size * size;
  mc_count_kernel<<<(unsigned)((n + MC_THREADS - 1) / MC_THREADS), MC_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      sdf, size, level, vert_count, tri_count);
  OF_LAUNCH_CHECK("of_mc_count");
  return OF_OK;
}

extern "C" int of_mc_emit(const float* sdf, int32_t size, float level, const int32_t* vert_scan, const int32_t* tri_scan,
                          float* verts, int32_t* faces, void* stream) {
  using namespace of;
  OF_REQUIRE(sdf && vert_scan && tri_scan && verts && faces, "of_mc_emit: null pointer");
  OF_REQUIRE(size >= 2 && size <= OF_MC_MAX_SIZE, "of_mc_emit: need 2 <= size <= %d (got %d)", OF_MC_MAX_SIZE, size);
  const int64_t n = (int64_t)size * size * size;
  mc_emit_kernel<<<(unsigned)((n + MC_THREADS - 1) / MC_THREADS), MC_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      sdf, size, level, vert_scan, tri_scan, verts, faces);
  OF_LAUNCH_CHECK("of_mc_emit");
  return OF_OK;
}

extern "C" int of_mesh_bbox(const float* verts, const int64_t* vert_offsets, int32_t batch, float* bbox, void* stream) {
  using namespace of;
  OF_REQUIRE(verts && vert_offsets && bbox, "of_mesh_bbox: null pointer");
  OF_REQUIRE(batch >= 0, "of_mesh_bbox: need batch >= 0 (got %d)", batch);
  if (batch == 0) return OF_OK;
  mesh_bbox_kernel<<<batch, MESH_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(verts, vert_offsets, bbox);
  OF_LAUNCH_CHECK("of_mesh_bbox");
  return OF_OK;
}

extern "C" int of_surface_sample(const float* verts, const int64_t* vert_offsets, const int32_t* faces,
                                 const int64_t* face_offsets, int32_t batch, int32_t count, uint64_t seed,
                                 double* area_scan, float* points, int32_t* face_index, void* stream) {
  using namespace of;
  OF_REQUIRE(verts && vert_offsets && faces && face_offsets && area_scan && points && face_index,
             "of_surface_sample: null pointer");
  OF_REQUIRE(batch >= 0 && count >= 1, "of_surface_sample: need batch >= 0 and count >= 1 (got %d, %d)", batch, count);
  if (batch == 0) return OF_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  area_scan_kernel<<<batch, MESH_THREADS, 0, st>>>(verts, vert_offsets, faces, face_offsets, area_scan);
  const int64_t n = (int64_t)batch * count;
  sample_kernel<<<(unsigned)((n + MESH_THREADS - 1) / MESH_THREADS), MESH_THREADS, 0, st>>>(
      verts, vert_offsets, faces, face_offsets, area_scan, batch, count, (unsigned long long)seed, points, face_index);
  add_launches(1);
  OF_LAUNCH_CHECK("of_surface_sample");
  return OF_OK;
}
