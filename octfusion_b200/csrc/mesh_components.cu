// Connected components of triangle meshes and the largest-component filter of export_mesh(clean=True) (reference
// models/octfusion_model_union.py:459-466: trimesh `split(only_watertight=False)`, then the component whose vertex
// bounding box has the largest extent).  The rules are restated in DESIGN.md §4.6; parity is unpinned at the trimesh
// boundary.
//
// One shape per call, scratch laid out from that shape's (nverts, nfaces) (of_mesh_components_bytes):
//   weld_insert_kernel  per vertex: open-addressing table keyed by the bit pattern of (x, y, z).  The slot keeps the
//                       smallest vertex id of its position (atomicMin), whatever order the inserts run in.
//   weld_find_kernel    canon[v] = that smallest id.
//   edge_insert_kernel  per face: its 3 edges on welded ids, key (min << 32) | max, in a second table; the key's count
//                       is an atomicAdd whose old value puts the first two faces into the slot's two face fields.
//   union_kernel        per slot with count exactly 2: lock-free union of its two faces, always hooking the larger
//                       root under the smaller (atomicCAS), so the final root of a component is its smallest face.
//   label_kernel        labels[f] = root of f; roots are counted.
//   bounds_kernel       per component: atomicMin / atomicMax of the order-preserving uint32 encoding of the
//                       coordinates of its faces' vertices (reduced per lane run and per warp first).
//   extent_kernel       per root: extent = max over axes of double(max) - double(min); the shape's largest extent by
//                       atomicMax on its fp64 bits (non-negative doubles order like their bits),
//   select_kernel       then the smallest root with exactly that extent by atomicMin.
//   mark_kernel         per face of the kept component: flags its welded vertices and counts the face.
//   vert_map_kernel     after an exclusive scan of the flags: vert_map[v] = new id of canon[v], or -1.
//   keep_flags_kernel, compact_faces_kernel, compact_verts_kernel
//                       after the caller has read the sizes: kept faces in order (exclusive scan of label == kept),
//                       vertices to their vert_map ids.
// Only integer atomics: every result is a function of the input alone, bit for bit, whatever the launch configuration.
#include "common.cuh"

namespace of {

constexpr int CC_T = 256;
constexpr int CC_RUN = 8;                      // faces per lane in bounds_kernel
constexpr int32_t CC_EMPTY_V = -1;
constexpr uint64_t CC_EMPTY_E = ~0ull;         // no valid key: ids are < 2^31

static inline size_t cc_align(size_t v) { return (v + 255) & ~(size_t)255; }

struct CcHeader {
  unsigned long long best_ext;                 // fp64 bits of the largest extent
  int32_t best_label;
  int32_t kept_faces;
};

// scratch layout of one shape, a pure function of (nverts, nfaces) and monotone in both
struct CcLayout {
  int64_t vcap, ecap, n;
  size_t hdr, vtab, canon, ekey, ecnt, eface, parent, blo, bhi, flags, scan, scan_tmp, total;
};

static CcLayout cc_layout(int64_t nv, int64_t nf) {
  CcLayout L;
  L.vcap = 2 * nv + 1;                          // load <= 1/2
  L.ecap = 4 * nf + 1;                          // <= 3 nf distinct edges: load <= 3/4 (3/8 on a closed mesh)
  L.n = nv > nf ? nv : nf;
  size_t off = 0;
  L.hdr = off; off += cc_align(sizeof(CcHeader));
  L.vtab = off; off += cc_align((size_t)L.vcap * 4);
  L.canon = off; off += cc_align((size_t)nv * 4);
  L.ekey = off; off += cc_align((size_t)L.ecap * 8);
  L.ecnt = off; off += cc_align((size_t)L.ecap * 4);
  L.eface = off; off += cc_align((size_t)L.ecap * 8);
  L.parent = off; off += cc_align((size_t)nf * 4);
  L.blo = off; off += cc_align((size_t)nf * 12);
  L.bhi = off; off += cc_align((size_t)nf * 12);
  L.flags = off; off += cc_align((size_t)L.n * 4);
  L.scan = off; off += cc_align((size_t)(L.n + 1) * 4);
  L.scan_tmp = off; off += cc_align((size_t)of_scan_scratch_bytes(L.n));
  L.total = off;
  return L;
}

template <typename T> static inline T* at(void* base, size_t off) {
  return reinterpret_cast<T*>(static_cast<char*>(base) + off);
}

__device__ __forceinline__ uint64_t mix64(uint64_t h) {
  h ^= h >> 33; h *= 0xff51afd7ed558ccdull;
  h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ull;
  h ^= h >> 33;
  return h;
}

// slot of a hash in [0, cap)
__device__ __forceinline__ int64_t home(uint64_t h, int64_t cap) { return (int64_t)__umul64hi(h, (uint64_t)cap); }

__device__ __forceinline__ uint64_t vert_hash(uint32_t x, uint32_t y, uint32_t z) {
  return mix64(mix64(((uint64_t)x << 32) | y) ^ z);
}

__device__ __forceinline__ bool same_bits(const float* __restrict__ verts, int32_t o, uint32_t x, uint32_t y, uint32_t z) {
  const float* p = verts + (int64_t)o * 3;
  return __float_as_uint(p[0]) == x && __float_as_uint(p[1]) == y && __float_as_uint(p[2]) == z;
}

// the three vertex ids of face f, false when one lies outside [0, nv)
__device__ __forceinline__ bool load_face(const int32_t* __restrict__ faces, int64_t f, int nv, int32_t* id) {
  bool ok = true;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    id[k] = faces[f * 3 + k];
    ok &= (unsigned)id[k] < (unsigned)nv;
  }
  return ok;
}

// order-preserving uint32 encoding of a non-NaN float, and back
__device__ __forceinline__ uint32_t ord_f32(float x) {
  const uint32_t u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float unord_f32(uint32_t u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

__global__ void __launch_bounds__(CC_T) weld_insert_kernel(const float* __restrict__ verts, int nv, int64_t vcap,
                                                           int32_t* __restrict__ vtab, int32_t* __restrict__ status) {
  const int64_t v = (int64_t)blockIdx.x * CC_T + threadIdx.x;
  if (v >= nv) return;
  const float* p = verts + v * 3;
  if (!(isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]))) atomicOr(status, 1);
  const uint32_t x = __float_as_uint(p[0]), y = __float_as_uint(p[1]), z = __float_as_uint(p[2]);
  for (int64_t s = home(vert_hash(x, y, z), vcap);; s = s + 1 == vcap ? 0 : s + 1) {
    const int32_t old = atomicCAS(vtab + s, CC_EMPTY_V, (int32_t)v);
    if (old == CC_EMPTY_V) break;
    if (same_bits(verts, old, x, y, z)) {       // every id in the slot has these bits, so the slot stays valid
      atomicMin(vtab + s, (int32_t)v);
      break;
    }
  }
}

__global__ void __launch_bounds__(CC_T) weld_find_kernel(const float* __restrict__ verts, int nv, int64_t vcap,
                                                         const int32_t* __restrict__ vtab, int32_t* __restrict__ canon) {
  const int64_t v = (int64_t)blockIdx.x * CC_T + threadIdx.x;
  if (v >= nv) return;
  const float* p = verts + v * 3;
  const uint32_t x = __float_as_uint(p[0]), y = __float_as_uint(p[1]), z = __float_as_uint(p[2]);
  // v itself was inserted: no empty slot lies between the home slot and the position's slot
  for (int64_t s = home(vert_hash(x, y, z), vcap);; s = s + 1 == vcap ? 0 : s + 1) {
    const int32_t o = vtab[s];
    if (same_bits(verts, o, x, y, z)) {
      canon[v] = o;
      return;
    }
  }
}

__global__ void __launch_bounds__(CC_T) edge_insert_kernel(const int32_t* __restrict__ faces, int nf, int nv,
                                                           const int32_t* __restrict__ canon, int64_t ecap,
                                                           unsigned long long* __restrict__ ekey,
                                                           int32_t* __restrict__ ecnt, int32_t* __restrict__ eface,
                                                           int32_t* __restrict__ parent, int32_t* __restrict__ status) {
  const int64_t f = (int64_t)blockIdx.x * CC_T + threadIdx.x;
  if (f >= nf) return;
  parent[f] = (int32_t)f;
  int32_t id[3];
  if (!load_face(faces, f, nv, id)) {
    atomicOr(status, 2);
    return;
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) id[k] = canon[id[k]];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const uint32_t a = (uint32_t)id[k], b = (uint32_t)id[k == 2 ? 0 : k + 1];
    const unsigned long long key = a < b ? ((uint64_t)a << 32) | b : ((uint64_t)b << 32) | a;
    int64_t s = home(mix64(key), ecap);
    for (;; s = s + 1 == ecap ? 0 : s + 1) {
      const unsigned long long old = atomicCAS(ekey + s, CC_EMPTY_E, key);
      if (old == CC_EMPTY_E || old == key) break;
    }
    const int32_t c = atomicAdd(ecnt + s, 1);
    if (c < 2) eface[2 * s + c] = (int32_t)f;
  }
}

// root of x.  parent[x] <= x always holds and only decreases; roots are written only by the CAS of unite, and the
// halving stores only write non-roots, each with one of its ancestors.
__device__ __forceinline__ int32_t find_root(int32_t* parent, int32_t x) {
  volatile int32_t* p = parent;
  int32_t cur = p[x];
  if (cur != x) {
    int32_t prev = x, next;
    while (cur > (next = p[cur])) {
      p[prev] = next;
      prev = cur;
      cur = next;
    }
  }
  return cur;
}

__device__ void unite(int32_t* parent, int32_t a, int32_t b) {
  int32_t ra = find_root(parent, a), rb = find_root(parent, b);
  while (ra != rb) {
    if (ra < rb) { const int32_t t = ra; ra = rb; rb = t; }
    const int32_t old = atomicCAS(parent + ra, ra, rb);     // hook the larger root under the smaller
    if (old == ra) return;
    ra = find_root(parent, old);                            // ra was hooked meanwhile: retry from both roots
    rb = find_root(parent, rb);
  }
}

__global__ void __launch_bounds__(CC_T) union_kernel(int64_t ecap, const int32_t* __restrict__ ecnt,
                                                     const int32_t* __restrict__ eface, int32_t* parent) {
  const int64_t s = (int64_t)blockIdx.x * CC_T + threadIdx.x;
  if (s >= ecap || ecnt[s] != 2) return;
  unite(parent, eface[2 * s], eface[2 * s + 1]);
}

__global__ void __launch_bounds__(CC_T) label_kernel(int nf, int32_t* parent, int32_t* __restrict__ labels,
                                                     int32_t* __restrict__ ncomp) {
  const int64_t f = (int64_t)blockIdx.x * CC_T + threadIdx.x;
  bool root = false;
  if (f < nf) {
    const int32_t r = find_root(parent, (int32_t)f);
    labels[f] = r;
    root = r == f;
  }
  const int n = __syncthreads_count(root);
  if (threadIdx.x == 0 && n) atomicAdd(ncomp, n);
}

__device__ __forceinline__ void flush_bounds(uint32_t* __restrict__ blo, uint32_t* __restrict__ bhi, int32_t l,
                                             const uint32_t* lo, const uint32_t* hi) {
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    atomicMin(blo + (int64_t)l * 3 + a, lo[a]);
    atomicMax(bhi + (int64_t)l * 3 + a, hi[a]);
  }
}

// one warp per 32 * CC_RUN consecutive faces, lane-strided.  A lane keeps a running box while the label stays the
// same, and a warp whose lanes all end on one label reduces before the atomics: a large component costs few atomics.
__global__ void __launch_bounds__(CC_T) bounds_kernel(const float* __restrict__ verts, const int32_t* __restrict__ faces,
                                                      int nf, int nv, const int32_t* __restrict__ labels,
                                                      uint32_t* __restrict__ blo, uint32_t* __restrict__ bhi) {
  const int lane = threadIdx.x & 31;
  const int64_t base = ((int64_t)blockIdx.x * (CC_T / 32) + (threadIdx.x >> 5)) * (32 * CC_RUN);
  if (base >= nf) return;                                   // whole warps leave together
  int32_t cur = -1;
  uint32_t lo[3] = {~0u, ~0u, ~0u}, hi[3] = {0u, 0u, 0u};
  for (int r = 0; r < CC_RUN; ++r) {
    const int64_t f = base + (int64_t)r * 32 + lane;
    if (f >= nf) break;
    int32_t id[3];
    if (!load_face(faces, f, nv, id)) continue;
    const int32_t l = labels[f];
    if (l != cur) {
      if (cur >= 0) flush_bounds(blo, bhi, cur, lo, hi);
      cur = l;
#pragma unroll
      for (int a = 0; a < 3; ++a) { lo[a] = ~0u; hi[a] = 0u; }
    }
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        const uint32_t e = ord_f32(verts[(int64_t)id[k] * 3 + a]);
        lo[a] = min(lo[a], e);
        hi[a] = max(hi[a], e);
      }
  }
  const int32_t first = __shfl_sync(0xffffffffu, cur, 0);
  if (__all_sync(0xffffffffu, cur == first || cur < 0)) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      lo[a] = __reduce_min_sync(0xffffffffu, lo[a]);
      hi[a] = __reduce_max_sync(0xffffffffu, hi[a]);
    }
    if (lane == 0 && first >= 0) flush_bounds(blo, bhi, first, lo, hi);
  } else if (cur >= 0) {
    flush_bounds(blo, bhi, cur, lo, hi);
  }
}

__device__ __forceinline__ unsigned long long extent_bits(const uint32_t* __restrict__ blo,
                                                          const uint32_t* __restrict__ bhi, int64_t l) {
  double e = 0.0;
#pragma unroll
  for (int a = 0; a < 3; ++a)
    e = fmax(e, (double)unord_f32(bhi[l * 3 + a]) - (double)unord_f32(blo[l * 3 + a]));
  return (unsigned long long)__double_as_longlong(e);
}

__global__ void __launch_bounds__(CC_T) extent_kernel(int nf, const int32_t* __restrict__ labels,
                                                      const uint32_t* __restrict__ blo, const uint32_t* __restrict__ bhi,
                                                      CcHeader* __restrict__ hdr) {
  const int64_t f = (int64_t)blockIdx.x * CC_T + threadIdx.x;
  unsigned long long e = 0;
  if (f < nf && labels[f] == f) e = extent_bits(blo, bhi, f);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long u = __shfl_xor_sync(0xffffffffu, e, o);
    e = u > e ? u : e;
  }
  if ((threadIdx.x & 31) == 0 && e) atomicMax(&hdr->best_ext, e);
}

__global__ void __launch_bounds__(CC_T) select_kernel(int nf, const int32_t* __restrict__ labels,
                                                      const uint32_t* __restrict__ blo, const uint32_t* __restrict__ bhi,
                                                      CcHeader* __restrict__ hdr) {
  const int64_t f = (int64_t)blockIdx.x * CC_T + threadIdx.x;
  if (f >= nf || labels[f] != f) return;
  if (extent_bits(blo, bhi, f) == hdr->best_ext) atomicMin(&hdr->best_label, (int32_t)f);
}

__global__ void __launch_bounds__(CC_T) mark_kernel(const int32_t* __restrict__ faces, int nf, int nv,
                                                    const int32_t* __restrict__ labels,
                                                    const int32_t* __restrict__ canon, int32_t* __restrict__ flags,
                                                    CcHeader* __restrict__ hdr) {
  const int64_t f = (int64_t)blockIdx.x * CC_T + threadIdx.x;
  bool kept = false;
  if (f < nf && labels[f] == hdr->best_label) {
    int32_t id[3];
    if (load_face(faces, f, nv, id)) {
      kept = true;
#pragma unroll
      for (int k = 0; k < 3; ++k) flags[canon[id[k]]] = 1;
    }
  }
  const int n = __syncthreads_count(kept);
  if (threadIdx.x == 0 && n) atomicAdd(&hdr->kept_faces, n);
}

__global__ void __launch_bounds__(CC_T) vert_map_kernel(int nv, const int32_t* __restrict__ canon,
                                                        const int32_t* __restrict__ flags,
                                                        const int32_t* __restrict__ scan,
                                                        const CcHeader* __restrict__ hdr, int32_t* __restrict__ vert_map,
                                                        int32_t* __restrict__ info) {
  const int64_t v = (int64_t)blockIdx.x * CC_T + threadIdx.x;
  if (v == 0) {
    info[2] = hdr->best_label;
    info[3] = hdr->kept_faces;
  }
  if (v >= nv) return;
  const int32_t c = canon[v];
  vert_map[v] = flags[c] ? scan[c] : -1;
}

__global__ void cc_header_kernel(CcHeader* hdr) {
  hdr->best_ext = 0;
  hdr->best_label = 0x7fffffff;
  hdr->kept_faces = 0;
}

__global__ void __launch_bounds__(CC_T) keep_flags_kernel(int nf, const int32_t* __restrict__ labels, int32_t label,
                                                          int32_t* __restrict__ flags) {
  const int64_t f = (int64_t)blockIdx.x * CC_T + threadIdx.x;
  if (f < nf) flags[f] = labels[f] == label;
}

__global__ void __launch_bounds__(CC_T) compact_faces_kernel(const int32_t* __restrict__ faces, int nf, int nv,
                                                             const int32_t* __restrict__ flags,
                                                             const int32_t* __restrict__ scan,
                                                             const int32_t* __restrict__ vert_map,
                                                             int32_t* __restrict__ out_faces) {
  const int64_t f = (int64_t)blockIdx.x * CC_T + threadIdx.x;
  if (f >= nf || !flags[f]) return;
  int32_t* o = out_faces + (int64_t)scan[f] * 3;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int32_t v = faces[f * 3 + k];
    o[k] = (unsigned)v < (unsigned)nv ? vert_map[v] : -1;
  }
}

// vertices welded together map to one id and carry the same bits, so their identical stores race harmlessly
__global__ void __launch_bounds__(CC_T) compact_verts_kernel(const float* __restrict__ verts, int nv,
                                                             const int32_t* __restrict__ vert_map,
                                                             float* __restrict__ out_verts) {
  const int64_t v = (int64_t)blockIdx.x * CC_T + threadIdx.x;
  if (v >= nv) return;
  const int32_t k = vert_map[v];
  if (k < 0) return;
#pragma unroll
  for (int a = 0; a < 3; ++a) out_verts[(int64_t)k * 3 + a] = verts[v * 3 + a];
}

static inline unsigned cc_blocks(int64_t n) { return (unsigned)((n + CC_T - 1) / CC_T); }

}  // namespace of

using namespace of;

extern "C" int64_t of_mesh_components_bytes(int64_t nverts, int64_t nfaces) {
  OF_REQUIRE(nverts >= 0 && nfaces >= 0 && nverts < ((int64_t)1 << 31) && nfaces < ((int64_t)1 << 31),
             "of_mesh_components_bytes: need 0 <= nverts, nfaces < 2^31 (got %lld, %lld)", (long long)nverts,
             (long long)nfaces);
  return (int64_t)cc_layout(nverts, nfaces).total;
}

extern "C" int of_mesh_components(const float* verts, int32_t nverts, const int32_t* faces, int32_t nfaces,
                                  void* scratch, int32_t* labels, int32_t* info, void* stream) {
  OF_REQUIRE(scratch && info && (verts || nverts == 0) && ((faces && labels) || nfaces == 0),
             "of_mesh_components: null pointer");
  OF_REQUIRE(nverts >= 0 && nfaces >= 0, "of_mesh_components: need nverts, nfaces >= 0 (got %d, %d)", nverts, nfaces);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const CcLayout L = cc_layout(nverts, nfaces);
  if (cudaMemsetAsync(info, 0, 2 * sizeof(int32_t), st) != cudaSuccess) {
    set_error("of_mesh_components: cudaMemsetAsync failed");
    return OF_E_CUDA;
  }
  if (nverts > 0) {
    int32_t* vtab = at<int32_t>(scratch, L.vtab);
    if (cudaMemsetAsync(vtab, 0xff, (size_t)L.vcap * 4, st) != cudaSuccess) {
      set_error("of_mesh_components: cudaMemsetAsync failed");
      return OF_E_CUDA;
    }
    weld_insert_kernel<<<cc_blocks(nverts), CC_T, 0, st>>>(verts, nverts, L.vcap, vtab, info);
    weld_find_kernel<<<cc_blocks(nverts), CC_T, 0, st>>>(verts, nverts, L.vcap, vtab, at<int32_t>(scratch, L.canon));
    add_launches(1);
    OF_LAUNCH_CHECK("of_mesh_components");
  }
  if (nfaces > 0) {
    unsigned long long* ekey = at<unsigned long long>(scratch, L.ekey);
    int32_t* ecnt = at<int32_t>(scratch, L.ecnt);
    int32_t* eface = at<int32_t>(scratch, L.eface);
    int32_t* parent = at<int32_t>(scratch, L.parent);
    if (cudaMemsetAsync(ekey, 0xff, (size_t)L.ecap * 8, st) != cudaSuccess ||
        cudaMemsetAsync(ecnt, 0, (size_t)L.ecap * 4, st) != cudaSuccess) {
      set_error("of_mesh_components: cudaMemsetAsync failed");
      return OF_E_CUDA;
    }
    edge_insert_kernel<<<cc_blocks(nfaces), CC_T, 0, st>>>(faces, nfaces, nverts, at<int32_t>(scratch, L.canon),
                                                           L.ecap, ekey, ecnt, eface, parent, info);
    union_kernel<<<cc_blocks(L.ecap), CC_T, 0, st>>>(L.ecap, ecnt, eface, parent);
    label_kernel<<<cc_blocks(nfaces), CC_T, 0, st>>>(nfaces, parent, labels, info + 1);
    add_launches(2);
    OF_LAUNCH_CHECK("of_mesh_components");
  }
  return OF_OK;
}

extern "C" int of_mesh_largest_component(const float* verts, int32_t nverts, const int32_t* faces, int32_t nfaces,
                                         void* scratch, const int32_t* labels, int32_t* vert_map, int32_t* info,
                                         void* stream) {
  OF_REQUIRE(scratch && info && ((verts && vert_map) || nverts == 0) && ((faces && labels) || nfaces == 0),
             "of_mesh_largest_component: null pointer");
  OF_REQUIRE(nverts >= 0 && nfaces >= 0, "of_mesh_largest_component: need nverts, nfaces >= 0 (got %d, %d)", nverts,
             nfaces);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const CcLayout L = cc_layout(nverts, nfaces);
  if (nfaces == 0) {
    // nothing kept: label -1, no faces, no vertices
    if ((nverts > 0 && cudaMemsetAsync(vert_map, 0xff, (size_t)nverts * 4, st) != cudaSuccess) ||
        cudaMemsetAsync(info + 2, 0xff, sizeof(int32_t), st) != cudaSuccess ||
        cudaMemsetAsync(info + 3, 0, 2 * sizeof(int32_t), st) != cudaSuccess) {
      set_error("of_mesh_largest_component: cudaMemsetAsync failed");
      return OF_E_CUDA;
    }
    return OF_OK;
  }
  CcHeader* hdr = at<CcHeader>(scratch, L.hdr);
  uint32_t* blo = at<uint32_t>(scratch, L.blo);
  uint32_t* bhi = at<uint32_t>(scratch, L.bhi);
  int32_t* canon = at<int32_t>(scratch, L.canon);
  int32_t* flags = at<int32_t>(scratch, L.flags);
  int32_t* scan = at<int32_t>(scratch, L.scan);
  if (cudaMemsetAsync(blo, 0xff, (size_t)nfaces * 12, st) != cudaSuccess ||
      cudaMemsetAsync(bhi, 0, (size_t)nfaces * 12, st) != cudaSuccess ||
      cudaMemsetAsync(flags, 0, (size_t)nverts * 4, st) != cudaSuccess) {
    set_error("of_mesh_largest_component: cudaMemsetAsync failed");
    return OF_E_CUDA;
  }
  cc_header_kernel<<<1, 1, 0, st>>>(hdr);
  const int64_t warps = (nfaces + 32 * CC_RUN - 1) / (32 * CC_RUN);
  bounds_kernel<<<(unsigned)((warps + CC_T / 32 - 1) / (CC_T / 32)), CC_T, 0, st>>>(verts, faces, nfaces, nverts, labels,
                                                                                    blo, bhi);
  extent_kernel<<<cc_blocks(nfaces), CC_T, 0, st>>>(nfaces, labels, blo, bhi, hdr);
  select_kernel<<<cc_blocks(nfaces), CC_T, 0, st>>>(nfaces, labels, blo, bhi, hdr);
  mark_kernel<<<cc_blocks(nfaces), CC_T, 0, st>>>(faces, nfaces, nverts, labels, canon, flags, hdr);
  add_launches(4);
  OF_LAUNCH_CHECK("of_mesh_largest_component");
  if (int rc = of_exclusive_scan_i32(flags, scan, nverts, info + 4, at<void>(scratch, L.scan_tmp), stream)) return rc;
  vert_map_kernel<<<cc_blocks(nverts > 0 ? nverts : 1), CC_T, 0, st>>>(nverts, canon, flags, scan, hdr, vert_map, info);
  OF_LAUNCH_CHECK("of_mesh_largest_component");
  return OF_OK;
}

extern "C" int of_mesh_compact(const float* verts, int32_t nverts, const int32_t* faces, int32_t nfaces,
                               const int32_t* labels, int32_t label, const int32_t* vert_map, void* scratch,
                               float* out_verts, int32_t* out_faces, void* stream) {
  OF_REQUIRE(verts && faces && labels && vert_map && scratch && out_verts && out_faces, "of_mesh_compact: null pointer");
  OF_REQUIRE(nverts > 0 && nfaces > 0 && label >= 0 && label < nfaces,
             "of_mesh_compact: need nverts, nfaces > 0 and 0 <= label < nfaces (got %d, %d, %d)", nverts, nfaces, label);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const CcLayout L = cc_layout(nverts, nfaces);
  int32_t* flags = at<int32_t>(scratch, L.flags);
  int32_t* scan = at<int32_t>(scratch, L.scan);
  keep_flags_kernel<<<cc_blocks(nfaces), CC_T, 0, st>>>(nfaces, labels, label, flags);
  OF_LAUNCH_CHECK("of_mesh_compact");
  if (int rc = of_exclusive_scan_i32(flags, scan, nfaces, nullptr, at<void>(scratch, L.scan_tmp), stream)) return rc;
  compact_faces_kernel<<<cc_blocks(nfaces), CC_T, 0, st>>>(faces, nfaces, nverts, flags, scan, vert_map, out_faces);
  compact_verts_kernel<<<cc_blocks(nverts), CC_T, 0, st>>>(verts, nverts, vert_map, out_verts);
  add_launches(1);
  OF_LAUNCH_CHECK("of_mesh_compact");
  return OF_OK;
}
