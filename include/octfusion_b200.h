/*
 * octfusion_b200 -- C ABI of the H100 (sm_90a) kernels behind the OctFusion denoising
 * U-Net hot path.
 *
 * The reference (octree-nn/octfusion) has NO native layer on this path: every operator below
 * is a sequence of ATen library calls issued from Python (SURVEY.md 2a).  This header is the
 * boundary a maintainer of the reference would bind (ctypes stub: INTEGRATION.md); each entry
 * point names the reference function (file:line under the reference tree) whose arithmetic it
 * replaces.
 *
 * Conventions
 *   - plain device pointers and sizes; no torch / ATen types; caller owns every buffer
 *     (outputs and workspaces included); nothing is allocated, freed or synchronised inside
 *   - every call is asynchronous on `stream` (a cudaStream_t passed as void*), re-entrant
 *     per stream, CUDA-graph capturable
 *   - return value: 0 = launched; negative = rejected before any launch (OF_E_*); the
 *     text of the last error of the calling thread is available from of_last_error()
 *   - dtype: OF_F32 (0) = float activations, OF_BF16 (1) = __nv_bfloat16 activations;
 *     accumulation is always fp32; norm statistics: fp32 partial sums per (32-row chunk, 4 channels), combined in fp64
 *   - all row strides (ld*) are in ELEMENTS
 */
#ifndef OCTFUSION_B200_H_
#define OCTFUSION_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OF_F32 0
#define OF_BF16 1

#define OF_OK 0
#define OF_E_ARG (-1)       /* inconsistent / unsupported argument combination            */
#define OF_E_UNSUPPORTED (-2) /* shape not supported by this entry point (use the other one) */
#define OF_E_CUDA (-3)      /* a CUDA runtime call failed (text in of_last_error)          */

const char* of_last_error(void);
int of_version(void);              /* ABI version, bumped on any signature change          */
int of_num_sms(void);              /* multiprocessor count of the current device           */
unsigned long long of_launch_count(void); /* kernels launched by this library so far (process-wide) */
/* ABI guards: sizeof(of_gemm_args) / sizeof(of_octree_levels) as compiled into the library -- a binding whose struct
 * mirror has a different size must refuse to run (a stale .so would otherwise read garbage pointers) */
int of_abi_sizeof_gemm_args(void);
int of_abi_sizeof_octree_levels(void);

/* ------------------------------------------------------------------------------------------
 * Tap-gather GEMM:   out[m, :] = sum_tap  mean_{j in nbr(m, tap)} [ A[j, :] | onehot(type_j) ] . W[tap]
 *                                 (+ bias) (+ row_add[row_add_idx[m]]) (+ resid[m])
 *
 * One operator covers
 *   GraphConv.forward                 models/networks/modules.py:194-220  (7 taps, mean over the
 *                                     1/4/16 finer neighbours = scatter_mean, utils/scatter.py:42-66,
 *                                     one-hot node type of the NEIGHBOUR appended :199-202)
 *   Conv1x1 / nn.Linear / Conv1d k=1  modules.py:332-339, 523-525 (taps = 1, identity)
 *   Downsample / Upsample GEMMs       modules.py:392-395, 440-443 (identity, in_rows / out_rows maps)
 *   dense Conv3d 3^3, stride 2, and nearest-upsample+conv  modules.py:63-95, 493-502
 *                                     (27 taps over a Morton-ordered voxel table)
 *   the "+ emb_out[batch_id]" loop    modules.py:757-758   (row_add)
 *   the residual / skip add           modules.py:513, 763  (resid)
 *
 * Neighbour table `tap_tab` [M, taps] int32 (row-major), the one encoding every reader uses:
 *      v >= 0 : exactly one source row v
 *      v == -1: no neighbour (slot contributes zero; count clamps to 1, scatter.py:60)
 *      v <= -2: several sources: multi-neighbour slot o = -(v+2), 0 <= o < n_multi, numbered in slot order
 *   `tap_extra` int32 [n_multi + 1 + words] lists the sources of the multi slots in CSR form: tap_extra[0..n_multi]
 *   are offsets into tap_extra itself, and the rows of slot o are tap_extra[tap_extra[o] .. tap_extra[o+1]), in the
 *   order of_graph_fill enumerates them.  May be NULL when the table has no multi slot.
 *   tap_tab == NULL: identity (taps must be 1); source row = in_rows ? in_rows[m] : m
 * A is the channel concatenation of up to two sources (a0 | a1) -- the torch.cat of the skip
 * stack (graph_unet_hr.py:266) is never materialised.
 * ------------------------------------------------------------------------------------------ */
typedef struct of_gemm_args {
  const void* a0; int64_t lda0; int32_t c0;
  const void* a1; int64_t lda1; int32_t c1;      /* a1 may be NULL (c1 = 0)                   */
  const int32_t* tap_tab; const int32_t* tap_extra;
  const int32_t* in_rows;                        /* identity mode only, may be NULL           */
  int32_t taps;
  const uint8_t* node_type; int32_t ntype;       /* ntype = 0: no one-hot columns             */
  /* B: fp32 path  -> canonical fp32 [K, N] row-major, K = taps*(c0+c1+ntype), k = tap*(c0+c1+ntype)+c
   *    (exactly GraphConv.weights; other layouts go through of_repack_weight once)
   *    tensor-core path -> bf16 tile image produced by of_pack_weight_tc                         */
  const void* w;
  const float* bias;                             /* [N] or NULL                               */
  const float* row_add; int64_t ld_row_add; const int32_t* row_add_idx;
  const void* resid; int64_t ld_resid;           /* dtype = activation dtype                  */
  const int32_t* out_rows;                       /* optional scatter of output rows           */
  void* out; int64_t ldo;
  int32_t out_f32;                               /* 1: write fp32 regardless of dtype         */
  int32_t M, N;
  int32_t dtype;                                 /* activation dtype of a0/a1/resid/out       */
  /* tensor-core path only: multi slot o reads row o of a_multi, its pre-averaged sources (built per input tensor
   * by of_gather_mean_rows).                                                                                 */
  const void* a_multi; int64_t ld_multi;
  /* tensor-core path with ntype > 0 (required there): the node-type K block as a precomputed bf16 [M, 64] tensor
   * (of_graph_type_block)                                                                                    */
  const void* nt_block;
  /* tensor-core path: 1 = walk the row tiles from the last to the first.  Alternating the direction from one kernel to
   * the next lets each kernel start on the rows its producer wrote last, which are still in the 50 MB L2.  */
  int32_t reverse;
  /* tensor-core path, optional: group-norm partial statistics of the OUTPUT, computed in the epilogue from the fp32
   * values before they are rounded to bf16 (the statistics pass of the following DualOctreeGroupNorm,
   * modules.py:291-326, then never reads the tensor).  Rows are cut into 32-row chunks; a chunk is split into
   * SEGMENTS at every change of sample id; stat_chunk_seg [ceil(M/32)+1] is the exclusive prefix sum of segments
   * per chunk (ops.StatPlan in the Python layer builds it once per graph depth).  stat_out [n_segments, N/G, 2]
   * fp32 receives (sum, sum of squares) per G-channel granule of every segment, G = 4 when N %% 128 == 0 else 2 (a
   * 64-channel norm has 2 channels per group) -- one plain store per value, no atomics, fixed summation order:
   * bit-reproducible.  Sample of row m: stat_sample[m], or m / stat_rows_per_sample
   * when stat_sample is NULL.  Requires N % 32 == 0 and out_rows == NULL.  NULL = off.                        */
  float* stat_out;
  const int32_t* stat_chunk_seg;
  const int32_t* stat_seg_slot;                  /* [n_segments] row of stat_out that segment s writes: segments are
                                                  * stored SAMPLE-MAJOR so that of_gn_finalize streams contiguous rows  */
  const int32_t* stat_sample;
  int32_t stat_rows_per_sample;
} of_gemm_args;

/* CUDA-core FFMA path: any shape, fp32-exact accumulation order-insensitive to 1e-6. */
int of_gather_gemm_simt(const of_gemm_args* args, void* stream);

/* Tensor-core path (wgmma, bf16 operands, fp32 accumulate). Requires dtype = OF_BF16,
 * (c0 % 64 == 0), (c1 % 64 == 0), N % 16 == 0 and w packed by of_pack_weight_tc. */
int of_gather_gemm_tc(const of_gemm_args* args, void* stream);
/* size in bytes of the packed image for K_feat = taps*(c0+c1) feature rows + ntype one-hot rows */
int64_t of_pack_weight_tc_bytes(int32_t taps, int32_t c, int32_t ntype, int32_t N);
/* w_canonical: fp32 [taps*(c+ntype), N]; out: packed bf16 image */
int of_pack_weight_tc(const float* w_canonical, int32_t taps, int32_t c, int32_t ntype, int32_t N,
                      void* out, void* stream);

/* dst[(tap*c + ci)*N + n] = src[tap*s_tap + ci*s_c + n*s_n]   (element strides).
 * nn.Linear [N,K]: taps=1,s_c=1,s_n=K.  Conv3d [N,C,27]: s_tap=1,s_c=27,s_n=27*C.
 * Downsample [C,C,8] (modules.py:393): taps=1, c=8C, s_c=1, s_n=8C.                        */
int of_repack_weight(const float* src, int64_t s_tap, int64_t s_c, int64_t s_n,
                     int32_t taps, int32_t c, int32_t N, float* dst, void* stream);

/* ------------------------------------------------------------------------------------------
 * Group normalisation over ragged per-sample node sets
 *   DualOctreeGroupNorm.forward   models/networks/modules.py:291-326  (count_eps = 1e-5: eps is
 *                                 added to the element count :302 as well as to the variance :310)
 *   GroupNorm32 (dense)           modules.py:26-28                    (count_eps = 0)
 * followed (fused) by SiLU (modules.py:743, 760, graph_unet_hr.py:272) and the channel concat.
 * x is the virtual concatenation (x0 | x1).  sample_id [rows] int32 (NULL => row / rows_per_sample).
 * Statistics are deterministic (no atomics): rows are cut into 32-row chunks, chunks into per-sample SEGMENTS
 * (see of_gemm_args.stat_out), and every segment owns one slot of a partial buffer.
 *   stats:    part [n_segments, C/gran, 2] fp32 = (sum x, sum x^2) per granule of `gran` (2 or 4) channels of each segment, one thread
 *             per (chunk, channel vector), rows added in order.  The tensor-core GEMM writes the same buffer from its
 *             epilogue (stat_out), in which case this pass is skipped.
 *             Slot of segment s in `part`: seg_slot[s] -- the segments of a sample occupy CONSECUTIVE slots (sample-major,
 *             row order inside the sample).
 *   finalize: for sample b the slots sample_seg_off[b] .. sample_seg_off[b+1] are summed in that order in fp64
 *             (contiguous, coalesced reads) -> mean / variance per group -> scale/shift [B, C] fp32 (gamma, beta folded in).
 *             The normalised tensor is the concat (x0 | x1): part0 / part1 are the partial buffers of the two
 *             tensors with their granule widths (c1 = 0: one tensor).  C/groups and c0 must be multiples of the granules.
 *   apply:    y[r, c] = act(x[r, c] * scale[b, c] + shift[b, c])   act: 0 none, 1 SiLU, 2 GELU (erf)
 * ------------------------------------------------------------------------------------------ */
int of_gn_stats(const void* x0, int64_t ld0, int32_t c0, const void* x1, int64_t ld1, int32_t c1,
                const int32_t* chunk_seg, const int32_t* seg_slot, const int32_t* sample_id, int32_t rows_per_sample,
                int64_t rows, int32_t dtype, int32_t gran, float* part, void* stream);
#define OF_GN_FINALIZE_SPLIT 8   /* CTAs per sample; scratch: batch * OF_GN_FINALIZE_SPLIT * C doubles; ticket: batch
                                  * int32, zero on first use (the kernel leaves them zero); both may be NULL (one CTA) */
int of_gn_finalize(const float* part0, int32_t c0, int32_t gran0, const float* part1, int32_t c1, int32_t gran1,
                   const int32_t* sample_seg_off, int32_t n_segments,
                   const int32_t* rows_of_sample, int32_t rows_per_sample,
                   const float* gamma, const float* beta, int32_t batch, int32_t groups, float eps,
                   float count_eps, float* scale, float* shift, double* scratch, int32_t* ticket, void* stream);
int of_gn_apply(const void* x0, int64_t ld0, int32_t c0, const void* x1, int64_t ld1, int32_t c1,
                const int32_t* sample_id, int32_t rows_per_sample, int64_t rows,
                const float* scale, const float* shift, int32_t act, int32_t dtype,
                void* y, int64_t ldy, int32_t reverse, void* stream);

/* ------------------------------------------------------------------------------------------
 * QKVAttention.forward   models/networks/modules.py:538-547
 * qkv [B*T, 3*C] channels-last, head-major legacy split: head h owns columns
 * [h*3*ch, (h+1)*3*ch) = q | k | v, ch = C / heads; q and k are both scaled by ch^-1/4; softmax
 * over keys in fp32; out [B*T, C] with column h*ch + c.
 * ------------------------------------------------------------------------------------------ */
int of_attention(const void* qkv, int64_t ld_qkv, void* out, int64_t ld_out, int32_t batch,
                 int32_t tokens, int32_t heads, int32_t ch, int32_t dtype, void* stream);

/* ------------------------------------------------------------------------------------------
 * Small per-step pieces
 * ------------------------------------------------------------------------------------------ */
/* out[b,:] = act(x[b,:]) . W^T + bias for a few rows (B <= a few dozen): the nn.Linear layers of the
 * timestep-embedding path (graph_unet_hr.py:107-111, modules.py:709-715 emb_layers, :479-482 time_mlp).
 * w_nk is the nn.Linear weight in its native [N, K] layout; a_silu applies SiLU to x on load. */
int of_linear_small(const float* x, int64_t ldx, const float* w_nk, const float* bias, int32_t B, int32_t K,
                    int32_t N, int32_t a_silu, float* out, int64_t ldo, void* stream);
/* timestep_embedding  diffusion_networks/ldm_diffusion_util.py:171-191  ->  out [B, dim] fp32 */
int of_timestep_embedding(const float* t, int32_t batch, int32_t dim, float max_period, float* out,
                          void* stream);
/* LearnedSinusoidalPosEmb.forward  modules.py:558-563  -> out [B, 2*half+1] fp32 */
int of_learned_sinusoidal(const float* t, const float* w, int32_t batch, int32_t half, float* out,
                          void* stream);
/* out[b,:] += table[label[b],:]   (nn.Embedding add, graph_unet_hr.py:232-234) */
int of_embedding_add(const float* table, const int32_t* label, int32_t batch, int32_t dim, float* out,
                     void* stream);
/* eps-DDIM update of sample_loop, models/octfusion_model_union.py:345-350.
 * log_snr / log_snr_next are device scalars (so the step is graph-capturable).
 * x (fp32, [n]) is updated in place; x_act (activation dtype copy fed to the first conv) is
 * refreshed when not NULL. */
int of_ddim_eps_update(float* x, const float* eps, const float* log_snr, const float* log_snr_next,
                       int64_t n, void* x_act, int32_t act_dtype, void* stream);
/* "x0" branch of sample_loop (stage 1), models/octfusion_model_union.py:324-344: optional sign() of the
 * prediction (truncation, :324-325), ancestral mean + sqrt(variance) * noise.  noise == NULL: no noise term. */
int of_ddpm_x0_update(float* x, float* pred, const float* noise, const float* log_snr, const float* log_snr_next,
                      int64_t n, int32_t do_sign, void* stream);
/* dtype conversion / strided row copy: dst[r, 0:c] = src[src_rows ? src_rows[r] : r, 0:c]
 * written to row (dst_rows ? dst_rows[r] : r) */
int of_copy_rows(const void* src, int64_t lds, int32_t src_dtype, const int32_t* src_rows,
                 void* dst, int64_t ldd, int32_t dst_dtype, const int32_t* dst_rows,
                 int64_t rows, int32_t c, void* stream);

/* ------------------------------------------------------------------------------------------
 * Dual-octree graph build   models/networks/dualoctree_networks/dual_octree.py:19-63,119-239,
 * 241-271,332-341,381-409  (DualOctree.__init__ + post_processing_for_docnn), for ONE graph depth.
 *
 * Inputs: the octree levels full_depth..depth: keys[d] (int64 Morton | batch<<48, sorted),
 * children[d] (int32, -1 = leaf else rank among non-empty), node counts nnum[d].
 * The graph at depth D has rows  [leaves of full_depth .. leaves of D-1, all nodes of D]
 * (remap_node_idx, dual_octree.py:265-271).
 *
 * of_leaf_rank / of_compact_idx   per level: rank of every leaf among the leaves of its depth, and the
 *                 index lists of leaf / non-empty nodes (row maps of GraphDownsample / GraphUpsample)
 * of_graph_count  pass 1: per slot, the rows it lists in tap_extra and whether it is a multi slot
 * of_exclusive_scan_i32 over both
 * of_graph_fill   pass 2: final tap_tab [rows, 7] (dir 6 = self loop, dual_octree.py:241-249) and
 *                 tap_extra; also node_type [rows] uint8 (:381-389) and batch_id [rows] int32 (:65-79)
 * ------------------------------------------------------------------------------------------ */
typedef struct of_octree_levels {
  const int64_t* keys[16];      /* indexed by depth; only full_depth..depth are read          */
  const int32_t* children[16];
  const int32_t* leaf_rank[16]; /* exclusive scan of (children < 0), from of_leaf_rank         */
  int32_t nnum[16];
  int32_t full_depth, depth, batch;
} of_octree_levels;

/* out[i] = number of j < i with in-flag set (children[j] < 0); *total_out (device) = #leaves.
 * scratch: >= of_scan_scratch_bytes(n) bytes. */
int64_t of_scan_scratch_bytes(int64_t n);
int of_leaf_rank(const int32_t* children, int32_t n, int32_t* rank_out, int32_t* total_out,
                 void* scratch, void* stream);
int of_exclusive_scan_i32(const int32_t* in, int32_t* out, int64_t n, int32_t* total_out,
                          void* scratch, void* stream);
/* leaf_idx[leaf_rank[i]] = i for leaves, nonempty_idx[children[i]] = i for the others */
int of_compact_idx(const int32_t* children, const int32_t* leaf_rank, int32_t n,
                   int32_t* leaf_idx, int32_t* nonempty_idx, void* stream);
/* number of rows of the depth-D graph (host arithmetic on nnum; no device work) */
int64_t of_graph_rows(const of_octree_levels* oct, int32_t D);
/* Multi-neighbour slots: a coarse leaf next to a subdivided cell, 4..16 finer neighbours averaged by scatter_mean
 * (utils/scatter.py:42-66); up to 4^k for k adaptive levels.
 * pass 1: need[row*7 + dir] = number of neighbours of a multi slot, else 0; multi[row*7 + dir] = 1 for a multi slot,
 * else 0. */
int of_graph_count(const of_octree_levels* oct, int32_t D, int32_t* need, int32_t* multi, void* stream);
/* pass 2: need_off / multi_ord = exclusive scans of need / multi, n_multi = total of multi; tap_extra holds
 * n_multi + 1 + (total of need) words. */
int of_graph_fill(const of_octree_levels* oct, int32_t D, const int32_t* need_off, const int32_t* multi_ord,
                  int32_t n_multi, int32_t* tap_tab, int32_t* tap_extra, uint8_t* node_type, int32_t* batch_id,
                  void* stream);
/* Node-type K block of the tensor-core GEMM, a per-graph constant: out [rows, 64] bf16, column tap*ntype + type =
 * (#neighbours of that type in slot (row, tap)) / (#neighbours) = the scatter_mean of the one-hot columns that
 * GraphConv.forward appends to the features (models/networks/modules.py:199-202, 208-210); zero elsewhere.
 * Requires taps*ntype <= 64, ntype <= 8. */
int of_graph_type_block(const int32_t* tap_tab, const int32_t* tap_extra, const uint8_t* node_type, int64_t rows,
                        int32_t taps, int32_t ntype, void* out_bf16, void* stream);
/* out[o, :] = mean over the rows of multi slot o of (a0|a1)[row, :], o < count (once per input tensor) */
int of_gather_mean_rows(const void* a0, int64_t lda0, int32_t c0, const void* a1, int64_t lda1, int32_t c1,
                        const int32_t* tap_extra, int32_t count, int32_t dtype, void* out, int64_t ldo, void* stream);
/* hist[v] += 1 for v = values[i] (caller zeroes hist) -- rows per sample for the norm count */
int of_histogram_i32(const int32_t* values, int64_t n, int32_t bins, int32_t* hist, void* stream);
/* reference-format edge list (edge_idx [2,E], edge_dir [E] int64, sorted by row*7+dir:
 * dual_octree.py:332-341) from a tap table.  per_slot[row*taps+tap] = #edges, then edges are
 * written at slot_off (exclusive scan of per_slot). */
int of_graph_edge_count(const int32_t* tap_tab, const int32_t* tap_extra, int64_t slots,
                        int32_t* per_slot, void* stream);
int of_graph_edges(const int32_t* tap_tab, const int32_t* tap_extra, int64_t slots, int32_t taps,
                   const int32_t* slot_off, int64_t* edge_row, int64_t* edge_col, int64_t* edge_dir,
                   void* stream);

/* 3^3 neighbour table of the third-party operator ocnn.nn.OctreeConv (BASELINE.json configs[0]; the reference never
 * calls it -- SURVEY.md section 0 -- its semantics are restated from ocnn-pytorch 2.2.x, SURVEY.md Appendix B: parity
 * is UNPINNED at the ocnn boundary): neigh [nnum[depth], 27] int32, entry (dx+1)*9 + (dy+1)*3 + (dz+1) = index within
 * `depth` of the node at (x+dx, y+dy, z+dz), -1 outside the volume or where no node exists.  The table is a tap table
 * of the tap-gather GEMM (taps = 27, weights [27, Cin, Cout] flattened to [27*Cin, Cout]).  Only keys / children / nnum
 * / full_depth / depth / batch of `oct` are read. */
int of_octree_neigh27(const of_octree_levels* oct, int32_t depth, int32_t* neigh, void* stream);

/* Dense voxel neighbour tables in Morton order for the LR middle U-Net (graph_unet_lr.py):
 * mode 0: 3^3 conv, same resolution `res_log2`        (Conv3d padding=1, modules.py:493-502)
 * mode 1: 3^3 stride-2 conv, out res = in res / 2      (ConvDownsample, modules.py:80-95)
 * mode 2: nearest x2 upsample then 3^3 conv            (ConvUpsample, modules.py:63-77)
 * tap = (dx+1)*9 + (dy+1)*3 + (dz+1); rows = batch * 8^out_res_log2; table values are rows of
 * the INPUT tensor (batch * 8^in_res_log2 rows), -1 outside the grid. */
int of_dense_tap_table(int32_t mode, int32_t out_res_log2, int32_t batch, int32_t* tap_tab,
                       void* stream);

/* ------------------------------------------------------------------------------------------
 * NeuralMPU: the implicit function defined by the GraphVAE decoder's regression values
 * (reference models/networks/dualoctree_networks/mpu.py:55-140 `octree_linear_pts` + `get_linear_pred`,
 *  utils/spmm.py `spmm` / `modulated_spmm`).
 *   pos   [npts, 4] fp32: x, y, z in [-1, 1] and the batch index
 *   reg   [sum_{d=full_depth..depth} nnum[d], 4] fp32: per octree node (gradient xyz, value) -- `reg_voxs[depth]` of
 *         GraphVAE.octree_decoder (graph_vae.py:214-221), padded over all nodes
 *   fval  [npts] fp32 = sum_w (F . [offset, 1]) / (sum_w + 1e-8) over the existing cells around the point at depths
 *         full_depth..depth (leaves only below `depth`), w = prod(1 - |offset|) * d^2 / 50
 *   touched [npts] uint8 = 1 when a depth-`depth` cell surrounds the point (the `flgs` mask, mpu.py:139)
 * Only `children`, `nnum`, `full_depth`, `depth`, `batch` of `oct` are read.
 * ------------------------------------------------------------------------------------------ */
int of_mpu_eval(const of_octree_levels* oct, int32_t depth, const float* pos, int64_t npts, const float* reg,
                float* fval, uint8_t* touched, void* stream);
/* The same evaluation on the regular sampling grid of `calc_sdf` (reference utils/util_dualoctree.py:99-118 with
 * get_mgrid :23-42; the 256^3 grid marching cubes consumes): point p of the size^3 grid of shape `batch_idx` is
 * (p / size^2, (p / size) % size, p % size) * ((bbmax - bbmin) / size) + bbmin, generated inside the kernel (no
 * coordinate tensor).  Points [head, head + count) are written to fval[head ..]; fval is the [size^3] array. */
int of_mpu_eval_grid(const of_octree_levels* oct, int32_t depth, int32_t batch_idx, int32_t size, float bbmin,
                     float bbmax, int64_t head, int64_t count, const float* reg, float* fval, void* stream);

/* ------------------------------------------------------------------------------------------
 * Octree build from point clouds: ocnn.octree.Octree.build_octree (third-party; the reference calls it at
 * models/octfusion_model_vae.py:135-146 and models/octfusion_model_union.py:200-212), restated from ocnn-pytorch 2.2.x
 * in SURVEY.md Appendix B -- parity is UNPINNED at the ocnn boundary.
 *   xyz [npts, 3] fp32 in [-1, 1] (values outside wrap: the integer coordinate is masked to `depth` bits), normals
 *   [npts, 3] fp32 or NULL; the points of shape b are rows shape_offsets[b] .. shape_offsets[b+1] (int64 [batch + 1]
 *   on the device).  Cell of a point: trunc((p + 1) * 2^(depth-1)) & (2^depth - 1) per axis; key = Morton | b << 48.
 *   Limits: 0 <= full_depth < depth <= 16, 1 <= batch < 1024, npts < 2^31, batch * 8^full_depth < 2^31.
 * Sequence: of_octree_build_levels (keys, stable radix sort, node ranks of depths full_depth..depth) -> the caller
 * reads level_counts (its one host synchronisation) and allocates -> of_octree_build_fill per depth ->
 * of_octree_build_signal.  The scratch (of_octree_build_bytes) carries the sorted keys between the calls and must not
 * be reused until the last of them has run.  Results are bit-reproducible and independent of the launch configuration.
 * ------------------------------------------------------------------------------------------ */
/* scratch bytes of one build (O(npts)); OF_E_ARG when the arguments are out of range */
int64_t of_octree_build_bytes(int64_t npts, int32_t batch, int32_t depth, int32_t full_depth);
/* level_counts [depth + 2] int32: [d] = number of non-empty (distinct) nodes at depth d for full_depth <= d <= depth,
 * 0 below full_depth; [depth + 1] = 1 when shape_offsets are not a partition of 0..npts (then nothing else is valid) */
int of_octree_build_levels(const float* xyz, const int64_t* shape_offsets, int64_t npts, int32_t batch, int32_t depth,
                           int32_t full_depth, void* scratch, int32_t* level_counts, void* stream);
/* depth d = full_depth: children_d [batch * 8^full_depth] = rank among the non-empty nodes, -1 elsewhere (keys_d may be
 * NULL: the full layer's keys are the octree_grow_full ones).  full_depth < d <= depth: nnum_d = 8 * level_counts[d-1];
 * keys_d [nnum_d] = the 8 children of every non-empty depth-(d-1) node in key order, children_d [nnum_d] = rank of the
 * child among the non-empty depth-d nodes, -1 when no point falls into it. */
int of_octree_build_fill(const void* scratch, int64_t npts, int32_t batch, int32_t depth, int32_t full_depth, int32_t d,
                         int64_t nnum_d, int64_t* keys_d, int32_t* children_d, void* stream);
/* per non-empty depth-`depth` node r (level_counts[depth] rows): points [r, 3] = mean of (p + 1) * 2^(depth-1) over its
 * points, normals [r, 3] = F.normalize(sum of its normals, eps = 1e-12); fp32 sums in input order.  normals_in and
 * normals are both NULL or both set. */
int of_octree_build_signal(const void* scratch, int64_t npts, int32_t batch, int32_t depth, int32_t full_depth,
                           const float* xyz, const float* normals_in, float* points, float* normals, void* stream);
/* ocnn InputFeature('ND', nempty=False) written as depth-D graph rows (DualOctree.get_input_feature, reference
 * dual_octree.py:343-360): rows [0, leaf_rows) are zero (the leaves of full_depth..D-1), row leaf_rows + j is
 * [normals[r] | sum((frac(points[r]) - 0.5) * normals[r])] with r = children[j], zero where r < 0.
 * out [leaf_rows + nnum, >= 4] of dtype OF_F32 / OF_BF16, columns 0..3 written. */
int of_input_feature_nd(const float* points, const float* normals, const int32_t* children, int64_t nnum,
                        int64_t leaf_rows, int32_t dtype, void* out, int64_t ldo, void* stream);

/* ------------------------------------------------------------------------------------------
 * Point-cloud shape metrics (reference metrics/evaluation_metrics.py: MMD, COV and 1-NNA with Chamfer distance and
 * approximate EMD).  Clouds are contiguous fp32 [count, points, 3].  "All pairs" entries compute every (i, j) of
 * a [na] x b [nb] into row-major [na, nb] outputs without copying any cloud; an entry is bit-identical to the same
 * pair computed in paired mode, and every result is identical from run to run (no float atomics, fixed sum order).
 * ------------------------------------------------------------------------------------------ */
#define OF_EMD_MAX_POINTS 4096            /* largest n of of_match_cost / of_emd_cd_pairwise                  */
#define OF_CD_PAIRWISE_MAX_POINTS 49152   /* largest P + Q of of_chamfer_pairwise                              */
/* nndistance (metrics/pytorch_structural_losses/src/nndistance.cu:125-128) for `batch` pairs (a[i], b[i]):
 * dist1 [batch, P]: dist1[i, k] = min_l |b_il - a_ik|^2, dist2 [batch, Q]: dist2[i, l] = min_k |b_il - a_ik|^2, with
 * the reference's fp32 expression (bit-identical values); cd [batch] = mean(dist1[i]) + mean(dist2[i]), may be NULL.
 * Any P, Q >= 1. */
int of_nn_distance(const float* a, const float* b, int32_t batch, int32_t P, int32_t Q, float* dist1, float* dist2,
                   float* cd, void* stream);
/* all-pairs Chamfer distance of _pairwise_EMD_CD_ (metrics/evaluation_metrics.py:111-154, CD arm :133-137):
 * cd [na, nb] = mean_k dist1 + mean_l dist2 of the pair (a_i, b_j).  P + Q <= OF_CD_PAIRWISE_MAX_POINTS. */
int of_chamfer_pairwise(const float* a, int32_t na, int32_t P, const float* b, int32_t nb, int32_t Q, float* cd,
                        void* stream);
/* approxmatch + matchcost (metrics/pytorch_structural_losses/src/approxmatch.cu:299-316) for `batch` pairs
 * (xyz1 = a[i], xyz2 = b[i]) of n points each: cost [batch] = sum_kl match_kl |b_l - a_k|, the reference's
 * un-normalised cost (9 levels -4^7 .. -4^-1), without a match matrix.  cd [batch] (may be NULL) = the Chamfer
 * distance of the same pair, as of_nn_distance computes it up to summation order.  1 <= n <= OF_EMD_MAX_POINTS. */
int of_match_cost(const float* a, const float* b, int32_t batch, int32_t n, float* cost, float* cd, void* stream);
/* all pairs of _pairwise_EMD_CD_ (metrics/evaluation_metrics.py:111-154) in one launch: cost [na, nb] as
 * of_match_cost (emd = cost / n) and cd [na, nb] as of_match_cost's cd, for xyz1 = a_i, xyz2 = b_j. */
int of_emd_cd_pairwise(const float* a, int32_t na, const float* b, int32_t nb, int32_t n, float* cost, float* cd,
                       void* stream);

/* ------------------------------------------------------------------------------------------
 * Meshes and metric point clouds.  Marching cubes replaces skimage.measure.marching_cubes(sdf, level) of export_mesh
 * (models/octfusion_model_union.py:452-455); surface sampling replaces trimesh mesh.sample(count) and the bounding box
 * feeds scale_to_unit_cube (metrics/generate_pointclouds.py:14-37).
 *
 * Grid: one [size, size, size] fp32 array of calc_sdf, sdf[i, j, k], i (x) slowest.  A corner is inside when
 * f < level (f == level and NaN are outside).  Grid point p owns its edges p -> p + e_axis inside the grid; a crossing
 * edge (one end inside) has one vertex at the lower-index end a plus t = (level - f_a) / (f_b - f_a) along the axis,
 * in fp32 with correctly rounded sub, div and add, in index space.  Vertex ids run in (point linear index, axis)
 * order; faces are int32 vertex-id triples in (cell linear index, table order), the table being generated by
 * octfusion_b200/mc_table.py.  Faces wind so that (v1 - v0) x (v2 - v0) points from inside to outside.  The output
 * is bit-reproducible and does not depend on the launch configuration.
 * ------------------------------------------------------------------------------------------ */
#define OF_MC_MAX_SIZE 512                /* largest grid side of of_mc_count / of_mc_emit                      */
/* pass 1: vert_count[p] = crossing edges point p owns (0..3), tri_count[p] = triangles of the cell whose lowest corner
 * is p (0..5; 0 on the far faces of the grid).  Both [size^3]. */
int of_mc_count(const float* sdf, int32_t size, float level, int32_t* vert_count, int32_t* tri_count, void* stream);
/* pass 2, after exclusive scans (of_exclusive_scan_i32) of both counts: verts [V, 3] fp32 and faces [F, 3] int32 of
 * the grid, with V = vert_scan[size^3] and F = tri_scan[size^3]. */
int of_mc_emit(const float* sdf, int32_t size, float level, const int32_t* vert_scan, const int32_t* tri_scan,
               float* verts, int32_t* faces, void* stream);
/* packed meshes: shape b has vertices verts[vert_offsets[b] .. vert_offsets[b+1]) and faces
 * faces[face_offsets[b] .. face_offsets[b+1]) with shape-local vertex ids; offsets are int64 [batch + 1] on the device.
 * bbox [batch, 6] = (min xyz, max xyz) of each shape's vertices (+inf / -inf for an empty shape). */
int of_mesh_bbox(const float* verts, const int64_t* vert_offsets, int32_t batch, float* bbox, void* stream);
/* trimesh sample_surface: per shape `count` points [batch, count, 3] fp32 and face_index [batch, count] int32.  The face
 * is searchsorted(side='left') of u * total area in the fp64 inclusive prefix sum of the face areas (written to
 * area_scan [face_offsets[batch]]), u in (0, 1], so zero-area faces are never chosen; the point is
 * v0 + r1 (v1 - v0) + r2 (v2 - v0), with r1, r2 replaced by |r1 - 1|, |r2 - 1| when r1 + r2 > 1.  u (53 bits), r1
 * and r2 (24 bits) come from Philox4x32-10 keyed by seed, counter (shape, sample): results depend on nothing else.  A
 * shape without faces gets NaN points and face_index -1. */
int of_surface_sample(const float* verts, const int64_t* vert_offsets, const int32_t* faces, const int64_t* face_offsets,
                      int32_t batch, int32_t count, uint64_t seed, double* area_scan, float* points,
                      int32_t* face_index, void* stream);

/* ------------------------------------------------------------------------------------------
 * Mesh connected components and the largest-component filter of export_mesh(clean=True)
 * (models/octfusion_model_union.py:459-466, models/octfusion_model_vae.py:242-250: trimesh split(only_watertight=False),
 * then the component with the largest vertex bounding-box extent).  Rules restated from trimesh in DESIGN.md §4.6 --
 * parity is UNPINNED at the trimesh boundary.  One shape per call: verts [nverts, 3] fp32, faces [nfaces, 3] int32 with
 * shape-local ids.
 *   weld       vertices with bit-identical (x, y, z) are one vertex, represented by the smallest id among them
 *   adjacency  the edges (v0,v1), (v1,v2), (v2,v0) of every face on welded ids, unordered; an edge occurring exactly
 *              twice in the shape links its two faces (once, or three times and more: no link)
 *   labels     int32 [nfaces]: the smallest face index of the face's component (isolated faces are their own)
 *   selection  extent = max over axes of (max - min) of the vertices the component's faces reference, in fp64 from the
 *              fp32 coordinates; the largest extent is kept, the smaller label on a tie
 *   output     the kept faces in their original order; their welded vertices in ascending id, renumbered from 0
 * Sequence: of_mesh_components -> of_mesh_largest_component (same scratch, nothing in between) -> the caller reads the
 * sizes in info (its one host synchronisation) and allocates -> of_mesh_compact.  Only integer atomics are used: the
 * results are bit-reproducible and do not depend on the launch configuration.
 * ------------------------------------------------------------------------------------------ */
/* scratch bytes of one shape (O(nverts + nfaces), monotone in both); OF_E_ARG unless 0 <= nverts, nfaces < 2^31 */
int64_t of_mesh_components_bytes(int64_t nverts, int64_t nfaces);
/* labels [nfaces] as above.  info int32 [5]: [0] status, bit 0 = a coordinate is not finite, bit 1 = a face id lies
 * outside [0, nverts) (no result is valid when status != 0); [1] number of components. */
int of_mesh_components(const float* verts, int32_t nverts, const int32_t* faces, int32_t nfaces, void* scratch,
                       int32_t* labels, int32_t* info, void* stream);
/* after of_mesh_components on the same shape and scratch: info [2] kept label (-1 without faces), [3] kept faces,
 * [4] kept vertices; vert_map [nverts] = output id of the vertex (every vertex welded to a kept one), -1 otherwise */
int of_mesh_largest_component(const float* verts, int32_t nverts, const int32_t* faces, int32_t nfaces, void* scratch,
                              const int32_t* labels, int32_t* vert_map, int32_t* info, void* stream);
/* out_faces [info[3], 3] = vert_map of the faces with labels == label, in order; out_verts [info[4], 3] = the vertex
 * each id came from.  Needs nverts, nfaces > 0; scratch as above (only its scan area is used). */
int of_mesh_compact(const float* verts, int32_t nverts, const int32_t* faces, int32_t nfaces, const int32_t* labels,
                    int32_t label, const int32_t* vert_map, void* scratch, float* out_verts, int32_t* out_faces,
                    void* stream);

#ifdef __cplusplus
}
#endif
#endif /* OCTFUSION_B200_H_ */
