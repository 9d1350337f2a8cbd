/*
 * diffdock_b200 - C ABI of the H100-native (sm_90a) DiffDock score-model hot path.
 *
 * The reference (gcorso/DiffDock @ b4704d9) is pure Python: it has no FFI of its own.  Each entry point below
 * replaces the op sequence of the cited reference lines; the Python host code in diffdock_b200/ binds them with
 * ctypes (INTEGRATION.md shows the stub a reference maintainer would add).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer owned by the caller (PyTorch caching allocator); nothing is freed here;
 *   - every launch goes to the caller-supplied `stream` (cudaStream_t passed as void*), no implicit sync;
 *   - return value: 0 = ok, otherwise a cudaError_t value or a negative DDB200_E* code; nothing throws;
 *   - indices are int32 (N, E < 2^31); the Python wrappers convert the reference's int64 indices;
 *   - floating point is fp32 everywhere (the reference path is fp32, TF32 disabled).
 */
#ifndef DIFFDOCK_B200_H
#define DIFFDOCK_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DDB200_EINVAL (-1) /* bad argument (alignment, size, null pointer)           */
#define DDB200_ETABLE (-2) /* malformed tensor-product table blob                    */
#define DDB200_ESMEM  (-3) /* table needs more shared memory than one SM offers      */

/* library / build information: "diffdock_b200 <version> sm_90a" */
const char* ddb200_version(void);

/* ---------------------------------------------------------------------------------------------------------------
 * Tensor-product table (one per TensorProductConvLayer; immutable after creation, shareable between streams).
 * Blob layout (produced by diffdock_b200/tp_table.py; int32 words):
 *   hdr[32] : 0 magic 'DB20' | 1 n_paths | 2 n_tiles | 3 n_chunks | 4 n_mentries | 5 n_terms | 6 D_in | 7 D_sh |
 *             8 D_out | 9 sh_lmax (-1: spherical harmonics are given per edge) | 10 z_total | 11 m_total |
 *             12 n_acc | 13 weight_numel (padded, multiple of 4) | 14 stage_floats |
 *             15..20 word offsets of the sections below | 21 total words
 *   paths   [n_paths][6] : in_off, mul_in, d_in, d_out, z_off, m_off
 *   tiles   [n_tiles][8] : w_local, row_stride, n_rows, z_base, d_out, width, row_groups, acc_base
 *   chunks  [n_chunks][4]: tile_begin, tile_end, w_offset, n_floats      (one TMA bulk copy each)
 *   mentries[n_ment][3]  : m_index, term_begin, term_count
 *   terms_y [n_terms]    : index into the per-edge spherical-harmonics vector
 *   outmap  [D_out][3]   : accumulator slot, lane stride between row groups, row groups
 * fblob: terms_val[n_terms] = path coefficient * Clebsch-Gordan entry.
 * Replaces: the e3nn code-generated o3.FullyConnectedTensorProduct / FasterTensorProduct instances built at
 * models/tensor_layers.py:295-299.
 * ------------------------------------------------------------------------------------------------------------- */
typedef struct ddb200_tp_table ddb200_tp_table;

int  ddb200_tp_table_create(const int32_t* iblob_host, int n_ints, const float* fblob_host, int n_floats,
                            ddb200_tp_table** out);
void ddb200_tp_table_destroy(ddb200_tp_table* t);
/* 0: D_in, 1: D_sh, 2: D_out, 3: weight_numel (padded), 4: sh_lmax, 5: dynamic shared memory bytes per CTA,
 * 6: warps per CTA, 7: pipeline stages per warp */
int  ddb200_tp_table_info(const ddb200_tp_table* t, int what);

/* ---------------------------------------------------------------------------------------------------------------
 * Fused tensor-product convolution, accumulate phase.
 *   for every edge e:   sum[edge_dst[e], :] += TP(x[edge_src[e], :], Y(geo[e]), w[e, :]) * edge_weight[e]
 *                       cnt[edge_dst[e]]    += 1
 * x        [n_src, x_stride]   gathered node irreps (x_stride >= D_in floats)
 * edge_src [E], edge_dst [E]   int32; performance (not correctness) wants edges sorted by edge_dst (CSR order)
 * geo      sh_lmax >= 0: edge vectors [E,3] (spherical harmonics evaluated in-kernel, component normalisation);
 *          sh_lmax == -1: precomputed spherical harmonics [E, D_sh]
 * edge_weight [E] or NULL
 * w        [E, w_stride] per-edge tensor-product weights in table layout (w 16-byte aligned, w_stride % 4 == 0)
 * sum      [n_dst, D_out] fp32 accumulator, cnt [n_dst] fp32 (may be NULL); caller zero-initialises both
 * Replaces: models/tensor_layers.py:139-144 and :204-221 (gather, tensor product, scatter-sum, bincount), plus the
 * o3.spherical_harmonics calls at models/cg_model.py:494,511,556-557,622,636.
 * ------------------------------------------------------------------------------------------------------------- */
int ddb200_tpconv_accumulate(const ddb200_tp_table* t, const float* x, int64_t x_stride, const int32_t* edge_src,
                             const int32_t* edge_dst, const float* geo, const float* edge_weight, const float* w,
                             int64_t w_stride, int64_t n_edges, float* sum, float* cnt, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Convolution epilogue:  out[n, c] = (sum[n, c] / max(cnt[n], eps) if mean else sum[n, c]) * bn_scale[c] + bn_shift[c]
 *                                    + (c < res_dim ? residual[n, c] : 0)
 * bn_scale / bn_shift: eval-mode e3nn BatchNorm folded per column (NULL = identity); residual may be NULL.
 * Replaces: models/tensor_layers.py:227-229 (mean), :327-328 (BatchNorm), :330-332 (zero-padded residual).
 * ------------------------------------------------------------------------------------------------------------- */
int ddb200_tpconv_finalize(const float* sum, const float* cnt, int64_t n_rows, int d_out, int mean,
                           const float* bn_scale, const float* bn_shift, const float* residual,
                           int64_t res_stride, int res_dim, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Batched fixed-radius neighbour search, two passes (count -> caller's exclusive scan -> fill).
 * x [n_x,3] candidates, batch-sorted, x_ptr [B+1] their per-complex segment offsets; y [n_y,3] queries with
 * y_batch [n_y] complex ids.  r_per_graph != NULL: coordinates are divided by r_per_graph[b] and compared with r
 * (the reference's radius(x / c, y / c, 1) formulation of a per-complex cutoff); else plain radius r.
 * Strict test d^2 < r^2; at most max_neighbors hits per query, first ones in candidate order; exclude_self drops
 * i == j after it was counted against the cap (radius_graph semantics).  Output sorted by (query, candidate).
 * Replaces: torch_cluster.radius / radius_graph at models/cg_model.py:477,543-548,630.
 * ------------------------------------------------------------------------------------------------------------- */
int ddb200_radius_count(const float* x, const float* y, const int32_t* x_ptr, const int32_t* y_batch,
                        const float* r_per_graph, float r, int64_t n_y, int max_neighbors, int exclude_self,
                        int32_t* count, void* stream);
int ddb200_radius_fill(const float* x, const float* y, const int32_t* x_ptr, const int32_t* y_batch,
                       const float* r_per_graph, float r, int64_t n_y, int max_neighbors, int exclude_self,
                       const int32_t* row_start, int32_t* out_row, int32_t* out_col, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * One reverse-diffusion pose update for n_poses copies of one ligand (n_atoms atoms, n_bonds rotatable bonds):
 *   tr  = coef[0] * tr_score  + coef[1] * tr_z        rot = coef[2] * rot_score + coef[3] * rot_z
 *   tor = coef[4] * tor_score + coef[5] * tor_z       (z pointers may be NULL = no noise; coef6 is a HOST array)
 *   rigid move about the ligand centroid, sequential torsion rotations (bond_u/bond_v [n_bonds], mask_rotate
 *   [n_bonds, n_atoms] bytes), Kabsch re-alignment of the flexed pose onto the rigid one.
 * pos / out_pos [n_poses * n_atoms, 3]; tr/rot [n_poses, 3]; tor [n_poses * n_bonds].  use_torsion = 0 skips the
 * torsion + Kabsch part (model_args.no_torsion).
 * Replaces: utils/sampling.py:133-186 (perturbations), utils/diffusion_utils.py:60-78, utils/torsion.py:75-90,
 * utils/geometry.py:72-86,246-276.
 * ------------------------------------------------------------------------------------------------------------- */
int ddb200_pose_update(const float* pos, int64_t n_poses, int n_atoms, int n_bonds, const int32_t* bond_u,
                       const int32_t* bond_v, const uint8_t* mask_rotate, const float* tr_score,
                       const float* rot_score, const float* tor_score, const float* tr_z, const float* rot_z,
                       const float* tor_z, const float* coef6, int use_torsion, float* out_pos, void* stream);

/* Same update for a step loop that never returns to the host: the SDE coefficients come from row *step_dev (NULL = row 0)
 * of a DEVICE table coef_table [n_steps, 6]; with pose_key != NULL the noise is drawn in-kernel from Philox4x32-10 keyed by
 * (seed, pose_key[b] = (complex id << 32) | pose id) at counter (step, dof block) - the noise of a pose is then independent of
 * batch composition and of the number of GPUs the poses are sharded over (SURVEY.md section 8(e)); otherwise tr_z / rot_z /
 * tor_z (may be NULL) as above.  out_pos may alias pos. */
int ddb200_pose_update_dev(const float* pos, int64_t n_poses, int n_atoms, int n_bonds, const int32_t* bond_u,
                           const int32_t* bond_v, const uint8_t* mask_rotate, const float* tr_score,
                           const float* rot_score, const float* tor_score, const float* tr_z, const float* rot_z,
                           const float* tor_z, const float* coef_table, const int32_t* step_dev, uint64_t seed,
                           const int64_t* pose_key, int use_torsion, float* out_pos, void* stream);
/* ddb200_pose_update_dev for a batch whose poses belong to different ligands (several complexes sampled in one step).  Row b
 * of the DEVICE descriptor layout [n_poses, 6] (int32) gives pose b's
 *   atom_off, n_atoms   its rows of pos / out_pos;
 *   bond_off, n_bonds   its rows of bond_u / bond_v, in the pose's local atom numbering;
 *   tor_off             its first entry of tor_score / tor_z (the score model's bond order, pose-major);
 *   mask_off            the first byte of its [n_bonds, n_atoms] block of the concatenated uint8 masks.
 * tr_score / rot_score / tr_z / rot_z stay [n_poses, 3].  Coefficients, Philox keys and in-place use as in
 * ddb200_pose_update_dev.  The host does not read the descriptor: max_atoms (>= every pose's n_atoms) sizes the shared
 * memory.  A pose with n_atoms outside [1, max_atoms] or a negative n_bonds is left untouched and sets *err (device
 * int32) to 1; the caller zeroes it and reads it when convenient.  use_torsion needs bond_u, bond_v, mask_rotate and
 * tor_score. */
int ddb200_pose_update_packed(const float* pos, int64_t n_poses, const int32_t* layout, int max_atoms, const int32_t* bond_u,
                              const int32_t* bond_v, const uint8_t* mask_rotate, const float* tr_score,
                              const float* rot_score, const float* tor_score, const float* tr_z, const float* rot_z,
                              const float* tor_z, const float* coef_table, const int32_t* step_dev, uint64_t seed,
                              const int64_t* pose_key, int use_torsion, int32_t* err, float* out_pos, void* stream);
/* Test hook: the four normals (and optionally the raw 4 x uint32 words) of Philox blocks block0 .. block0 + n_blocks - 1. */
int ddb200_philox_probe(uint64_t seed, int64_t pose_key, uint32_t step, uint32_t block0, int n_blocks,
                        float* out_normals, uint32_t* out_raw, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Sync-free graph construction: fill pass that writes into caller-sized (upper-bound) buffers; the edge total stays in
 * device memory (last element of the caller's inclusive scan) and is handed to the convolution as n_edges_dev.
 *   row_start [n_y]   exclusive scan of (pre_ptr[q+1] - pre_ptr[q]) + radius count (ddb200_radius_count)
 *   pre_ptr / pre_col optional CSR of static edges listed first for every query (the ligand bond edges of
 *                     models/cg_model.py:478-483); out_eid [E] = index into pre_col, or -1 for radius edges
 *   out_vec [E, 3]    x[col] - y[row]  (models/cg_model.py:491,508,552), optional
 *   slot_out          optional dense table: slot_out[q * slot_ld + (i - x_ptr[b])] = edge position (forward pass of a
 *                     bipartite graph);  slot_in / y_ptr / out_perm: reverse pass (queries and candidates swapped) emits
 *                     out_perm[pos] = slot_in[i * slot_ld + (q - y_ptr[b])], the position of the same pair in the forward
 *                     list, which ddb200_fused_conv takes as edge_perm (same pairs in both directions, :555-557).
 *   row_offset / col_offset are added to the indices written to out_row / out_col (the model numbers ligand and receptor
 *                     nodes jointly, models/cg_model.py:329-338).
 * ------------------------------------------------------------------------------------------------------------- */
int ddb200_graph_fill(const float* x, const float* y, const int32_t* x_ptr, const int32_t* y_batch,
                      const float* r_per_graph, float r, int64_t n_y, int max_neighbors, int exclude_self,
                      const int32_t* row_start, const int32_t* pre_ptr, const int32_t* pre_col, int32_t* out_row,
                      int32_t* out_col, float* out_vec, int32_t* out_eid, int32_t* slot_out, const int32_t* slot_in,
                      const int32_t* y_ptr, int slot_ld, int32_t* out_perm, int row_offset, int col_offset, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * CSR order of an arbitrary edge list: stable sort by target (keys tgt [n_edges] int32 in [0, n_rows)), device only.
 *   tgt_sorted [n_edges], perm [n_edges] (perm[p] = original position of the edge now at p), row_ptr [n_rows + 1] or NULL.
 * Two-call workspace protocol (nothing is allocated here): workspace == NULL writes the required size to *workspace_bytes;
 * otherwise *workspace_bytes is the size of the caller's device buffer.
 * Replaces: the per-layer implicit ordering work of torch_scatter (models/tensor_layers.py:220); SURVEY.md section 8(b).
 * ------------------------------------------------------------------------------------------------------------- */
int ddb200_csr_sort_by_target(const int32_t* tgt, int64_t n_edges, int32_t n_rows, int32_t* tgt_sorted, int32_t* perm,
                              int32_t* row_ptr, void* workspace, size_t* workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Ligand-receptor edge embedding, one kernel, live edge count on the device:
 *   h = relu(u[edge_row[e]] + W1_rbf . rbf(|edge_vec[e]|)),  out[e] = W2 . h + b2,   rbf_k(d) = exp(coeff (d - offset_k)^2)
 * u [n_rows, ns] = W1[:, :S] . sigma_emb + b1 per ligand node (the sigma-embedding half of the first Linear, computed once
 * per node instead of once per edge); w1_rbf [ns, rbf_dim] = W1[:, S:]; w2 [ns, ns]; out [capacity, ns].
 * Replaces: models/cg_model.py:553-554 (edge_attr = cat[sigma_emb, GaussianSmearing(d)]) + cross_edge_embedding at :326
 * (models/layers.py:20-30 + Linear/ReLU/Linear).  Unsupported (rbf_dim, ns) -> DDB200_EINVAL.
 * ------------------------------------------------------------------------------------------------------------- */
int ddb200_edge_embed(const float* edge_vec, const int32_t* edge_row, const float* u, const float* w1_rbf, const float* w2,
                      const float* b2, int rbf_dim, int ns, const float* rbf_offset, float rbf_coeff, int64_t capacity,
                      const int32_t* n_edges_dev, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Radial-MLP output layer on the Hopper tensor cores (wgmma):  out[e, n] = sum_k h[e, k] * W2[n, k] + bias[n], fp32-accurate
 * through a split-bf16 (hi/lo) product evaluated as one bf16 GEMM over K' = 3K.
 * h [n_edges, ldh] fp32 (K <= 149); b_images: bf16, [n_tiles_n][ceil(3K/64)][256 rows][64] pre-split
 * ([hi | lo | hi] of W2 rows, zero padded) and 128B-swizzled shared-memory images built by
 * diffdock_b200/radial.py:build_b_images (128-byte aligned); bias [n_tiles_n*256]; out [n_edges, ldo] fp32 with
 * ldo >= n_tiles_n*256, ldo % 4 == 0, 16-byte aligned.  Columns are in the tensor-product table's weight-row layout.
 * Replaces: the last nn.Linear of FCBlock (models/layers.py:16) applied at models/tensor_layers.py:140,211.
 * ------------------------------------------------------------------------------------------------------------- */
int ddb200_radial_gemm(const float* h, int64_t ldh, int64_t n_edges, int K, const void* b_images, const float* bias,
                       int n_tiles_n, float* out, int64_t ldo, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Whole radial MLP of one edge group in one kernel (FCBlock with two Linear layers and ReLU):
 *   a[e, :] = [edge_attr[e, :ne] | node[tgt[e], :ns] | node[src[e], :ns]]            (the torch.cat / gathers of
 *                                                                                    models/cg_model.py:342-349; ns = 0: none)
 *   h       = relu(a @ W1^T + b1)            (hidden units, also a split-bf16 wgmma GEMM, kept on chip)
 *   out     = h @ W2^T + b2                  (as ddb200_radial_gemm)
 * w1_images: build_b_images(W1 [hidden, ne + 2 ns]) (one N tile), w2_images / b2 / n_tiles_n / out / ldo as above.
 * Replaces: models/layers.py:10-17 (FCBlock, tp_weights_layers == 2) and the edge_attr_ assembly feeding it.
 * ------------------------------------------------------------------------------------------------------------- */
int ddb200_radial_mlp(const float* edge_attr, int64_t ld_ea, int ne, const float* node, int64_t ld_node, int ns,
                      const int32_t* tgt, const int32_t* src, const void* w1_images, const float* b1, int hidden,
                      const void* w2_images, const float* b2, int n_tiles_n, int64_t n_edges, float* out, int64_t ldo,
                      void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Fully fused convolution of one edge group: radial MLP (as ddb200_radial_mlp) whose output tiles are contracted with the
 * edge irreps from an on-chip accumulator tile and scatter-added - the [E, weight_numel] weights never reach HBM.
 *   r = edge_perm ? edge_perm[e] : e                                      (row of the per-edge input arrays)
 *   a = [edge_attr[r] (+ ea_add[ea_add_idx[e]]) | node[tgt[e], :ns] | node[src[e], :ns]]
 *   sum[tgt[e], :] += TP(x[src[e], :], Y(vec_sign * edge_vec[r]), FCBlock(a)) * edge_weight[r]
 *   cnt[tgt[e]]    += 1
 * for e < min(n_edges, *n_edges_dev): the edge count may live on the device (neighbour lists built without a host round
 * trip); n_edges is then the capacity of the arrays.  edge_perm / vec_sign let one stored edge list serve both directions
 * of a bipartite graph (the reverse direction reads the same attribute rows in another order with the vector negated,
 * models/cg_model.py:556-557) and let poses share one copy of the static receptor edge attributes; ea_add carries the
 * per-complex sigma-embedding term of models/cg_model.py:298-301 without materialising edge_attr + sigma per step.
 * w1_images / w2_images / tiles / mtab: the plan built by diffdock_b200/fused.py (operand images [hi | lo | bias] with
 * 16-column-aligned sections, N tiles = whole rows of one path block, dense Clebsch-Gordan tables [path][3][3][5] padded to
 * 48 floats).  FCBlock = Linear(W1) -> ReLU -> [Linear(Wh_l) -> ReLU for l < n_hidden] -> Linear(W2): wh_images holds the
 * n_hidden extra H x H layers (tp_weights_layers - 2 of them) as [n_hidden] one-N-tile images of the W2 layout, 128-byte
 * aligned; n_hidden = 0 with wh_images = NULL is the two-layer FCBlock.  Supported shapes: (mul_out, 2l_out+1) in {(48,1),(10,3),(16,1),(4,3),(10,1),(4,1)}, l_in <= 1, at most
 * 16 paths, spherical harmonics from edge vectors (sh_lmax <= 2), ne + 2 ns <= 144, hidden <= 144.
 * Any base pointer and row stride is accepted.  The rows of a are read with 16-byte loads when ne % 8 == 0, ns % 8 == 0,
 * ld_ea % 4 == 0, edge_attr 16-byte aligned, and (ns > 0) ld_node % 4 == 0 and node 16-byte aligned, and (ea_add given)
 * ea_add 16-byte aligned; otherwise element by element.  x is read with 8-byte loads when x_pairs_ok, ld_x is even and x
 * is 8-byte aligned; otherwise element by element.
 * Replaces: models/tensor_layers.py:139-144 / :204-221 including fc_layer(edge_attr) and the edge_attr_ assembly of
 * models/cg_model.py:342-349.  Follow with ddb200_tpconv_finalize.
 * ------------------------------------------------------------------------------------------------------------- */
typedef struct ddb200_fused_args {
  const float*   edge_attr;   int64_t ld_ea;   int32_t ne;     /* [rows, ld_ea] per-edge attributes, ne columns used   */
  const float*   node;        int64_t ld_node; int32_t ns;     /* node scalars of both end points (ns = 0: none)       */
  const int32_t* tgt;         const int32_t* src;              /* [n_edges] scatter target / gathered node             */
  const int32_t* edge_perm;                                    /* [n_edges] or NULL                                    */
  const float*   ea_add;      const int32_t* ea_add_idx;       /* [*, ne] and [n_edges], both or neither               */
  float          vec_sign;                                     /* +1 / -1 (0 is read as +1)                            */
  const void*    w1_images;   int32_t hidden;
  const void*    w2_images;
  const int32_t* tiles;       int32_t n_tiles;                 /* [n_tiles][8]                                         */
  const float*   mtab;        int32_t n_paths;                 /* [n_paths][48]                                        */
  const float*   x;           int64_t ld_x;    int32_t x_pairs_ok;   /* x_pairs_ok: every tile offset / count is even  */
  const float*   edge_vec;    const float* edge_weight;        /* [rows, 3]; [rows] or NULL                            */
  int32_t        sh_lmax;
  int64_t        n_edges;     const int32_t* n_edges_dev;      /* capacity (or count if n_edges_dev == NULL)           */
  float*         sum;         int32_t d_out;   float* cnt;     /* [n_dst, d_out] fp32, [n_dst] fp32 or NULL            */
  const void*    wh_images;   int32_t n_hidden;                /* extra H x H hidden layers (NULL / 0: two-layer FCBlock) */
} ddb200_fused_args;

int ddb200_fused_conv(const ddb200_fused_args* args, void* stream);
/* Second-order instantiation (node irreps with l = 2 blocks, use_second_order_repr): same arguments, additionally
 * (mul_out, 2l_out+1) in {(10,5),(4,5)} and l_in <= 2, at most 32 paths, mtab = [n_paths][5][5][5] padded to 128 floats;
 * x is read element by element (x_pairs_ok is ignored). */
int ddb200_fused_conv_so(const ddb200_fused_args* args, void* stream);
/* Execution: one CTA per SM, persistent over tiles of 64 edges; one warpgroup issues wgmma, one contracts. */

/* Diagnostics, no reference counterpart: with DDB200_FUSED_DEBUG=1 in the environment the fused kernel accumulates clock
 * counters per edge tile; this copies the 32 counters to `out` (host, uint64_t[32]) and clears them.  DDB200_EINVAL when disabled. */
int ddb200_fused_debug_read(uint64_t* out);

/* ---------------------------------------------------------------------------------------------------------------
 * Input side: receptor contact graph (residues or atoms of ONE complex) on the device, two passes around the caller's
 * exclusive scan of `count` (as ddb200_radius_count / _fill).  For every centre i over pos [n, 3]:
 *   hits = { j != i : d(i, j) < cutoff }        d = torch.cdist(pos, pos)[i, j]: squared distance in ATen's fp32 operation
 *                                               order (bit-identical), correctly rounded square root
 *   |hits| <= max_neighbors : the hits in ascending index order
 *   |hits| >  max_neighbors : the max_neighbors nearest points, ascending (distance, index) - np.argsort order with
 *                             exact-distance ties (unspecified there) broken by index
 *   |hits| == 0             : the nearest other point
 *   knn_only != 0           : the max_neighbors nearest points regardless of cutoff (knn_graph)
 * out_nbr / out_ctr [E] = edge_index[0] / edge_index[1] ([neighbour, centre], centre by centre).
 * Replaces: the cdist + Python loop of datasets/process_mols.py:168-192 (residues) and :205-224 (atoms).
 * ------------------------------------------------------------------------------------------------------------- */
int ddb200_contact_count(const float* pos, int32_t n, float cutoff, int32_t max_neighbors, int32_t knn_only,
                         int32_t* count, void* stream);
int ddb200_contact_fill(const float* pos, int32_t n, float cutoff, int32_t max_neighbors, int32_t knn_only,
                        const int32_t* row_start, int32_t* out_nbr, int32_t* out_ctr, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Per-step receptor cropping, masked form (the receptor arrays keep their size; a dropped residue loses its edges).
 * ddb200_crop_flags: for every residue r of complex b = rec_batch[r]
 *   keep[r] = any over the ligand atoms j of b (segment lig_ptr[b] .. lig_ptr[b+1]) of
 *             (lx - rx)^2 + (ly - ry)^2 + (lz - rz)^2 < cutoff2_table[*step_dev]      (step_dev NULL: row 0)
 *   with three rounded products added left to right (no FMA) and a strict test, bit-compatible with the reference's
 *   sum((lig - rec) ** 2, -1) < cutoff ** 2 on float32 tensors when the table holds cutoff^2 rounded to float32;
 *   rec_pos_masked [n_rec, 3] = rec_pos, with +inf in every coordinate of a dropped residue (handed to the radius kernels
 *   as candidates or queries, a dropped residue then has no neighbour: d^2 < r^2 is false).
 * ddb200_crop_select_edges: the edges e of a static list (tgt / src [n_edges] receptor indices, gid [n_edges] any int32
 *   payload, may be NULL together with out_gid) with keep[tgt[e]] && keep[src[e]] && need[tgt[e]] (keep NULL / need NULL:
 *   that condition holds for every edge), in their original order:
 *   out_perm[k] = e, out_tgt[k] = tgt[e] + offset, out_src[k] = src[e] + offset, out_gid[k] = gid[e] for k < *n_selected;
 *   the output arrays have n_edges rows, rows at and beyond *n_selected are unspecified; the count stays in device memory.
 *   Workspace protocol as ddb200_csr_sort_by_target (workspace == NULL: size query).
 * Replaces: utils/utils.py:388-413 (crop_beyond, all_atoms=False) as called at utils/sampling.py:104-109, without the
 * deep copy / to_data_list / re-collate of the batch.
 * ------------------------------------------------------------------------------------------------------------- */
/* ---------------------------------------------------------------------------------------------------------------
 * ddb200_receptor_need: the residues whose features after an interaction layer can still reach a ligand atom.
 *   need [n_levels, n_rec] bytes (0 / 1), row k = R_{k+1}:
 *   R_1     = { cross_tgt[e] - offset : e < min(*n_cross, cross_cap) }   (the targets of the step's receptor <- ligand
 *             edges in the joint numbering; offset = number of ligand atoms)
 *   R_{k+1} = R_k | { src[e] : tgt[e] in R_k, and keep[tgt[e]] && keep[src[e]] (keep NULL: every edge) }
 *   over the static contact list tgt / src [n_edges] (receptor indices).  One memset, one seed launch and one launch per
 *   further level; no host value is read, so the call can be captured in a CUDA graph.
 * ------------------------------------------------------------------------------------------------------------- */
int ddb200_crop_flags(const float* lig_pos, const int32_t* lig_ptr, const float* rec_pos, const int32_t* rec_batch,
                      int64_t n_rec, const float* cutoff2_table, const int32_t* step_dev, uint8_t* keep,
                      float* rec_pos_masked, void* stream);
int ddb200_crop_select_edges(const int32_t* tgt, const int32_t* src, const int32_t* gid, int64_t n_edges,
                             const uint8_t* keep, const uint8_t* need, int32_t offset, int32_t* out_tgt, int32_t* out_src,
                             int32_t* out_perm, int32_t* out_gid, int32_t* n_selected, void* workspace,
                             size_t* workspace_bytes, void* stream);
int ddb200_receptor_need(const int32_t* cross_tgt, const int32_t* n_cross, int64_t cross_cap, int32_t offset,
                         const int32_t* tgt, const int32_t* src, int64_t n_edges, const uint8_t* keep, int64_t n_rec,
                         int32_t n_levels, uint8_t* need, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * ddb200_confidence_head: the confidence head of the confidence models, one CTA per pose b, atoms lig_ptr[b] ..
 * lig_ptr[b+1] of x [n_lig, n_cols] (row stride ld_x):
 *   s[a]   = [x[a, 0:n_head] | x[a, tail_off:tail_off + n_tail]]                       (the selected scalar columns)
 *   with atom_mlp:  y[a] = atom_mlp(s[a]) [n_atom_out + n_in];  atom_confidence[a, 0:n_atom_out] = y[a, 0:n_atom_out];
 *                   s[a] = y[a, n_atom_out:]
 *   confidence[b, 0:n_out] = mlp(mean over the pose's atoms of s[a])          (an empty pose: mean = 0)
 * A packed MLP is Linear -> BN -> ReLU -> Linear -> BN -> ReLU -> Linear in eval mode (Dropout = identity), float32:
 *   W1 [h, in] row-major | b1 [h] | scale1 [h] | shift1 [h] | W2 [h, h] | b2 | scale2 | shift2 | W3 [out, h] | b3 [out]
 *   with BatchNorm folded to y = (W x + b) * scale + shift (nn.Identity: scale 1, shift 0).  For atom_mlp: in = n_head +
 *   n_tail, h = atom_hidden, out = n_atom_out + n_in; for mlp: in = n_in (= n_head + n_tail without atom_mlp), h = n_hidden.
 * Fixed summation order, no atomics: bit-identical results across calls.  No host synchronisation.
 * Limits (DDB200_EINVAL beyond them): n_head + n_tail and n_in <= DDB200_CONF_MAX_IN; n_hidden, atom_hidden <=
 *   DDB200_CONF_MAX_HIDDEN; n_out, n_atom_out <= DDB200_CONF_MAX_OUT.  atom_mlp NULL: no atom head (atom_confidence unused).
 * Replaces: models/cg_model.py:354-366 / models/aa_model.py:434-455 (scatter_mean + the two nn.Sequential heads) and
 * models/old_cg_model.py:296-299 / models/old_aa_model.py:283-286.
 * ------------------------------------------------------------------------------------------------------------- */
#define DDB200_CONF_MAX_IN 256
#define DDB200_CONF_MAX_HIDDEN 128
#define DDB200_CONF_MAX_OUT 16
int ddb200_confidence_head(const float* x, int64_t ld_x, int64_t n_cols, const int32_t* lig_ptr, int32_t n_poses,
                           int32_t n_head, int32_t tail_off, int32_t n_tail, const float* atom_mlp, int32_t atom_hidden,
                           int32_t n_atom_out, const float* mlp, int32_t n_in, int32_t n_hidden, int32_t n_out,
                           float* confidence, float* atom_confidence, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DIFFDOCK_B200_H */
