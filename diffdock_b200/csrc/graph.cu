// Batched fixed-radius neighbour search (replaces torch_cluster.radius / radius_graph on the hot path:
// models/cg_model.py:477 ligand radius graph, :543-548 cross graph with per-complex cutoff, :630 bond graph).
//
// One warp per query point y_j.  The candidates are the points x_i of the same complex (segment
// [x_ptr[b], x_ptr[b+1]) of the batch-sorted x array); lanes test 32 candidates at a time and the survivors are
// ranked with ballot/popc, so the output is deterministic and sorted by (query, candidate) - i.e. already CSR-sorted
// by the convolution's target node.  Semantics follow torch_cluster's CUDA kernel: strict squared-distance test
// d^2 < r^2, at most max_neighbors hits per query, the first ones in candidate order.
#include <cuda_runtime.h>
#include <stdint.h>

#include <cub/device/device_radix_sort.cuh>

#include "../../include/diffdock_b200.h"

namespace {

__global__ void iota_kernel(int* p, long long n) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n) p[i] = (int)i;
}
// row_ptr[v] = first position of a key >= v in the sorted key array (v = 0 .. n_rows)
__global__ void row_ptr_kernel(const int* __restrict__ keys, long long n, int n_rows, int* __restrict__ row_ptr) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v > n_rows) return;
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (keys[mid] < v) lo = mid + 1; else hi = mid;
  }
  row_ptr[v] = (int)lo;
}

template <bool FILL>
__global__ void radius_kernel(const float* __restrict__ x, const float* __restrict__ y, const int* __restrict__ x_ptr,
                              const int* __restrict__ y_batch, const float* __restrict__ r_per_graph, float r_scalar,
                              int n_y, int max_neighbors, int exclude_self, int* __restrict__ count,
                              const int* __restrict__ row_start, int* __restrict__ out_row, int* __restrict__ out_col) {
  const int lane = threadIdx.x & 31;
  const int q = (int)((blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5);
  if (q >= n_y) return;
  const int b = y_batch[q];
  // per-complex cutoff c: the reference calls radius(x / c, y / c, r=1) (models/cg_model.py:543-545); the same
  // arithmetic is used here (IEEE division of every coordinate, unfused multiply/add) so that borderline pairs
  // fall on the same side of the strict test as in the reference formulation.
  const float c = r_per_graph ? r_per_graph[b] : 1.0f;
  const float r2 = __fmul_rn(r_scalar, r_scalar);
  const float qx = __fdiv_rn(y[3 * q], c), qy = __fdiv_rn(y[3 * q + 1], c), qz = __fdiv_rn(y[3 * q + 2], c);
  const int beg = x_ptr[b], end = x_ptr[b + 1];
  int found = 0;      // hits so far, including a skipped self hit (torch_cluster counts it against the cap)
  int written = 0;
  const int base = FILL ? row_start[q] : 0;
  for (int i0 = beg; i0 < end && found < max_neighbors; i0 += 32) {
    const int i = i0 + lane;
    bool hit = false;
    if (i < end) {
      const float dx = __fsub_rn(__fdiv_rn(x[3 * i], c), qx), dy = __fsub_rn(__fdiv_rn(x[3 * i + 1], c), qy),
                  dz = __fsub_rn(__fdiv_rn(x[3 * i + 2], c), qz);
      hit = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)) < r2;
    }
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    const int before = __popc(m & ((1u << lane) - 1u));
    const bool keep = hit && (found + before) < max_neighbors;
    const bool emit = keep && !(exclude_self && i == q);
    const unsigned em = __ballot_sync(0xffffffffu, emit);
    if (FILL && emit) {
      const int pos = base + written + __popc(em & ((1u << lane) - 1u));
      out_row[pos] = q;
      out_col[pos] = i;
    }
    written += __popc(em);
    found += __popc(m);
  }
  if (!FILL && lane == 0) count[q] = written;
}


// ---- sync-free graph construction (no host round trip for the edge counts) ------------------------------------------------
// Same search as radius_kernel<true>, plus what the convolution needs so that nothing has to be re-sorted or gathered on
// the host side of the step:
//   * optional static edges listed FIRST for every query (the ligand's bond edges, models/cg_model.py:478-483: the
//     reference concatenates bonds and radius edges; sorted by target that is "bonds of the atom, then its radius hits"),
//     out_eid = index of the static edge or -1;
//   * the edge vector x[col] - y[row] (models/cg_model.py:491,508,552);
//   * forward pass of a bipartite graph: slot_out[q * slot_ld + (i - x_ptr[b])] = edge position, so that
//   * the reverse pass (queries and candidates swapped) can emit perm[pos] = slot_in[i * slot_ld + (q - y_ptr[b])]: the
//     position of the same pair in the forward list (models/cg_model.py:555-557 uses the same pairs in both directions).
struct FillArgs {
  const float* x; const float* y; const int* x_ptr; const int* y_batch; const float* r_per_graph; float r;
  int n_y, max_neighbors, exclude_self;
  const int* row_start; const int* pre_ptr; const int* pre_col;
  int* out_row; int* out_col; float* out_vec; int* out_eid;
  int* slot_out; const int* slot_in; const int* y_ptr; int slot_ld; int* out_perm;
  int row_off, col_off;          // added to the indices written to out_row / out_col (joint node numbering of the model)
};

__global__ void graph_fill_kernel(const FillArgs a) {
  const int lane = threadIdx.x & 31;
  const int q = (int)((blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5);
  if (q >= a.n_y) return;
  const int b = a.y_batch[q];
  const float c = a.r_per_graph ? a.r_per_graph[b] : 1.0f;
  const float r2 = __fmul_rn(a.r, a.r);
  const float yx = a.y[3 * q], yy = a.y[3 * q + 1], yz = a.y[3 * q + 2];
  const float qx = __fdiv_rn(yx, c), qy = __fdiv_rn(yy, c), qz = __fdiv_rn(yz, c);
  const int beg = a.x_ptr[b], end = a.x_ptr[b + 1];
  int base = a.row_start[q];
  if (a.pre_ptr) {          // static edges of this query first
    const int p0 = a.pre_ptr[q], p1 = a.pre_ptr[q + 1];
    for (int p = p0 + lane; p < p1; p += 32) {
      const int i = a.pre_col[p], pos = base + (p - p0);
      a.out_row[pos] = q + a.row_off;
      a.out_col[pos] = i + a.col_off;
      if (a.out_eid) a.out_eid[pos] = p;
      if (a.out_vec) {
        a.out_vec[3 * pos] = a.x[3 * i] - yx; a.out_vec[3 * pos + 1] = a.x[3 * i + 1] - yy; a.out_vec[3 * pos + 2] = a.x[3 * i + 2] - yz;
      }
    }
    base += p1 - p0;
  }
  int found = 0, written = 0;
  for (int i0 = beg; i0 < end && found < a.max_neighbors; i0 += 32) {
    const int i = i0 + lane;
    bool hit = false;
    float xx = 0.f, xy = 0.f, xz = 0.f;
    if (i < end) {
      xx = a.x[3 * i]; xy = a.x[3 * i + 1]; xz = a.x[3 * i + 2];
      const float dx = __fsub_rn(__fdiv_rn(xx, c), qx), dy = __fsub_rn(__fdiv_rn(xy, c), qy), dz = __fsub_rn(__fdiv_rn(xz, c), qz);
      hit = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)) < r2;
    }
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    const int before = __popc(m & ((1u << lane) - 1u));
    const bool keep = hit && (found + before) < a.max_neighbors;
    const bool emit = keep && !(a.exclude_self && i == q);
    const unsigned em = __ballot_sync(0xffffffffu, emit);
    if (emit) {
      const int pos = base + written + __popc(em & ((1u << lane) - 1u));
      a.out_row[pos] = q + a.row_off;
      a.out_col[pos] = i + a.col_off;
      if (a.out_eid) a.out_eid[pos] = -1;
      if (a.out_vec) { a.out_vec[3 * pos] = xx - yx; a.out_vec[3 * pos + 1] = xy - yy; a.out_vec[3 * pos + 2] = xz - yz; }
      if (a.slot_out) a.slot_out[(long long)q * a.slot_ld + (i - beg)] = pos;
      if (a.out_perm) a.out_perm[pos] = a.slot_in[(long long)i * a.slot_ld + (q - a.y_ptr[b])];
    }
    written += __popc(em);
    found += __popc(m);
  }
}

// Edge-embedding MLP of the ligand-receptor edges (models/cg_model.py:553-554 edge_attr = [sigma_emb[lig] | RBF(d)] followed
// by cross_edge_embedding = Linear -> ReLU -> Linear at :326), one thread per edge, weights in shared memory:
//   h   = relu(u[row[e]] + W1r . rbf(|vec[e]|)),   u[n] = W1s . sigma_emb[n] + b1  (per ligand node, precomputed by the caller)
//   out = W2 . h + b2
// rbf_k(d) = exp(coeff * (d - mu_k)^2), k < D, mu = the module's `offset` buffer  (models/layers.py:20-30, GaussianSmearing).
// Live edge count read from device memory; one thread keeps its edge's D Gaussians and NS hidden units in registers.
template <int D, int NS>
__global__ void __launch_bounds__(128) edge_embed_kernel(const float* __restrict__ vec, const int* __restrict__ row,
                                                         const float* __restrict__ u, const float* __restrict__ w1r,
                                                         const float* __restrict__ w2, const float* __restrict__ b2,
                                                         const float* __restrict__ mu, float coeff, long long cap,
                                                         const int* __restrict__ n_dev, float* __restrict__ out) {
  __shared__ __align__(16) float sW1[D * NS];     // [k][o]: transposed so that one k feeds NS consecutive outputs
  __shared__ __align__(16) float sW2[NS * NS];    // [h][o]
  __shared__ float sB2[NS];
  __shared__ float sMu[D];
  for (int i = threadIdx.x; i < D; i += blockDim.x) sMu[i] = mu[i];
  for (int i = threadIdx.x; i < D * NS; i += blockDim.x) { const int o = i / D, k = i - o * D; sW1[k * NS + o] = w1r[i]; }
  for (int i = threadIdx.x; i < NS * NS; i += blockDim.x) { const int o = i / NS, h = i - o * NS; sW2[h * NS + o] = w2[i]; }
  for (int i = threadIdx.x; i < NS; i += blockDim.x) sB2[i] = b2[i];
  __syncthreads();
  long long n = cap;
  if (n_dev) { const long long nd = *n_dev; n = nd < n ? (nd < 0 ? 0 : nd) : n; }
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const float vx = vec[3 * e], vy = vec[3 * e + 1], vz = vec[3 * e + 2];
    const float d = sqrtf(vx * vx + vy * vy + vz * vz);
    float h[NS];
    const float* ur = u + (long long)row[e] * NS;
#pragma unroll
    for (int o = 0; o < NS; o += 4) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(ur + o));
      h[o] = t.x; h[o + 1] = t.y; h[o + 2] = t.z; h[o + 3] = t.w;
    }
#pragma unroll 4
    for (int k = 0; k < D; ++k) {
      const float t = d - sMu[k];
      const float g = expf(coeff * t * t);
      const float4* wr = reinterpret_cast<const float4*>(sW1 + k * NS);
#pragma unroll
      for (int o = 0; o < NS; o += 4) {
        const float4 w = wr[o >> 2];
        h[o] = fmaf(g, w.x, h[o]); h[o + 1] = fmaf(g, w.y, h[o + 1]); h[o + 2] = fmaf(g, w.z, h[o + 2]); h[o + 3] = fmaf(g, w.w, h[o + 3]);
      }
    }
    float acc[NS];
#pragma unroll
    for (int o = 0; o < NS; ++o) acc[o] = sB2[o];
#pragma unroll
    for (int j = 0; j < NS; ++j) {
      const float hv = fmaxf(h[j], 0.f);
      const float4* wr = reinterpret_cast<const float4*>(sW2 + j * NS);
#pragma unroll
      for (int o = 0; o < NS; o += 4) {
        const float4 w = wr[o >> 2];
        acc[o] = fmaf(hv, w.x, acc[o]); acc[o + 1] = fmaf(hv, w.y, acc[o + 1]); acc[o + 2] = fmaf(hv, w.z, acc[o + 2]); acc[o + 3] = fmaf(hv, w.w, acc[o + 3]);
      }
    }
    float4* orow = reinterpret_cast<float4*>(out + e * NS);
#pragma unroll
    for (int o = 0; o < NS; o += 4) orow[o >> 2] = make_float4(acc[o], acc[o + 1], acc[o + 2], acc[o + 3]);
  }
}

}  // namespace

extern "C" {

// Pass 1: count[j] = number of neighbours of y_j (after cap / self exclusion).
int ddb200_radius_count(const float* x, const float* y, const int32_t* x_ptr, const int32_t* y_batch,
                        const float* r_per_graph, float r, int64_t n_y, int max_neighbors, int exclude_self,
                        int32_t* count, void* stream) {
  if (!x || !y || !x_ptr || !y_batch || !count || n_y < 0 || max_neighbors <= 0) return DDB200_EINVAL;
  if (n_y == 0) return 0;
  const int threads = 256;
  const long long blocks = (n_y * 32 + threads - 1) / threads;
  radius_kernel<false><<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(
      x, y, x_ptr, y_batch, r_per_graph, r, (int)n_y, max_neighbors, exclude_self, count, nullptr, nullptr, nullptr);
  return (int)cudaGetLastError();
}

// Pass 2: row_start = exclusive scan of count; writes out_row[e] = query index, out_col[e] = candidate index.
int ddb200_radius_fill(const float* x, const float* y, const int32_t* x_ptr, const int32_t* y_batch,
                       const float* r_per_graph, float r, int64_t n_y, int max_neighbors, int exclude_self,
                       const int32_t* row_start, int32_t* out_row, int32_t* out_col, void* stream) {
  if (!x || !y || !x_ptr || !y_batch || !row_start || !out_row || !out_col || n_y < 0 || max_neighbors <= 0)
    return DDB200_EINVAL;
  if (n_y == 0) return 0;
  const int threads = 256;
  const long long blocks = (n_y * 32 + threads - 1) / threads;
  radius_kernel<true><<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(
      x, y, x_ptr, y_batch, r_per_graph, r, (int)n_y, max_neighbors, exclude_self, nullptr, row_start, out_row, out_col);
  return (int)cudaGetLastError();
}


// Fill pass of the sync-free graph builders (see graph_fill_kernel).  Optional arguments may be NULL.
int ddb200_graph_fill(const float* x, const float* y, const int32_t* x_ptr, const int32_t* y_batch,
                      const float* r_per_graph, float r, int64_t n_y, int max_neighbors, int exclude_self,
                      const int32_t* row_start, const int32_t* pre_ptr, const int32_t* pre_col, int32_t* out_row,
                      int32_t* out_col, float* out_vec, int32_t* out_eid, int32_t* slot_out, const int32_t* slot_in,
                      const int32_t* y_ptr, int slot_ld, int32_t* out_perm, int row_offset, int col_offset, void* stream) {
  if (!x || !y || !x_ptr || !y_batch || !row_start || !out_row || !out_col || n_y < 0 || max_neighbors <= 0)
    return DDB200_EINVAL;
  if ((pre_ptr == nullptr) != (pre_col == nullptr)) return DDB200_EINVAL;
  if (out_perm && (!slot_in || !y_ptr || slot_ld <= 0)) return DDB200_EINVAL;
  if (slot_out && slot_ld <= 0) return DDB200_EINVAL;
  if (n_y == 0) return 0;
  FillArgs a = {x, y, x_ptr, y_batch, r_per_graph, r, (int)n_y, max_neighbors, exclude_self, row_start, pre_ptr, pre_col,
                out_row, out_col, out_vec, out_eid, slot_out, slot_in, y_ptr, slot_ld, out_perm, row_offset, col_offset};
  const int threads = 256;
  const long long blocks = (n_y * 32 + threads - 1) / threads;
  graph_fill_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(a);
  return (int)cudaGetLastError();
}

// Ligand-receptor edge embedding (see edge_embed_kernel).  rbf_dim in {32, 64}, ns in {16, 24, 32, 48}; other shapes:
// DDB200_EINVAL (the caller then runs the library MLP).
int ddb200_edge_embed(const float* edge_vec, const int32_t* edge_row, const float* u, const float* w1_rbf, const float* w2,
                      const float* b2, int rbf_dim, int ns, const float* rbf_offset, float rbf_coeff, int64_t capacity,
                      const int32_t* n_edges_dev, float* out, void* stream) {
  if (!edge_vec || !edge_row || !u || !w1_rbf || !w2 || !b2 || !rbf_offset || !out || capacity < 0) return DDB200_EINVAL;
  if (capacity == 0) return 0;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  long long blocks = (capacity + 127) / 128;
  if (blocks > (long long)sms * 8) blocks = (long long)sms * 8;
  cudaStream_t st = (cudaStream_t)stream;
#define DDB200_EMBED_CASE(D_, NS_)                                                                                        \
  if (rbf_dim == D_ && ns == NS_) {                                                                                       \
    edge_embed_kernel<D_, NS_><<<(unsigned)blocks, 128, 0, st>>>(edge_vec, edge_row, u, w1_rbf, w2, b2, rbf_offset,       \
                                                                  rbf_coeff, capacity, n_edges_dev, out);                 \
    return (int)cudaGetLastError();                                                                                       \
  }
  DDB200_EMBED_CASE(64, 48) DDB200_EMBED_CASE(32, 48) DDB200_EMBED_CASE(64, 32) DDB200_EMBED_CASE(32, 32)
  DDB200_EMBED_CASE(64, 24) DDB200_EMBED_CASE(32, 24) DDB200_EMBED_CASE(64, 16) DDB200_EMBED_CASE(32, 16)
  DDB200_EMBED_CASE(16, 16) DDB200_EMBED_CASE(8, 16) DDB200_EMBED_CASE(16, 24) DDB200_EMBED_CASE(8, 24)
#undef DDB200_EMBED_CASE
  return DDB200_EINVAL;
}


// Stable sort of an edge list by its convolution target (CSR order) without any host round trip: LSD radix sort of the
// int32 keys with the edge ids as values (cub::DeviceRadixSort::SortPairs, stable), then the CSR row pointer by binary search.
int ddb200_csr_sort_by_target(const int32_t* tgt, int64_t n_edges, int32_t n_rows, int32_t* tgt_sorted, int32_t* perm,
                              int32_t* row_ptr, void* workspace, size_t* workspace_bytes, void* stream) {
  if (!workspace_bytes || n_edges < 0 || n_rows < 0 || n_edges > 0x7fffffffLL) return DDB200_EINVAL;
  size_t cub_bytes = 0;
  int end_bit = 1;
  while (end_bit < 31 && (1LL << end_bit) <= (long long)n_rows) ++end_bit;
  cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const int*)nullptr, (int*)nullptr, (const int*)nullptr,
                                                  (int*)nullptr, (int)n_edges, 0, end_bit, (cudaStream_t)stream);
  if (e != cudaSuccess) return (int)e;
  const size_t ids_bytes = ((size_t)n_edges * sizeof(int) + 255) / 256 * 256;
  const size_t need = ids_bytes + cub_bytes;
  if (!workspace) {                       // size query
    *workspace_bytes = need;
    return 0;
  }
  if (*workspace_bytes < need || (n_edges > 0 && (!tgt || !tgt_sorted || !perm))) return DDB200_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  if (n_edges > 0) {
    int* ids = reinterpret_cast<int*>(workspace);
    iota_kernel<<<(unsigned)((n_edges + 255) / 256), 256, 0, st>>>(ids, n_edges);
    e = cub::DeviceRadixSort::SortPairs(reinterpret_cast<char*>(workspace) + ids_bytes, cub_bytes, tgt, tgt_sorted, ids, perm,
                                        (int)n_edges, 0, end_bit, st);
    if (e != cudaSuccess) return (int)e;
  }
  if (row_ptr) row_ptr_kernel<<<(unsigned)((n_rows + 1 + 255) / 256), 256, 0, st>>>(tgt_sorted, n_edges, n_rows, row_ptr);
  return (int)cudaGetLastError();
}

}  // extern "C"
