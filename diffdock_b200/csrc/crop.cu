// Per-step receptor cropping on the device (utils/utils.py:388-413, called per step at utils/sampling.py:104-109), in the
// masked form: the receptor arrays keep their full size, a dropped residue gets no edges.  Every shape stays static for a
// batch and nothing is read back to the host, so the cropped step can be captured in a CUDA graph.
//   crop_flags_kernel     keep[r] and a copy of the receptor positions with +inf at dropped residues (the cross-graph search
//                         then never sees them: d^2 < r^2 is false for an infinite coordinate);
//   ddb200_crop_select_edges  the static contact graph restricted to edges whose two ends are kept and whose target is
//                         needed, original order;
//   ddb200_receptor_need  the residues whose features can still reach a ligand atom, one set per remaining layer: the
//                         targets of the step's receptor <- ligand edges, then one contact hop back per level.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <cub/device/device_select.cuh>

#include "../../include/diffdock_b200.h"

namespace {

// One warp per residue; lanes walk the ligand atoms of the residue's complex 32 at a time.  The distance test is the
// reference's expression sum((lig - rec) ** 2, -1) < cutoff ** 2 evaluated as torch does on float32 tensors: three rounded
// squares added left to right (no FMA contraction), strict comparison with the float32-rounded cutoff^2.
__global__ void crop_flags_kernel(const float* __restrict__ lig, const int* __restrict__ lig_ptr,
                                  const float* __restrict__ rec, const int* __restrict__ rec_batch, int n_rec,
                                  const float* __restrict__ cut2_table, const int* __restrict__ step_dev,
                                  uint8_t* __restrict__ keep, float* __restrict__ rec_masked) {
  const int lane = threadIdx.x & 31;
  const int r = (int)((blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5);
  if (r >= n_rec) return;
  const float c2 = cut2_table[step_dev ? *step_dev : 0];
  const int b = rec_batch[r];
  const float rx = rec[3 * r], ry = rec[3 * r + 1], rz = rec[3 * r + 2];
  const int beg = lig_ptr[b], end = lig_ptr[b + 1];
  bool any = false;
  for (int j0 = beg; j0 < end && !any; j0 += 32) {
    const int j = j0 + lane;
    bool hit = false;
    if (j < end) {
      const float dx = __fsub_rn(lig[3 * j], rx), dy = __fsub_rn(lig[3 * j + 1], ry), dz = __fsub_rn(lig[3 * j + 2], rz);
      hit = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)) < c2;
    }
    any = __any_sync(0xffffffffu, hit);
  }
  if (lane == 0) keep[r] = any ? 1 : 0;
  if (lane < 3) rec_masked[3 * r + lane] = any ? rec[3 * r + lane] : INFINITY;
}

// keep / need NULL: no condition from that array.
__global__ void edge_flags_kernel(const int* __restrict__ tgt, const int* __restrict__ src, const uint8_t* __restrict__ keep,
                                  const uint8_t* __restrict__ need, long long n, uint8_t* __restrict__ flags,
                                  int* __restrict__ ids) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int t = tgt[e];
  uint8_t f = need ? need[t] : 1;
  if (keep) f &= keep[t] & keep[src[e]];
  flags[e] = f;
  ids[e] = (int)e;
}

// need[cross_tgt[e] - offset] = 1 for e < *n_cross: the residues a ligand atom sends a message to.  Only ones are written,
// so concurrent writes to one residue agree.
__global__ void need_seed_kernel(const int* __restrict__ cross_tgt, const int* __restrict__ n_cross, long long cap,
                                 int offset, uint8_t* __restrict__ need) {
  const long long n = *n_cross < cap ? *n_cross : cap;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x)
    need[cross_tgt[e] - offset] = 1;
}

// One contact hop back: out = in | {src[e] : in[tgt[e]]}, over the edges whose two ends are kept (keep NULL: all).  Threads
// 0 .. n_rec - 1 carry the set over, the rest walk the edges; out starts zeroed and only ones are written.
__global__ void need_expand_kernel(const int* __restrict__ tgt, const int* __restrict__ src, long long n_edges, int n_rec,
                                   const uint8_t* __restrict__ keep, const uint8_t* __restrict__ in,
                                   uint8_t* __restrict__ out) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n_rec) {
    if (in[i]) out[i] = 1;
    return;
  }
  const long long e = i - n_rec;
  if (e >= n_edges) return;
  const int t = tgt[e], s = src[e];
  if (in[t] && (!keep || (keep[t] && keep[s]))) out[s] = 1;
}

// Rows of the selected edges, for e < *n_sel: perm[e] is the position in the static list.
__global__ void edge_gather_kernel(const int* __restrict__ tgt, const int* __restrict__ src, const int* __restrict__ gid,
                                   const int* __restrict__ perm, const int* __restrict__ n_sel, long long cap, int offset,
                                   int* __restrict__ out_tgt, int* __restrict__ out_src, int* __restrict__ out_gid) {
  const long long n = *n_sel < cap ? *n_sel : cap;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const int p = perm[e];
    out_tgt[e] = tgt[p] + offset;
    out_src[e] = src[p] + offset;
    if (out_gid) out_gid[e] = gid[p];
  }
}

size_t align256(size_t b) { return (b + 255) / 256 * 256; }

}  // namespace

extern "C" {

int ddb200_crop_flags(const float* lig_pos, const int32_t* lig_ptr, const float* rec_pos, const int32_t* rec_batch,
                      int64_t n_rec, const float* cutoff2_table, const int32_t* step_dev, uint8_t* keep,
                      float* rec_pos_masked, void* stream) {
  if (!lig_pos || !lig_ptr || !rec_pos || !rec_batch || !cutoff2_table || !keep || !rec_pos_masked || n_rec < 0 ||
      n_rec > 0x7fffffffLL / 32)
    return DDB200_EINVAL;
  if (n_rec == 0) return 0;
  const int threads = 256;
  const long long blocks = (n_rec * 32 + threads - 1) / threads;
  crop_flags_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(lig_pos, lig_ptr, rec_pos, rec_batch, (int)n_rec,
                                                                            cutoff2_table, step_dev, keep, rec_pos_masked);
  return (int)cudaGetLastError();
}

// Stream compaction with cub::DeviceSelect::Flagged (stable) over the edge ids (flag: both ends kept, target needed), then a gather of the selected rows bounded
// by the device-side count.  Workspace: flags [n] bytes | ids [n] int32 | cub temporary storage.
int ddb200_crop_select_edges(const int32_t* tgt, const int32_t* src, const int32_t* gid, int64_t n_edges,
                             const uint8_t* keep, const uint8_t* need, int32_t offset, int32_t* out_tgt, int32_t* out_src,
                             int32_t* out_perm, int32_t* out_gid, int32_t* n_selected, void* workspace,
                             size_t* workspace_bytes, void* stream) {
  if (!workspace_bytes || n_edges < 0 || n_edges > 0x7fffffffLL) return DDB200_EINVAL;
  size_t cub_bytes = 0;
  cudaError_t e = cub::DeviceSelect::Flagged(nullptr, cub_bytes, (const int*)nullptr, (const uint8_t*)nullptr, (int*)nullptr,
                                             (int*)nullptr, (int)n_edges, (cudaStream_t)stream);
  if (e != cudaSuccess) return (int)e;
  const size_t flags_bytes = align256((size_t)n_edges), ids_bytes = align256((size_t)n_edges * sizeof(int));
  const size_t ws_bytes = flags_bytes + ids_bytes + cub_bytes;
  if (!workspace) {                       // size query
    *workspace_bytes = ws_bytes;
    return 0;
  }
  if (*workspace_bytes < ws_bytes || !n_selected) return DDB200_EINVAL;
  if (n_edges > 0 && (!tgt || !src || !out_tgt || !out_src || !out_perm || (out_gid && !gid))) return DDB200_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  if (n_edges == 0) return (int)cudaMemsetAsync(n_selected, 0, sizeof(int32_t), st);
  uint8_t* flags = reinterpret_cast<uint8_t*>(workspace);
  int* ids = reinterpret_cast<int*>(reinterpret_cast<char*>(workspace) + flags_bytes);
  void* tmp = reinterpret_cast<char*>(workspace) + flags_bytes + ids_bytes;
  const unsigned blocks = (unsigned)((n_edges + 255) / 256);
  edge_flags_kernel<<<blocks, 256, 0, st>>>(tgt, src, keep, need, n_edges, flags, ids);
  e = cub::DeviceSelect::Flagged(tmp, cub_bytes, ids, flags, out_perm, n_selected, (int)n_edges, st);
  if (e != cudaSuccess) return (int)e;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const unsigned gblocks = (unsigned)(blocks < (unsigned)sms * 8 ? blocks : (unsigned)sms * 8);
  edge_gather_kernel<<<gblocks, 256, 0, st>>>(tgt, src, gid, out_perm, n_selected, n_edges, offset, out_tgt, out_src, out_gid);
  return (int)cudaGetLastError();
}

// need [n_levels][n_rec]: one memset, the seed, then one expansion launch per further level.
int ddb200_receptor_need(const int32_t* cross_tgt, const int32_t* n_cross, int64_t cross_cap, int32_t offset,
                         const int32_t* tgt, const int32_t* src, int64_t n_edges, const uint8_t* keep, int64_t n_rec,
                         int32_t n_levels, uint8_t* need, void* stream) {
  if (cross_cap < 0 || n_edges < 0 || n_rec < 0 || n_levels < 0 || n_edges + n_rec > 0x7fffffffLL ||
      cross_cap > 0x7fffffffLL)
    return DDB200_EINVAL;
  if (n_levels == 0 || n_rec == 0) return 0;
  if (!need || (cross_cap > 0 && (!cross_tgt || !n_cross)) || (n_edges > 0 && (!tgt || !src))) return DDB200_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(need, 0, (size_t)n_levels * (size_t)n_rec, st);
  if (e != cudaSuccess) return (int)e;
  if (cross_cap > 0) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const long long b = (cross_cap + 255) / 256;
    need_seed_kernel<<<(unsigned)(b < sms * 8LL ? b : sms * 8LL), 256, 0, st>>>(cross_tgt, n_cross, cross_cap, offset, need);
  }
  const unsigned blocks = (unsigned)((n_edges + n_rec + 255) / 256);
  for (int k = 1; k < n_levels; ++k)
    need_expand_kernel<<<blocks, 256, 0, st>>>(tgt, src, n_edges, (int)n_rec, keep, need + (size_t)(k - 1) * n_rec,
                                               need + (size_t)k * n_rec);
  return (int)cudaGetLastError();
}

}  // extern "C"
