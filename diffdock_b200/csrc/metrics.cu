// Pose metrics of evaluation (evaluate.py:474-486, :503-505) as one kernel: the symmetry-corrected RMSD of every sampled
// pose against every crystal pose over a precomputed automorphism table, the centroid distance and the minimum
// self-distance.  One CTA per pose; the pose and one crystal pose at a time sit in shared memory as float64, and the warps
// split the automorphisms: warp w sweeps a = w, w + 8, ... reading each table row with consecutive lanes on consecutive
// atoms, so a table of thousands of rows costs no more registers than one.  Every sum has a fixed order (lane-strided,
// then a butterfly), every arg-min keeps the lowest index among equal values, and there are no atomics.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/diffdock_b200_metrics.h"

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

__device__ __forceinline__ double warp_sum(double v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// min that keeps a NaN once it has met one (numpy's min propagates NaN)
__device__ __forceinline__ double nan_min(double a, double b) { return (b < a || b != b) ? b : a; }

// Sum over atoms of one coordinate array, by warp 0 (every lane gets the same value).
__device__ __forceinline__ double atom_sum(const double* v, int n, int lane) {
  double s = 0.0;
  for (int i = lane; i < n; i += 32) s += v[i];
  return warp_sum(s);
}

__global__ void __launch_bounds__(kThreads, 2) pose_metrics_kernel(
    const float* __restrict__ pos, const double* __restrict__ refs, const int* __restrict__ aut,
    const int* __restrict__ layout, int max_atoms, double* __restrict__ rmsd, double* __restrict__ rmsd_min,
    double* __restrict__ centroid_dist, double* __restrict__ min_self_dist, int* __restrict__ best_aut,
    int* __restrict__ err) {
  extern __shared__ double sm[];
  double* px = sm;
  double* py = px + max_atoms;
  double* pz = py + max_atoms;
  double* rx = pz + max_atoms;
  double* ry = rx + max_atoms;
  double* rz = ry + max_atoms;
  __shared__ double w_best[kWarps];
  __shared__ int w_arg[kWarps];
  __shared__ int bad;

  const int b = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int* row = layout + 8 * (long long)b;
  const int pos_off = row[0], n = row[1], ref_off = row[2], n_refs = row[3], aut_off = row[4], n_aut = row[5];
  const int rmsd_off = row[6], rmsd_ld = row[7];
  const double nan = __longlong_as_double(0x7ff8000000000000ll);

  if (n < 1 || n > max_atoms || n_refs < 1 || n_aut < 1) {
    if (tid == 0) {
      *err = 1;
      for (int g = 0; g < n_refs; ++g) rmsd[rmsd_off + (long long)g * rmsd_ld] = nan;
      rmsd_min[b] = centroid_dist[b] = min_self_dist[b] = nan;
      best_aut[b] = -1;
    }
    return;
  }
  if (tid == 0) bad = 0;
  for (int i = tid; i < n; i += kThreads) {
    const float* p = pos + 3 * ((long long)pos_off + i);
    px[i] = (double)p[0];
    py[i] = (double)p[1];
    pz[i] = (double)p[2];
  }
  __syncthreads();

  double pcx = 0.0, pcy = 0.0, pcz = 0.0;          // pose centroid, held by warp 0
  if (warp == 0) {
    pcx = atom_sum(px, n, lane) / n;
    pcy = atom_sum(py, n, lane) / n;
    pcz = atom_sum(pz, n, lane) / n;
  }
  double best_all = INFINITY, cdist = INFINITY;     // thread 0's running minima over the crystal poses
  int arg_all = -1;

  for (int g = 0; g < n_refs; ++g) {
    const double* r = refs + 3 * ((long long)ref_off + (long long)g * n);
    for (int i = tid; i < n; i += kThreads) {
      rx[i] = r[3 * i];
      ry[i] = r[3 * i + 1];
      rz[i] = r[3 * i + 2];
    }
    __syncthreads();

    double best = INFINITY;
    int arg = -1;
    bool oob = false;
    for (int a = warp; a < n_aut; a += kWarps) {
      const int* perm = aut + (long long)aut_off + (long long)a * n;
      double s = 0.0;
      for (int i = lane; i < n; i += 32) {
        int j = __ldg(perm + i);
        if ((unsigned)j >= (unsigned)n) {
          oob = true;
          j = 0;
        }
        const double dx = rx[i] - px[j], dy = ry[i] - py[j], dz = rz[i] - pz[j];
        s += dx * dx + dy * dy + dz * dz;
      }
      s = warp_sum(s);
      if (s < best) {                                 // a ascends within the warp: the first of equal values stays
        best = s;
        arg = a;
      }
    }
    if (oob) bad = 1;
    if (lane == 0) {
      w_best[warp] = best;
      w_arg[warp] = arg;
    }
    double rcx = 0.0, rcy = 0.0, rcz = 0.0;
    if (warp == 0) {
      rcx = atom_sum(rx, n, lane) / n;
      rcy = atom_sum(ry, n, lane) / n;
      rcz = atom_sum(rz, n, lane) / n;
    }
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < kWarps; ++w)
        if (w_best[w] < best || (w_best[w] == best && w_arg[w] >= 0 && (arg < 0 || w_arg[w] < arg))) {
          best = w_best[w];
          arg = w_arg[w];
        }
      rmsd[rmsd_off + (long long)g * rmsd_ld] = sqrt(best / n);
      if (best < best_all) {
        best_all = best;
        arg_all = arg;
      }
      const double dx = pcx - rcx, dy = pcy - rcy, dz = pcz - rcz;
      cdist = g == 0 ? sqrt(dx * dx + dy * dy + dz * dz) : nan_min(cdist, sqrt(dx * dx + dy * dy + dz * dz));
    }
    __syncthreads();                                  // rx.. are overwritten by the next crystal pose
  }

  // minimum over pairs i < j of the squared distance; a min is exact in any order
  double d2 = INFINITY;
  for (int i = tid; i < n; i += kThreads)
    for (int j = i + 1; j < n; ++j) {
      const double dx = px[i] - px[j], dy = py[i] - py[j], dz = pz[i] - pz[j];
      d2 = nan_min(d2, dx * dx + dy * dy + dz * dz);
    }
  for (int o = 16; o > 0; o >>= 1) d2 = nan_min(d2, __shfl_xor_sync(0xffffffffu, d2, o));
  if (lane == 0) w_best[warp] = d2;
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < kWarps; ++w) d2 = nan_min(d2, w_best[w]);
    if (bad) {
      *err = 1;
      for (int g = 0; g < n_refs; ++g) rmsd[rmsd_off + (long long)g * rmsd_ld] = nan;
      rmsd_min[b] = nan;
      arg_all = -1;
    } else {
      rmsd_min[b] = sqrt(best_all / n);
    }
    best_aut[b] = arg_all;
    centroid_dist[b] = cdist;
    min_self_dist[b] = sqrt(d2);
  }
}

}  // namespace

extern "C" int ddb200_pose_metrics(const float* pos, const double* refs, const int32_t* aut, const int32_t* layout,
                                   int64_t n_poses, int32_t max_atoms, double* rmsd, double* rmsd_min,
                                   double* centroid_dist, double* min_self_dist, int32_t* best_aut, int32_t* err,
                                   void* stream) {
  if (n_poses < 0 || n_poses > 0x7fffffff) return DDB200_EINVAL;
  if (n_poses == 0) return 0;
  if (!pos || !refs || !aut || !layout || !rmsd || !rmsd_min || !centroid_dist || !min_self_dist || !best_aut || !err)
    return DDB200_EINVAL;
  if (max_atoms < 1 || max_atoms > DDB200_METRICS_MAX_ATOMS) return DDB200_EINVAL;
  const size_t smem = 6 * sizeof(double) * (size_t)max_atoms;
  pose_metrics_kernel<<<(unsigned)n_poses, kThreads, smem, (cudaStream_t)stream>>>(
      pos, refs, aut, layout, max_atoms, rmsd, rmsd_min, centroid_dist, min_self_dist, best_aut, err);
  return (int)cudaGetLastError();
}
