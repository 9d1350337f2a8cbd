// Fused tensor-product graph convolution for sm_90a (H100).
//
// One warp owns a run of 32 consecutive edges (edges are CSR-sorted by destination).  For every edge it
//   1. gathers the source node's irreps row (L2-resident) into shared memory,
//   2. evaluates the real spherical harmonics of the edge vector in registers,
//   3. folds Clebsch-Gordan blocks x Y into small per-path matrices M and forms z[u,k] = sum_i x[u,i] M[i,k],
//   4. streams the edge's weight row (the dominant HBM stream, 11-28 KB per edge) through a private ring of shared
//      memory stages filled by 1-D TMA bulk copies (cp.async.bulk + mbarrier complete_tx) and contracts it with z,
//      each weight being used for 1..5 FMAs and never re-read,
//   5. keeps the running sum of a destination row in a lane-distributed shared accumulator and flushes it with
//      fp32 reductions (RED.ADD) when the destination changes.
// Everything that depends on the irreps (paths, CG entries, tile -> lane mapping, TMA chunking) comes from the table
// blob built by diffdock_b200/tp_table.py, so one binary serves every (ns, nv, sh_lmax, ...) configuration.
//
// Reference semantics: models/tensor_layers.py:125-231 (tp_scatter_simple / tp_scatter_multigroup).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/diffdock_b200.h"
#include "../../include/diffdock_b200_fixed.h"

namespace {

constexpr int WARP = 32;
constexpr int HDR = 32;
constexpr int ERUN = 32;          // edges per work unit (one lane holds one edge's indices/geometry)
constexpr int MAX_XREG = 8;       // register prefetch of the next source row covers D_in <= 256
constexpr uint32_t MAGIC = 0x44423232u;
template <int N>
struct IC { static constexpr int value = N; };

struct KParams {
  const float* x; long long x_stride;
  const int* esrc; const int* edst;
  const float* geo; const float* ew;
  const float* w; long long w_stride;
  long long n_edges;
  float* sum; float* cnt;
  long long* sum_fx; int* err;    // deterministic kernel: int64 accumulator in units of 2^-32, sticky error word
  const int* iblob; const float* fblob;
  int n_ints, n_terms;
  int stages, warps;
  int warp_floats;    // per-warp scratch size in floats
  int warp_base_off;  // byte offset of the first warp's scratch inside dynamic shared memory
  int stage_floats;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// 1-D TMA bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
      ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}
__device__ __forceinline__ bool elect_one() {   // exactly one lane of the (converged) warp gets true
  uint32_t pred;
  asm volatile("{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.u32 %0, 1, 0, P;\n\t}" : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ uint64_t policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}

// ---- deterministic scatter: every edge's output values are converted to 64-bit fixed point (v * 2^32, rounded to nearest)
// and a row is summed as integers, so that its sum does not depend on the order of its edges or on how they are split
// over warps, launches or kernels.  |v| >= 2^31 and non-finite values saturate and set the sticky error word (bit 0).
constexpr int MAX_FX = 8;         // output values per lane: D_out <= 256
__device__ __forceinline__ long long to_fixed(float v, int* err) {
  const float s = v * 0x1p32f;
  if (fabsf(s) < 0x1p63f) return __float2ll_rn(s);
  atomicOr(err, 1);
  return v > 0.f ? 0x7fffffffffffffffLL : (v < 0.f ? -0x7fffffffffffffffLL : 0LL);
}
__device__ __forceinline__ void red_add_u64(long long* addr, long long v) {
  asm volatile("red.global.add.u64 [%0], %1;" ::"l"(addr), "l"((unsigned long long)v) : "memory");
}

// ---- weight-tile contraction: acc[v*DOUT+k] += W[u, c*VEC+v] * z[u, k] over this lane's rows of the tile -----------
// Lane (r, c) owns VEC consecutive output channels and every R-th row; W comes from the TMA stage with one
// LDS.128/LDS.64 per row, z[u, :] with one LDS (DOUT=1) or one LDS.128 (DOUT=3, rows padded to 4 floats).
template <int VEC, int DOUT>
__device__ __forceinline__ void fma_row(const float* __restrict__ wp, const float* __restrict__ zp, float* __restrict__ acc) {
  float w[VEC], z[DOUT];
  if constexpr (VEC == 4) {
    const float4 t = *reinterpret_cast<const float4*>(wp);
    w[0] = t.x; w[1] = t.y; w[2] = t.z; w[3] = t.w;
  } else {
    const float2 t = *reinterpret_cast<const float2*>(wp);
    w[0] = t.x; w[1] = t.y;
  }
  if constexpr (DOUT == 1) {
    z[0] = *zp;
  } else {
    const float4 t = *reinterpret_cast<const float4*>(zp);
    z[0] = t.x; z[1] = t.y; z[2] = t.z;
  }
#pragma unroll
  for (int v = 0; v < VEC; ++v)
#pragma unroll
    for (int k = 0; k < DOUT; ++k) acc[v * DOUT + k] = fmaf(w[v], z[k], acc[v * DOUT + k]);
}

template <int VEC, int DOUT>
__device__ __forceinline__ void run_rows(const float* __restrict__ wp, const float* __restrict__ zp, int n_it, int wstep,
                                         int zstep, float* __restrict__ acc) {
  int it = 0;
  for (; it + 2 <= n_it; it += 2) {     // two independent rows in flight
    fma_row<VEC, DOUT>(wp, zp, acc);
    fma_row<VEC, DOUT>(wp + wstep, zp + zstep, acc);
    wp += 2 * wstep;
    zp += 2 * zstep;
  }
  if (it < n_it) fma_row<VEC, DOUT>(wp, zp, acc);
}

// generic fallback (any 2l+1 <= 9, scalar weight loads): second-order representations, odd multiplicities
__device__ __noinline__ void run_rows_generic(const float* __restrict__ wp, const float* __restrict__ zp, int n_it,
                                              int wstep, int zstep, int dout, float* __restrict__ acc) {
  for (int it = 0; it < n_it; ++it) {
    const float wv = *wp;
    for (int k = 0; k < dout; ++k) acc[k] = fmaf(wv, zp[k], acc[k]);
    wp += wstep;
    zp += zstep;
  }
}

template <bool FIXED>
__device__ __forceinline__ void tpconv_accumulate_body(const KParams& p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  // ---- CTA-shared: table copy ---------------------------------------------------------------------------------
  int* tb = reinterpret_cast<int*>(smem_raw);
  for (int i = threadIdx.x; i < p.n_ints; i += blockDim.x) tb[i] = p.iblob[i];
  float* tval = reinterpret_cast<float*>(tb + ((p.n_ints + 3) & ~3));
  for (int i = threadIdx.x; i < p.n_terms; i += blockDim.x) tval[i] = p.fblob[i];
  uint64_t* bars = reinterpret_cast<uint64_t*>(tval + ((p.n_terms + 3) & ~3));
  float* warp_base = reinterpret_cast<float*>(smem_raw + p.warp_base_off);   // offset planned on the host (128-B aligned)
  if (lane == 0)
    for (int s = 0; s < p.stages; ++s) mbar_init(&bars[warp * p.stages + s], 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();

  const int n_paths = tb[1], n_chunks = tb[3], n_ment = tb[4];
  const int D_in = tb[6], D_sh = tb[7], D_out = tb[8], lmax = tb[9];
  const int z_total = tb[10], m_total = tb[11], n_acc = tb[12];
  const int* paths = tb + tb[15];
  const int* tiles = tb + tb[16];
  const int* chunks = tb + tb[17];
  const int* ment = tb + tb[18];
  const int* terms_y = tb + tb[19];
  const int* outmap = tb + tb[20];

  // lane -> (row group r, column slot c) for the (at most four) lanes-per-row values the table uses
  int lr[4], lc[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int lpr = tb[22 + q] > 0 ? tb[22 + q] : 32;
    lr[q] = lane / lpr;
    lc[q] = lane - lr[q] * lpr;
  }

  // ---- per-warp scratch ---------------------------------------------------------------------------------------
  float* wsm = warp_base + (size_t)warp * p.warp_floats;
  float* stage_base = wsm;                                     // stages * stage_floats
  float* zs = stage_base + (size_t)p.stages * p.stage_floats;  // z_total (16-byte aligned rows)
  float* racc = zs + ((z_total + 3) & ~3);                     // n_acc * 32
  float* xs = racc + n_acc * WARP;                             // D_in
  float* ys = xs + ((D_in + 3) & ~3);                          // D_sh
  float* ms = ys + ((D_sh + 3) & ~3);                          // m_total
  uint64_t* mybar = bars + warp * p.stages;
  for (int i = lane; i < n_acc * WARP; i += WARP) racc[i] = 0.f;
  for (int i = lane; i < m_total; i += WARP) ms[i] = 0.f;   // structurally-zero CG entries are never rewritten
  for (int i = lane; i < z_total; i += WARP) zs[i] = 0.f;   // padding lanes of z rows stay zero
  __syncwarp();

  const long long E = p.n_edges;
  const long long n_units = (E + ERUN - 1) / ERUN;
  const long long TW = (long long)gridDim.x * p.warps;
  const long long gw = (long long)blockIdx.x * p.warps + warp;
  const uint64_t policy = policy_evict_first();

  // ---- producer cursor: warp-uniform state, one elected lane issues ------------------------------------------
  // Kept cheap on purpose: it runs once per TMA chunk (~16 times per edge).  Row pointer and edge countdown are
  // advanced incrementally; stage / barrier operands are 32-bit shared-window addresses.
  const uint32_t stage_u32 = smem_u32(stage_base), bar_u32 = smem_u32(mybar);
  const uint32_t stage_bytes = (uint32_t)p.stage_floats * 4u;
  const long long row_bytes = p.w_stride * 4;
  const char* const w_bytes = reinterpret_cast<const char*>(p.w);
  long long p_unit = gw;
  bool p_valid = gw < n_units;
  const char* p_row = w_bytes + gw * ERUN * row_bytes;
  int p_left = p_valid ? (int)((E - gw * ERUN) < ERUN ? (E - gw * ERUN) : ERUN) : 0;
  int p_c = 0;
  uint32_t p_stage = 0;
  auto issue_next = [&]() {
    if (p_valid) {
      const int goff = chunks[4 * p_c + 2], nfl = chunks[4 * p_c + 3];
      if (elect_one()) {
        const uint32_t bar = bar_u32 + p_stage * 8u, bytes = (uint32_t)nfl * 4u;
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
        asm volatile(
            "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
            ::"r"(stage_u32 + p_stage * stage_bytes), "l"(p_row + (long long)goff * 4), "r"(bytes), "r"(bar), "l"(policy)
            : "memory");
      }
      if (++p_c == n_chunks) {
        p_c = 0;
        p_row += row_bytes;
        if (--p_left == 0) {
          p_unit += TW;
          p_valid = p_unit < n_units;
          p_row = w_bytes + p_unit * ERUN * row_bytes;
          const long long rem = E - p_unit * ERUN;
          p_left = (int)(rem < ERUN ? rem : ERUN);
        }
      }
      p_stage = (p_stage + 1 == (uint32_t)p.stages) ? 0u : p_stage + 1;
    }
  };
  for (int s = 0; s < p.stages; ++s) issue_next();

  int c_stage = 0;
  uint32_t c_par = 0;
  const int nxr = (D_in + WARP - 1) / WARP;

  long long fx[FIXED ? MAX_FX : 1];          // FIXED: this lane's output values o = lane + 32 j of the current row
#pragma unroll
  for (int j = 0; j < (FIXED ? MAX_FX : 1); ++j) fx[j] = 0;
  auto flush_row = [&](int row, int row_edges) {
    __syncwarp();
    if constexpr (FIXED) {
      long long* srow = p.sum_fx + (long long)row * D_out;
#pragma unroll
      for (int j = 0; j < MAX_FX; ++j) {
        if (lane + WARP * j < D_out) red_add_u64(srow + lane + WARP * j, fx[j]);
        fx[j] = 0;
      }
    } else {
      float* srow = p.sum + (long long)row * D_out;
      for (int o = lane; o < D_out; o += WARP) {
        const int* om = outmap + 3 * o;
        float v = 0.f;
        for (int r = 0; r < om[2]; ++r) v += racc[om[0] + r * om[1]];
        atomicAdd(srow + o, v);
      }
    }
    if (p.cnt && lane == 0) atomicAdd(p.cnt + row, (float)row_edges);
    if constexpr (!FIXED) {       // FIXED: the accumulators were cleared after the row's last edge
      __syncwarp();
      for (int j = lane; j < n_acc * WARP; j += WARP) racc[j] = 0.f;
    }
  };

  for (long long unit = gw; unit < n_units; unit += TW) {
    const long long e0 = unit * ERUN;
    const int ne = (int)((E - e0) < ERUN ? (E - e0) : ERUN);
    // one edge per lane: indices + geometry
    int l_src = 0, l_dst = -1;
    float l_vx = 0.f, l_vy = 0.f, l_vz = 0.f, l_ew = 1.f;
    if (lane < ne) {
      l_src = p.esrc[e0 + lane];
      l_dst = p.edst[e0 + lane];
      if (lmax >= 0) {
        const float* g = p.geo + 3 * (e0 + lane);
        l_vx = g[0]; l_vy = g[1]; l_vz = g[2];
      }
      if (p.ew) l_ew = p.ew[e0 + lane];
    }
    int cur_row = -1, row_edges = 0;
    float xr[MAX_XREG];
    {  // source row of the first edge
      const int s0 = __shfl_sync(0xffffffffu, l_src, 0);
      const float* xrow = p.x + (long long)s0 * p.x_stride;
#pragma unroll
      for (int j = 0; j < MAX_XREG; ++j) xr[j] = (j < nxr && lane + WARP * j < D_in) ? __ldg(xrow + lane + WARP * j) : 0.f;
    }
    for (int i = 0; i < ne; ++i) {
      const int dst = __shfl_sync(0xffffffffu, l_dst, i);
      const int src = __shfl_sync(0xffffffffu, l_src, i);
      const float ewt = __shfl_sync(0xffffffffu, l_ew, i);
      if (dst != cur_row) {
        if (cur_row >= 0) flush_row(cur_row, row_edges);
        cur_row = dst;
        row_edges = 0;
      }
      ++row_edges;
      // ---- stage x row (prefetched registers -> smem); large rows fall back to direct loads -------------------
#pragma unroll
      for (int j = 0; j < MAX_XREG; ++j)
        if (j < nxr && lane + WARP * j < D_in) xs[lane + WARP * j] = xr[j];
      if (nxr > MAX_XREG) {
        const float* xrow = p.x + (long long)src * p.x_stride;
        for (int j = MAX_XREG * WARP + lane; j < D_in; j += WARP) xs[j] = __ldg(xrow + j);
      }
      // ---- spherical harmonics -----------------------------------------------------------------------------------
      if (lmax >= 0) {
        float vx = __shfl_sync(0xffffffffu, l_vx, i), vy = __shfl_sync(0xffffffffu, l_vy, i),
              vz = __shfl_sync(0xffffffffu, l_vz, i);
        const float nrm = fmaxf(sqrtf(vx * vx + vy * vy + vz * vz), 1e-12f);
        vx /= nrm; vy /= nrm; vz /= nrm;
        if (lane == 0) {
          ys[0] = 1.f;
          if (lmax >= 1) {
            const float s3 = 1.7320508075688772f;
            ys[1] = s3 * vx; ys[2] = s3 * vy; ys[3] = s3 * vz;
          }
          if (lmax >= 2) {
            const float s5 = 2.23606797749979f, s15 = 3.872983346207417f;
            ys[4] = s15 * vx * vz;
            ys[5] = s15 * vx * vy;
            ys[6] = s5 * (vy * vy - 0.5f * (vx * vx + vz * vz));
            ys[7] = s15 * vy * vz;
            ys[8] = 0.5f * s15 * (vz * vz - vx * vx);
          }
        }
      } else {
        const float* g = p.geo + (e0 + i) * (long long)D_sh;
        for (int j = lane; j < D_sh; j += WARP) ys[j] = __ldg(g + j);
      }
      __syncwarp();
      // ---- M[i,k] = edge_weight * sum_j (coef*C[i,j,k]) * Y[j] --------------------------------------------------
      for (int m = lane; m < n_ment; m += WARP) {
        const int* me = ment + 3 * m;
        float a = 0.f;
        for (int q = me[1]; q < me[1] + me[2]; ++q) a = fmaf(tval[q], ys[terms_y[q]], a);
        ms[me[0]] = a * ewt;
      }
      __syncwarp();
      // ---- z[u,k] = sum_i x[u,i] * M[i,k] -----------------------------------------------------------------------
      for (int q = 0; q < n_paths; ++q) {
        const int* pa = paths + 8 * q;
        const int mul_in = pa[1];
        const float* xp = xs + pa[0];
        const float* mp = ms + pa[5];
        float* zp = zs + pa[4];
        switch (pa[7]) {
          case 1:   // 0 x l -> 0 : z[u] = x[u] M
            for (int u = lane; u < mul_in; u += WARP) zp[u] = xp[u] * mp[0];
            break;
          case 2: { // scalar in, vector out: z[u,:] = x[u] M[0,:]
            const float m0 = mp[0], m1 = mp[1], m2 = mp[2];
            for (int u = lane; u < mul_in; u += WARP) {
              const float xv = xp[u];
              *reinterpret_cast<float4*>(zp + 4 * u) = make_float4(xv * m0, xv * m1, xv * m2, 0.f);
            }
          } break;
          case 3: { // vector in, scalar out: z[u] = x[u,:] . M[:,0]
            const float m0 = mp[0], m1 = mp[1], m2 = mp[2];
            for (int u = lane; u < mul_in; u += WARP)
              zp[u] = fmaf(xp[3 * u], m0, fmaf(xp[3 * u + 1], m1, xp[3 * u + 2] * m2));
          } break;
          case 4: { // vector in, vector out: z[u,:] = x[u,:] M (3x3)
            for (int u = lane; u < mul_in; u += WARP) {
              const float x0 = xp[3 * u], x1 = xp[3 * u + 1], x2 = xp[3 * u + 2];
              *reinterpret_cast<float4*>(zp + 4 * u) =
                  make_float4(fmaf(x0, mp[0], fmaf(x1, mp[3], x2 * mp[6])), fmaf(x0, mp[1], fmaf(x1, mp[4], x2 * mp[7])),
                              fmaf(x0, mp[2], fmaf(x1, mp[5], x2 * mp[8])), 0.f);
            }
          } break;
          default: {
            const int din = pa[2], dout = pa[3], zstr = pa[6];
            const int n = mul_in * dout;
            for (int idx = lane; idx < n; idx += WARP) {
              const int u = idx / dout, k = idx - u * dout;
              float a = 0.f;
              for (int ii = 0; ii < din; ++ii) a = fmaf(xp[u * din + ii], mp[ii * dout + k], a);
              zp[u * zstr + k] = a;
            }
          }
        }
      }
      __syncwarp();
      // ---- prefetch the next edge's source row while the weights are contracted --------------------------------
      if (i + 1 < ne) {
        const int s1 = __shfl_sync(0xffffffffu, l_src, i + 1);
        const float* xrow = p.x + (long long)s1 * p.x_stride;
#pragma unroll
        for (int j = 0; j < MAX_XREG; ++j)
          xr[j] = (j < nxr && lane + WARP * j < D_in) ? __ldg(xrow + lane + WARP * j) : 0.f;
      }
      // ---- weight contraction: one accumulator run per output irrep, tiles = row pieces of the weight blocks --------
      {
        const int n_tiles = tb[2];
        const int4* tiles4 = reinterpret_cast<const int4*>(tiles);
        const float* st = stage_base;
        int t = 0;
        // tile loop of one accumulator run, specialised on (vector width, 2l+1); also drives the TMA ring
        auto run_group = [&](auto vec_c, auto dout_c, int woff, int zoff, int wstep, int zstep, bool active, int r,
                             float* as) {
          constexpr int VEC = decltype(vec_c)::value, DOUT = decltype(dout_c)::value;
          float acc[VEC * DOUT];
#pragma unroll
          for (int q = 0; q < VEC * DOUT; ++q) acc[q] = 0.f;
          for (;;) {
            const int4 ta = tiles4[4 * t];
            if (ta.w & 4) {      // first tile of a TMA chunk: wait for its stage
              while (!mbar_try_wait(&mybar[c_stage], c_par)) {}
              st = stage_base + c_stage * p.stage_floats;
            }
            const int n_it = active ? (ta.z & 0xffff) + (r < (ta.z >> 16) ? 1 : 0) : 0;
            run_rows<VEC, DOUT>(st + ta.x + woff, zs + ta.y + zoff, n_it, wstep, zstep, acc);
            if (ta.w & 8) {      // last tile of the chunk: hand the stage back to the TMA producer
              __syncwarp();
              issue_next();
              if (++c_stage == p.stages) { c_stage = 0; c_par ^= 1u; }
            }
            ++t;
            if (ta.w & 2) break;
          }
#pragma unroll
          for (int q = 0; q < VEC * DOUT; ++q) as[q * WARP] += acc[q];
        };
        while (t < n_tiles) {
          const int4 gb = tiles4[4 * t + 1], gc = tiles4[4 * t + 2];
          const int rs = gb.x, dout = gb.y, vec = gb.z, li = gb.w, R = gc.x, accb = gc.y, zstr = gc.z, kind = gc.w;
          const int r = li == 0 ? lr[0] : (li == 1 ? lr[1] : (li == 2 ? lr[2] : lr[3]));
          const int cc = li == 0 ? lc[0] : (li == 1 ? lc[1] : (li == 2 ? lc[2] : lc[3]));
          const bool active = r < R;
          const int woff = r * rs + cc * vec, zoff = r * zstr, wstep = R * rs, zstep = R * zstr;
          float* as = racc + accb + lane;
          switch (kind) {
            case 1: run_group(IC<4>{}, IC<1>{}, woff, zoff, wstep, zstep, active, r, as); break;
            case 2: run_group(IC<4>{}, IC<3>{}, woff, zoff, wstep, zstep, active, r, as); break;
            case 3: run_group(IC<2>{}, IC<1>{}, woff, zoff, wstep, zstep, active, r, as); break;
            case 4: run_group(IC<2>{}, IC<3>{}, woff, zoff, wstep, zstep, active, r, as); break;
            default: {   // generic: scalar weight loads, any 2l+1 <= 9, accumulators in a private (stack) array
              float acc[9];
#pragma unroll
              for (int q = 0; q < 9; ++q) acc[q] = 0.f;
              for (;;) {
                const int4 ta = tiles4[4 * t];
                if (ta.w & 4) {
                  while (!mbar_try_wait(&mybar[c_stage], c_par)) {}
                  st = stage_base + c_stage * p.stage_floats;
                }
                const int n_it = active ? (ta.z & 0xffff) + (r < (ta.z >> 16) ? 1 : 0) : 0;
                run_rows_generic(st + ta.x + woff, zs + ta.y + zoff, n_it, wstep, zstep, dout, acc);
                if (ta.w & 8) {
                  __syncwarp();
                  issue_next();
                  if (++c_stage == p.stages) { c_stage = 0; c_par ^= 1u; }
                }
                ++t;
                if (ta.w & 2) break;
              }
              for (int q = 0; q < vec * dout; ++q) as[q * WARP] += acc[q];
            } break;
          }
        }
      }
      if constexpr (FIXED) {      // this edge's output values alone (racc was clear before it), converted and summed
        __syncwarp();
#pragma unroll
        for (int j = 0; j < MAX_FX; ++j) {
          const int o = lane + WARP * j;
          if (o < D_out) {
            const int* om = outmap + 3 * o;
            float v = 0.f;
            for (int r = 0; r < om[2]; ++r) v += racc[om[0] + r * om[1]];
            fx[j] += to_fixed(v, p.err);
          }
        }
        __syncwarp();
        for (int j = lane; j < n_acc * WARP; j += WARP) racc[j] = 0.f;
        __syncwarp();
      }
    }
    if (cur_row >= 0) flush_row(cur_row, row_edges);   // last row of this run
  }
}

__global__ void __launch_bounds__(512, 1) tpconv_accumulate_kernel(const KParams p) { tpconv_accumulate_body<false>(p); }
// deterministic instantiation (ddb200_tpconv_accumulate_fixed)
__global__ void __launch_bounds__(512, 1) tpconv_accumulate_fixed_kernel(const KParams p) { tpconv_accumulate_body<true>(p); }

__global__ void tpconv_finalize_kernel(const float* __restrict__ sum, const float* __restrict__ cnt, long long n_rows,
                                       int d_out, int mean, const float* __restrict__ bn_scale,
                                       const float* __restrict__ bn_shift, const float* __restrict__ residual,
                                       long long res_stride, int res_dim, float* __restrict__ out) {
  const long long total = n_rows * d_out;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / d_out;
    const int c = (int)(i - n * d_out);
    float v = sum[i];
    if (mean) v = v / fmaxf(cnt[n], 1.1920928955078125e-07f);   // torch.finfo(float32).eps, tensor_layers.py:228
    if (bn_scale) v = fmaf(v, bn_scale[c], bn_shift[c]);
    if (residual && c < res_dim) v += residual[n * res_stride + c];
    out[i] = v;
  }
}

// the epilogue over fixed-point sums: the mean is formed in double from the exact integer sum and rounded once to fp32
__global__ void tpconv_finalize_fixed_kernel(const long long* __restrict__ sum, const float* __restrict__ cnt,
                                             long long n_rows, int d_out, int mean, const float* __restrict__ bn_scale,
                                             const float* __restrict__ bn_shift, const float* __restrict__ residual,
                                             long long res_stride, int res_dim, float* __restrict__ out) {
  const long long total = n_rows * d_out;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / d_out;
    const int c = (int)(i - n * d_out);
    const double s = (double)sum[i] * 0x1p-32;
    float v = mean ? (float)(s / (double)fmaxf(cnt[n], 1.1920928955078125e-07f)) : (float)s;
    if (bn_scale) v = fmaf(v, bn_scale[c], bn_shift[c]);
    if (residual && c < res_dim) v += residual[n * res_stride + c];
    out[i] = v;
  }
}

}  // namespace

struct ddb200_tp_table {
  int* d_iblob;
  float* d_fblob;
  int hdr[HDR];
  int n_ints, n_terms;
  int warps, stages, warp_floats, smem_bytes, warp_base_off;
};

static int plan_smem(ddb200_tp_table* t) {
  const int* h = t->hdr;
  const int D_in = h[6], D_sh = h[7], m_total = h[11], z_total = h[10], n_acc = h[12], stage_floats = h[14];
  auto al4 = [](int v) { return (v + 3) & ~3; };
  const int fixed = al4(D_in) + al4(D_sh) + al4(m_total) + al4(z_total) + n_acc * WARP;
  int dev = 0, max_smem = 0;
  cudaGetDevice(&dev);
  if (cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess || max_smem <= 0)
    max_smem = 227 * 1024;
  const int shared_bytes = (al4(t->n_ints) + al4(t->n_terms)) * 4 + 256;
  // as many warps as fit (latency hiding), then as many ring stages as fit (bytes in flight), at least 2
  static const int warp_opts[] = {16, 14, 12, 10, 8, 6, 4, 2, 1};
  const char* env_w = getenv("DDB200_TPCONV_WARPS");
  const char* env_s = getenv("DDB200_TPCONV_STAGES");
  for (int warps : warp_opts) {
    if (env_w && atoi(env_w) > 0 && warps > atoi(env_w)) continue;
    for (int stages = (env_s && atoi(env_s) >= 2) ? atoi(env_s) : 4; stages >= 2; --stages) {
      const int wf = (stages * stage_floats + fixed + 31) & ~31;
      // [table ints | term values | mbarriers | (128-B aligned) per-warp scratch]
      const long long bars_off = 4LL * (al4(t->n_ints) + al4(t->n_terms));
      const long long base_off = (bars_off + 8LL * ((warps * stages + 1) & ~1) + 127) & ~127LL;
      const long long need = base_off + 4LL * wf * warps;
      if (need <= max_smem) {
        t->warps = warps; t->stages = stages; t->warp_floats = wf; t->smem_bytes = (int)need;
        t->warp_base_off = (int)base_off;
        return 0;
      }
    }
  }
  return DDB200_ESMEM;
}

extern "C" {

const char* ddb200_version(void) { return "diffdock_b200 0.1.0 sm_90a"; }

int ddb200_tp_table_create(const int32_t* ib, int n_ints, const float* fb, int n_floats, ddb200_tp_table** out) {
  if (!ib || !fb || !out || n_ints < HDR) return DDB200_EINVAL;
  if ((uint32_t)ib[0] != MAGIC || ib[21] != n_ints || ib[5] > n_floats) return DDB200_ETABLE;
  if (ib[13] % 4 || ib[14] % 4 || ib[1] <= 0 || ib[3] <= 0) return DDB200_ETABLE;
  ddb200_tp_table* t = (ddb200_tp_table*)calloc(1, sizeof(ddb200_tp_table));
  if (!t) return DDB200_EINVAL;
  memcpy(t->hdr, ib, sizeof(int) * HDR);
  t->n_ints = n_ints;
  t->n_terms = ib[5];
  int rc = plan_smem(t);
  if (rc) { free(t); return rc; }
  cudaError_t e = cudaMalloc(&t->d_iblob, sizeof(int) * n_ints);
  if (e == cudaSuccess) e = cudaMalloc(&t->d_fblob, sizeof(float) * (n_floats > 0 ? n_floats : 1));
  if (e == cudaSuccess) e = cudaMemcpy(t->d_iblob, ib, sizeof(int) * n_ints, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(t->d_fblob, fb, sizeof(float) * n_floats, cudaMemcpyHostToDevice);
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(tpconv_accumulate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(tpconv_accumulate_fixed_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  if (e != cudaSuccess) { ddb200_tp_table_destroy(t); return (int)e; }
  *out = t;
  return 0;
}

void ddb200_tp_table_destroy(ddb200_tp_table* t) {
  if (!t) return;
  if (t->d_iblob) cudaFree(t->d_iblob);
  if (t->d_fblob) cudaFree(t->d_fblob);
  free(t);
}

int ddb200_tp_table_info(const ddb200_tp_table* t, int what) {
  if (!t) return DDB200_EINVAL;
  switch (what) {
    case 0: return t->hdr[6];
    case 1: return t->hdr[7];
    case 2: return t->hdr[8];
    case 3: return t->hdr[13];
    case 4: return t->hdr[9];
    case 5: return t->smem_bytes;
    case 6: return t->warps;
    case 7: return t->stages;
    default: return DDB200_EINVAL;
  }
}

}  // extern "C"

static int tpconv_accumulate_launch(const ddb200_tp_table* t, const float* x, int64_t x_stride, const int32_t* edge_src,
                                    const int32_t* edge_dst, const float* geo, const float* edge_weight, const float* w,
                                    int64_t w_stride, int64_t n_edges, float* sum, long long* sum_fx, int* err, float* cnt,
                                    void* stream) {
  const bool fixed = sum_fx != nullptr;
  if (!t || !x || !edge_src || !edge_dst || !geo || !w || !(fixed ? (err != nullptr) : (sum != nullptr)) || n_edges < 0)
    return DDB200_EINVAL;
  if (fixed && t->hdr[8] > WARP * MAX_FX) return DDB200_EINVAL;
  if (n_edges == 0) return 0;
  if ((reinterpret_cast<uintptr_t>(w) & 15) || (w_stride & 3) || w_stride < t->hdr[13] || x_stride < t->hdr[6])
    return DDB200_EINVAL;
  KParams p;
  p.x = x; p.x_stride = x_stride; p.esrc = edge_src; p.edst = edge_dst; p.geo = geo; p.ew = edge_weight;
  p.w = w; p.w_stride = w_stride; p.n_edges = n_edges; p.sum = sum; p.cnt = cnt; p.sum_fx = sum_fx; p.err = err;
  p.iblob = t->d_iblob; p.fblob = t->d_fblob; p.n_ints = t->n_ints; p.n_terms = t->n_terms;
  p.stages = t->stages; p.warps = t->warps; p.warp_floats = t->warp_floats; p.stage_floats = t->hdr[14];
  p.warp_base_off = t->warp_base_off;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const long long units = (n_edges + ERUN - 1) / ERUN;
  long long ctas = (units + t->warps - 1) / t->warps;
  if (ctas > sms) ctas = sms;   // persistent: one CTA per SM, warps stride over the edge runs
  if (fixed)
    tpconv_accumulate_fixed_kernel<<<(unsigned)ctas, t->warps * WARP, t->smem_bytes, (cudaStream_t)stream>>>(p);
  else
    tpconv_accumulate_kernel<<<(unsigned)ctas, t->warps * WARP, t->smem_bytes, (cudaStream_t)stream>>>(p);
  return (int)cudaGetLastError();
}

extern "C" {

int ddb200_tpconv_accumulate(const ddb200_tp_table* t, const float* x, int64_t x_stride, const int32_t* edge_src,
                             const int32_t* edge_dst, const float* geo, const float* edge_weight, const float* w,
                             int64_t w_stride, int64_t n_edges, float* sum, float* cnt, void* stream) {
  return tpconv_accumulate_launch(t, x, x_stride, edge_src, edge_dst, geo, edge_weight, w, w_stride, n_edges, sum, nullptr,
                                  nullptr, cnt, stream);
}

int ddb200_tpconv_accumulate_fixed(const ddb200_tp_table* t, const float* x, int64_t x_stride, const int32_t* edge_src,
                                   const int32_t* edge_dst, const float* geo, const float* edge_weight, const float* w,
                                   int64_t w_stride, int64_t n_edges, int64_t* sum, float* cnt, int32_t* err,
                                   void* stream) {
  if (!sum) return DDB200_EINVAL;
  return tpconv_accumulate_launch(t, x, x_stride, edge_src, edge_dst, geo, edge_weight, w, w_stride, n_edges, nullptr,
                                  reinterpret_cast<long long*>(sum), err, cnt, stream);
}

int ddb200_tpconv_finalize(const float* sum, const float* cnt, int64_t n_rows, int d_out, int mean,
                           const float* bn_scale, const float* bn_shift, const float* residual, int64_t res_stride,
                           int res_dim, float* out, void* stream) {
  if (!sum || !out || n_rows < 0 || d_out <= 0 || (mean && !cnt) || ((bn_scale == nullptr) != (bn_shift == nullptr)))
    return DDB200_EINVAL;
  if (n_rows == 0) return 0;
  const long long total = n_rows * (long long)d_out;
  long long blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  tpconv_finalize_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(sum, cnt, n_rows, d_out, mean, bn_scale,
                                                                            bn_shift, residual, res_stride, res_dim, out);
  return (int)cudaGetLastError();
}

int ddb200_tpconv_finalize_fixed(const int64_t* sum, const float* cnt, int64_t n_rows, int d_out, int mean,
                                 const float* bn_scale, const float* bn_shift, const float* residual, int64_t res_stride,
                                 int res_dim, float* out, void* stream) {
  if (!sum || !out || n_rows < 0 || d_out <= 0 || (mean && !cnt) || ((bn_scale == nullptr) != (bn_shift == nullptr)))
    return DDB200_EINVAL;
  if (n_rows == 0) return 0;
  const long long total = n_rows * (long long)d_out;
  long long blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  tpconv_finalize_fixed_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const long long*>(sum), cnt, n_rows, d_out, mean, bn_scale, bn_shift, residual, res_stride, res_dim,
      out);
  return (int)cudaGetLastError();
}

}  // extern "C"
