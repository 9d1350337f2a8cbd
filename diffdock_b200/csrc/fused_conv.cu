// Fully fused equivariant convolution for one edge group (sm_90a): radial MLP on the Hopper tensor cores (wgmma) +
// tensor-product contraction + scatter - the per-edge weight tensor [E, weight_numel] never exists in HBM.
//
//   for a tile of 128 CSR-sorted edges (one CTA, persistent over tiles; warpgroup g owns edges 64 g .. 64 g + 63 and does
//   all of their work; the B' images are streamed once per CTA by TMA bulk copies through a 3-stage ring both read):
//     A0' = split-bf16([edge_attr (+ per-graph term) | node[tgt,:ns] | node[src,:ns]])   the warpgroup's own image in shared
//                                      memory (128B swizzle)
//     H   = relu(A0' x W1'^T)          wgmma -> registers -> A' image (bias folded via two constant-one columns)
//     H   = relu(A' x Wh'^T)           for every extra H x H hidden layer (tp_weights_layers > 2), in place over A'
//     for every N tile (whole rows u of one path block [mul_in, mul_out], <= 192 columns):
//        z_e[u,k] = sum_i x[src_e][u,i] M_e[i,k],  M_e = edge_weight * coef * C . Y(vec_e)   built by each quad of threads
//                                      for its two edges in a per-warpgroup shared-memory buffer
//        Wt = A' x W2'^T[tile]         wgmma m64nNk16 into registers
//        acc[w,k] += Wt[e, (u,w)] * z_e[u,k]   straight from the accumulator registers (partial sums per thread)
//     at the end of an output irrep: sum[tgt_e, irrep] += acc  (the partial sums are staged in shared memory, runs of
//                                                              equal targets reduced, then one coalesced RED.ADD per run
//                                                              and output value)
//
// Operand layout: BOTH operand images hold each split part once - activation [hi | lo | 1 1 0..], static operand
// [hi | lo | b_hi b_lo 0..] (2 Kp + 16 columns, Kp = K rounded up to 16).  The three products hi.hi + hi.lo + lo.hi (+ bias)
// are formed by an MMA schedule over 16-column steps: a `hi` step of B is multiplied with the hi AND the lo columns of A (two
// MMAs on one staged block), a `lo` step with the hi columns, the bias step with the constant-one columns.  Compared with
// concatenating [hi | hi | lo] x [hi | lo | hi] along K this stages 5 instead of 7 k-blocks of B per tile and a third fewer
// activation stores.
//
// Replaces models/tensor_layers.py:139-144 / :204-221 *including* the FCBlock at :140/:211 and the edge_attr_ assembly of
// models/cg_model.py:342-349 (and the per-call sigma-embedding add of :298-301 through `ea_add`).
// Plan (tiles, operand images, dense Clebsch-Gordan tables) is built by diffdock_b200/fused.py.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include "../../include/diffdock_b200.h"
#include "../../include/diffdock_b200_fixed.h"
#include "sm90.cuh"

namespace {

using namespace ddb200_sm90;

constexpr int BM = 64, BK = 64;                  // edges of one warpgroup = one wgmma M; BK bf16 = one 128-byte swizzle row
constexpr int CTA_EDGES = 2 * BM;                // edge tile of the CTA: one 64-edge half per warpgroup
constexpr int A_KB_BYTES = BM * BK * 2;          // 8 KB
constexpr int B_IMAGE_BYTES = 256 * BK * 2;      // 32 KB: one k-block image of an N tile in global memory
constexpr int MAX_N = 192;                       // widest N tile of a plan (and widest hidden layer)
constexpr int STAGES = 4;                        // every stage feeds both warpgroups' chains
constexpr int STAGE_BYTES = MAX_N * BK * 2;      // 24 KB: the rows of an image the MMA reads
constexpr int MAX_KB = 5;                        // k-blocks of either operand image: 2 Kp + 16 <= 320  (Kp <= 144)
constexpr int MAX_KA = MAX_KB;
constexpr int A_IMAGE_BYTES = MAX_KA * A_KB_BYTES;    // 40 KB: one warpgroup's activation image
constexpr int OPS_PER_KB = 8;                    // MMAs that read one staged k-block of B (4 steps x up to 2 A partners)
constexpr int THREADS = 256;                     // two warpgroups, each with its own 64 edges
constexpr int MAX_TILES = 128, MAX_PATHS = 16, MTAB = 48;     // per path: dense [3][3][5] table, padded to 48 floats
constexpr int BAR_WG = 1;                        // named barrier BAR_WG + g: the 128 threads of warpgroup g
// Second-order instantiation (SO, node irreps with l = 2 blocks: use_second_order_repr): 5-component inputs and outputs, up
// to 32 paths whose dense [5][5][5] tables (padded to 128 floats, 16 KB) are read through L1 instead of being staged, and
// 3 B stages, so that the larger z buffer fits beside the two A images under the 227 KB opt-in.
constexpr int SO_STAGES = 3, SO_MAX_PATHS = 32, SO_MTAB = 128;

// fire-and-forget global reduction (atomicAdd here may be compiled to an atomic that returns its old value)
__device__ __forceinline__ void red_add(float* addr, float v) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(addr), "f"(v) : "memory");
}
// 64-bit integer reduction: the fixed-point accumulators of the deterministic instantiations (two's complement, so a
// signed sum is an unsigned one)
__device__ __forceinline__ void red_add_u64(long long* addr, long long v) {
  asm volatile("red.global.add.u64 [%0], %1;" ::"l"(addr), "l"((unsigned long long)v) : "memory");
}
// v * 2^32 rounded to nearest (even), as a 64-bit integer.  |v| >= 2^31 and non-finite values saturate and set the sticky
// error word *err (bit 0), which the host reads after the work is done.
__device__ __forceinline__ long long to_fixed(float v, int* err) {
  const float s = v * 0x1p32f;
  if (fabsf(s) < 0x1p63f) return __float2ll_rn(s);
  atomicOr(err, 1);
  return v > 0.f ? 0x7fffffffffffffffLL : (v < 0.f ? -0x7fffffffffffffffLL : 0LL);
}
__device__ __forceinline__ void wgmma_wait_one() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }

__device__ __forceinline__ void put_a(unsigned char* sA, int r, int col, __nv_bfloat16 v) {
  const int kb = col >> 6, c = (col & 63) >> 3, j = col & 7;
  *reinterpret_cast<__nv_bfloat16*>(sA + (size_t)kb * A_KB_BYTES + r * 128 + ((c ^ (r & 7)) << 4) + j * 2) = v;
}
// columns col, col + 1 (col even) of row r
__device__ __forceinline__ void put_a2(unsigned char* sA, int r, int col, uint32_t v) {
  const int kb = col >> 6, c = (col & 63) >> 3, j = col & 7;
  *reinterpret_cast<uint32_t*>(sA + (size_t)kb * A_KB_BYTES + r * 128 + ((c ^ (r & 7)) << 4) + j * 2) = v;
}
// 8 consecutive columns col0..col0+7 (col0 % 8 == 0) of row r = one 16-byte chunk of the swizzled image
__device__ __forceinline__ void put_a8(unsigned char* sA, int r, int col0, const uint4& v) {
  const int kb = col0 >> 6, c = (col0 & 63) >> 3;
  *reinterpret_cast<uint4*>(sA + (size_t)kb * A_KB_BYTES + r * 128 + ((c ^ (r & 7)) << 4)) = v;
}
__device__ __forceinline__ void split1(float f, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16(f);
  lo = __float2bfloat16(f - __bfloat162float(hi));
}
// split 8 floats into bf16 hi / lo parts, packed as two 16-byte chunks
__device__ __forceinline__ void split8(const float* f, uint4& hi, uint4& lo) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __nv_bfloat16 h0, h1, l0, l1;
    split1(f[2 * i], h0, l0);
    split1(f[2 * i + 1], h1, l1);
    h[i] = (uint32_t)__bfloat16_as_ushort(h0) | ((uint32_t)__bfloat16_as_ushort(h1) << 16);
    l[i] = (uint32_t)__bfloat16_as_ushort(l0) | ((uint32_t)__bfloat16_as_ushort(l1) << 16);
  }
  hi = make_uint4(h[0], h[1], h[2], h[3]);
  lo = make_uint4(l[0], l[1], l[2], l[3]);
}
// The tail of an operand image row: zero the padding of the hi / lo sections (K..Kp), write the two constant-one columns
// that carry the folded bias and zero the rest of their 16-column step.
__device__ __forceinline__ void put_a_tail(unsigned char* sA, int r, int K, int Kp) {
  const __nv_bfloat16 zero = __float2bfloat16(0.f);
  for (int c = K; c < Kp; ++c) { put_a(sA, r, c, zero); put_a(sA, r, Kp + c, zero); }
  const uint32_t ones = 0x3F803F80u;     // two bf16 1.0
  put_a8(sA, r, 2 * Kp, make_uint4(ones, 0u, 0u, 0u));
  put_a8(sA, r, 2 * Kp + 8, make_uint4(0u, 0u, 0u, 0u));
}

struct FusedParams {
  const float* ea; long long ld_ea; int ne;          // per-edge attributes
  const float* node; long long ld_node; int ns;      // node scalars for the radial MLP (both end points)
  const int* tgt; const int* src;                    // scatter target / gathered node of every edge
  const int* perm;                                   // optional: row of ea / vec / ew that belongs to edge e
  const float* ea_add; const int* ea_add_idx;        // optional: ea row += ea_add[ea_add_idx[e], :ne]
  int a0_vec;                                        // A0' rows gathered with 16-byte loads (decided by the host)
  float vec_sign;
  const __nv_bfloat16* w1img; int K1, K1p, n_kb1, H, Hp, n_kb;
  const __nv_bfloat16* w2img;                        // [n_tiles][n_kb][256][64]
  const __nv_bfloat16* whimg; int n_hidden;          // [n_hidden][n_kb][256][64]: extra H x H hidden layers, in order
  const int* tiles; int n_tiles;                     // [n_tiles][8]: kind, N_mma, x_off, rows, d_in, out_off, flags | sh_off << 8, path
  const float* mtab; int n_paths;                    // [n_paths][48]: coef * C[i, j, k] as [i][k][j], i,k < 3, j < 5
  const float* x; long long ld_x; int x_vec2;        // node irreps gathered by src
  const float* vec; const float* ew; int lmax;
  float* sum; int d_out; float* cnt;
  long long* sum_fx; int* err;                       // deterministic instantiations: int64 accumulator (2^-32 units), error word
  long long n_edges; const int* n_edges_dev;
  unsigned long long* dbg;                           // optional [32] clock counters (DDB200_FUSED_DEBUG=1), else nullptr
};

// ---- contraction straight from the wgmma accumulators.  Thread t of a warpgroup holds rows r0 = 16 (t / 32) + (t % 32) / 4
// and r0 + 8 (its two edges h = 0, 1) and columns c = 8 j + 2 q + b (q = t % 4, b = 0, 1) of the weight tile as
// d[4 j + 2 h + b]; column c is row u = c / MULOUT and output channel w = c % MULOUT of the tile.  The thread keeps its
// partial sums per slot (j mod P, b), P = MULOUT / gcd(MULOUT, 8): the slots of one thread hold distinct channels (slot ->
// channel is fixed up to a shift by 2 q, so every index into the partial sums is known at compile time), and NCOPY =
// 8 / gcd(MULOUT, 8) threads of a quad hold partial sums of the same channel.
template <int MULOUT> struct Slots {
  static_assert(MULOUT % 2 == 0 && MULOUT >= 4, "a column pair (b = 0, 1) lies in one row u; w() wraps at most once");
  static constexpr int G = MULOUT % 8 == 0 ? 8 : (MULOUT % 4 == 0 ? 4 : 2);
  static constexpr int P = MULOUT / G, N = 2 * P, NCOPY = 8 / G;
  // (8 (slot >> 1) + (slot & 1) + 2 q) mod MULOUT as a compile-time channel plus a shift: 2 q <= 6 wraps at most once
  static __device__ __forceinline__ int w(int slot, int q) {
    const int c = (8 * (slot >> 1) + (slot & 1)) % MULOUT;
    return c + 2 * q - (2 * q >= MULOUT - c ? MULOUT : 0);
  }
};
constexpr int NACC_MAX = 60;                     // partial sums per thread: slots x d_out x 2 edges, at most 10 x 3 x 2
constexpr int ZLD = 68;                          // z buffer row of one edge: [16 rows u][4]; 8 edges' 16-byte reads hit 8 bank groups
constexpr int WG_BUF = 64 * ZLD;                 // floats per warpgroup: z [64][ZLD], or the scatter staging [copies][64][nacc + 1]
// SO: components 3, 4 of a 5-component z row lie in a second plane [64][ZLDB] behind the first ([16 rows u][2]; 8 edges'
// 8-byte reads hit 16 distinct banks).  The scatter staging still fits in the first plane.
constexpr int ZLDB = 34;
constexpr int WG_BUF_SO = 64 * (ZLD + ZLDB);

using Acc = float[MAX_N / 2];

// acc[(slot d_out + k) 2 + h] += d[edge h, columns of the slot] * z[edge h][u][K0 + k] over the tile's first `nch` 32-column
// chunks; z = the row of this thread's first edge in the z buffer (the second edge lies 8 rows further), zb its row in the
// second plane (SO only: K0 + DOUT > 3)
template <int MULOUT, int DOUT, int ROWS, int K0 = 0>
__device__ __forceinline__ void contract(const Acc& d, const float* __restrict__ z, int nch, int q, float* __restrict__ acc,
                                         const float* __restrict__ zb = nullptr) {
  using S = Slots<MULOUT>;
  constexpr int NCOL = MULOUT * ROWS;
  static_assert(NCOL % 32 == 0 && NCOL <= MAX_N && S::N * DOUT * 2 <= NACC_MAX, "tile width");
  static_assert((K0 == 0 && (DOUT <= 3 || DOUT == 5)) || (K0 == 3 && DOUT == 2), "a z row is read as (0..2 | 3..4)");
#pragma unroll
  for (int j = 0; j < NCOL / 8; ++j) {
    if ((j >> 2) < nch) {
      // u = (8 j + 2 q) / MULOUT: 8 j splits into a compile-time row and remainder, and 2 q < 8 adds at most one row
      const int JR = (8 * j) % MULOUT;
      const int u = (8 * j) / MULOUT + ((MULOUT % 8 != 0 && 2 * q >= MULOUT - JR) ? 1 : 0);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float zk[DOUT];
        if constexpr (K0 == 3) {
          const float2 v = *reinterpret_cast<const float2*>(zb + h * 8 * ZLDB + u * 2);
          zk[0] = v.x; zk[1] = v.y;
        } else if constexpr (DOUT == 1) {
          zk[0] = z[h * 8 * ZLD + u * 4];
        } else {
          const float4 v = *reinterpret_cast<const float4*>(z + h * 8 * ZLD + u * 4);
          zk[0] = v.x; zk[1] = v.y; zk[2] = v.z;
          if constexpr (DOUT == 5) {
            const float2 w = *reinterpret_cast<const float2*>(zb + h * 8 * ZLDB + u * 2);
            zk[3] = w.x; zk[4] = w.y;
          }
        }
#pragma unroll
        for (int b = 0; b < 2; ++b) {
          const int slot = (j % S::P) * 2 + b;
#pragma unroll
          for (int k = 0; k < DOUT; ++k)
            acc[(slot * DOUT + k) * 2 + h] = fmaf(d[4 * j + 2 * h + b], zk[k], acc[(slot * DOUT + k) * 2 + h]);
        }
      }
    }
  }
}

// z[u][k] = sum_i x[u d_in + i] M[i][k] for this thread's edge and the tile rows u0 .. u0 + 7 (< ROWS), into its row `zrow`
// of the z buffer; xn = the node values of these rows, prefetched one tile ahead (zero past the tile's rows)
template <int DOUT, int ROWS>
__device__ __forceinline__ void build_z(const float* __restrict__ xn, int d_in, const float* __restrict__ M,
                                        float* __restrict__ zrow, int u0) {
  constexpr int NU = ROWS < 8 ? ROWS : 8;
  if (u0 >= ROWS) return;
#pragma unroll
  for (int r = 0; r < NU; ++r) {
    float z[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < DOUT; ++k) {
      if (d_in == 1) z[k] = xn[r] * M[k];
      else z[k] = fmaf(xn[3 * r + 2], M[6 + k], fmaf(xn[3 * r + 1], M[3 + k], xn[3 * r] * M[k]));
    }
    *reinterpret_cast<float4*>(zrow + (u0 + r) * 4) = make_float4(z[0], z[1], z[2], 0.f);
  }
}

// SO: as build_z for d_in in {1, 3, 5} and DOUT in {1, 3, 5}, M = [5][5] (row-major, zero where i >= d_in or k >= d_out);
// xs = the node values of rows u0 .. u0 + nrows - 1, read here rather than prefetched: the prefetch would hold 40 values
// through the MMAs, while here they live beside the free accumulator registers only
template <int DOUT, int ROWS>
__device__ __forceinline__ void build_z_so(const float* __restrict__ xs, int nrows, int d_in, const float* __restrict__ M,
                                           float* __restrict__ zrow, float* __restrict__ zrowb, int u0) {
  constexpr int NU = ROWS < 8 ? ROWS : 8;
  if (u0 >= ROWS) return;
  float xv[NU][5];
#pragma unroll
  for (int r = 0; r < NU; ++r)
#pragma unroll
    for (int i = 0; i < 5; ++i) xv[r][i] = (r < nrows && i < d_in) ? __ldg(xs + r * d_in + i) : 0.f;
#pragma unroll
  for (int r = 0; r < NU; ++r) {
    float z[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < DOUT; ++k)
#pragma unroll
      for (int i = 0; i < 5; ++i) z[k] = fmaf(xv[r][i], M[5 * i + k], z[k]);
    *reinterpret_cast<float4*>(zrow + (u0 + r) * 4) = make_float4(z[0], z[1], z[2], 0.f);
    if (DOUT == 5) *reinterpret_cast<float2*>(zrowb + (u0 + r) * 2) = make_float2(z[3], z[4]);
  }
}

constexpr int XN = 24;     // node values one thread gathers per tile: 8 rows x at most 3 components
__device__ __forceinline__ void prefetch_x(const float* __restrict__ src, int cnt, int vec2, float* __restrict__ xn) {
  if (vec2) {          // 8-byte loads: every tile offset and count of the plan is even
#pragma unroll
    for (int j = 0; j < XN / 2; ++j) {
      float2 v = make_float2(0.f, 0.f);
      if (2 * j < cnt) v = __ldg(reinterpret_cast<const float2*>(src) + j);
      xn[2 * j] = v.x; xn[2 * j + 1] = v.y;
    }
  } else {
#pragma unroll
    for (int j = 0; j < XN; ++j) xn[j] = (j < cnt) ? __ldg(src + j) : 0.f;
  }
}
// node values of tile `ti`'s rows u0 .. u0 + 7 for the source row xrow
__device__ __forceinline__ void prefetch_tile(const float* xrow, const int* ti, int u0, int vec2, float* xn) {
  const int d_in = ti[4], rows = min(max(ti[3] - u0, 0), 8);
  prefetch_x(xrow + ti[2] + u0 * d_in, rows * d_in, vec2, xn);
}

// End of an output irrep: scatter-add of the warpgroup's 64 edges.  Every thread stages its partial sums in shared memory
// (over the z buffer, at most two copies: with four, the pairs q, q ^ 1 are first added by a shuffle); warp w4 then takes edges 32 (w4 & 1) .. + 31 and output value i = 32 (w4 >> 1) + lane,
// adds the copies, sums runs of equal targets (CSR order makes them contiguous; unsorted input just yields runs of length
// one) and issues ONE fully coalesced RED.ADD per run for output value i.  A slice (SO: components K0 .. K0 + DOUT - 1 of a
// DFULL-component block) lands at w DFULL + K0 + k of the block.
template <int MULOUT, int DOUT, int DFULL = DOUT, int K0 = 0, bool FIXED = false>
__device__ __forceinline__ void flush(const FusedParams& p, float* __restrict__ acc, float* buf, int r0, int q, int w4,
                                      int lane, int dst_s, uint32_t head_mask, int out_off, int bar) {
  using S = Slots<MULOUT>;
  constexpr int NACC = MULOUT * DOUT, LD = NACC + 1, NCOPY = S::NCOPY == 4 ? 2 : S::NCOPY;
  static_assert(NCOPY * 64 * LD <= WG_BUF, "staging area");
  bool writes = true;
  if constexpr (S::NCOPY == 4) {
    // slot (j + 1) mod 5 of thread q + 1 holds the channel of slot j of thread q (8 = -2 mod 10): the even threads add
    // their odd partner's partial sums and stage them, the odd ones stage nothing
    static_assert(MULOUT == 10 && S::P == 5, "quad reduction");
    const bool odd = q & 1;
    writes = !odd;
#pragma unroll
    for (int j = 0; j < 5; ++j)
#pragma unroll
      for (int b = 0; b < 2; ++b)
#pragma unroll
        for (int k = 0; k < DOUT; ++k)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int own = ((j * 2 + b) * DOUT + k) * 2 + h;
            const int up = ((((j + 1) % 5) * 2 + b) * DOUT + k) * 2 + h;
            const float r = __shfl_xor_sync(0xffffffffu, odd ? acc[up] : 0.f, 1);
            if (!odd) acc[own] += r;
          }
  }
  named_bar(bar, 128);                           // every warp is done with its z rows
  float* st = buf + (NCOPY == 1 ? 0 : q >> 1) * 64 * LD;
  if (writes) {
#pragma unroll
    for (int slot = 0; slot < S::N; ++slot) {
      const int w = S::w(slot, q);
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int k = 0; k < DOUT; ++k) st[(r0 + 8 * h) * LD + w * DOUT + k] = acc[(slot * DOUT + k) * 2 + h];
    }
  }
  named_bar(bar, 128);
  const int half = w4 >> 1, i = 32 * half + lane;
  if (32 * half < NACC) {
    const bool act = i < NACC;
    const float* col = buf + 32 * (w4 & 1) * LD + (act ? i : 0);
    if constexpr (FIXED) {
      // deterministic: each edge's value (its copies added in a fixed order) is converted on its own and the run is
      // summed as integers, so the sum depends neither on the edge order nor on where runs cross tile boundaries
      const uint32_t live = __ballot_sync(0xffffffffu, dst_s >= 0);
      long long s = 0;
#pragma unroll
      for (int le = 0; le < 32; ++le) {
        float v = 0.f;
#pragma unroll
        for (int c = 0; c < NCOPY; ++c) v += col[(c * 64 + le) * LD];
        if (act && ((live >> le) & 1)) s += to_fixed(v, p.err);
        if (le == 31 || ((head_mask >> (le + 1)) & 1)) {        // warp-uniform: last edge of a run
          const int dst = __shfl_sync(0xffffffffu, dst_s, le);
          if constexpr (DFULL == DOUT) {
            if (dst >= 0 && act) red_add_u64(p.sum_fx + (long long)dst * p.d_out + out_off + i, s);
          } else {
            const int w = i / DOUT;
            if (dst >= 0 && act)
              red_add_u64(p.sum_fx + (long long)dst * p.d_out + out_off + w * DFULL + K0 + (i - w * DOUT), s);
          }
          s = 0;
        }
      }
    } else {
      float s = 0.f;
#pragma unroll
      for (int le = 0; le < 32; ++le) {
#pragma unroll
        for (int c = 0; c < NCOPY; ++c) s += col[(c * 64 + le) * LD];
        if (le == 31 || ((head_mask >> (le + 1)) & 1)) {          // warp-uniform: last edge of a run
          const int dst = __shfl_sync(0xffffffffu, dst_s, le);
          if constexpr (DFULL == DOUT) {
            if (dst >= 0 && act) red_add(p.sum + (long long)dst * p.d_out + out_off + i, s);
          } else {
            const int w = i / DOUT;
            if (dst >= 0 && act) red_add(p.sum + (long long)dst * p.d_out + out_off + w * DFULL + K0 + (i - w * DOUT), s);
          }
          s = 0.f;
        }
      }
    }
  }
  named_bar(bar, 128);                           // the staging area is free for the next z rows
}

// MMA schedule of one staged k-block of B (4 steps of 16 columns; images [hi | lo | bias], S = Kp / 16 steps per part):
// step c < S (hi): x A hi (column block c) and x A lo (block S + c);  S <= c < 2S (lo): x A hi (block c - S);
// c == 2S (bias): x A ones (block 2S).  Per k-block OPS_PER_KB slots of two words, stored as [A words 0-7 | B words 0-7]:
// A word = low descriptor word of the A column block (absolute: one schedule per warpgroup image), B word = offset of the B step
// inside the stage in 16-byte units; the first n slots are used.  After the MAX_KB k-blocks: n of every k-block
// (1 <= n <= 8 for every k-block of an image: the last one holds at least the bias step).
constexpr int SCHED_WORDS = MAX_KB * (2 * OPS_PER_KB + 1);
__device__ __forceinline__ uint32_t a_block_offset(int c) { return (uint32_t)((c >> 2) * (A_KB_BYTES >> 4) + (c & 3) * 2); }
__device__ __forceinline__ void build_ops(uint32_t* ops, int S, uint32_t a_lo0) {     // ops[SCHED_WORDS]
  for (int kb = 0; kb < MAX_KB; ++kb) {
    uint32_t* oa = ops + kb * 2 * OPS_PER_KB;
    uint32_t* ob = oa + OPS_PER_KB;
    int n = 0;
    for (int j = 0; j < 4; ++j) {
      const int c = kb * 4 + j;
      if (c < S) {
        oa[n] = a_lo0 + a_block_offset(c); ob[n++] = (uint32_t)j * 2;
        oa[n] = a_lo0 + a_block_offset(S + c); ob[n++] = (uint32_t)j * 2;
      } else if (c < 2 * S) { oa[n] = a_lo0 + a_block_offset(c - S); ob[n++] = (uint32_t)j * 2; }
      else if (c == 2 * S) { oa[n] = a_lo0 + a_block_offset(2 * S); ob[n++] = (uint32_t)j * 2; }
    }
    ops[MAX_KB * 2 * OPS_PER_KB + kb] = (uint32_t)n;
    for (; n < OPS_PER_KB; ++n) { oa[n] = a_lo0; ob[n] = 0u; }
  }
}

// B stream of a CTA: per edge tile the W1' k-blocks, then the Wh' k-blocks of every extra hidden layer in order, then
// every N tile's W2' k-blocks; item i goes to stage i % NST and is read by both warpgroups
template <int NST> struct Stream {
  unsigned char* sB; uint64_t* full; uint32_t* rel; const int* tiles;
  int n1, per_unit; uint32_t len;
  __device__ __forceinline__ void issue(const FusedParams& p, uint32_t i) const {
    if (i >= len) return;
    const int j = (int)(i % (uint32_t)per_unit);
    const int jh = j - p.n_kb1, j2 = jh - p.n_hidden * p.n_kb;
    const unsigned char* src;
    uint32_t bytes;
    if (j < p.n_kb1) {
      src = reinterpret_cast<const unsigned char*>(p.w1img) + (size_t)j * B_IMAGE_BYTES;
      bytes = (uint32_t)n1 * 128u;
    } else if (j2 < 0) {        // image (l, kb) of the Wh' set lies at (l * n_kb + kb) = jh; its H rows as for W1'
      src = reinterpret_cast<const unsigned char*>(p.whimg) + (size_t)jh * B_IMAGE_BYTES;
      bytes = (uint32_t)n1 * 128u;
    } else {                    // image (t, kb) of the W2' set lies at (t * n_kb + kb) = j2
      src = reinterpret_cast<const unsigned char*>(p.w2img) + (size_t)j2 * B_IMAGE_BYTES;
      bytes = (uint32_t)tiles[(j2 / p.n_kb) * 8 + 1] * 128u;
    }
    const uint32_t s = i % NST;
    bulk_load(sB + (size_t)s * STAGE_BYTES, src, bytes, &full[s]);
  }
  // item i has been read by every MMA of this warpgroup (its group is complete in every warp): the second warpgroup to
  // release it refills its stage with item i + NST (rel[s] counts two releases per use of stage s)
  __device__ __forceinline__ void release(const FusedParams& p, uint32_t i, int bar, int t) const {
    named_bar(bar, 128);
    if (t == 0) {
      __threadfence_block();
      if (atomicAdd(rel + i % NST, 1u) & 1u) issue(p, i + NST);
    }
  }
};

// ---- MMAs of a warpgroup.  Every product is issued MAX_N wide into the warpgroup's 96 accumulators, k-block after k-block
// of the CTA's B stream, counted by mc.

// the n MMAs of one staged k-block as one chain: one register fence in front, one commit group.  The descriptors are read
// before the fence, so that nothing but the MMAs lies between the fence and the commit.  The first MMA of a product
// (FIRST) overwrites d and does not read it: the accumulators are dead between products.
template <int NOPS, bool FIRST>
__device__ __forceinline__ void mma_chain(Acc& d, const uint32_t* oa, const uint32_t* ob, uint32_t b_lo) {
  uint32_t a[NOPS], b[NOPS];
#pragma unroll
  for (int i = 0; i < NOPS; ++i) { a[i] = oa[i]; b[i] = b_lo + ob[i]; }
  wgmma_fence();
#pragma unroll
  for (int i = 0; i < NOPS; ++i) {
    if (FIRST && i == 0) wgmma192_first(d, gmma_desc(a[i]), gmma_desc(b[i]));
    else Wgmma<MAX_N>::mma(d, gmma_desc(a[i]), gmma_desc(b[i]), 1u);
  }
  wgmma_commit();
}

// k-block kb of the schedule `ops` from stage mc % NST into d; dwait (debug, one thread per warpgroup) collects the
// clocks spent waiting for the stage to land
template <bool FIRST, int NST>
__device__ __forceinline__ void mma_kblock(Acc& d, const Stream<NST>& st, const uint32_t* ops, int kb, uint32_t mc,
                                           unsigned long long* dwait) {
  const uint32_t s = mc % NST;
  const long long c0 = dwait ? clock64() : 0;
  mbar_wait(&st.full[s], (mc / NST) & 1);
  if (dwait) *dwait += (unsigned long long)(clock64() - c0);
  const uint32_t* oa = ops + kb * 2 * OPS_PER_KB;
  const uint32_t* ob = oa + OPS_PER_KB;
  const uint32_t b_lo = gmma_desc_lo(smem_u32(st.sB)) + s * (STAGE_BYTES >> 4);
  switch (ops[MAX_KB * 2 * OPS_PER_KB + kb]) {      // uniform: the chain length follows from the plan's shapes
    case 1: mma_chain<1, FIRST>(d, oa, ob, b_lo); break;
    case 2: mma_chain<2, FIRST>(d, oa, ob, b_lo); break;
    case 3: mma_chain<3, FIRST>(d, oa, ob, b_lo); break;
    case 4: mma_chain<4, FIRST>(d, oa, ob, b_lo); break;
    case 5: mma_chain<5, FIRST>(d, oa, ob, b_lo); break;
    case 6: mma_chain<6, FIRST>(d, oa, ob, b_lo); break;
    case 7: mma_chain<7, FIRST>(d, oa, ob, b_lo); break;
    case 8: mma_chain<8, FIRST>(d, oa, ob, b_lo); break;
    default: __trap();     // unreachable: build_ops gives every k-block of an image 1..8 MMAs (n_kb = ceil((2S + 1) / 4))
  }
}

// one product, k-blocks 0 .. nkb - 1, into d.  Once a k-block is committed the previous one is waited for and released;
// on return every group is complete, every stage the product read released and d readable.
template <int NST>
__device__ __forceinline__ void mma_product(Acc& d, const FusedParams& p, const Stream<NST>& st, const uint32_t* ops, int nkb, uint32_t& mc, int bar, int t, unsigned long long* dwait) {
  mma_kblock<true>(d, st, ops, 0, mc++, dwait);
  for (int kb = 1; kb < nkb; ++kb, ++mc) {
    mma_kblock<false>(d, st, ops, kb, mc, dwait);
    wgmma_wait_one();
    st.release(p, mc - 1, bar, t);
  }
  wgmma_wait_all();
  st.release(p, mc - 1, bar, t);
  wgmma_fence_regs(d);                           // d is read only after the wait that completed it
}

// hidden layer -> A': ReLU, bf16 split, written back over the warpgroup's operand image; complete and visible to the async
// proxy before the first weight-tile MMA reads it
__device__ __forceinline__ void store_hidden(const Acc& d, const FusedParams& p, unsigned char* sA, int t, int bar) {
  const int lane = t & 31, r0 = (t >> 5) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
  const int K = p.H, Kp = p.Hp;
#pragma unroll
  for (int j = 0; j < MAX_N / 8; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int c = 8 * j + c0, r = r0 + 8 * h;
      __nv_bfloat16 h0, l0, h1, l1;
      split1(fmaxf(d[4 * j + 2 * h], 0.f), h0, l0);
      split1(fmaxf(d[4 * j + 2 * h + 1], 0.f), h1, l1);
      if (c + 1 < K) {
        put_a2(sA, r, c, (uint32_t)__bfloat16_as_ushort(h0) | ((uint32_t)__bfloat16_as_ushort(h1) << 16));
        put_a2(sA, r, Kp + c, (uint32_t)__bfloat16_as_ushort(l0) | ((uint32_t)__bfloat16_as_ushort(l1) << 16));
      } else if (c < K) {
        put_a(sA, r, c, h0);
        put_a(sA, r, Kp + c, l0);
      }
    }
  if (t < BM) put_a_tail(sA, t, K, Kp);
  fence_proxy_async();
  named_bar(bar, 128);
}

// ---- A0' image of the warpgroup's 64 edges e0 .. e0 + 63, built by its 128 threads: [hi | lo | 1 1 0..] of
// [edge_attr (+ per-graph term) | node[tgt,:ns] | node[src,:ns]]
__device__ __forceinline__ void build_a0(const FusedParams& p, unsigned char* sA, long long e0, long long n_edges, int t) {
  const int Kin = p.K1, Kp = p.K1p;
  if (t < BM) put_a_tail(sA, t, Kin, Kp);
  if (p.a0_vec) {
    // vector path: four (virtual) threads per edge row, each converting a contiguous quarter of the row's 8-column groups
    // (<= 5 groups = 10 independent 16-byte loads); the 128 threads take two passes over the 64 rows.  The row's indices
    // (attribute row, per-graph term, both end points) are loaded once per pass, then ALL data loads of the pass are
    // issued - including the per-graph term's - then the conversions: two dependent global-memory round trips per pass.
    constexpr int TPR = 4;
    const int groups = Kin >> 3, gh = (groups + TPR - 1) / TPR;
    constexpr int PER = (144 / 8 + TPR - 1) / TPR;      // Kp <= 144 (MAX_KB k-blocks)
#pragma unroll 1
    for (int vt = t; vt < BM * TPR; vt += 128) {
      const int r = vt / TPR, g0 = (vt % TPR) * gh, g1 = min(groups, g0 + gh);
      const long long e = e0 + r;
      const bool live = e < n_edges;
      const int ge = p.ne >> 3, gs = p.ns >> 3;           // groups of the attribute / of one node section
      long long er = e;
      int ai = -1, it = 0, is = 0;
      if (live) {
        if (g0 < ge) {
          if (p.perm) er = (long long)__ldg(p.perm + e);
          if (p.ea_add) ai = __ldg(p.ea_add_idx + e);
        }
        if (g0 < ge + gs && g1 > ge) it = __ldg(p.tgt + e);
        if (g1 > ge + gs) is = __ldg(p.src + e);
      }
      const float* ea_row = p.ea + er * p.ld_ea;
      const float* add_row = ai >= 0 ? p.ea_add + (long long)ai * p.ne : nullptr;
      const float* t_row = p.node + (long long)it * p.ld_node - p.ne;
      const float* s_row = p.node + (long long)is * p.ld_node - p.ne - p.ns;
      float4 f[PER][2], ad[PER][2];
#pragma unroll
      for (int u = 0; u < PER; ++u) {
        const int g = g0 + u, k = g << 3;
        f[u][0] = f[u][1] = ad[u][0] = ad[u][1] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (live && g < g1) {
          const float* src = (g < ge) ? ea_row + k : (g < ge + gs ? t_row + k : s_row + k);
          const float4* s4 = reinterpret_cast<const float4*>(src);
          f[u][0] = __ldg(s4);
          f[u][1] = __ldg(s4 + 1);
          if (g < ge && add_row) {
            const float4* a4 = reinterpret_cast<const float4*>(add_row + k);
            ad[u][0] = __ldg(a4);
            ad[u][1] = __ldg(a4 + 1);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < PER; ++u) {
        const int g = g0 + u;
        if (g < g1) {
          f[u][0].x += ad[u][0].x; f[u][0].y += ad[u][0].y; f[u][0].z += ad[u][0].z; f[u][0].w += ad[u][0].w;
          f[u][1].x += ad[u][1].x; f[u][1].y += ad[u][1].y; f[u][1].z += ad[u][1].z; f[u][1].w += ad[u][1].w;
          uint4 hi, lo;
          split8(reinterpret_cast<const float*>(&f[u][0]), hi, lo);
          put_a8(sA, r, g << 3, hi);
          put_a8(sA, r, Kp + (g << 3), lo);
        }
      }
    }
  } else {
    for (int idx = t; idx < BM * Kin; idx += 128) {
      const int r = idx / Kin, k = idx - r * Kin;
      const long long e = e0 + r;
      float v = 0.f;
      if (e < n_edges) {
        if (k < p.ne) {
          const long long er = p.perm ? (long long)__ldg(p.perm + e) : e;
          v = __ldg(p.ea + er * p.ld_ea + k);
          if (p.ea_add) v += __ldg(p.ea_add + (long long)__ldg(p.ea_add_idx + e) * p.ne + k);
        } else if (k < p.ne + p.ns) v = __ldg(p.node + (long long)__ldg(p.tgt + e) * p.ld_node + (k - p.ne));
        else v = __ldg(p.node + (long long)__ldg(p.src + e) * p.ld_node + (k - p.ne - p.ns));
      }
      const __nv_bfloat16 hi = __float2bfloat16(v);
      const __nv_bfloat16 lo = __float2bfloat16(v - __bfloat162float(hi));
      put_a(sA, r, k, hi);
      put_a(sA, r, Kp + k, lo);
    }
  }
  fence_proxy_async();
}

// Shared-memory budget of an instantiation (the launcher checks it against the 227 KB opt-in): the two A images, the B
// stages, the z / staging buffers, Y, the staged Clebsch-Gordan tables (first order only), tiles, barriers and schedules,
// plus the 1 KB alignment slack.
template <bool SO> constexpr size_t smem_bytes() {
  constexpr int NST = SO ? SO_STAGES : STAGES;
  return 2 * (size_t)A_IMAGE_BYTES + (size_t)NST * STAGE_BYTES +
         (2 * (SO ? WG_BUF_SO : WG_BUF) + 2 * BM * 9 + (SO ? 0 : MAX_PATHS * MTAB)) * 4 + MAX_TILES * 8 * 4 +
         (NST + 4) * sizeof(uint64_t) + (4 * SCHED_WORDS + NST) * 4 + 1024;
}

// SO = false: the first-order kernel (d_in, d_out <= 3, kinds 0-5, <= 16 paths).  SO = true: the second-order one (d_in,
// d_out <= 5, kinds 0-7, <= 32 paths); a (10, 5) tile (kind 6) would need 100 partial sums beside the 96 accumulator
// registers, so it contracts its block in two slices, components 0-2 then 3-4, from the same accumulator tile and scatters
// each slice at the end of the tile (not of the output irrep): 60 and 40 partial sums, the budget of kind 1.
template <bool SO, bool FIXED>
__device__ __forceinline__ void fused_conv_body(const FusedParams& p) {
  constexpr int NST = SO ? SO_STAGES : STAGES;
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  unsigned char* sA = smem;                                      // [2 warpgroups][MAX_KA x 8 KB]
  unsigned char* sB = smem + 2 * (size_t)A_IMAGE_BYTES;          // ring of B stages
  float* sBuf = reinterpret_cast<float*>(sB + NST * STAGE_BYTES);      // [2 warpgroups][WG_BUF]: z rows / scatter staging
  float* sY = sBuf + 2 * (SO ? WG_BUF_SO : WG_BUF);              // [2][64][9] edge_weight * spherical harmonics per edge
  float* sMtab = sY + 2 * BM * 9;                                // [MAX_PATHS][48] (first order)
  int* sTiles = reinterpret_cast<int*>(sMtab + (SO ? 0 : MAX_PATHS * MTAB));   // [MAX_TILES][8]
  uint64_t* full = reinterpret_cast<uint64_t*>(sTiles + MAX_TILES * 8);   // B stage s has landed (TMA complete_tx)
  unsigned long long* sDbg = reinterpret_cast<unsigned long long*>(full + NST);   // [2][2] debug clocks per warpgroup
  uint32_t* sOps = reinterpret_cast<uint32_t*>(sDbg + 4);       // [2 warpgroups][W1', W2'][SCHED_WORDS] MMA schedules
  uint32_t* sRel = sOps + 4 * SCHED_WORDS;                       // [NST] releases of each stage

  const int tid = threadIdx.x;
  const int S1 = p.K1p >> 4, S2 = p.Hp >> 4;
  for (int i = tid; i < p.n_tiles * 8; i += THREADS) sTiles[i] = p.tiles[i];
  if constexpr (!SO)
    for (int i = tid; i < p.n_paths * MTAB; i += THREADS) sMtab[i] = p.mtab[i];
  if (tid % 32 == 0 && tid < 128) {
    const int wg = tid >> 6, which = (tid >> 5) & 1;
    build_ops(sOps + (2 * wg + which) * SCHED_WORDS, which ? S2 : S1, gmma_desc_lo(smem_u32(sA + wg * A_IMAGE_BYTES)));
  }
  if (tid < NST) sRel[tid] = 0u;
  if (tid < 4) sDbg[tid] = 0ull;
  if (tid == 0) {
    for (int s = 0; s < NST; ++s) mbar_init(&full[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int n1 = ((p.H + 15) / 16) * 16;

  // the edge count may live on the device (neighbour lists built without a host round trip): p.n_edges is then its bound
  long long n_edges = p.n_edges;
  if (p.n_edges_dev) { const long long nd = __ldg(p.n_edges_dev); n_edges = nd < n_edges ? (nd < 0 ? 0 : nd) : n_edges; }
  const long long n_mtiles = (n_edges + CTA_EDGES - 1) / CTA_EDGES;
  const long long my_units = blockIdx.x < n_mtiles ? (n_mtiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  // debug clocks: a span is counted by subtracting its start from the counter and adding its end (modulo 2^64), so no start
  // value is held in registers through the kernel
  if (p.dbg && blockIdx.x == 0 && tid == 0) {      // effective SM clock of this launch: clock64 ticks per globaltimer ns
    unsigned long long g0;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g0));
    atomicAdd(p.dbg + 25, 0ull - (unsigned long long)clock64());
    atomicAdd(p.dbg + 26, 0ull - g0);
  }

  Stream<NST> st;
  st.sB = sB; st.full = full; st.rel = sRel; st.tiles = sTiles; st.n1 = n1;
  st.per_unit = p.n_kb1 + p.n_hidden * p.n_kb + p.n_tiles * p.n_kb;
  st.len = (uint32_t)(my_units * st.per_unit);
  // the ring runs ahead across edge tiles: the next tile's W1' blocks are requested while this one is contracted
  if (tid == 0)
    for (int i = 0; i < NST; ++i) st.issue(p, (uint32_t)i);

  // Warpgroup g owns edges 64 g .. 64 g + 63 of every 128-edge tile and does all of their work; the two warpgroups meet
  // only at the stages of the shared B stream.
  const int g = __shfl_sync(0xffffffffu, tid >> 7, 0);          // warp-uniform for the compiler
  const int t = tid & 127, w4 = t >> 5, lane = tid & 31, q = lane & 3, bar = BAR_WG + g;
  const int r0 = 16 * w4 + (lane >> 2);                          // this thread's accumulator rows (edges) r0, r0 + 8
  const int rb = r0 + 8 * (q >> 1), ub = 8 * (q & 1);            // its z rows: edge rb, tile rows ub .. ub + 7
  unsigned char* sAg = sA + (size_t)g * A_IMAGE_BYTES;
  float* buf = sBuf + g * (SO ? WG_BUF_SO : WG_BUF);
  float* zrow = buf + rb * ZLD;
  const float* zcon = buf + r0 * ZLD;
  float* zrowb = buf + 64 * ZLD + rb * ZLDB;                     // SO: components 3, 4
  const float* zconb = buf + 64 * ZLD + r0 * ZLDB;
  unsigned long long* dwait = (p.dbg && t == 0) ? sDbg + 2 * g : nullptr;
  const uint32_t* ops1 = sOps + 2 * g * SCHED_WORDS;
  const uint32_t* ops2 = ops1 + SCHED_WORDS;
  uint32_t mc = 0;
  for (long long mt = blockIdx.x; mt < n_mtiles; mt += gridDim.x) {
    const long long e0 = mt * CTA_EDGES + g * BM;
    if (p.dbg && tid == 0) atomicAdd(p.dbg + 11, 0ull - (unsigned long long)clock64());
    build_a0(p, sAg, e0, n_edges, t);
    named_bar(bar, 128);
    // this thread's z edge: its source node's values, edge weight and spherical harmonics (component normalisation, e3nn
    // polynomials); rows past the end see zero node values and scatter nothing
    const long long eb = e0 + rb;
    const bool vb = eb < n_edges;
    const int src_b = vb ? __ldg(p.src + eb) : 0;
    const long long erb = (vb && p.perm) ? (long long)__ldg(p.perm + eb) : eb;
    const float ew_b = (vb && p.ew) ? __ldg(p.ew + erb) : 1.f;
    float* Y = sY + (g * BM + rb) * 9;
    if (ub == 0) {
      float vx = vb ? p.vec_sign * __ldg(p.vec + 3 * erb) : 1.f, vy = vb ? p.vec_sign * __ldg(p.vec + 3 * erb + 1) : 0.f,
            vz = vb ? p.vec_sign * __ldg(p.vec + 3 * erb + 2) : 0.f;
      const float nrm = fmaxf(sqrtf(vx * vx + vy * vy + vz * vz), 1e-12f);
      vx /= nrm; vy /= nrm; vz /= nrm;
      const float s3 = 1.7320508075688772f, s5 = 2.23606797749979f, s15 = 3.872983346207417f;
      Y[0] = ew_b;
      Y[1] = ew_b * (s3 * vx); Y[2] = ew_b * (s3 * vy); Y[3] = ew_b * (s3 * vz);
      Y[4] = ew_b * (s15 * vx * vz);
      Y[5] = ew_b * (s15 * vx * vy);
      Y[6] = ew_b * (s5 * (vy * vy - 0.5f * (vx * vx + vz * vz)));
      Y[7] = ew_b * (s15 * vy * vz);
      Y[8] = ew_b * (0.5f * s15 * (vz * vz - vx * vx));
    }
    __syncwarp();
    // this lane's scatter edge: runs of equal targets inside the warp (rows past the end form their own, never flushed, runs)
    const long long es = e0 + 32 * (w4 & 1) + lane;
    const bool vs = es < n_edges;
    const int dst_s = vs ? __ldg(p.tgt + es) : -1;
    const int key_up = __shfl_up_sync(0xffffffffu, dst_s, 1);
    const uint32_t head_mask = __ballot_sync(0xffffffffu, lane == 0 || key_up != dst_s || !vs);

    const float* xrow = p.x + (long long)src_b * p.ld_x;
    float xn[SO ? 1 : XN], M[SO ? 25 : 9], acc[NACC_MAX];
    if constexpr (!SO) prefetch_tile(xrow, sTiles, ub, p.x_vec2, xn);
    Acc d;
    // the hidden stack, one product loop: W1' from A0' (schedule ops1, n_kb1 k-blocks), then each extra H x H layer Wh'
    // from the A' image (ops2, n_kb k-blocks, the geometry of the W2' products).  store_hidden writes each layer's ReLU
    // over the image its product read: mma_product returns only once every group of the product is complete in all four
    // warps (the release's barrier follows the last wait), and store_hidden fences to the async proxy and meets at the
    // barrier before the next product reads the image.
#pragma unroll 1
    for (int l = 0; l <= p.n_hidden; ++l) {
      mma_product(d, p, st, l ? ops2 : ops1, l ? p.n_kb : p.n_kb1, mc, bar, t, dwait);
      store_hidden(d, p, sAg, t, bar);
    }
    for (int ti = 0; ti < p.n_tiles; ++ti) {
      const int* tt = sTiles + ti * 8;
      const int kind = tt[0], d_in = tt[4], out_off = tt[5], flags = tt[6];
      if (flags & 1) {
#pragma unroll
        for (int i = 0; i < NACC_MAX; ++i) acc[i] = 0.f;
      }
      // M[i,k] = edge_weight * sum_j coef*C[i,j,k] * Y[sh_off + j]  (at most 3x3 for the supported paths; row-major,
      // stride 3), rebuilt only when the tile belongs to another path than its predecessor: dense table, fully unrolled
      if (SO && (flags & 4)) {    // [5][5] from the [5][5][5] table in global memory (L1), stride 5
        const float* T = p.mtab + tt[7] * SO_MTAB;
        const int sh_off = (flags >> 8) & 0xff;
        float yb[5];
#pragma unroll
        for (int j = 0; j < 5; ++j) yb[j] = Y[min(sh_off + j, 8)];
#pragma unroll
        for (int ik = 0; ik < 25; ++ik) {
          float a = 0.f;
#pragma unroll
          for (int j = 0; j < 5; ++j) a = fmaf(__ldg(T + ik * 5 + j), yb[j], a);
          M[ik] = a;
        }
      } else if (flags & 4) {
        const float* T = sMtab + tt[7] * MTAB;
        const int sh_off = (flags >> 8) & 0xff;
        float yb[5];
#pragma unroll
        for (int j = 0; j < 5; ++j) yb[j] = Y[min(sh_off + j, 8)];
#pragma unroll
        for (int ik = 0; ik < 9; ++ik) {
          float a = 0.f;
#pragma unroll
          for (int j = 0; j < 5; ++j) a = fmaf(T[ik * 5 + j], yb[j], a);
          M[ik] = a;
        }
      }
      // z of this tile from the node values prefetched one tile ahead; then the next tile's values are requested, so that
      // their latency hides behind this tile's MMAs (SO: read by build_z_so itself)
      __syncwarp();                             // the quad has read the previous tile's z rows
      if constexpr (SO) {
        const float* xs = xrow + tt[2] + ub * d_in;
        const int nr = min(max(tt[3] - ub, 0), 8);
        switch (kind) {
          case 0: build_z_so<1, 4>(xs, nr, d_in, M, zrow, zrowb, ub); break;
          case 1: case 3: build_z_so<3, 16>(xs, nr, d_in, M, zrow, zrowb, ub); break;
          case 2: build_z_so<1, 8>(xs, nr, d_in, M, zrow, zrowb, ub); break;
          case 4: case 5: build_z_so<1, 16>(xs, nr, d_in, M, zrow, zrowb, ub); break;
          case 6: case 7: build_z_so<5, 16>(xs, nr, d_in, M, zrow, zrowb, ub); break;
          default: __trap();   // unreachable: FusedPlan writes kinds 0-7 only (fused.py:CONSUMER_KINDS)
        }
      } else switch (kind) {
        case 0: build_z<1, 4>(xn, d_in, M, zrow, ub); break;
        case 1: build_z<3, 16>(xn, d_in, M, zrow, ub); break;
        case 2: build_z<1, 8>(xn, d_in, M, zrow, ub); break;
        case 3: build_z<3, 16>(xn, d_in, M, zrow, ub); break;
        case 4: case 5: build_z<1, 16>(xn, d_in, M, zrow, ub); break;
        default: __trap();     // unreachable: FusedPlan writes kinds 0-5 only (fused.py:CONSUMER_KINDS)
      }
      __syncwarp();
      if (!SO && ti + 1 < p.n_tiles) prefetch_tile(xrow, tt + 8, ub, p.x_vec2, xn);
      mma_product(d, p, st, ops2, p.n_kb, mc, bar, t, dwait);
      const long long c0 = dwait ? clock64() : 0;
      const int nch = tt[1] >> 5;
      if constexpr (SO) {
        switch (kind) {
          case 0: contract<48, 1, 4>(d, zcon, nch, q, acc); break;
          case 1: contract<10, 3, 16>(d, zcon, nch, q, acc); break;
          case 2: contract<16, 1, 8>(d, zcon, nch, q, acc); break;
          case 3: contract<4, 3, 16>(d, zcon, nch, q, acc); break;
          case 4: contract<10, 1, 16>(d, zcon, nch, q, acc); break;
          case 5: contract<4, 1, 16>(d, zcon, nch, q, acc); break;
          case 6:                  // (10, 5): components 0-2, scattered, then 3-4 from the same accumulator tile
#pragma unroll
            for (int i = 0; i < NACC_MAX; ++i) acc[i] = 0.f;
            contract<10, 3, 16>(d, zcon, nch, q, acc);
            flush<10, 3, 5, 0, FIXED>(p, acc, buf, r0, q, w4, lane, dst_s, head_mask, out_off, bar);
#pragma unroll
            for (int i = 0; i < NACC_MAX; ++i) acc[i] = 0.f;
            contract<10, 2, 16, 3>(d, zcon, nch, q, acc, zconb);
            flush<10, 2, 5, 3, FIXED>(p, acc, buf, r0, q, w4, lane, dst_s, head_mask, out_off, bar);
            break;
          case 7: contract<4, 5, 16>(d, zcon, nch, q, acc, zconb); break;
          default: __trap();
        }
        if ((flags & 2) && kind != 6) {
          switch (kind) {
            case 0: flush<48, 1, 1, 0, FIXED>(p, acc, buf, r0, q, w4, lane, dst_s, head_mask, out_off, bar); break;
            case 1: flush<10, 3, 3, 0, FIXED>(p, acc, buf, r0, q, w4, lane, dst_s, head_mask, out_off, bar); break;
            case 2: flush<16, 1, 1, 0, FIXED>(p, acc, buf, r0, q, w4, lane, dst_s, head_mask, out_off, bar); break;
            case 3: flush<4, 3, 3, 0, FIXED>(p, acc, buf, r0, q, w4, lane, dst_s, head_mask, out_off, bar); break;
            case 4: flush<10, 1, 1, 0, FIXED>(p, acc, buf, r0, q, w4, lane, dst_s, head_mask, out_off, bar); break;
            case 5: flush<4, 1, 1, 0, FIXED>(p, acc, buf, r0, q, w4, lane, dst_s, head_mask, out_off, bar); break;
            case 7: flush<4, 5, 5, 0, FIXED>(p, acc, buf, r0, q, w4, lane, dst_s, head_mask, out_off, bar); break;
            default: __trap();
          }
        }
      } else {
        switch (kind) {
          case 0: contract<48, 1, 4>(d, zcon, nch, q, acc); break;
          case 1: contract<10, 3, 16>(d, zcon, nch, q, acc); break;
          case 2: contract<16, 1, 8>(d, zcon, nch, q, acc); break;
          case 3: contract<4, 3, 16>(d, zcon, nch, q, acc); break;
          case 4: contract<10, 1, 16>(d, zcon, nch, q, acc); break;
          case 5: contract<4, 1, 16>(d, zcon, nch, q, acc); break;
          default: __trap();
        }
        if (flags & 2) {
          switch (kind) {
            case 0: flush<48, 1, 1, 0, FIXED>(p, acc, buf, r0, q, w4, lane, dst_s, head_mask, out_off, bar); break;
            case 1: flush<10, 3, 3, 0, FIXED>(p, acc, buf, r0, q, w4, lane, dst_s, head_mask, out_off, bar); break;
            case 2: flush<16, 1, 1, 0, FIXED>(p, acc, buf, r0, q, w4, lane, dst_s, head_mask, out_off, bar); break;
            case 3: flush<4, 3, 3, 0, FIXED>(p, acc, buf, r0, q, w4, lane, dst_s, head_mask, out_off, bar); break;
            case 4: flush<10, 1, 1, 0, FIXED>(p, acc, buf, r0, q, w4, lane, dst_s, head_mask, out_off, bar); break;
            case 5: flush<4, 1, 1, 0, FIXED>(p, acc, buf, r0, q, w4, lane, dst_s, head_mask, out_off, bar); break;
            default: __trap();
          }
        }
      }
      if (dwait) dwait[1] += (unsigned long long)(clock64() - c0);
    }
    if (p.cnt && w4 < 2) {         // edge counts per target: one atomic per run, issued by the run's first lane
      const bool head = (head_mask >> lane) & 1;
      const uint32_t above = (lane == 31) ? 0u : (head_mask >> (lane + 1));
      const int run_len = above ? __ffs(above) : 32 - lane;
      if (head && vs) red_add(p.cnt + dst_s, (float)run_len);
    }
    if (p.dbg && tid == 0) { atomicAdd(p.dbg + 11, (unsigned long long)clock64()); atomicAdd(p.dbg + 12, 2ull); }
    if (dwait) {
      atomicAdd(p.dbg + 13, dwait[0]);
      atomicAdd(p.dbg + 14, dwait[1]);
      dwait[0] = dwait[1] = 0ull;
    }
  }
  if (p.dbg && blockIdx.x == 0 && tid == 0) {
    unsigned long long g1;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g1));
    atomicAdd(p.dbg + 25, (unsigned long long)clock64());
    atomicAdd(p.dbg + 26, g1);
  }
}

__global__ void __launch_bounds__(THREADS, 1) fused_conv_kernel(const FusedParams p) { fused_conv_body<false, false>(p); }
__global__ void __launch_bounds__(THREADS, 1) fused_conv_kernel_so(const FusedParams p) { fused_conv_body<true, false>(p); }
// deterministic instantiations: the scatter adds 64-bit fixed-point values (ddb200_fused_conv_fixed / _so_fixed)
__global__ void __launch_bounds__(THREADS, 1) fused_conv_fixed_kernel(const FusedParams p) { fused_conv_body<false, true>(p); }
__global__ void __launch_bounds__(THREADS, 1) fused_conv_fixed_kernel_so(const FusedParams p) { fused_conv_body<true, true>(p); }

// per-device state: debug counters and the one-time opt-in to > 48 KB of dynamic shared memory
constexpr int MAX_DEVICES = 64;
struct DeviceState {
  bool attr_done[2][2] = {};                      // [SO][FIXED]
  bool dbg_init = false;
  unsigned long long* dbg = nullptr;
};
DeviceState g_dev[MAX_DEVICES];

unsigned long long* fused_debug_buffer(int dev) {
  if (dev < 0 || dev >= MAX_DEVICES) return nullptr;
  DeviceState& st = g_dev[dev];
  if (!st.dbg_init) {
    st.dbg_init = true;
    const char* e = getenv("DDB200_FUSED_DEBUG");
    if (e && atoi(e) != 0 && cudaMalloc(&st.dbg, 32 * sizeof(unsigned long long)) == cudaSuccess)
      cudaMemset(st.dbg, 0, 32 * sizeof(unsigned long long));
  }
  return st.dbg;
}

}  // namespace


// Diagnostics (DDB200_FUSED_DEBUG=1 only): copies the 32 clock counters of the fused kernel (current device) to `out` and
// clears them.  [11] clocks spent per 128-edge tile by warpgroup 0 (summed over tiles), [12] 64-edge units (two per
// 128-edge tile), [13] clocks the warpgroups spent waiting for a B stage to land, [14] clocks they spent contracting and
// scattering (both summed over the two warpgroups), [25] / [26] clock64 ticks / ns of CTA 0 over the launch.  Synchronises
// the device.
extern "C" int ddb200_fused_debug_read(uint64_t* out) {
  int dev = 0;
  cudaGetDevice(&dev);
  unsigned long long* b = fused_debug_buffer(dev);
  if (!b || !out) return DDB200_EINVAL;
  cudaError_t e = cudaDeviceSynchronize();
  if (e == cudaSuccess) e = cudaMemcpy(out, b, 32 * sizeof(unsigned long long), cudaMemcpyDeviceToHost);
  if (e == cudaSuccess) e = cudaMemset(b, 0, 32 * sizeof(unsigned long long));
  return (int)e;
}

namespace {

template <bool SO, bool FIXED>
int fused_conv_launch(const ddb200_fused_args* a, long long* sum_fx, int* err, void* stream) {
  if (FIXED && (!sum_fx || !err)) return DDB200_EINVAL;
  if (!a || !a->edge_attr || !a->w1_images || !a->w2_images || !a->tiles || !a->mtab || !a->x || !a->edge_vec ||
      (!FIXED && !a->sum) ||
      !a->tgt || !a->src || a->n_edges < 0 || a->ne <= 0 || a->ns < 0 || a->hidden <= 0 || a->n_tiles <= 0 || a->d_out <= 0)
    return DDB200_EINVAL;
  if (a->ns > 0 && (!a->node || a->ld_node < a->ns)) return DDB200_EINVAL;
  if (a->n_tiles > MAX_TILES || a->n_paths <= 0 || a->n_paths > (SO ? SO_MAX_PATHS : MAX_PATHS) || a->sh_lmax < 0 ||
      a->sh_lmax > 2)
    return DDB200_EINVAL;
  if ((a->ea_add == nullptr) != (a->ea_add_idx == nullptr)) return DDB200_EINVAL;
  const int K1 = a->ne + 2 * a->ns, H = a->hidden;
  const int K1p = (K1 + 15) / 16 * 16, Hp = (H + 15) / 16 * 16;
  const int n_kb = (2 * Hp + 16 + BK - 1) / BK, n_kb1 = (2 * K1p + 16 + BK - 1) / BK;
  if (n_kb > MAX_KB || n_kb1 > MAX_KB || H > MAX_N) return DDB200_EINVAL;
  if ((reinterpret_cast<uintptr_t>(a->w1_images) & 127) || (reinterpret_cast<uintptr_t>(a->w2_images) & 127)) return DDB200_EINVAL;
  if (a->n_hidden < 0 || (a->n_hidden > 0 && (!a->wh_images || (reinterpret_cast<uintptr_t>(a->wh_images) & 127))))
    return DDB200_EINVAL;
  if (a->n_edges == 0) return 0;
  FusedParams p = {};
  p.ea = a->edge_attr; p.ld_ea = a->ld_ea; p.ne = a->ne; p.node = a->node; p.ld_node = a->ld_node; p.ns = a->ns;
  p.tgt = a->tgt; p.src = a->src; p.perm = a->edge_perm; p.ea_add = a->ea_add; p.ea_add_idx = a->ea_add_idx;
  // 16-byte loads of whole 8-column groups: every row that is read (edge_attr, ea_add, both node sections) must start on a
  // 16-byte boundary, so the base pointers as well as the widths and row strides are checked
  const auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  p.a0_vec = ((a->ne | a->ns) & 7) == 0 && ((a->ld_ea | (a->ns ? a->ld_node : 0)) & 3) == 0 && al16(a->edge_attr) &&
             (a->ns == 0 || al16(a->node)) && (a->ea_add == nullptr || al16(a->ea_add));
  p.vec_sign = a->vec_sign == 0.f ? 1.f : a->vec_sign;
  p.w1img = reinterpret_cast<const __nv_bfloat16*>(a->w1_images); p.K1 = K1; p.K1p = K1p; p.n_kb1 = n_kb1;
  p.H = H; p.Hp = Hp; p.n_kb = n_kb;
  p.w2img = reinterpret_cast<const __nv_bfloat16*>(a->w2_images); p.tiles = a->tiles; p.n_tiles = a->n_tiles;
  p.whimg = reinterpret_cast<const __nv_bfloat16*>(a->wh_images); p.n_hidden = a->n_hidden;
  p.mtab = a->mtab; p.n_paths = a->n_paths;
  p.x = a->x; p.ld_x = a->ld_x; p.x_vec2 = (a->x_pairs_ok && (a->ld_x & 1) == 0 && (reinterpret_cast<uintptr_t>(a->x) & 7) == 0) ? 1 : 0;
  p.vec = a->edge_vec; p.ew = a->edge_weight; p.lmax = a->sh_lmax; p.sum = a->sum; p.d_out = a->d_out; p.cnt = a->cnt;
  p.n_edges = a->n_edges; p.n_edges_dev = a->n_edges_dev;
  p.sum_fx = sum_fx; p.err = err;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= MAX_DEVICES) return DDB200_EINVAL;
  p.dbg = fused_debug_buffer(dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const long long n_mtiles = (a->n_edges + CTA_EDGES - 1) / CTA_EDGES;
  const size_t smem = smem_bytes<SO>();
  if (smem > 227 * 1024) return DDB200_ESMEM;
  auto kernel = FIXED ? (SO ? fused_conv_fixed_kernel_so : fused_conv_fixed_kernel) : (SO ? fused_conv_kernel_so : fused_conv_kernel);
  bool& attr_done = g_dev[dev].attr_done[SO][FIXED];
  if (!attr_done) {                 // the opt-in is a per-device, per-kernel attribute
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    attr_done = true;
  }
  const unsigned grid = (unsigned)(n_mtiles < sms ? n_mtiles : sms);
  kernel<<<grid, THREADS, smem, (cudaStream_t)stream>>>(p);
  return (int)cudaGetLastError();
}

}  // namespace

extern "C" int ddb200_fused_conv(const ddb200_fused_args* a, void* stream) {
  return fused_conv_launch<false, false>(a, nullptr, nullptr, stream);
}

// The second-order instantiation: plans with a 5-component input or output block (fused.py:FusedPlan.second_order); the
// Clebsch-Gordan tables are [n_paths][5][5][5] padded to 128 floats.
extern "C" int ddb200_fused_conv_so(const ddb200_fused_args* a, void* stream) {
  return fused_conv_launch<true, false>(a, nullptr, nullptr, stream);
}

// Deterministic instantiations (include/diffdock_b200.h): a->sum is ignored; the sums go to sum_fx in units of 2^-32.
extern "C" int ddb200_fused_conv_fixed(const ddb200_fused_args* a, int64_t* sum_fx, int32_t* err, void* stream) {
  return fused_conv_launch<false, true>(a, reinterpret_cast<long long*>(sum_fx), err, stream);
}
extern "C" int ddb200_fused_conv_so_fixed(const ddb200_fused_args* a, int64_t* sum_fx, int32_t* err, void* stream) {
  return fused_conv_launch<true, true>(a, reinterpret_cast<long long*>(sum_fx), err, stream);
}
