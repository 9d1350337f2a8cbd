// Fully fused equivariant convolution for one edge group (sm_90a): radial MLP on the Hopper tensor cores (wgmma) +
// tensor-product contraction + scatter - the per-edge weight tensor [E, weight_numel] never exists in HBM.
//
//   for a tile of 64 CSR-sorted edges (one CTA, persistent over tiles; warpgroup 0 multiplies, warpgroup 1 contracts):
//     A0' = split-bf16([edge_attr (+ per-graph term) | node[tgt,:ns] | node[src,:ns]])   built in shared memory (128B swizzle)
//     H   = relu(A0' x W1'^T)          wgmma -> registers -> A' image (bias folded via two constant-one columns)
//     for every N tile (whole rows u of one path block [mul_in, mul_out], <= 192 columns):
//        Wt = A' x W2'^T[tile]         wgmma m64nNk16 into registers (B' images streamed by TMA bulk copies through a
//                                      4-stage ring), then stored to a padded shared-memory tile C [64][196] once the
//                                      consumers have drained the previous one: the next tile's MMAs overlap the contraction
//        consumer thread pair (e, half): acc[w,k] += Wt[e, (u,w)] * z_e[u,k] over its half of the 32-column chunks,
//                                        z_e[u,k] = sum_i x[src_e][u,i] M_e[i,k],  M_e = edge_weight * coef * C . Y(vec_e)
//     at the end of an output irrep: sum[tgt_e, irrep] += acc  (the pair's partial sums are added and runs of equal
//                                                              targets reduced through shared memory, then one coalesced
//                                                              RED.ADD per run and 32 output values)
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
#include "sm90.cuh"

namespace {

using namespace ddb200_sm90;

constexpr int BM = 64, BK = 64;                  // CTA tile = one wgmma M; BK bf16 = one 128-byte swizzle row
constexpr int A_KB_BYTES = BM * BK * 2;          // 8 KB
constexpr int B_IMAGE_BYTES = 256 * BK * 2;      // 32 KB: one k-block image of an N tile in global memory
constexpr int MAX_N = 192;                       // widest N tile of a plan (and widest hidden layer)
constexpr int STAGES = 4;
constexpr int STAGE_BYTES = MAX_N * BK * 2;      // 24 KB: the rows of an image the MMA reads
constexpr int MAX_KB = 5;                        // k-blocks of either operand image: 2 Kp + 16 <= 320  (Kp <= 144)
constexpr int MAX_KA = MAX_KB;
constexpr int OPS_PER_KB = 8;                    // MMAs that read one staged k-block of B (4 steps x up to 2 A partners)
constexpr int THREADS = 256;                     // warpgroup 0: MMA, warpgroup 1: consumers (two threads per edge)
constexpr int MAX_TILES = 128, MAX_PATHS = 16, MTAB = 48;     // per path: dense [3][3][5] table, padded to 48 floats
constexpr int FLUSH_LD = 33;                     // padded row of the per-warp scatter staging buffer [48][33]
constexpr int CLD = 196;                         // row of the accumulator tile: 16-byte reads of 8 rows hit 8 bank groups
constexpr int BAR_MMA = 1, BAR_PAIR = 2;         // named barriers: the MMA warpgroup, the two consumer warp pairs

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
  const int* tiles; int n_tiles;                     // [n_tiles][8]: kind, N_mma, x_off, rows, d_in, out_off, flags | sh_off << 8, path
  const float* mtab; int n_paths;                    // [n_paths][48]: coef * C[i, j, k] as [i][k][j], i,k < 3, j < 5
  const float* x; long long ld_x; int x_vec2;        // node irreps gathered by src
  const float* vec; const float* ew; int lmax;
  float* sum; int d_out; float* cnt;
  long long n_edges; const int* n_edges_dev;
  unsigned long long* dbg;                           // optional [32] clock counters (DDB200_FUSED_DEBUG=1), else nullptr
};

// ---- consumer: this thread's half (alternate 32-column chunks) of one accumulator tile (ROWS rows u of a [mul_in, MULOUT]
// block) times z -> acc.  Only the first `nch` chunks hold MMA results (the last tile of a path block may be narrower).
template <int MULOUT, int DOUT, int ROWS>
__device__ __forceinline__ void consume_tile(const float* __restrict__ crow, int nch, int half, const float* __restrict__ z,
                                             float* __restrict__ acc) {
  constexpr int NCOL = MULOUT * ROWS;
  static_assert(NCOL % 32 == 0 && NCOL <= MAX_N, "tile width");
#pragma unroll
  for (int c = 0; c < NCOL / 32; ++c) {
    if (c < nch && (c & 1) == half) {
      float v[32];
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float4 f = reinterpret_cast<const float4*>(crow + c * 32)[q];
        v[4 * q] = f.x; v[4 * q + 1] = f.y; v[4 * q + 2] = f.z; v[4 * q + 3] = f.w;
      }
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int col = c * 32 + j, row = col / MULOUT, w = col % MULOUT;     // compile-time after unrolling
#pragma unroll
        for (int k = 0; k < DOUT; ++k) acc[w * DOUT + k] = fmaf(v[j], z[row * DOUT + k], acc[w * DOUT + k]);
      }
    }
  }
}

// z[r, k] = sum_i x[x_off + r*DIN + i] * M[i, k] for the tile's rows; xv = the tile's gathered node values (prefetched into
// registers one tile ahead, zero beyond the valid rows)
template <int DIN, int DOUT, int ROWS>
__device__ __forceinline__ void make_z(const float* __restrict__ xv, const float* __restrict__ M, float* __restrict__ z) {
#pragma unroll
  for (int r = 0; r < ROWS; ++r) {
#pragma unroll
    for (int k = 0; k < DOUT; ++k) {
      float a = 0.f;
#pragma unroll
      for (int i = 0; i < DIN; ++i) a = fmaf(xv[r * DIN + i], M[i * 3 + k], a);
      z[r * DOUT + k] = a;
    }
  }
}

constexpr int XN = 48;     // gathered node values of one tile: at most 16 rows x 3 components
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

// z is formed from the node values prefetched during the previous tile before waiting for the accumulator tile
template <int MULOUT, int DOUT, int ROWS>
__device__ __forceinline__ void tile_body(const float* crow, int nch, int half, const float* xn, int d_in, const float* M,
                                          float* acc, uint64_t* cfull, uint32_t parity) {
  float z[ROWS * DOUT];
  if (d_in == 1) make_z<1, DOUT, ROWS>(xn, M, z);
  else make_z<3, DOUT, ROWS>(xn, M, z);
  mbar_wait(cfull, parity);
  consume_tile<MULOUT, DOUT, ROWS>(crow, nch, half, z, acc);
}

// MMA schedule of one staged k-block of B (4 steps of 16 columns; images [hi | lo | bias], S = Kp / 16 steps per part):
// step c < S (hi): x A hi (column block c) and x A lo (block S + c);  S <= c < 2S (lo): x A hi (block c - S);
// c == 2S (bias): x A ones (block 2S).  Per k-block OPS_PER_KB slots of two words, stored as [A words 0-7 | B words 0-7]:
// A word = low descriptor word of the A column block (absolute), B word = offset of the B step inside the stage in 16-byte
// units; the first n slots are used.  After the MAX_KB k-blocks: n of every k-block (1 <= n <= 8 for every k-block of an
// image: the last one holds at least the bias step).
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

// B stream of a CTA: per edge tile the W1' k-blocks, then every N tile's W2' k-blocks; item i goes to stage i % STAGES
struct Stream {
  unsigned char* sB; uint64_t* full; const int* tiles;
  int n1, per_unit; uint32_t len;
  __device__ __forceinline__ void issue(const FusedParams& p, uint32_t i) const {
    if (i >= len) return;
    const int j = (int)(i % (uint32_t)per_unit);
    const unsigned char* src;
    uint32_t bytes;
    if (j < p.n_kb1) {
      src = reinterpret_cast<const unsigned char*>(p.w1img) + (size_t)j * B_IMAGE_BYTES;
      bytes = (uint32_t)n1 * 128u;
    } else {                    // image (t, kb) of the W2' set lies at (t * n_kb + kb) = j - n_kb1
      src = reinterpret_cast<const unsigned char*>(p.w2img) + (size_t)(j - p.n_kb1) * B_IMAGE_BYTES;
      bytes = (uint32_t)tiles[((j - p.n_kb1) / p.n_kb) * 8 + 1] * 128u;
    }
    const uint32_t s = i % STAGES;
    bulk_load(sB + (size_t)s * STAGE_BYTES, src, bytes, &full[s]);
  }
};

// ---- MMA warpgroup.  Every product is issued MAX_N wide into one of two register sets of accumulators (Acc); k-block after
// k-block of the CTA's B stream, counted by mc.  One MMA group stays in flight while the previous k-block's stage is
// refilled.
using Acc = float[MAX_N / 2];

// the n MMAs of one staged k-block as one chain: one register fence in front, one commit group.  The descriptors are read
// before the fence, so that nothing but the MMAs lies between the fence and the commit; acc0 == 0 overwrites d.
template <int NOPS>
__device__ __forceinline__ void mma_chain(Acc& d, const uint32_t* oa, const uint32_t* ob, uint32_t b_lo, uint32_t acc0) {
  uint32_t a[NOPS], b[NOPS];
#pragma unroll
  for (int i = 0; i < NOPS; ++i) { a[i] = oa[i]; b[i] = b_lo + ob[i]; }
  wgmma_fence();
#pragma unroll
  for (int i = 0; i < NOPS; ++i) Wgmma<MAX_N>::mma(d, gmma_desc(a[i]), gmma_desc(b[i]), i == 0 ? acc0 : 1u);
  wgmma_commit();
}

// k-block kb of the schedule `ops` from stage mc % STAGES into d
__device__ __forceinline__ void mma_kblock(Acc& d, const Stream& st, const uint32_t* ops, int kb, uint32_t mc) {
  const uint32_t s = mc % STAGES;
  mbar_wait(&st.full[s], (mc / STAGES) & 1);
  const uint32_t* oa = ops + kb * 2 * OPS_PER_KB;
  const uint32_t* ob = oa + OPS_PER_KB;
  const uint32_t b_lo = gmma_desc_lo(smem_u32(st.sB)) + s * (STAGE_BYTES >> 4);
  const uint32_t acc0 = kb != 0;
  switch (ops[MAX_KB * 2 * OPS_PER_KB + kb]) {      // uniform: the chain length follows from the plan's shapes
    case 1: mma_chain<1>(d, oa, ob, b_lo, acc0); break;
    case 2: mma_chain<2>(d, oa, ob, b_lo, acc0); break;
    case 3: mma_chain<3>(d, oa, ob, b_lo, acc0); break;
    case 4: mma_chain<4>(d, oa, ob, b_lo, acc0); break;
    case 5: mma_chain<5>(d, oa, ob, b_lo, acc0); break;
    case 6: mma_chain<6>(d, oa, ob, b_lo, acc0); break;
    case 7: mma_chain<7>(d, oa, ob, b_lo, acc0); break;
    case 8: mma_chain<8>(d, oa, ob, b_lo, acc0); break;
    default: __trap();     // unreachable: build_ops gives every k-block of an image 1..8 MMAs (n_kb = ceil((2S + 1) / 4))
  }
}

// k-blocks kb0 .. nkb - 1 of one product into d.  Once a k-block is committed, every older group is waited for and the
// previous k-block's stage refilled (for kb0 only when `release_first`: that k-block belongs to another product).
__device__ __forceinline__ void mma_kblocks(Acc& d, const FusedParams& p, const Stream& st, const uint32_t* ops, int kb0,
                                            int nkb, bool release_first, uint32_t& mc, int t) {
  for (int kb = kb0; kb < nkb; ++kb, ++mc) {
    mma_kblock(d, st, ops, kb, mc);
    if (kb > kb0 || release_first) {
      wgmma_wait_one();
      named_bar(BAR_MMA, 128);                   // every warp is done with the previous k-block's stage
      if (t == 0) st.issue(p, mc - 1 + STAGES);
    }
  }
}

// every group complete: the last k-block's stage is refilled
__device__ __forceinline__ void mma_drain(const FusedParams& p, const Stream& st, uint32_t mc, int t) {
  wgmma_wait_all();
  named_bar(BAR_MMA, 128);
  if (t == 0) st.issue(p, mc - 1 + STAGES);
}

// hidden layer -> A': ReLU, bf16 split, written back over the operand image; complete and visible to the async proxy
// before the first weight-tile MMA reads it
__device__ __forceinline__ void store_hidden(const Acc& d, const FusedParams& p, unsigned char* sA, int t) {
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
  named_bar(BAR_MMA, 128);
}

// a complete weight tile -> the accumulator tile C, once the consumers have drained the previous one
__device__ __forceinline__ void store_weights(Acc& d, float* sC, uint64_t* cfull, uint64_t* cempty, uint32_t& cc, int t) {
  wgmma_fence_regs(d);                           // d is read only after the wait that completed it
  const int lane = t & 31, r0 = (t >> 5) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
  mbar_wait(cempty, (cc & 1) ^ 1);
#pragma unroll
  for (int j = 0; j < MAX_N / 8; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h)
      *reinterpret_cast<float2*>(sC + (r0 + 8 * h) * CLD + 8 * j + c0) = make_float2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
  mbar_arrive(cfull);
  ++cc;
}

// weight tile t, every k-block committed into `cur`, is followed by another one: that tile's first k-block is committed
// into `nxt` first and only `cur`'s groups are waited for, so the tensor pipe works through that k-block while C is
// written; then its remaining k-blocks are issued.
__device__ __forceinline__ void weight_tile_next(Acc& cur, Acc& nxt, const FusedParams& p, const Stream& st,
                                                 const uint32_t* ops, uint32_t& mc, float* sC, uint64_t* cfull,
                                                 uint64_t* cempty, uint32_t& cc, int t) {
  mma_kblocks(nxt, p, st, ops, 0, 1, true, mc, t);
  store_weights(cur, sC, cfull, cempty, cc, t);
  mma_kblocks(nxt, p, st, ops, 1, p.n_kb, true, mc, t);
}

// ---- A0' image of edge tile mt, built by all threads: [hi | lo | 1 1 0..] of [edge_attr (+ per-graph term) | node[tgt,:ns] |
// node[src,:ns]]
__device__ __forceinline__ void build_a0(const FusedParams& p, unsigned char* sA, long long mt, long long n_edges, int tid) {
  const long long e0 = mt * BM;
  const int Kin = p.K1, Kp = p.K1p;
  if (tid < BM) put_a_tail(sA, tid, Kin, Kp);
  if (p.a0_vec) {
    // vector path: four threads per edge row, each converting a contiguous quarter of the row's 8-column groups (<= 5
    // groups = 10 independent 16-byte loads).  The row's indices (attribute row, per-graph term, both end points) are
    // loaded once per thread, then ALL data loads of the thread are issued - including the per-graph term's - then the
    // conversions: two dependent global-memory round trips per tile.
    constexpr int TPR = THREADS / BM;
    const int groups = Kin >> 3, gh = (groups + TPR - 1) / TPR;
    constexpr int PER = (144 / 8 + TPR - 1) / TPR;      // Kp <= 144 (MAX_KB k-blocks)
    const int r = tid / TPR, g0 = (tid % TPR) * gh, g1 = min(groups, g0 + gh);
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
  } else {
    for (int idx = tid; idx < BM * Kin; idx += THREADS) {
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

__global__ void __launch_bounds__(THREADS, 1) fused_conv_kernel(const FusedParams p) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  unsigned char* sA = smem;                                      // MAX_KA x 8 KB
  unsigned char* sB = smem + (size_t)MAX_KA * A_KB_BYTES;        // ring of B stages
  float* sC = reinterpret_cast<float*>(sB + STAGES * STAGE_BYTES);    // [64][CLD] accumulator tile
  float* sY = sC + BM * CLD;                                     // [2][9][64] spherical harmonics per consumer thread
  float* sFlush = sY + 2 * 9 * BM;                               // [4 warps][48][33] scatter staging
  float* sMtab = sFlush + 4 * 48 * FLUSH_LD;                     // [MAX_PATHS][48]
  int* sTiles = reinterpret_cast<int*>(sMtab + MAX_PATHS * MTAB);   // [MAX_TILES][8]
  uint32_t* sOps = reinterpret_cast<uint32_t*>(sTiles + MAX_TILES * 8);   // [2][SCHED_WORDS] MMA schedules
  uint64_t* bars = reinterpret_cast<uint64_t*>(sOps + 2 * SCHED_WORDS);
  uint64_t* full = bars;                 // B stage s has landed (TMA complete_tx)
  uint64_t* cfull = bars + STAGES;       // C holds a weight tile (128 MMA threads arrive)
  uint64_t* cempty = cfull + 1;          // the consumers have drained C (128 consumer threads arrive)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int S1 = p.K1p >> 4, S2 = p.Hp >> 4;
  for (int i = tid; i < p.n_tiles * 8; i += THREADS) sTiles[i] = p.tiles[i];
  for (int i = tid; i < p.n_paths * MTAB; i += THREADS) sMtab[i] = p.mtab[i];
  if (tid == 32) build_ops(sOps, S1, gmma_desc_lo(smem_u32(sA)));
  if (tid == 64) build_ops(sOps + SCHED_WORDS, S2, gmma_desc_lo(smem_u32(sA)));
  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) mbar_init(&full[s], 1);
    mbar_init(cfull, 128);
    mbar_init(cempty, 128);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int n1 = ((p.H + 15) / 16) * 16;

  // the edge count may live on the device (neighbour lists built without a host round trip): p.n_edges is then its bound
  long long n_edges = p.n_edges;
  if (p.n_edges_dev) { const long long nd = __ldg(p.n_edges_dev); n_edges = nd < n_edges ? (nd < 0 ? 0 : nd) : n_edges; }
  const long long n_mtiles = (n_edges + BM - 1) / BM;
  const long long my_units = blockIdx.x < n_mtiles ? (n_mtiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  // debug clocks: a span is counted by subtracting its start from the counter and adding its end (modulo 2^64), so no start
  // value is held in registers through the kernel
  if (p.dbg && blockIdx.x == 0 && tid == 0) {      // effective SM clock of this launch: clock64 ticks per globaltimer ns
    unsigned long long g0;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g0));
    atomicAdd(p.dbg + 25, 0ull - (unsigned long long)clock64());
    atomicAdd(p.dbg + 26, 0ull - g0);
  }

  // Each warpgroup runs its own loop over the CTA's edge tiles, so that the state one of them carries from tile to tile is
  // not held in registers through the other's work (together they would not fit in 255 registers).  Both loops meet at
  // the same two block-wide barriers per edge tile, around the A0' image that all threads build.
  if (__shfl_sync(0xffffffffu, tid >> 7, 0) == 0) {     // warp-uniform for the compiler
    Stream st;
    st.sB = sB; st.full = full; st.tiles = sTiles; st.n1 = n1;
    st.per_unit = p.n_kb1 + p.n_tiles * p.n_kb;
    st.len = (uint32_t)(my_units * st.per_unit);
    // the ring runs ahead across edge tiles: the next tile's W1' blocks are requested while this one is contracted
    if (tid == 0)
      for (int i = 0; i < STAGES; ++i) st.issue(p, (uint32_t)i);
    uint32_t mc = 0, cc = 0;
    for (long long mt = blockIdx.x; mt < n_mtiles; mt += gridDim.x) {
      __syncthreads();
      if (p.dbg && tid == 0) atomicAdd(p.dbg + 11, 0ull - (unsigned long long)clock64());
      build_a0(p, sA, mt, n_edges, tid);
      __syncthreads();
      // ===== MMA warpgroup: hidden layer, then every N tile.  Every product is issued MAX_N wide: the stage rows past a
      // tile's width hold stale data whose columns are never read, and one width keeps both accumulator sets in
      // registers.  The tile loop is unrolled by two so that the set each tile uses is known at compile time.
      Acc d0, d1;
      const uint32_t* ops2 = sOps + SCHED_WORDS;
      mma_kblocks(d0, p, st, sOps, 0, p.n_kb1, false, mc, tid);
      mma_drain(p, st, mc, tid);
      wgmma_fence_regs(d0);
      store_hidden(d0, p, sA, tid);
      mma_kblocks(d0, p, st, ops2, 0, p.n_kb, false, mc, tid);
      for (int tile = 0;; tile += 2) {     // the last tile drains the pipe on the path that leaves the loop
        if (tile + 1 >= p.n_tiles) {
          mma_drain(p, st, mc, tid);
          store_weights(d0, sC, cfull, cempty, cc, tid);
          break;
        }
        weight_tile_next(d0, d1, p, st, ops2, mc, sC, cfull, cempty, cc, tid);
        if (tile + 2 >= p.n_tiles) {
          mma_drain(p, st, mc, tid);
          store_weights(d1, sC, cfull, cempty, cc, tid);
          break;
        }
        weight_tile_next(d1, d0, p, st, ops2, mc, sC, cfull, cempty, cc, tid);
      }
      if (p.dbg && tid == 0) { atomicAdd(p.dbg + 11, (unsigned long long)clock64()); atomicAdd(p.dbg + 12, 1ull); }
    }
  } else {
    uint32_t cc_con = 0;
    for (long long mt = blockIdx.x; mt < n_mtiles; mt += gridDim.x) {
      __syncthreads();
      build_a0(p, sA, mt, n_edges, tid);
      __syncthreads();
      // ===== consumers: two threads per edge (warps q and q ^ 2), each contracting alternate 32-column chunks ========
      const int q = warp & 3, half = q >> 1, ct = (q & 1) * 32 + lane;     // ct = row of the edge tile
      const long long e = mt * BM + ct;
      const bool valid = e < n_edges;
      const int src_e = valid ? __ldg(p.src + e) : 0, dst_e = valid ? __ldg(p.tgt + e) : -1;
      const long long er = (valid && p.perm) ? (long long)__ldg(p.perm + e) : e;
      const float ew_e = (valid && p.ew) ? __ldg(p.ew + er) : 1.f;
      // runs of equal scatter targets inside the warp (rows past the end form their own, never flushed, runs)
      const int key_up = __shfl_up_sync(0xffffffffu, dst_e, 1);
      const uint32_t head_mask = __ballot_sync(0xffffffffu, lane == 0 || key_up != dst_e || !valid);
      float* sF = sFlush + q * 48 * FLUSH_LD;
      const float* sFp = sFlush + (q ^ 2) * 48 * FLUSH_LD;     // the partner warp's partial sums
      float* sYh = sY + half * 9 * BM;
      {   // real spherical harmonics of the edge vector, component normalisation (e3nn polynomials)
        float vx = valid ? p.vec_sign * __ldg(p.vec + 3 * er) : 1.f, vy = valid ? p.vec_sign * __ldg(p.vec + 3 * er + 1) : 0.f,
              vz = valid ? p.vec_sign * __ldg(p.vec + 3 * er + 2) : 0.f;
        const float nrm = fmaxf(sqrtf(vx * vx + vy * vy + vz * vz), 1e-12f);
        vx /= nrm; vy /= nrm; vz /= nrm;
        const float s3 = 1.7320508075688772f, s5 = 2.23606797749979f, s15 = 3.872983346207417f;
        sYh[0 * BM + ct] = 1.f;
        sYh[1 * BM + ct] = s3 * vx; sYh[2 * BM + ct] = s3 * vy; sYh[3 * BM + ct] = s3 * vz;
        sYh[4 * BM + ct] = s15 * vx * vz;
        sYh[5 * BM + ct] = s15 * vx * vy;
        sYh[6 * BM + ct] = s5 * (vy * vy - 0.5f * (vx * vx + vz * vz));
        sYh[7 * BM + ct] = s15 * vy * vz;
        sYh[8 * BM + ct] = 0.5f * s15 * (vz * vz - vx * vx);
      }
      const float* xrow = p.x + (long long)src_e * p.ld_x;
      const float* crow = sC + ct * CLD;
      float acc[48], xn[XN], M[9];
      prefetch_x(xrow + sTiles[2], sTiles[3] * sTiles[4], p.x_vec2, xn);
      for (int t = 0; t < p.n_tiles; ++t, ++cc_con) {
        const int* ti = sTiles + t * 8;
        const int kind = ti[0], d_in = ti[4], out_off = ti[5], flags = ti[6];
        const int tn = (t + 1 < p.n_tiles) ? t + 1 : t;          // next tile (the last one requests nothing)
        const float* xnext = xrow + sTiles[tn * 8 + 2];
        const int cnt_next = (t + 1 < p.n_tiles) ? sTiles[tn * 8 + 3] * sTiles[tn * 8 + 4] : 0;
        if (flags & 1) {
#pragma unroll
          for (int i = 0; i < 48; ++i) acc[i] = 0.f;
        }
        // M[i,k] = edge_weight * sum_j coef*C[i,j,k] * Y[sh_off + j]  (at most 3x3 for the supported paths; row-major,
        // stride 3), rebuilt only when the tile belongs to another path than its predecessor: dense table, fully unrolled
        if (flags & 4) {
          const float* T = sMtab + ti[7] * MTAB;
          const int sh_off = (flags >> 8) & 0xff;
          float yb[5];
#pragma unroll
          for (int j = 0; j < 5; ++j) yb[j] = sYh[min(sh_off + j, 8) * BM + ct];
#pragma unroll
          for (int ik = 0; ik < 9; ++ik) {
            float a = 0.f;
#pragma unroll
            for (int j = 0; j < 5; ++j) a = fmaf(T[ik * 5 + j], yb[j], a);
            M[ik] = a * ew_e;
          }
        }
        const uint32_t par = cc_con & 1;
        const int nch = ti[1] >> 5;
        switch (kind) {
          case 0: tile_body<48, 1, 4>(crow, nch, half, xn, d_in, M, acc, cfull, par); break;
          case 1: tile_body<10, 3, 16>(crow, nch, half, xn, d_in, M, acc, cfull, par); break;
          case 2: tile_body<16, 1, 8>(crow, nch, half, xn, d_in, M, acc, cfull, par); break;
          default: tile_body<4, 3, 16>(crow, nch, half, xn, d_in, M, acc, cfull, par); break;
        }
        mbar_arrive(cempty);
        // the next tile's node values are requested only now, so that they are not held in registers through the
        // contraction; their latency overlaps the scatter and the wait for the next accumulator tile
        prefetch_x(xnext, cnt_next, p.x_vec2, xn);
        if (flags & 2) {
          // end of an output irrep: scatter-add.  Both warps of the pair stage their 32 x nacc partial results in shared
          // memory (padded rows: conflict-free both ways); lane i of warp `half` then walks the 32 edges adding the two
          // partial sums, sums runs of equal targets (CSR order makes them contiguous; unsorted input just yields runs of
          // length one) and issues ONE fully coalesced RED.ADD per run for output value 32 half + i.
          const int nacc = (kind == 0) ? 48 : (kind == 1 ? 30 : (kind == 2 ? 16 : 12));
#pragma unroll
          for (int i = 0; i < 48; ++i)
            if (i < nacc) sF[i * FLUSH_LD + lane] = acc[i];
          named_bar(BAR_PAIR + (q & 1), 64);
          const int i = 32 * half + lane;
          if (32 * half < nacc) {
            const bool act = i < nacc;
            const float* col = sF + (act ? i : 0) * FLUSH_LD;
            const float* colp = sFp + (act ? i : 0) * FLUSH_LD;
            float s = 0.f;
#pragma unroll
            for (int le = 0; le < 32; ++le) {
              s += col[le] + colp[le];
              if (le == 31 || ((head_mask >> (le + 1)) & 1)) {          // warp-uniform: last edge of a run
                const int d = __shfl_sync(0xffffffffu, dst_e, le);
                if (d >= 0 && act) atomicAdd(p.sum + (long long)d * p.d_out + out_off + i, s);
                s = 0.f;
              }
            }
          }
          named_bar(BAR_PAIR + (q & 1), 64);
        }
      }
      if (p.cnt && half == 0) {       // edge counts per target: one atomic per run, issued by the run's first lane
        const bool head = (head_mask >> lane) & 1;
        const uint32_t above = (lane == 31) ? 0u : (head_mask >> (lane + 1));
        const int run_len = above ? __ffs(above) : 32 - lane;
        if (head && valid) atomicAdd(p.cnt + dst_e, (float)run_len);
      }
    }
  }
  if (p.dbg && blockIdx.x == 0 && tid == 0) {
    unsigned long long g1;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g1));
    atomicAdd(p.dbg + 25, (unsigned long long)clock64());
    atomicAdd(p.dbg + 26, g1);
  }
}

// per-device state: debug counters and the one-time opt-in to > 48 KB of dynamic shared memory
constexpr int MAX_DEVICES = 64;
struct DeviceState {
  bool attr_done = false;
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
// clears them.  [11] clocks spent per edge tile (summed over tiles), [12] edge tiles, [25] / [26] clock64 ticks / ns of
// CTA 0 over the launch.  Synchronises the device.
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

extern "C" int ddb200_fused_conv(const ddb200_fused_args* a, void* stream) {
  if (!a || !a->edge_attr || !a->w1_images || !a->w2_images || !a->tiles || !a->mtab || !a->x || !a->edge_vec || !a->sum ||
      !a->tgt || !a->src || a->n_edges < 0 || a->ne <= 0 || a->ns < 0 || a->hidden <= 0 || a->n_tiles <= 0 || a->d_out <= 0)
    return DDB200_EINVAL;
  if (a->ns > 0 && (!a->node || a->ld_node < a->ns)) return DDB200_EINVAL;
  if (a->n_tiles > MAX_TILES || a->n_paths <= 0 || a->n_paths > MAX_PATHS || a->sh_lmax < 0 || a->sh_lmax > 2)
    return DDB200_EINVAL;
  if ((a->ea_add == nullptr) != (a->ea_add_idx == nullptr)) return DDB200_EINVAL;
  const int K1 = a->ne + 2 * a->ns, H = a->hidden;
  const int K1p = (K1 + 15) / 16 * 16, Hp = (H + 15) / 16 * 16;
  const int n_kb = (2 * Hp + 16 + BK - 1) / BK, n_kb1 = (2 * K1p + 16 + BK - 1) / BK;
  if (n_kb > MAX_KB || n_kb1 > MAX_KB || H > MAX_N) return DDB200_EINVAL;
  if ((reinterpret_cast<uintptr_t>(a->w1_images) & 127) || (reinterpret_cast<uintptr_t>(a->w2_images) & 127)) return DDB200_EINVAL;
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
  p.mtab = a->mtab; p.n_paths = a->n_paths;
  p.x = a->x; p.ld_x = a->ld_x; p.x_vec2 = (a->x_pairs_ok && (a->ld_x & 1) == 0 && (reinterpret_cast<uintptr_t>(a->x) & 7) == 0) ? 1 : 0;
  p.vec = a->edge_vec; p.ew = a->edge_weight; p.lmax = a->sh_lmax; p.sum = a->sum; p.d_out = a->d_out; p.cnt = a->cnt;
  p.n_edges = a->n_edges; p.n_edges_dev = a->n_edges_dev;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= MAX_DEVICES) return DDB200_EINVAL;
  p.dbg = fused_debug_buffer(dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const long long n_mtiles = (a->n_edges + BM - 1) / BM;
  const size_t fixed = (BM * CLD + 2 * 9 * BM + 4 * 48 * FLUSH_LD + MAX_PATHS * MTAB) * 4 + MAX_TILES * 8 * 4 +
                       2 * SCHED_WORDS * 4 + (STAGES + 2) * sizeof(uint64_t) + 1024;
  const size_t smem = (size_t)MAX_KA * A_KB_BYTES + (size_t)STAGES * STAGE_BYTES + fixed;
  if (smem > 227 * 1024) return DDB200_ESMEM;
  if (!g_dev[dev].attr_done) {      // the opt-in is a per-device attribute
    const cudaError_t e = cudaFuncSetAttribute(fused_conv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    g_dev[dev].attr_done = true;
  }
  const unsigned grid = (unsigned)(n_mtiles < sms ? n_mtiles : sms);
  fused_conv_kernel<<<grid, THREADS, smem, (cudaStream_t)stream>>>(p);
  return (int)cudaGetLastError();
}
