/* diffdock_b200: deterministic (fixed-point) convolutions - C ABI.
 *
 * What diffdock_b200 runs under torch.use_deterministic_algorithms(True).  The convolutions of include/diffdock_b200.h
 * add fp32 messages into shared accumulators with float reductions, whose order (and so whose last bits) varies from run
 * to run.  These entry points convert every edge's message value to 64-bit fixed point (units of 2^-32) and add
 * integers, so a sum is the same whatever order its terms arrive in.  Same library, same conventions (return codes,
 * device pointers, stream) as include/diffdock_b200.h; their ctypes signatures are diffdock_b200/_lib.py:FIXED_SIGNATURES.
 */
#ifndef DIFFDOCK_B200_FIXED_H
#define DIFFDOCK_B200_FIXED_H

#include "diffdock_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---------------------------------------------------------------------------------------------------------------
 * Deterministic accumulate phase: as ddb200_tpconv_accumulate, but every edge's output values are converted on their
 * own to 64-bit fixed point,
 *   q = round_to_nearest_even(v * 2^32)      (v the edge's fp32 message value)
 * and sum [n_dst, D_out] int64 receives the integer sums.  Integer addition is associative, so the sums do not depend on
 * the edge order, on how the edges are split over launches, or on which kernel (this one or ddb200_fused_conv_fixed)
 * added them.  A value with |v| >= 2^31 (or not finite) saturates to +-(2^63 - 1) and sets bit 0 of the sticky error
 * word *err (int32, device; never cleared here).  Sums must stay below 2^31 in magnitude.  D_out <= 256.
 * cnt as for ddb200_tpconv_accumulate (fp32 edge counts, exact below 2^24).  Follow with ddb200_tpconv_finalize_fixed.
 * ------------------------------------------------------------------------------------------------------------- */
int ddb200_tpconv_accumulate_fixed(const ddb200_tp_table* t, const float* x, int64_t x_stride, const int32_t* edge_src,
                                   const int32_t* edge_dst, const float* geo, const float* edge_weight, const float* w,
                                   int64_t w_stride, int64_t n_edges, int64_t* sum, float* cnt, int32_t* err,
                                   void* stream);

/* Epilogue over fixed-point sums: as ddb200_tpconv_finalize with
 *   mean = (double)sum[n, c] * 2^-32 / max(cnt[n], eps)   (no mean: (double)sum[n, c] * 2^-32), rounded once to fp32,
 * then BatchNorm and the residual in fp32 exactly as ddb200_tpconv_finalize applies them. */
int ddb200_tpconv_finalize_fixed(const int64_t* sum, const float* cnt, int64_t n_rows, int d_out, int mean,
                                 const float* bn_scale, const float* bn_shift, const float* residual,
                                 int64_t res_stride, int res_dim, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Deterministic fused convolution: ddb200_fused_conv / ddb200_fused_conv_so with the same MMAs, staging and
 * contraction; the scatter converts each edge's output value to 64-bit fixed point (round_to_nearest_even(v * 2^32)), sums a run of equal targets as integers and adds it to
 * sum_fx [n_dst, d_out] int64 with one 64-bit integer reduction (args->sum is not used).  Saturation, the error word and
 * the range are those of ddb200_tpconv_accumulate_fixed, whose sums these can share.  Follow with
 * ddb200_tpconv_finalize_fixed.
 * ------------------------------------------------------------------------------------------------------------- */
int ddb200_fused_conv_fixed(const ddb200_fused_args* args, int64_t* sum_fx, int32_t* err, void* stream);
int ddb200_fused_conv_so_fixed(const ddb200_fused_args* args, int64_t* sum_fx, int32_t* err, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* DIFFDOCK_B200_FIXED_H */
