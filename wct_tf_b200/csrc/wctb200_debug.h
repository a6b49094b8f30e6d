/* Tuning / probe hooks of libwctb200 -- PRIVATE: used by tools/ and tests/ only, not part of the stable C-ABI
 * (include/wctb200.h).  They set process-global knobs and are not thread-safe. */
#ifndef WCTB200_DEBUG_H
#define WCTB200_DEBUG_H
#include "../../include/wctb200.h"
#ifdef __cplusplus
extern "C" {
#endif
/* force the conv output-channel tile (64/128; 256 runs as 128; 0 = built-in heuristic) */
WCTB200_API int wctb200_debug_set_conv_bn(int bn);
/* CTAs per SM in the persistent conv grid (default 4; 1 = exactly one CTA per SM) */
WCTB200_API int wctb200_debug_set_conv_oversub(int k);
/* fuse the a_hi*b_hi and a_hi*b_lo products into one N = 2*tile MMA at the 64-wide tile: -1 / 1 on (default), 0 off */
WCTB200_API int wctb200_debug_set_conv_fuse(int mode);
/* Jacobi cross-phase schedule: 2^lg_groups warp groups (0..4) started stagger_cycles apart; negative = per-size default */
WCTB200_API int wctb200_debug_set_jacobi(int lg_groups, int stagger_cycles);
/* Jacobi: largest pair cosine of a sweep below which no verification sweep follows (default 1e-4) */
WCTB200_API int wctb200_debug_set_jacobi_tolq(float tolq);
/* covariance kernel: cap on the depth of the tile ring (default 12 = 192 KB in flight at every stage size) */
WCTB200_API int wctb200_debug_set_cov_stages(int n);
/* EXPERIMENT (VERDICT r1 next #6): split-fp16 products per MAC in the encoder / decoder convs: 3 = a_hi b_hi + a_hi b_lo +
 * a_lo b_hi (default, fp32-class), 2 = without a_lo b_hi (activations effectively fp16), 1 = a_hi b_hi only.  Returns the
 * value now selected.  With the fused MMA (N = 2*tile) 2 and 1 cost the same: a_hi [b_hi|b_lo] is one instruction. */
WCTB200_API int wctb200_debug_set_conv_products(int n);
/* decoder tail (64 -> 3): 1 = transposed tensor-core product (conv_tail_tc.cu, default), 0 = SIMT kernels of layers.cu */
WCTB200_API int wctb200_debug_set_conv_tail_tc(int on);
/* whitening / colouring matrices: mode 1 (default) = coupled Newton-Schulz on the tensor cores where the threshold keeps
 * every eigenvalue (matfun_tc.cu), Jacobi eigensolver otherwise; mode 0 = always the eigensolver.  max_it: iteration budget
 * (0 = leave unchanged).  Returns the mode. */
WCTB200_API int wctb200_debug_set_matfun(int mode, int max_it);
/* the fast path alone: A [count][C][C] fp32 (device) -> out = A^-1/2 for the first n_first matrices, A^+1/2 for the rest;
 * ok[b] = 1 where the guard accepted the result (device int[count]); info (device float[count][4], may be null) receives
 * (iteration of convergence or -1, last residual max|I - ZY|, lower bound of lambda_min, ||A||_F) */
WCTB200_API int wctb200_debug_matfun(const float* A, int C, int count, int n_first, float thresh, float eps_eig, float* out, int* ok,
                                     float* info, void* stream);
/* encoder head (3 -> 64): 1 = tensor cores with an operand built in shared memory (conv_head_tc.cu, default), 0 = SIMT */
WCTB200_API int wctb200_debug_set_conv_head_tc(int on);
/* where wctb200_style_swap_prepare / _apply leave each stage's result, for reading back after the apply (no stage
 * overwrites another's).  out[11] = n_patches, cout_pad, ho, wo (the VALID score grid), then byte offsets
 *   into the state:           whitened style SPF16 [1,Hs,Ws,C] | fp32 1/||tap|| [P*P][C] | split-fp16 filters [2][cout_pad][P*P*C]
 *   into the apply workspace: whitened content SPF16 [Nc,Hc,Wc,C] | scores SPF16 [Nc,Hc,Wc,cout_pad] (the top-left anchored
 *                             correlation at every pixel) | int32 arg-max [Nc][ho][wo] | gathered feature SPF16 [Nc,Hc,Wc,C] */
WCTB200_API int wctb200_debug_style_swap_layout(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int patch, int stride,
                                                long long* out);
#ifdef __cplusplus
}
#endif
#endif
