// Rotation arithmetic shared by the two one-sided Jacobi kernels (wct.cu: k_jacobi<C>, jacobi_s.cu: k_jacobi_s).
#pragma once
#include "common.cuh"

namespace wctb {

// ---- register-blocked pair rotation: operands live in registers as PACKED fp32 pairs
// (as fp32 pairs), column norms are cached ----
// single-MUFU approximations (the CUDA intrinsics wrap these in range/denormal fix-ups: measured 25 FMUL +
// 12 FSETP + 7 MUFU per rotation in the SASS of the previous version)
__device__ __forceinline__ float rsqrt_ap(float x) {
    float y;
    asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float rcp_ap(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// Rotation parameters of one Hestenes step from g = x.y, a = |x|^2, b = |y|^2.
//   * convergence test without a division:  |g| > tol*sqrt(ab)  <=>  g^2 > tol^2 * ab ; `flag` collects
//     1 (some pair above tol: a further sweep is needed to VERIFY) and 2 (some pair above tol_q, the level
//     from which one more quadratically convergent sweep cannot be trusted to land below tol);
//   * t = tan(theta) = sgn(d) 2g / (|d| + sqrt(d^2 + 4g^2)),  d = b - a  (no zeta = d/2g, so nothing overflows
//     for tiny g).  Approximate MUFU arithmetic is fine for t: ANY t gives an exact rotation as long as (c,s)
//     is orthonormal, an inexact t only leaves a residual for the next sweep;
//   * (c,s): r = h^-1/2 refined by one Newton step, s = t r, and c is applied as 1 + cm1 with
//     cm1 = -s^2/(1+r), so that small angles neither shrink nor grow the columns (no eigenvalue bias).
//   * a pair whose columns are BOTH at the rounding-noise floor (|col|^2 < null2 of the previous sweep, k_jacobi:
//     |col| < min(3.16e-6 max|col|, max(thresh / 2, 16 * 2^-24 max|col|))) is left alone and not counted: such columns
//     span the null space of a rank-deficient map, their mutual cosines are O(1) noise that never converges (26 sweeps
//     instead of 13 on a rank-299 512x512 matrix), and their directions inside the null space do not matter.  What the
//     floor guarantees: a kept column (|col| ~ lambda > thresh) is live whenever lambda > 16 * 2^-24 lambda_max, i.e.
//     wherever fp32 determines its direction; the noise columns (~7 * 2^-24 lambda_max) are not.  Pairs of a noise
//     column with a live column are still rotated: that is what keeps the noise columns' Rayleigh quotients
//     second-order small.
__device__ __forceinline__ void rot_scalars(float g, float a, float b, float tol2, float tolq2, float null2, float& flag,
                                            float& t, float& s, float& cm1) {
    const float ab = a * b, gg = g * g;
    const bool live = fmaxf(a, b) > null2;
    const bool rot = live && gg > tol2 * ab;
    flag = fmaxf(flag, (live && gg > tolq2 * ab) ? 2.f : (rot ? 1.f : 0.f));
    const float d = b - a, g2 = g + g;
    const float w2 = fmaf(d, d, g2 * g2);
    const float w = w2 * rsqrt_ap(w2);
    float tt = (d < 0.f ? -g2 : g2) * rcp_ap(fabsf(d) + w);
    tt = rot ? tt : 0.f;                                   // (select, not arithmetic: discards the NaN of d = g = 0)
    const float h = fmaf(tt, tt, 1.f);
    float r = rsqrt_ap(h);
    r = r * fmaf(-0.5f * h, r * r, 1.5f);
    t = tt;
    s = tt * r;
    cm1 = -(s * s) * rcp_ap(1.f + r);
}


}  // namespace wctb
