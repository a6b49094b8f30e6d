// Whiten-colour transform (ops.py:24-140) and AdaIN (ops.py:282-294) for one relu level,
// batched over frames.
//
// Stage A  channel moments / covariance     HBM-bound streaming kernels (fp32 FFMA, fp64 combine)
// Stage B  C x C symmetric eigendecomposition: one-sided (Hestenes) Jacobi, one pair per warp,
//          columns staged in shared memory, a thread-block CLUSTER of C/64 CTAs per matrix
// Stage C  W_c = E_c D_c^-1/2 E_c^T, C_s = E_s D_s^1/2 E_s^T, T = C_s W_c, M = aT + (1-a)I, bias
// Stage D  out = M x + bias : the 1-tap mode of the wgmma conv kernel (conv_tc.cu) with a
//          per-frame weight set, so the apply GEMM runs on the tensor cores.
#include <cfloat>
#include <cmath>
#include <cooperative_groups.h>

#include "common.cuh"
#include "jacobi_common.cuh"

namespace cg = cooperative_groups;

namespace wctb {

// ---------------------------------------------------------------------------
// Stage A.1 (AdaIN): per-channel moments over the interior pixels, centred on the shift t of k_sample_shift (cov_tc.cu)
//   grid (slices, frames); 256 threads; thread = (row lane, 8-channel group).  A slice is moments_slice(C) pixels, up to
//   32 per thread: the split of a frame depends on C and H x W only, never on the batch, so neither does any rounding.
//   Each CTA writes sum (x - t) and sum (x - t)^2 of its slice to its OWN slot [frame][slice][2][C]; k_moments_finalize
//   adds the slots in a fixed order.  Centring first keeps the sum of squares free of cancellation: a channel with a large
//   mean and a small spread (a flat region of the frame) would lose its variance in sum x^2 / HW - mean^2.
// ---------------------------------------------------------------------------
static inline int moments_slice(int C) { return 32 * (256 / (C / 8)); }

__global__ void __launch_bounds__(256)
k_chan_moments(const __half* __restrict__ act, ActGeom g, const float* __restrict__ shift, int slice, float* __restrict__ part) {
    __shared__ float red[256 * 8];
    __shared__ float red2[256 * 8];
    const int cgs = g.C / 8;
    const int rows = 256 / cgs;                 // pixel rows handled per iteration (C <= 2048)
    const int grp = threadIdx.x % cgs;
    const int rl = threadIdx.x / cgs;
    const int n = blockIdx.y;
    const long long HW = (long long)g.H * g.W;
    const long long q0 = (long long)blockIdx.x * slice;
    const long long q1 = min(q0 + slice, HW);
    float s[8], s2[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { s[j] = 0.f; s2[j] = 0.f; }
    if (rl < rows) {
        float t[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) t[j] = shift[(long long)n * g.C + grp * 8 + j];
        for (long long q = q0 + rl; q < q1; q += rows) {
            const int y = (int)((unsigned)q / (unsigned)g.W), x = (int)((unsigned)q - (unsigned)y * (unsigned)g.W);
            float v[8];
            load8(act, g, ((long long)n * g.Hp + y + 1) * g.Wp + x + 1, grp * 8, v);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float d = v[j] - t[j];
                s[j] += d;
                s2[j] = fmaf(d, d, s2[j]);
            }
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        red[threadIdx.x * 8 + j] = s[j];
        red2[threadIdx.x * 8 + j] = s2[j];
    }
    __syncthreads();
    // thread t < C reduces channel t over the row lanes, in order
    float* slot = part + ((long long)n * gridDim.x + blockIdx.x) * 2 * g.C;
    for (int c = threadIdx.x; c < g.C; c += 256) {
        const int gq = c / 8, j = c % 8;
        float a = 0.f, a2 = 0.f;
        for (int r = 0; r < rows; ++r) {
            a += red[(r * cgs + gq) * 8 + j];
            a2 += red2[(r * cgs + gq) * 8 + j];
        }
        slot[c] = a;
        slot[g.C + c] = a2;
    }
}

// mean = t + s / HW, var = S / HW - (s / HW)^2 (biased, tf.nn.moments) with s, S the slot sums of k_chan_moments added in
// slot order in fp64
// (shared with the statistics record of a rectangle, k_moments_record / k_record_moments_finalize)
__device__ __forceinline__ void moments_slot_sums(const float* __restrict__ p, int C, int nslices, double& s, double& S) {
    s = 0.0;
    S = 0.0;
#pragma unroll 8
    for (int b = 0; b < nslices; ++b) {
        s += (double)p[(long long)b * 2 * C];
        S += (double)p[(long long)b * 2 * C + C];
    }
}
__device__ __forceinline__ void moments_from_sums(float shift, double s, double S, long long HW, float& mean, float& var) {
    const double m = s / (double)HW;
    mean = (float)((double)shift + m);
    var = (float)fmax(S / (double)HW - m * m, 0.0);
}
__global__ void k_moments_finalize(const float* __restrict__ part, const float* __restrict__ shift, int C, int nslices, long long HW,
                                   int total, float* __restrict__ mean, float* __restrict__ var) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int n = i / C, c = i - n * C;
    double s, S;
    moments_slot_sums(part + (long long)n * nslices * 2 * C + c, C, nslices, s, S);
    moments_from_sums(shift[i], s, S, HW, mean[i], var[i]);
}
// the slots of k_chan_moments -> a statistics record with the diagonal S (layout: stats_record_layout)
__global__ void k_moments_record(const float* __restrict__ part, const float* __restrict__ shift, int C, int nslices, long long HW,
                                 int total, StatsRecord rec) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int n = i / C, c = i - n * C;
    moments_slot_sums(part + (long long)n * nslices * 2 * C + c, C, nslices, rec.s[i], rec.S[i]);
    rec.t[i] = (double)shift[i];
    if (c == 0) rec.n[n] = (double)HW;
}
__global__ void k_record_moments_finalize(StatsRecord rec, int C, int total, float* __restrict__ mean, float* __restrict__ var) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    moments_from_sums((float)rec.t[i], rec.s[i], rec.S[i], (long long)rec.n[i / C], mean[i], var[i]);
}

// Accumulate record B into record A (tiled stylisation): B's sums are re-centred on A's shift in fp64,
//   s_B' = s_B + n_B D,  S_B' = S_B + (D s_B^T + s_B D^T) + n_B D D^T,  D = t_B - t_A,
// and added to A's.  A record with n = 0 takes B as it is (one accumulate into an empty record is the identity).  Two
// launches: the S entries read n_A, t_A and s_B before k_record_fold_vec changes A's n, t and s (one block per frame).
// Explicitly rounded products: no contraction, so entry (i, j) and (j, i) are the same bits.
__global__ void k_record_fold_S(StatsRecord a, StatsRecord b, int C, int N, int diag) {
    const long long per = diag ? (long long)C : (long long)C * C;
    const long long total = (long long)N * per;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const long long n = t / per;
        const int i = diag ? (int)(t - n * per) : (int)((t - n * per) / C);
        const int j = diag ? i : (int)((t - n * per) % C);
        if (a.n[n] == 0.0) {
            a.S[t] = b.S[t];
            continue;
        }
        const double di = __dsub_rn(b.t[n * C + i], a.t[n * C + i]), dj = __dsub_rn(b.t[n * C + j], a.t[n * C + j]);
        const double cross = __dadd_rn(__dmul_rn(di, b.s[n * C + j]), __dmul_rn(b.s[n * C + i], dj));
        const double sb = __dadd_rn(__dadd_rn(b.S[t], cross), __dmul_rn(b.n[n], __dmul_rn(di, dj)));
        a.S[t] = __dadd_rn(a.S[t], sb);
    }
}
__global__ void __launch_bounds__(256) k_record_fold_vec(StatsRecord a, StatsRecord b, int C) {
    const int n = blockIdx.x;
    const bool empty = a.n[n] == 0.0;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const long long i = (long long)n * C + c;
        if (empty) {
            a.s[i] = b.s[i];
            a.t[i] = b.t[i];
        } else {
            const double d = __dsub_rn(b.t[i], a.t[i]);
            a.s[i] = __dadd_rn(a.s[i], __dadd_rn(b.s[i], __dmul_rn(b.n[n], d)));
        }
    }
    __syncthreads();                            // every thread has read a.n[n]
    if (threadIdx.x == 0) a.n[n] = __dadd_rn(a.n[n], b.n[n]);
}

// ---------------------------------------------------------------------------
// Stage B: one-sided Jacobi.  Matrix n x n (n = 64*P), columns contiguous
//   (symmetric input, so row-major == column-major).  A cluster of P CTAs owns one
//   matrix; the 2P column blocks (32 columns each) are paired by a round-robin
//   tournament; a CTA stages its two blocks in shared memory, orthogonalises
//   all 32x32 cross pairs (one pair per warp, 32 warps), writes them back, and
//   the cluster barriers.  On convergence column i = sigma_i * u_i.
// ---------------------------------------------------------------------------
template <int NN>
struct JacobiCfg {
    static constexpr int P = NN / 64;
    static constexpr int VEC = NN >= 128 ? 4 : 2;        // floats per lane per load
    static constexpr int NV = NN / (32 * VEC);           // vector loads per lane per column
    static constexpr int SMEM_BYTES = 64 * NN * 4 + 64;
};

// Two INDEPENDENT rotations (x0,y0) and (x1,y1) fused and branch-free so their long
// dependency chains (dot -> 5-step shuffle reduction -> MUFU chain -> rotation) interleave:
// the kernel is latency bound (ncu: 38 % issue utilisation with 16 warps per SM).
template <int HP>
__device__ __forceinline__ void rot_regs2(f32x2 (&x0)[HP], f32x2 (&y0)[HP], float& a0, float& b0, f32x2 (&x1)[HP],
                                          f32x2 (&y1)[HP], float& a1, float& b1, float tol2, float tolq2, float null2,
                                          float& flag) {
    f32x2 d00 = pack2(0.f, 0.f), d01 = d00, d10 = d00, d11 = d00;
#pragma unroll
    for (int i = 0; i < HP; ++i) {
        if (i & 1) { d01 = fma2(x0[i], y0[i], d01); d11 = fma2(x1[i], y1[i], d11); }
        else { d00 = fma2(x0[i], y0[i], d00); d10 = fma2(x1[i], y1[i], d10); }
    }
    float p0, p1, p2, p3, q0, q1, q2, q3;
    unpack2(d00, p0, p1); unpack2(d01, p2, p3);
    unpack2(d10, q0, q1); unpack2(d11, q2, q3);
    float g0 = (p0 + p1) + (p2 + p3);
    float g1 = (q0 + q1) + (q2 + q3);
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
        g0 += __shfl_xor_sync(0xffffffffu, g0, o);
        g1 += __shfl_xor_sync(0xffffffffu, g1, o);
    }
    float t0, s0, c0, t1, s1, c1;
    rot_scalars(g0, a0, b0, tol2, tolq2, null2, flag, t0, s0, c0);
    rot_scalars(g1, a1, b1, tol2, tolq2, null2, flag, t1, s1, c1);
    if (t0 != 0.f || t1 != 0.f) {          // warp-uniform: skip the FMAs only when BOTH pairs are already orthogonal
        const f32x2 s20 = pack2(s0, s0), ns20 = pack2(-s0, -s0), c20 = pack2(c0, c0);
        const f32x2 s21 = pack2(s1, s1), ns21 = pack2(-s1, -s1), c21 = pack2(c1, c1);
#pragma unroll
        for (int i = 0; i < HP; ++i) {
            const f32x2 xa = x0[i], ya = y0[i], xb = x1[i], yb = y1[i];
            x0[i] = fma2(c20, xa, fma2(ns20, ya, xa));       // x' = x + cm1*x - s*y
            y0[i] = fma2(c20, ya, fma2(s20, xa, ya));        // y' = y + cm1*y + s*x
            x1[i] = fma2(c21, xb, fma2(ns21, yb, xb));
            y1[i] = fma2(c21, yb, fma2(s21, xb, yb));
        }
        a0 = fmaxf(fmaf(-t0, g0, a0), 0.f); b0 = fmaxf(fmaf(t0, g0, b0), 0.f);   // |x'|^2 = |x|^2 - t g , |y'|^2 = |y|^2 + t g
        a1 = fmaxf(fmaf(-t1, g1, a1), 0.f); b1 = fmaxf(fmaf(t1, g1, b1), 0.f);
    }
}

template <int NN>
__device__ __forceinline__ void load_col(const float* __restrict__ c, int lane, f32x2 (&r)[NN / 64]) {
    using Cfg = JacobiCfg<NN>;
#pragma unroll
    for (int v = 0; v < Cfg::NV; ++v) {
        const int off = (v * 32 + lane) * Cfg::VEC;
        if (Cfg::VEC == 4) {
            const f32x2x2 a = *reinterpret_cast<const f32x2x2*>(c + off);
            r[v * 2] = a.x;
            r[v * 2 + 1] = a.y;
        } else {
            r[v] = *reinterpret_cast<const f32x2*>(c + off);
        }
    }
}
template <int NN>
__device__ __forceinline__ void store_col(float* __restrict__ c, int lane, const f32x2 (&r)[NN / 64]) {
    using Cfg = JacobiCfg<NN>;
#pragma unroll
    for (int v = 0; v < Cfg::NV; ++v) {
        const int off = (v * 32 + lane) * Cfg::VEC;
        if (Cfg::VEC == 4) *reinterpret_cast<f32x2x2*>(c + off) = f32x2x2{r[v * 2], r[v * 2 + 1]};
        else *reinterpret_cast<f32x2*>(c + off) = r[v];
    }
}

__device__ __forceinline__ void group_bar(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// All pairs between the two columns x0,x1 held in REGISTERS by this warp (cached squared norms a0,a1) and the
// `npairs` column pairs of the shared-memory sub-block starting at bot0: npairs steps x 4 rotations.  Each bottom
// pair is loaded/stored once per 4 rotations, column norms are cached in nrm[] and updated analytically, so a
// rotation costs one dot product instead of three.  The `npairs` warps that share the sub-block form a ring
// (warp wsub starts at pair wsub) and synchronise on their own named barrier `bar` (32*npairs threads): groups
// working on disjoint sub-blocks run out of phase, so one group's FMA bursts fill the other's latency chains.
template <int NN>
__device__ __forceinline__ void ring_steps(float* cols, float* nrm, f32x2 (&x0)[NN / 64], f32x2 (&x1)[NN / 64], float& a0,
                                           float& a1, int bot0, int npairs, int wsub, int bar, int lane, float tol2,
                                           float tolq2, float null2, float& flag) {
    constexpr int HP = NN / 64;
    for (int s = 0; s < npairs; ++s) {
        const int j = bot0 + 2 * ((wsub + s) & (npairs - 1));
        float* cy0 = cols + j * NN;
        float* cy1 = cy0 + NN;
        f32x2 y0[HP], y1[HP];
        load_col<NN>(cy0, lane, y0);
        load_col<NN>(cy1, lane, y1);
        float b0 = nrm[j], b1 = nrm[j + 1];
        rot_regs2<HP>(x0, y0, a0, b0, x1, y1, a1, b1, tol2, tolq2, null2, flag);
        rot_regs2<HP>(x0, y1, a0, b1, x1, y0, a1, b0, tol2, tolq2, null2, flag);
        store_col<NN>(cy0, lane, y0);
        store_col<NN>(cy1, lane, y1);
        if (lane == 0) { nrm[j] = b0; nrm[j + 1] = b1; }
        if (npairs > 1) group_bar(bar, 32 * npairs);
        else __syncwarp();
    }
}

// tops (top, top+1) from shared memory, one ring pass, tops back to shared memory (the pairs INSIDE a block)
template <int NN>
__device__ __forceinline__ void cross_steps(float* cols, float* nrm, int top, int bot0, int npairs, int wsub, int bar,
                                            int lane, float tol2, float tolq2, float null2, float& flag) {
    constexpr int HP = NN / 64;
    f32x2 x0[HP], x1[HP];
    load_col<NN>(cols + top * NN, lane, x0);
    load_col<NN>(cols + (top + 1) * NN, lane, x1);
    float a0 = nrm[top], a1 = nrm[top + 1];
    ring_steps<NN>(cols, nrm, x0, x1, a0, a1, bot0, npairs, wsub, bar, lane, tol2, tolq2, null2, flag);
    store_col<NN>(cols + top * NN, lane, x0);
    store_col<NN>(cols + (top + 1) * NN, lane, x1);
    if (lane == 0) { nrm[top] = a0; nrm[top + 1] = a1; }
}

// 512 threads = 16 warps, 64 columns (a "top" and a "bottom" block of 32) in shared memory.
//   every round : the 32x32 cross pairs: warp w keeps top columns 2w,2w+1 in registers; the warps split into
//                 2^lg groups, group g walks bottom sub-block g^h in sub-round h (ring of 16>>lg warps on a named
//                 barrier), groups start `stagger` cycles apart so that they stay out of phase;
//   round 0     : additionally the pairs INSIDE both blocks, by recursive halving with the same register-blocked
//                 step (16|16 -> 8|8 -> 4|4 -> 2|2 -> 1|1 : 8+4+2+1+1 steps instead of 62 one-pair-per-warp steps).
__device__ float g_jacobi_tolq = 1e-4f;   // predicted-convergence level (see k_jacobi); device global so a probe can vary it

template <int NN>
__global__ void __launch_bounds__(512, 1)
k_jacobi(float* __restrict__ Gall, float* __restrict__ conv_ws, int* __restrict__ sweeps_out, int max_sweeps, float tol,
         int lg, int stagger, const int* __restrict__ skip, float thresh) {
    if (skip && skip[blockIdx.y]) {          // matrix handled by the matrix-function fast path (matfun_tc.cu): whole cluster leaves
        if (blockIdx.x == 0 && threadIdx.x == 0 && sweeps_out) sweeps_out[blockIdx.y] = 0;
        return;
    }
    using Cfg = JacobiCfg<NN>;
    constexpr int P = Cfg::P;
    constexpr int NB = 2 * P;
    constexpr int M = NB - 1;
    constexpr int HP = NN / 64;
    extern __shared__ __align__(16) float cols[];          // [64][NN]
    __shared__ float nrm[64];
    __shared__ unsigned int s_max, s_amax;

    const int rank = blockIdx.x;
    const int prob = blockIdx.y;
    float* G = Gall + (long long)prob * NN * NN;
    float* cw = conv_ws + (long long)prob * 16;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    cg::cluster_group cluster = cg::this_cluster();

    // Every pair is rotated, including columns that have collapsed to rounding noise: keeping the noise
    // columns orthogonal to the large ones is what makes their Rayleigh quotients (k_rayleigh) second-order
    // small.  (A variant that left columns below 4*eps*max|column| alone was measured: the untouched columns
    // keep large range-space components and their Rayleigh quotients are O(lambda).)
    const float tol2 = tol * tol;
    // Quadratic convergence: a sweep whose largest cosine was rho leaves ~rho^2 behind.  When a sweep saw
    // nothing above tol_q = 1e-4 (rho^2 = 1e-8 << tol ~ 2.7e-6) its own rotations already finished the job and
    // the verification sweep (no rotations, ~60 % of a sweep's cost) is skipped.
    const float tolq2 = g_jacobi_tolq * g_jacobi_tolq;

    float null2 = 0.f;                                 // noise floor of the previous sweep (0: every pair is live)
    int sweep = 0;
    for (; sweep < max_sweeps; ++sweep) {
        if (threadIdx.x == 0) { s_max = 0u; s_amax = 0u; }
        float flag = 0.f, amax = 0.f;
        for (int r = 0; r < (P == 1 ? 1 : M); ++r) {
            int bt, bb;
            if (P == 1) { bt = 0; bb = 1; }
            else if (rank == 0) { bt = NB - 1; bb = r; }
            else { bt = (r + rank) % M; bb = (r - rank + M) % M; }
            if (P > 1 || sweep == 0) {
                const float4* s0 = reinterpret_cast<const float4*>(G + (long long)bt * 32 * NN);
                const float4* s1 = reinterpret_cast<const float4*>(G + (long long)bb * 32 * NN);
                float4* d = reinterpret_cast<float4*>(cols);
                for (int i = threadIdx.x; i < 32 * NN / 4; i += 512) {
                    d[i] = __ldcg(s0 + i);                 // L2 (peers of the cluster wrote these columns)
                    d[32 * NN / 4 + i] = __ldcg(s1 + i);
                }
            }
            __syncthreads();
            // ---- column norms (fresh every round: the cached values never drift far)
            for (int c = warp * 4; c < warp * 4 + 4; ++c) {
                f32x2 v[HP];
                load_col<NN>(cols + c * NN, lane, v);
                f32x2 q = pack2(0.f, 0.f);
#pragma unroll
                for (int i = 0; i < HP; ++i) q = fma2(v[i], v[i], q);
                float q0, q1;
                unpack2(q, q0, q1);
                float ss = q0 + q1;
#pragma unroll
                for (int o = 16; o >= 1; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
                if (lane == 0) nrm[c] = ss;
                amax = fmaxf(amax, ss);
            }
            __syncthreads();
            // ---- pairs inside each 32-column block: once per sweep
            if (r == 0) {
                for (int lv = 3; lv >= 0; --lv) {          // sub-block halves of 16, 8, 4, 2 columns
                    const int wpg = 1 << lv;               // warps per sub-block pair = column pairs per half
                    const int base = (warp >> lv) * (4 << lv);
                    cross_steps<NN>(cols, nrm, base + 2 * (warp & (wpg - 1)), base + (2 << lv), wpg, warp & (wpg - 1),
                                    1 + (warp >> lv), lane, tol2, tolq2, null2, flag);
                    __syncthreads();
                }
                {   // 1|1 : columns (4w,4w+1) and (4w+2,4w+3)
                    f32x2 x0[HP], y0[HP], x1[HP], y1[HP];
                    float* c0 = cols + 4 * warp * NN;
                    load_col<NN>(c0, lane, x0);
                    load_col<NN>(c0 + NN, lane, y0);
                    load_col<NN>(c0 + 2 * NN, lane, x1);
                    load_col<NN>(c0 + 3 * NN, lane, y1);
                    float a0 = nrm[4 * warp], b0 = nrm[4 * warp + 1], a1 = nrm[4 * warp + 2], b1 = nrm[4 * warp + 3];
                    rot_regs2<HP>(x0, y0, a0, b0, x1, y1, a1, b1, tol2, tolq2, null2, flag);
                    store_col<NN>(c0, lane, x0);
                    store_col<NN>(c0 + NN, lane, y0);
                    store_col<NN>(c0 + 2 * NN, lane, x1);
                    store_col<NN>(c0 + 3 * NN, lane, y1);
                    if (lane == 0) { nrm[4 * warp] = a0; nrm[4 * warp + 1] = b0; nrm[4 * warp + 2] = a1; nrm[4 * warp + 3] = b1; }
                    __syncthreads();
                }
            }
            // ---- cross pairs: 16 steps x 4 rotations per warp
            {
                f32x2 x0[HP], x1[HP];
                load_col<NN>(cols + 2 * warp * NN, lane, x0);
                load_col<NN>(cols + (2 * warp + 1) * NN, lane, x1);
                float a0 = nrm[2 * warp], a1 = nrm[2 * warp + 1];
                const int ring = 16 >> lg;                         // warps per group = bottom pairs per sub-block
                const int grp = warp / ring, wsub = warp & (ring - 1);
                for (int h = 0; h < (1 << lg); ++h) {
                    if (stagger > 0 && grp > 0) {
                        const long long t0 = clock64();
                        while (clock64() - t0 < (long long)grp * stagger) {}
                    }
                    ring_steps<NN>(cols, nrm, x0, x1, a0, a1, 32 + 2 * ring * (grp ^ h), ring, wsub, 1 + grp, lane, tol2,
                                   tolq2, null2, flag);
                    __syncthreads();
                }
                store_col<NN>(cols + 2 * warp * NN, lane, x0);
                store_col<NN>(cols + (2 * warp + 1) * NN, lane, x1);
                __syncthreads();
            }
            if (P > 1) {
                float4* d0 = reinterpret_cast<float4*>(G + (long long)bt * 32 * NN);
                float4* d1 = reinterpret_cast<float4*>(G + (long long)bb * 32 * NN);
                const float4* sc = reinterpret_cast<const float4*>(cols);
                for (int i = threadIdx.x; i < 32 * NN / 4; i += 512) {
                    d0[i] = sc[i];
                    d1[i] = sc[32 * NN / 4 + i];
                }
                __threadfence();
                cluster.sync();   // release/acquire: next round reads what the peers just wrote
            }
        }
        // ---- convergence: worst pair class seen in this sweep (0 / 1 / 2), agreed across the cluster
        if (lane == 0) { atomicMax(&s_max, __float_as_uint(flag)); atomicMax(&s_amax, __float_as_uint(amax)); }
        __syncthreads();
        float gmax = __uint_as_float(s_max);
        float amx = __uint_as_float(s_amax);
        if (P > 1) {
            if (threadIdx.x == 0) {
                reinterpret_cast<volatile float*>(cw)[rank] = gmax;
                reinterpret_cast<volatile float*>(cw)[8 + rank] = amx;
                __threadfence();
            }
            cluster.sync();
            gmax = 0.f;
            amx = 0.f;
            for (int i = 0; i < P; ++i) {
                gmax = fmaxf(gmax, reinterpret_cast<volatile float*>(cw)[i]);
                amx = fmaxf(amx, reinterpret_cast<volatile float*>(cw)[8 + i]);
            }
            cluster.sync();   // everyone has read before the next sweep overwrites
        }
        // Null floor (rot_scalars): |column| below max(thresh / 2, 16 * 2^-24 * max|column|), and never above the
        // 3.16e-6 * max|column| of the original rule.  Kept columns (|g| ~ lambda > thresh) stay live as long as fp32
        // resolves them against lambda_max; the rounding-noise columns of a rank-deficient map (~4e-7 lambda_max, i.e.
        // ~7 x 2^-24 lambda_max) stay below it.  A floor of 3.16e-6 lambda_max alone froze a graded kept tail
        // between thresh and that level after sweep 0 and whitened it wrong by O(1) (tests/test_gpu_whitening.py).
        null2 = fminf(1e-11f * amx, fmaxf(0.25f * thresh * thresh, 9.1e-13f * amx));
        __syncthreads();
        if (gmax < 2.f) { ++sweep; break; }
    }
    if (P == 1) {
        float4* d = reinterpret_cast<float4*>(G);
        const float4* sc = reinterpret_cast<const float4*>(cols);
        for (int i = threadIdx.x; i < 64 * NN / 4; i += 512) d[i] = sc[i];
    }
    if (rank == 0 && threadIdx.x == 0 && sweeps_out) sweeps_out[prob] = sweep;
}

// Rayleigh quotients  lambda_i = g_i^T A g_i / |g_i|^2  of the converged columns against the ORIGINAL matrix.
// The column norm |g_i| is a first-order eigenvalue estimate: on a rank-deficient map the null columns
// keep the rounding noise of the cancellations that created them (measured 4e-7*lambda_max, i.e. above
// the 1e-5 cut for lambda_max > 25; LAPACK: 4e-8*lambda_max).  The Rayleigh quotient is second order in
// that noise: the same null columns give ~1e-8.   grid (C/16, problems), C threads.
__global__ void __launch_bounds__(512)
k_rayleigh(const float* __restrict__ A0all, const float* __restrict__ Gall, int C, float* __restrict__ lam,
           const int* __restrict__ skip) {
    if (skip && skip[blockIdx.y]) return;
    __shared__ __align__(16) float gs[512 * 16];
    __shared__ float red_q[16][17], red_s[16][17];     // [warp][column]: fixed-order (deterministic) reduction
    const int prob = blockIdx.y, j0 = blockIdx.x * 16, r = threadIdx.x;
    const float* A0 = A0all + (long long)prob * C * C;
    const float* G = Gall + (long long)prob * C * C;
    float mine[16];
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
        mine[jj] = G[(long long)(j0 + jj) * C + r];          // column j0+jj, row r (coalesced over r)
        gs[r * 16 + jj] = mine[jj];
    }
    __syncthreads();
    float acc[16];
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) acc[jj] = 0.f;
    // 8 rows of A in flight per thread: the loop is a chain of dependent L2 loads otherwise (measured 311 us per launch
    // of 16 matrices at C = 512 for 33 MB of traffic)
#pragma unroll 1
    for (int k8 = 0; k8 < C; k8 += 8) {
        float av[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) av[u] = __ldg(A0 + (long long)(k8 + u) * C + r);   // A symmetric: row k read as column k, coalesced over r
#pragma unroll
        for (int u = 0; u < 8; ++u) {
        const int k = k8 + u;
        const float a = av[u];
        const float4* g4 = reinterpret_cast<const float4*>(gs + k * 16);
        const float4 g0 = g4[0], g1 = g4[1], g2 = g4[2], g3 = g4[3];
        acc[0] = fmaf(a, g0.x, acc[0]); acc[1] = fmaf(a, g0.y, acc[1]); acc[2] = fmaf(a, g0.z, acc[2]); acc[3] = fmaf(a, g0.w, acc[3]);
        acc[4] = fmaf(a, g1.x, acc[4]); acc[5] = fmaf(a, g1.y, acc[5]); acc[6] = fmaf(a, g1.z, acc[6]); acc[7] = fmaf(a, g1.w, acc[7]);
        acc[8] = fmaf(a, g2.x, acc[8]); acc[9] = fmaf(a, g2.y, acc[9]); acc[10] = fmaf(a, g2.z, acc[10]); acc[11] = fmaf(a, g2.w, acc[11]);
        acc[12] = fmaf(a, g3.x, acc[12]); acc[13] = fmaf(a, g3.y, acc[13]); acc[14] = fmaf(a, g3.z, acc[14]); acc[15] = fmaf(a, g3.w, acc[15]);
        }
    }
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
        float q = mine[jj] * acc[jj], ss = mine[jj] * mine[jj];
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) {
            q += __shfl_xor_sync(0xffffffffu, q, o);
            ss += __shfl_xor_sync(0xffffffffu, ss, o);
        }
        if (lane == 0) { red_q[threadIdx.x >> 5][jj] = q; red_s[threadIdx.x >> 5][jj] = ss; }
    }
    __syncthreads();
    if (r < 16) {
        float q = 0.f, ss = 0.f;
        for (int w = 0; w < (C >> 5); ++w) { q += red_q[w][r]; ss += red_s[w][r]; }
        lam[(long long)prob * C + j0 + r] = ss > 0.f ? q / ss : 0.f;
    }
}

// eigenvalue estimate (Rayleigh quotient when `lam` is given, else |column i|); per-problem kept count;
// scaling d_i of the rank-k reconstruction
//   mode 0 (content, whitening): d = (sigma+eps_eig)^-1/2 / sigma^2
//   mode 1 (style, colouring)  : d = (sigma+eps_eig)^+1/2 / sigma^2
//   so that  E_k f(S_k) E_k^T = G diag(d) G^T  with G's columns = sigma_i u_i.
__global__ void k_eig_post(const float* __restrict__ Gall, const float* __restrict__ lam, int C, float thresh, float eps_eig,
                           int n_content, float* __restrict__ sigma, float* __restrict__ dvec, int* __restrict__ kcount,
                           const int* __restrict__ skip) {
    const int prob = blockIdx.y;
    if (skip && skip[prob]) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int col = blockIdx.x * (blockDim.x >> 5) + warp;
    if (col >= C) return;
    const float* g = Gall + ((long long)prob * C + col) * C;
    float ss = 0.f;
    for (int i = lane; i < C; i += 32) ss = fmaf(g[i], g[i], ss);
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if (lane == 0) {
        const float sg = lam ? fabsf(lam[(long long)prob * C + col]) : sqrtf(ss);   // |lambda| like the SVD of ops.py:54,110
        sigma[(long long)prob * C + col] = sg;
        float d = 0.f;
        if (sg > thresh) {                                       // ops.py:68-69,112,125
            const float f = (prob < n_content) ? rsqrtf(sg + eps_eig) : sqrtf(sg + eps_eig);
            d = f / ss;
            if (kcount) atomicAdd(&kcount[prob], 1);
        }
        if (dvec) dvec[(long long)prob * C + col] = d;
    }
}

// ---------------------------------------------------------------------------
// Stage C: small dense products  Cm[i][j] = sum_k A[k][i] * d[k] * B[k][j]   (all n x n, k-major)
//   grid (n/64, n/64, batch); 256 threads, 4x4 per thread
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_outer_gemm(const float* __restrict__ A, long long sa, const float* __restrict__ B, long long sb,
             const float* __restrict__ d, long long sd, float* __restrict__ Cm, long long sc, int n,
             const int* __restrict__ skip = nullptr, int amod = 0) {
    if (skip && skip[blockIdx.z]) return;      // this output was produced by the matrix-function fast path
    __shared__ __align__(16) float As[16][64];
    __shared__ __align__(16) float Bs[16][64];
    const int z = blockIdx.z;
    const float* a = A + (long long)(amod ? z % amod : z) * sa;     // amod: A cycles through amod matrices (regions: style z % R)
    const float* b = B + (long long)z * sb;
    const float* dd = d ? d + (long long)z * sd : nullptr;
    const int i0 = blockIdx.x * 64, j0 = blockIdx.y * 64;
    const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
    const int lk = threadIdx.x >> 4, lc = (threadIdx.x & 15) * 4;   // loader: 16 k-rows x 64 cols
    float acc[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] = 0.f;
    for (int k0 = 0; k0 < n; k0 += 16) {
        float4 av = *reinterpret_cast<const float4*>(a + (long long)(k0 + lk) * n + i0 + lc);
        const float4 bv = *reinterpret_cast<const float4*>(b + (long long)(k0 + lk) * n + j0 + lc);
        if (dd) {
            const float s = dd[k0 + lk];
            av.x *= s; av.y *= s; av.z *= s; av.w *= s;
        }
        __syncthreads();
        *reinterpret_cast<float4*>(&As[lk][lc]) = av;
        *reinterpret_cast<float4*>(&Bs[lk][lc]) = bv;
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < 16; ++kk) {
            const float4 x = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
            const float4 y = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
            const float xv[4] = {x.x, x.y, x.z, x.w};
            const float yv[4] = {y.x, y.y, y.z, y.w};
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) acc[r][c] = fmaf(xv[r], yv[c], acc[r][c]);
        }
    }
    float* cm = Cm + (long long)z * sc;
#pragma unroll
    for (int r = 0; r < 4; ++r)
        *reinterpret_cast<float4*>(cm + (long long)(i0 + ty * 4 + r) * n + j0 + tx * 4) =
            make_float4(acc[r][0], acc[r][1], acc[r][2], acc[r][3]);
}

// M = alpha*T + (1-alpha)*I  -> split-fp16 GEMM operand [frame][2][C][C] (row = output channel), row i stored times 2^e_i,
// e_i in mexp [frame][C]: the power of two that puts the row's max |m| into [512, 1024) (weight_scale_exp), so that no lo
// half that matters is an fp16 subnormal (DESIGN.md §3.1); the apply's epilogue multiplies by 2^-e_i exactly
// bias = alpha*ms - M*mc + (1-alpha)*readd*mc  from the unscaled M     (ops.py:80-83 / 131-133)
//   one warp per (frame, output channel); style mean z % Ns (Ns == 1: shared; regions: problem z = frame*R + r, Ns = R)
__global__ void k_finalize_transform(const float* __restrict__ T, int C, int Nc, int Ns, float alpha, int readd,
                                     const float* __restrict__ mean_c, const float* __restrict__ mean_s,
                                     __half* __restrict__ Msplit, int* __restrict__ mexp, float* __restrict__ bias) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int row = blockIdx.x * (blockDim.x >> 5) + warp;
    const int z = blockIdx.y;
    if (row >= C) return;
    const float* t = T + ((long long)z * C + row) * C;
    const float* mc = mean_c + (long long)z * C;
    const float* ms = mean_s + (long long)(Ns == 1 ? 0 : z % Ns) * C;
    __half* mh = Msplit + (((long long)z * 2 + 0) * C + row) * C;
    __half* ml = Msplit + (((long long)z * 2 + 1) * C + row) * C;
    float amax = 0.f;
    for (int j = lane; j < C; j += 32) amax = fmaxf(amax, fabsf(alpha * t[j] + (j == row ? 1.f - alpha : 0.f)));
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    const int e = weight_scale_exp(__float_as_uint(amax));
    const float sc = pow2i(e);
    if (lane == 0) mexp[(long long)z * C + row] = e;
    float dot = 0.f;
    for (int j = lane; j < C; j += 32) {
        const float m = alpha * t[j] + (j == row ? 1.f - alpha : 0.f);
        __half hi, lo;
        split_f32(m * sc, hi, lo);
        mh[j] = hi;
        ml[j] = lo;
        dot = fmaf(m, mc[j], dot);
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
    if (lane == 0) bias[(long long)z * C + row] = alpha * ms[row] - dot + (readd ? (1.f - alpha) * mc[row] : 0.f);
}

// ---------------------------------------------------------------------------
// AdaIN (ops.py:282-294): per-(frame,channel) affine map
// ---------------------------------------------------------------------------
// inv = rsqrt(vc + eps) * sqrt(vs) (batch_normalization with scale = sqrt(style_var)) and the style mean of each content frame
__global__ void k_adain_coeffs(const float* __restrict__ var_c, const float* __restrict__ mean_s, const float* __restrict__ var_s,
                               int C, int Nc, int Ns, float eps, float* __restrict__ inv, float* __restrict__ ms) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Nc * C) return;
    const int z = i / C, c = i % C;
    const int si = (Ns == 1 ? 0 : z) * C + c;
    inv[i] = rsqrtf(var_c[i] + eps) * sqrtf(var_s[si]);
    ms[i] = mean_s[si];
}
// y = (x - mc) * inv + ms, out = alpha * y + (1 - alpha) * x.  Centred first, as tf.nn.batch_normalization is: folded into
// x * scale + shift, the shift of a channel with a large mean and a small spread is the difference of two large fp32 terms.
__global__ void k_affine_apply(const __half* __restrict__ in, ActGeom g, const float* __restrict__ mean_c,
                               const float* __restrict__ inv, const float* __restrict__ ms, float alpha, __half* __restrict__ out) {
    const int cgs = g.C / 8;
    const long long total = (long long)g.N * g.H * g.W * cgs;
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < (unsigned)total; i += gridDim.x * blockDim.x) {
        const int c0 = (int)(i % (unsigned)cgs) * 8;
        unsigned pix = i / (unsigned)cgs;
        const int x = (int)(pix % (unsigned)g.W); pix /= (unsigned)g.W;
        const int y = (int)(pix % (unsigned)g.H);
        const int n = (int)(pix / (unsigned)g.H);
        float v[8];
        load8(in, g, ((long long)n * g.Hp + y + 1) * g.Wp + x + 1, c0, v);
        const float* mc = mean_c + (long long)n * g.C + c0;
        const float* iv = inv + (long long)n * g.C + c0;
        const float* m_s = ms + (long long)n * g.C + c0;
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = fmaf(alpha, fmaf(v[j] - mc[j], iv[j], m_s[j]), (1.f - alpha) * v[j]);
        Half8 hi, lo;
        split8(v, hi, lo);
        store8_with_halo(out, g, n, y, x, c0, hi, lo);
    }
}
// k_affine_apply with a strength map (soft spatial control): alpha s(p) in place of alpha, str [N][H][W]; s = 1 gives
// k_affine_apply's bits
__global__ void k_affine_apply_strength(const __half* __restrict__ in, ActGeom g, const float* __restrict__ mean_c,
                                        const float* __restrict__ inv, const float* __restrict__ ms, float alpha,
                                        const float* __restrict__ str, __half* __restrict__ out) {
    const int cgs = g.C / 8;
    const long long total = (long long)g.N * g.H * g.W * cgs;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c0 = (int)(i % cgs) * 8;
        const long long pix = i / cgs;
        const int x = (int)(pix % g.W);
        const int y = (int)((pix / g.W) % g.H);
        const int n = (int)(pix / ((long long)g.W * g.H));
        const float a = alpha * __ldg(str + pix);
        float v[8];
        load8(in, g, ((long long)n * g.Hp + y + 1) * g.Wp + x + 1, c0, v);
        const float* mc = mean_c + (long long)n * g.C + c0;
        const float* iv = inv + (long long)n * g.C + c0;
        const float* m_s = ms + (long long)n * g.C + c0;
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = fmaf(a, fmaf(v[j] - mc[j], iv[j], m_s[j]), (1.f - a) * v[j]);
        Half8 hi, lo;
        split8(v, hi, lo);
        store8_with_halo(out, g, n, y, x, c0, hi, lo);
    }
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

struct WctWs {
    size_t shift, dsum, mean, var, G, A0, lam, sigma, dvec, Wc, Cs, T, Msplit, Mexp, bias, conv, kcount, ok, inv, ms, total;
};
static WctWs wct_layout(int C, int Nc, int Ns) {
    WctWs w;
    const size_t np = (size_t)Nc + Ns;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o = align_up(o + bytes, 256); return r; };
    w.shift = take(np * C * 4);        // AdaIN: centring shift of the channel moments (k_sample_shift)
    w.dsum = take(np * C * 8);         // WCT: fp64 sums of the shifted features (cov_tc.cu)
    w.mean = take(np * C * 4);
    w.var = take(np * C * 4);
    w.G = take(np * C * C * 4);
    w.A0 = take(np * C * C * 4);
    w.lam = take(np * C * 4);
    w.sigma = take(np * C * 4);
    w.dvec = take(np * C * 4);
    w.Wc = take((size_t)Nc * C * C * 4);
    w.Cs = take((size_t)Ns * C * C * 4);
    w.T = take((size_t)Nc * C * C * 4);
    w.Msplit = take((size_t)Nc * 2 * C * C * 2);
    w.Mexp = take((size_t)Nc * C * 4);
    w.bias = take((size_t)Nc * C * 4);
    w.conv = take(np * 16 * 4);
    w.kcount = take(np * 2 * 4);
    w.ok = take(np * 4);               // matrices whose W / C_s came from the matrix-function fast path (matfun_tc.cu)
    w.inv = take((size_t)Nc * C * 4);  // AdaIN: rsqrt(vc + eps) sqrt(vs) and the style mean, per (frame, channel)
    w.ms = take((size_t)Nc * C * 4);
    w.total = o;
    return w;
}
size_t wct_workspace_bytes(int C, int Nc, int Ns) { return wct_layout(C, Nc, Ns).total; }

int launch_sample_shift(const __half* act, ActGeom g, float* shift, cudaStream_t st);   // cov_tc.cu

// per-channel mean and biased variance of a feature batch: shift, slot partials (`part`: [N][slices][2][C]), fixed-order finalize
static int launch_moments(const __half* act, ActGeom g, float* shift, float* part, float* mean, float* var, cudaStream_t st) {
    const long long HW = (long long)g.H * g.W;
    const int slice = moments_slice(g.C);
    const int nslices = cdiv(HW, slice);
    int rc = launch_sample_shift(act, g, shift, st);
    if (rc) return rc;
    k_chan_moments<<<dim3((unsigned)nslices, (unsigned)g.N), 256, 0, st>>>(act, g, shift, slice, part);
    WCTB_CHECK_LAUNCH("k_chan_moments");
    k_moments_finalize<<<cdiv((long long)g.N * g.C, 256), 256, 0, st>>>(part, shift, g.C, nslices, HW, g.N * g.C, mean, var);
    WCTB_CHECK_LAUNCH("k_moments_finalize");
    return 0;
}

// ---------------------------------------------------------------------------
// Statistics records (tiled stylisation, DESIGN.md §3.3.7): fp64 n [N] | t [N][C] | s [N][C] | S [N][C][C] (diag: [N][C])
// ---------------------------------------------------------------------------
size_t stats_record_layout(int C, int N, int diag, size_t* off_n, size_t* off_t, size_t* off_s, size_t* off_S) {
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o = align_up(o + bytes, 256); return r; };
    const size_t a = take((size_t)N * 8), b = take((size_t)N * C * 8), c = take((size_t)N * C * 8);
    const size_t d = take((size_t)N * (diag ? (size_t)C : (size_t)C * C) * 8);
    if (off_n) *off_n = a;
    if (off_t) *off_t = b;
    if (off_s) *off_s = c;
    if (off_S) *off_S = d;
    return o;
}
static StatsRecord stats_record_at(const void* rec, int C, int N, int diag) {
    size_t a, b, c, d;
    stats_record_layout(C, N, diag, &a, &b, &c, &d);
    uint8_t* p = static_cast<uint8_t*>(const_cast<void*>(rec));
    return StatsRecord{reinterpret_cast<double*>(p + a), reinterpret_cast<double*>(p + b), reinterpret_cast<double*>(p + c),
                       reinterpret_cast<double*>(p + d)};
}

int launch_cov_record(const __half* act, int N, int H, int W, int C, int y0, int x0, int h, int w, const StatsRecord& rec,
                      cudaStream_t st);   // cov_tc.cu
int launch_record_cov_finalize(const StatsRecord& rec, int C, int N, float eps_cov, float* mean, float* G, float* A0, cudaStream_t st);

int launch_wct_stats_rect(const __half* act, int N, int H, int W, int C, int y0, int x0, int h, int w, void* record, cudaStream_t st) {
    WCTB_REQUIRE(C == 64 || C == 128 || C == 256 || C == 512, "wct_stats_rect: C=%d not in {64,128,256,512}", C);
    return launch_cov_record(act, N, H, W, C, y0, x0, h, w, stats_record_at(record, C, N, 0), st);
}

// AdaIN's moments of a rectangle: k_sample_shift and k_chan_moments over a view of the padded planes (see launch_cov_record)
int launch_adain_stats_rect(const __half* act, int N, int H, int W, int C, int y0, int x0, int h, int w, void* record, cudaStream_t st) {
    WCTB_REQUIRE(C % 8 == 0 && C <= 2048, "adain_stats_rect: C=%d must be a multiple of 8 (<= 2048)", C);
    ActGeom v(N, H, W, C);
    v.H = h;
    v.W = w;
    const __half* base = act + ((long long)y0 * v.Wp + x0) * C;
    const long long HW = (long long)h * w;
    const int slice = moments_slice(C);
    const int nslices = cdiv(HW, slice);
    const size_t nshift = align_up((size_t)N * C, 64);
    float* scratch = nullptr;
    { int rc0 = scratch_alloc(reinterpret_cast<void**>(&scratch), (nshift + (size_t)N * nslices * 2 * C) * sizeof(float), st, 5); if (rc0) return rc0; }
    float* shift = scratch;
    float* part = scratch + nshift;
    int rc = launch_sample_shift(base, v, shift, st);
    if (rc) return rc;
    k_chan_moments<<<dim3((unsigned)nslices, (unsigned)N), 256, 0, st>>>(base, v, shift, slice, part);
    WCTB_CHECK_LAUNCH("k_chan_moments");
    k_moments_record<<<cdiv((long long)N * C, 256), 256, 0, st>>>(part, shift, C, nslices, HW, N * C, stats_record_at(record, C, N, 1));
    WCTB_CHECK_LAUNCH("k_moments_record");
    return 0;
}

int launch_stats_accumulate(void* rec_a, const void* rec_b, int C, int N, int diag, cudaStream_t st) {
    const StatsRecord a = stats_record_at(rec_a, C, N, diag), b = stats_record_at(rec_b, C, N, diag);
    const long long tot = (long long)N * (diag ? (long long)C : (long long)C * C);
    k_record_fold_S<<<(unsigned)(cdiv(tot, 256) > 4096 ? 4096 : cdiv(tot, 256)), 256, 0, st>>>(a, b, C, N, diag);
    WCTB_CHECK_LAUNCH("k_record_fold_S");
    k_record_fold_vec<<<(unsigned)N, 256, 0, st>>>(a, b, C);
    WCTB_CHECK_LAUNCH("k_record_fold_vec");
    return 0;
}

// cross-phase schedule of k_jacobi: 2^lg warp groups, started `stagger` cycles apart (wctb200_debug_set_jacobi)
// -1 = auto: chosen by measurement (tools/jacobi_bench.py): C=512 -> 4 groups 300 cycles apart (6.76 ms vs 7.80 ms for
// one group), smaller matrices -> 2 groups 600 cycles apart.
int g_jacobi_lg = -1;
int g_jacobi_stagger = -1;
int set_jacobi_tolq(float v) {
    return cudaMemcpyToSymbol(g_jacobi_tolq, &v, sizeof(float)) == cudaSuccess ? 0 : -1;
}

int launch_jacobi(float* G, int C, int count, float* conv_ws, int* sweeps, cudaStream_t st, const int* skip, float thresh) {
    const float tol = 2.f * sqrtf((float)C) * 5.96e-8f;
    const int max_sweeps = 40;
    const int lg = g_jacobi_lg >= 0 ? g_jacobi_lg : (C >= 512 ? 2 : 1);
    const int stagger = g_jacobi_stagger >= 0 ? g_jacobi_stagger : (C >= 512 ? 300 : 600);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(C / 64), (unsigned)count, 1);
    cfg.blockDim = dim3(512, 1, 1);
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = (unsigned)(C / 64);
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
#define WCTB_JACOBI_CASE(NN)                                                                                         \
    case NN: {                                                                                                       \
        WCTB_ENSURE_SMEM(k_jacobi<NN>, JacobiCfg<NN>::SMEM_BYTES);                                                   \
        cfg.dynamicSmemBytes = JacobiCfg<NN>::SMEM_BYTES;                                                            \
        WCTB_CUDA(cudaLaunchKernelEx(&cfg, k_jacobi<NN>, G, conv_ws, sweeps, max_sweeps, tol, lg, stagger, skip, thresh));         \
        break;                                                                                                       \
    }
    switch (C) {
        WCTB_JACOBI_CASE(64)
        WCTB_JACOBI_CASE(128)
        WCTB_JACOBI_CASE(256)
        WCTB_JACOBI_CASE(512)
        default:
            set_error("jacobi: C=%d not in {64,128,256,512}", C);
            return WCTB200_EINVAL;
    }
#undef WCTB_JACOBI_CASE
    return 0;
}

int launch_eig_post(const float* G, const float* A0, float* lam, int C, int count, float thresh, float eps_eig,
                    int n_content, float* sigma, float* dvec, int* kcount, cudaStream_t st, const int* skip = nullptr) {
    if (A0 && lam) {
        dim3 gr((unsigned)(C / 16), (unsigned)count);
        k_rayleigh<<<gr, C, 0, st>>>(A0, G, C, lam, skip);
        WCTB_CHECK_LAUNCH("k_rayleigh");
    } else {
        lam = nullptr;
    }
    dim3 grid((unsigned)cdiv(C, 8), (unsigned)count);
    k_eig_post<<<grid, 256, 0, st>>>(G, lam, C, thresh, eps_eig, n_content, sigma, dvec, kcount, skip);
    WCTB_CHECK_LAUNCH("k_eig_post");
    return 0;
}

// matfun_tc.cu: A^-1/2 / A^+1/2 by coupled Newton-Schulz on the tensor cores where every eigenvalue is kept; ok[b] = 1 there
int launch_matfun_ns(const float* A, int C, int count, int n_first, float thresh, float eps_eig, float* out, int* ok, int* kcount,
                     cudaStream_t st, float* info = nullptr);
// cov_tc.cu: per-channel means and covariance (+ eps_cov I) in one pass over the features
int launch_mean_cov(const __half* act, ActGeom g, float eps_cov, float* mean, float* G, float* A0, double* dsum, cudaStream_t st);

int launch_wct_level(const __half* content, int Nc, int Hc, int Wc, const __half* style, int Ns, int Hs, int Ws, int C,
                     float alpha, float eps_cov, float eps_eig, float thresh, int readd, __half* out, int32_t* k_out,
                     void* ws, size_t ws_bytes, cudaStream_t st) {
    WCTB_REQUIRE(C == 64 || C == 128 || C == 256 || C == 512, "wct_level: C=%d not in {64,128,256,512}", C);
    WCTB_REQUIRE(Ns == 1 || Ns == Nc, "wct_level: Ns must be 1 or Nc");
    WCTB_REQUIRE(Hc >= 2 && Wc >= 2 && Hs >= 2 && Ws >= 2 && (long long)Hc * Wc >= 2 && (long long)Hs * Ws >= 2, "wct_level: bad geometry");
    const WctWs L = wct_layout(C, Nc, Ns);
    if (ws_bytes < L.total) {
        set_error("wct_level: workspace %zu < %zu bytes", ws_bytes, L.total);
        return WCTB200_EWS;
    }
    uint8_t* w = static_cast<uint8_t*>(ws);
    const int np = Nc + Ns;
    double* dsum = reinterpret_cast<double*>(w + L.dsum);
    float* mean = reinterpret_cast<float*>(w + L.mean);
    float* G = reinterpret_cast<float*>(w + L.G);
    float* sigma = reinterpret_cast<float*>(w + L.sigma);
    float* dvec = reinterpret_cast<float*>(w + L.dvec);
    float* Wcm = reinterpret_cast<float*>(w + L.Wc);
    float* Csm = reinterpret_cast<float*>(w + L.Cs);
    float* T = reinterpret_cast<float*>(w + L.T);
    __half* Msplit = reinterpret_cast<__half*>(w + L.Msplit);
    float* bias = reinterpret_cast<float*>(w + L.bias);
    float* conv = reinterpret_cast<float*>(w + L.conv);
    int* kc = reinterpret_cast<int*>(w + L.kcount);
    const long long CC = (long long)C * C;

    WCTB_CUDA(cudaMemsetAsync(kc, 0, (size_t)np * 2 * 4, st));
    ActGeom gc(Nc, Hc, Wc, C), gs(Ns, Hs, Ws, C);
    float* A0 = reinterpret_cast<float*>(w + L.A0);
    float* lam = reinterpret_cast<float*>(w + L.lam);
    int rc = launch_mean_cov(content, gc, eps_cov, mean, G, A0, dsum, st);
    if (rc) return rc;
    rc = launch_mean_cov(style, gs, eps_cov, mean + (long long)Nc * C, G + Nc * CC, A0 + Nc * CC, dsum + (long long)Nc * C, st);
    if (rc) return rc;
    // fast path first: W_c = A^-1/2, C_s = A^+1/2 straight from the covariances where the threshold keeps every eigenvalue
    int* ok = reinterpret_cast<int*>(w + L.ok);
    rc = launch_matfun_ns(A0, C, np, Nc, thresh, eps_eig, Wcm, ok, kc, st);        // Wc and Cs are contiguous in ws (Wc then Cs)
    if (rc < 0) return rc;
    rc = launch_jacobi(G, C, np, conv, kc + np, st, ok, thresh);
    if (rc) return rc;
    rc = launch_eig_post(G, A0, lam, C, np, thresh, eps_eig, Nc, sigma, dvec, kc, st, ok);
    if (rc) return rc;
    // W_c (whitening) per content frame, C_s (colouring) per style
    dim3 gg((unsigned)(C / 64), (unsigned)(C / 64), (unsigned)np);
    k_outer_gemm<<<gg, 256, 0, st>>>(G, CC, G, CC, dvec, C, Wcm, CC, C, ok);
    WCTB_CHECK_LAUNCH("k_outer_gemm(W)");
    dim3 gt((unsigned)(C / 64), (unsigned)(C / 64), (unsigned)Nc);
    k_outer_gemm<<<gt, 256, 0, st>>>(Csm, Ns == 1 ? 0 : CC, Wcm, CC, nullptr, 0, T, CC, C);   // T = C_s W_c (C_s symmetric)
    WCTB_CHECK_LAUNCH("k_outer_gemm(T)");
    dim3 gf((unsigned)cdiv(C, 8), (unsigned)Nc);
    int* Mexp = reinterpret_cast<int*>(w + L.Mexp);
    k_finalize_transform<<<gf, 256, 0, st>>>(T, C, Nc, Ns, alpha, readd, mean, mean + (long long)Nc * C, Msplit, Mexp, bias);
    WCTB_CHECK_LAUNCH("k_finalize_transform");
    // out = M x + bias on the tensor cores (1-tap conv, per-frame weight set)
    rc = launch_conv_apply(content, Nc, Hc, Wc, C, Msplit, Nc, Mexp, bias, out, st);
    if (rc) return rc;
    if (k_out) WCTB_CUDA(cudaMemcpyAsync(k_out, kc, (size_t)np * 2 * 4, cudaMemcpyDeviceToDevice, st));
    return 0;
}

// ---------------------------------------------------------------------------
// Split form of the level transform: the style side (means, covariance, eigendecomposition,
// colouring matrix C_s) depends only on the style features, so the host runs it on a second
// stream where it overlaps the content encoder/decoder convolutions (the Jacobi kernel is
// latency bound and leaves the tensor cores idle), and caches it when a batch shares a style.
//   state layout: [Ns][C] mean_s | [Ns][C][C] C_s | [2*Ns] int32 (k_s, sweeps)
// ---------------------------------------------------------------------------
static size_t style_state_offsets(int C, int Ns, size_t* off_cs, size_t* off_k) {
    size_t o = align_up((size_t)Ns * C * 4, 256);
    *off_cs = o;
    o = align_up(o + (size_t)Ns * C * C * 4, 256);
    *off_k = o;
    return align_up(o + (size_t)Ns * 2 * 4, 256);
}
size_t wct_style_state_bytes(int C, int Ns) {
    size_t a, b;
    return style_state_offsets(C, Ns, &a, &b);
}
size_t wct_style_state_layout(int C, int Ns, size_t* off_mean, size_t* off_cs, size_t* off_k) {
    size_t a, b;
    const size_t total = style_state_offsets(C, Ns, &a, &b);
    if (off_mean) *off_mean = 0;
    if (off_cs) *off_cs = a;
    if (off_k) *off_k = b;
    return total;
}

int launch_wct_style_prepare(const __half* style, int Ns, int Hs, int Ws, int C, float eps_cov, float eps_eig, float thresh,
                             void* state, void* ws, size_t ws_bytes, cudaStream_t st) {
    WCTB_REQUIRE(C == 64 || C == 128 || C == 256 || C == 512, "wct_style_prepare: C=%d not in {64,128,256,512}", C);
    const WctWs L = wct_layout(C, 0, Ns);
    if (ws_bytes < L.total) {
        set_error("wct_style_prepare: workspace %zu < %zu bytes", ws_bytes, L.total);
        return WCTB200_EWS;
    }
    uint8_t* w = static_cast<uint8_t*>(ws);
    size_t off_cs, off_k;
    style_state_offsets(C, Ns, &off_cs, &off_k);
    uint8_t* sp = static_cast<uint8_t*>(state);
    float* mean_s = reinterpret_cast<float*>(sp);
    float* Cs = reinterpret_cast<float*>(sp + off_cs);
    int* kc = reinterpret_cast<int*>(sp + off_k);
    double* dsum = reinterpret_cast<double*>(w + L.dsum);
    float* G = reinterpret_cast<float*>(w + L.G);
    float* sigma = reinterpret_cast<float*>(w + L.sigma);
    float* dvec = reinterpret_cast<float*>(w + L.dvec);
    float* conv = reinterpret_cast<float*>(w + L.conv);
    const long long CC = (long long)C * C;
    WCTB_CUDA(cudaMemsetAsync(kc, 0, (size_t)Ns * 2 * 4, st));
    float* A0 = reinterpret_cast<float*>(w + L.A0);
    float* lam = reinterpret_cast<float*>(w + L.lam);
    int rc = launch_mean_cov(style, ActGeom(Ns, Hs, Ws, C), eps_cov, mean_s, G, A0, dsum, st);
    if (rc) return rc;
    int* ok = reinterpret_cast<int*>(w + L.ok);
    rc = launch_matfun_ns(A0, C, Ns, /*n_first=*/0, thresh, eps_eig, Cs, ok, kc, st);     // C_s = A^+1/2 where every eigenvalue is kept
    if (rc < 0) return rc;
    rc = launch_jacobi(G, C, Ns, conv, kc + Ns, st, ok, thresh);
    if (rc) return rc;
    rc = launch_eig_post(G, A0, lam, C, Ns, thresh, eps_eig, /*n_content=*/0, sigma, dvec, kc, st, ok);
    if (rc) return rc;
    dim3 gg((unsigned)(C / 64), (unsigned)(C / 64), (unsigned)Ns);
    k_outer_gemm<<<gg, 256, 0, st>>>(G, CC, G, CC, dvec, C, Cs, CC, C, ok);
    WCTB_CHECK_LAUNCH("k_outer_gemm(Cs)");
    return 0;
}

// Content side of the split transform (wct_apply, wct_apply_blend) in the workspace `w` of wct_layout(C, Nc, 0): means and
// covariances of the Nc frames, then W_c = A^-1/2 by the matrix-function fast path or the eigensolver.  The kcount slot
// receives [k_c x Nc | sweeps_c x Nc].
static int wct_whiten(int Nc, int C, float eps_eig, float thresh, uint8_t* w, const WctWs& L, cudaStream_t st);
static int wct_content_side(const __half* content, int Nc, int Hc, int Wc, int C, float eps_cov, float eps_eig, float thresh,
                            uint8_t* w, const WctWs& L, cudaStream_t st) {
    double* dsum = reinterpret_cast<double*>(w + L.dsum);
    float* mean = reinterpret_cast<float*>(w + L.mean);
    float* G = reinterpret_cast<float*>(w + L.G);
    int* kc = reinterpret_cast<int*>(w + L.kcount);
    WCTB_CUDA(cudaMemsetAsync(kc, 0, (size_t)Nc * 2 * 4, st));
    float* A0 = reinterpret_cast<float*>(w + L.A0);
    int rc = launch_mean_cov(content, ActGeom(Nc, Hc, Wc, C), eps_cov, mean, G, A0, dsum, st);
    if (rc) return rc;
    return wct_whiten(Nc, C, eps_eig, thresh, w, L, st);
}
// W_c from the covariances G / A0 of wct_content_side (or of a statistics record)
static int wct_whiten(int Nc, int C, float eps_eig, float thresh, uint8_t* w, const WctWs& L, cudaStream_t st) {
    float* G = reinterpret_cast<float*>(w + L.G);
    float* sigma = reinterpret_cast<float*>(w + L.sigma);
    float* dvec = reinterpret_cast<float*>(w + L.dvec);
    float* Wcm = reinterpret_cast<float*>(w + L.Wc);
    float* conv = reinterpret_cast<float*>(w + L.conv);
    int* kc = reinterpret_cast<int*>(w + L.kcount);
    const long long CC = (long long)C * C;
    float* A0 = reinterpret_cast<float*>(w + L.A0);
    float* lam = reinterpret_cast<float*>(w + L.lam);
    int* ok = reinterpret_cast<int*>(w + L.ok);
    int rc = launch_matfun_ns(A0, C, Nc, /*n_first=*/Nc, thresh, eps_eig, Wcm, ok, kc, st);   // W_c = A^-1/2 where every eigenvalue is kept
    if (rc < 0) return rc;
    rc = launch_jacobi(G, C, Nc, conv, kc + Nc, st, ok, thresh);
    if (rc) return rc;
    rc = launch_eig_post(G, A0, lam, C, Nc, thresh, eps_eig, Nc, sigma, dvec, kc, st, ok);
    if (rc) return rc;
    dim3 gg((unsigned)(C / 64), (unsigned)(C / 64), (unsigned)Nc);
    k_outer_gemm<<<gg, 256, 0, st>>>(G, CC, G, CC, dvec, C, Wcm, CC, C, ok);
    WCTB_CHECK_LAUNCH("k_outer_gemm(Wc)");
    return 0;
}

// Style side of the split transform after wct_content_side: T = C_s W_c, the split-fp16 operand M and the bias, then
// out = M x + bias on the tensor cores.  C_s [Ns][C][C] and mean_s [Ns][C] with Ns == 1 (shared) or Ns == Nc (per frame).
static int wct_colour_transform(int Nc, int C, const float* Cs, const float* mean_s, int Ns, float alpha, int readd, uint8_t* w,
                                const WctWs& L, __half* Msplit, int* Mexp, float* bias, cudaStream_t st) {
    const float* mean = reinterpret_cast<const float*>(w + L.mean);
    const float* Wcm = reinterpret_cast<const float*>(w + L.Wc);
    float* T = reinterpret_cast<float*>(w + L.T);
    const long long CC = (long long)C * C;
    dim3 gg((unsigned)(C / 64), (unsigned)(C / 64), (unsigned)Nc);
    k_outer_gemm<<<gg, 256, 0, st>>>(Cs, Ns == 1 ? 0 : CC, Wcm, CC, nullptr, 0, T, CC, C);   // T = C_s W_c
    WCTB_CHECK_LAUNCH("k_outer_gemm(T)");
    dim3 gf((unsigned)cdiv(C, 8), (unsigned)Nc);
    k_finalize_transform<<<gf, 256, 0, st>>>(T, C, Nc, Ns, alpha, readd, mean, mean_s, Msplit, Mexp, bias);
    WCTB_CHECK_LAUNCH("k_finalize_transform");
    return 0;
}
static int wct_colour_apply(const __half* content, int Nc, int Hc, int Wc, int C, const float* Cs, const float* mean_s, int Ns,
                            float alpha, int readd, uint8_t* w, const WctWs& L, __half* out, cudaStream_t st) {
    __half* Msplit = reinterpret_cast<__half*>(w + L.Msplit);
    int* Mexp = reinterpret_cast<int*>(w + L.Mexp);
    float* bias = reinterpret_cast<float*>(w + L.bias);
    int rc = wct_colour_transform(Nc, C, Cs, mean_s, Ns, alpha, readd, w, L, Msplit, Mexp, bias, st);
    if (rc) return rc;
    return launch_conv_apply(content, Nc, Hc, Wc, C, Msplit, Nc, Mexp, bias, out, st);
}

int launch_wct_apply(const __half* content, int Nc, int Hc, int Wc, int C, const void* state, int Ns, float alpha,
                     float eps_cov, float eps_eig, float thresh, int readd, __half* out, int32_t* k_out, void* ws,
                     size_t ws_bytes, cudaStream_t st) {
    WCTB_REQUIRE(C == 64 || C == 128 || C == 256 || C == 512, "wct_apply: C=%d not in {64,128,256,512}", C);
    WCTB_REQUIRE(Ns == 1 || Ns == Nc, "wct_apply: Ns must be 1 or Nc");
    const WctWs L = wct_layout(C, Nc, 0);
    if (ws_bytes < L.total) {
        set_error("wct_apply: workspace %zu < %zu bytes", ws_bytes, L.total);
        return WCTB200_EWS;
    }
    uint8_t* w = static_cast<uint8_t*>(ws);
    size_t off_cs, off_k;
    style_state_offsets(C, Ns, &off_cs, &off_k);
    const uint8_t* sp = static_cast<const uint8_t*>(state);
    const float* mean_s = reinterpret_cast<const float*>(sp);
    const float* Cs = reinterpret_cast<const float*>(sp + off_cs);
    const int* ks = reinterpret_cast<const int*>(sp + off_k);
    int* kc = reinterpret_cast<int*>(w + L.kcount);
    int rc = wct_content_side(content, Nc, Hc, Wc, C, eps_cov, eps_eig, thresh, w, L, st);
    if (rc) return rc;
    rc = wct_colour_apply(content, Nc, Hc, Wc, C, Cs, mean_s, Ns, alpha, readd, w, L, out, st);
    if (rc) return rc;
    if (k_out) {
        // k_out: [k_c x Nc | k_s x Ns | sweeps_c x Nc | sweeps_s x Ns]  (same order as wct_level)
        WCTB_CUDA(cudaMemcpyAsync(k_out, kc, (size_t)Nc * 4, cudaMemcpyDeviceToDevice, st));
        WCTB_CUDA(cudaMemcpyAsync(k_out + Nc, ks, (size_t)Ns * 4, cudaMemcpyDeviceToDevice, st));
        WCTB_CUDA(cudaMemcpyAsync(k_out + Nc + Ns, kc + Nc, (size_t)Nc * 4, cudaMemcpyDeviceToDevice, st));
        WCTB_CUDA(cudaMemcpyAsync(k_out + 2 * Nc + Ns, ks + Ns, (size_t)Ns * 4, cudaMemcpyDeviceToDevice, st));
    }
    return 0;
}

// ---------------------------------------------------------------------------
// Transforms from statistics records (tiled stylisation): wct_apply / adain_apply with the content statistics read from a
// record instead of summed over the content, cut after the transform.  The transform buffer is applied to any feature
// map of the frame (a tile and its halo).  The steps after the statistics are the ones wct_apply / adain_apply run.
//   WCT transform:   split-fp16 M [N][2][C][C] | bias fp32 [N][C] | int32 [k_c x N | sweeps_c x N]
//                    | int32 [N][C] e: row i of M is stored times 2^e_i (k_finalize_transform; 0 = as is)
//   AdaIN transform: fp32 mean_c [N][C] | var_c [N][C] | inv [N][C] | ms [N][C]
// ---------------------------------------------------------------------------
size_t wct_transform_layout(int C, int N, size_t* off_m, size_t* off_bias, size_t* off_k, size_t* off_exp) {
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o = align_up(o + bytes, 256); return r; };
    const size_t a = take((size_t)N * 2 * C * C * 2), b = take((size_t)N * C * 4), c = take((size_t)N * 2 * 4);
    const size_t d = take((size_t)N * C * 4);
    if (off_m) *off_m = a;
    if (off_bias) *off_bias = b;
    if (off_k) *off_k = c;
    if (off_exp) *off_exp = d;
    return o;
}
size_t adain_transform_layout(int C, int N, size_t* off_mean, size_t* off_var, size_t* off_inv, size_t* off_ms) {
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o = align_up(o + bytes, 256); return r; };
    const size_t a = take((size_t)N * C * 4), b = take((size_t)N * C * 4), c = take((size_t)N * C * 4), d = take((size_t)N * C * 4);
    if (off_mean) *off_mean = a;
    if (off_var) *off_var = b;
    if (off_inv) *off_inv = c;
    if (off_ms) *off_ms = d;
    return o;
}

// the k slot of a transform: k_c, or -1 for a problem that is skipped -- a record of n < 2 (a weighted problem of too
// little weight) or a style entry with k_s = -1 (an empty style-mask region) -- then the sweeps
__global__ void k_transform_kout(const int* __restrict__ kc, const double* __restrict__ rn, const int* __restrict__ ks, int Nc, int Ns,
                                 int* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Nc) return;
    out[i] = (rn[i] < 2.0 || ks[Ns == 1 ? 0 : i] == -1) ? -1 : kc[i];
    out[Nc + i] = kc[Nc + i];
}

int launch_wct_transform_from_stats(const void* record, int Nc, int C, const void* state, int Ns, float alpha, float eps_cov,
                                    float eps_eig, float thresh, int readd, void* transform, void* ws, size_t ws_bytes,
                                    cudaStream_t st) {
    WCTB_REQUIRE(C == 64 || C == 128 || C == 256 || C == 512, "wct_transform_from_stats: C=%d not in {64,128,256,512}", C);
    WCTB_REQUIRE(Ns == 1 || Ns == Nc, "wct_transform_from_stats: Ns must be 1 or Nc");
    const WctWs L = wct_layout(C, Nc, 0);
    if (ws_bytes < L.total) {
        set_error("wct_transform_from_stats: workspace %zu < %zu bytes", ws_bytes, L.total);
        return WCTB200_EWS;
    }
    uint8_t* w = static_cast<uint8_t*>(ws);
    size_t off_cs, off_k;
    style_state_offsets(C, Ns, &off_cs, &off_k);
    const uint8_t* sp = static_cast<const uint8_t*>(state);
    int* kc = reinterpret_cast<int*>(w + L.kcount);
    WCTB_CUDA(cudaMemsetAsync(kc, 0, (size_t)Nc * 2 * 4, st));
    int rc = launch_record_cov_finalize(stats_record_at(record, C, Nc, 0), C, Nc, eps_cov, reinterpret_cast<float*>(w + L.mean),
                                        reinterpret_cast<float*>(w + L.G), reinterpret_cast<float*>(w + L.A0), st);
    if (rc) return rc;
    rc = wct_whiten(Nc, C, eps_eig, thresh, w, L, st);
    if (rc) return rc;
    size_t om, ob, ok, oexp;
    wct_transform_layout(C, Nc, &om, &ob, &ok, &oexp);
    uint8_t* tp = static_cast<uint8_t*>(transform);
    rc = wct_colour_transform(Nc, C, reinterpret_cast<const float*>(sp + off_cs), reinterpret_cast<const float*>(sp), Ns, alpha, readd,
                              w, L, reinterpret_cast<__half*>(tp + om), reinterpret_cast<int*>(tp + oexp),
                              reinterpret_cast<float*>(tp + ob), st);
    if (rc) return rc;
    k_transform_kout<<<(unsigned)cdiv(Nc, 256), 256, 0, st>>>(kc, stats_record_at(record, C, Nc, 0).n,
                                                            reinterpret_cast<const int*>(sp + off_k), Nc, Ns,
                                                            reinterpret_cast<int*>(tp + ok));
    WCTB_CHECK_LAUNCH("k_transform_kout");
    return 0;
}
int launch_wct_transform_apply(const __half* act, int N, int H, int W, int C, const void* transform, __half* out, cudaStream_t st) {
    WCTB_REQUIRE(C == 64 || C == 128 || C == 256 || C == 512, "wct_transform_apply: C=%d not in {64,128,256,512}", C);
    size_t om, ob, oexp;
    wct_transform_layout(C, N, &om, &ob, nullptr, &oexp);
    const uint8_t* tp = static_cast<const uint8_t*>(transform);
    return launch_conv_apply(act, N, H, W, C, reinterpret_cast<const __half*>(tp + om), N,
                          reinterpret_cast<const int*>(tp + oexp), reinterpret_cast<const float*>(tp + ob), out, st);
}

// ---------------------------------------------------------------------------
// Optimal-transport transform (OST, DESIGN.md §3.3.8): the Monge map between the content and style Gaussians,
//   M = W_c B^1/2 W_c,   B = S_c C_s C_s S_c,   S_c = W_c (A_c + eps_eig I) = E_k (lambda + eps_eig)^+1/2 E_k^T,
// in place of T = C_s W_c.  The content side (W_c) is wct_apply's and the style state is the WCT state unchanged; B^1/2
// takes the matrix-function fast path where it converges (thresh = eps = 0: the guard reduces to convergence) and the
// one-sided Jacobi solver on P = S_c C_s elsewhere (k_root_post: B^1/2 = sum sigma_i u_i u_i^T).  The products are
// k_outer_gemm's A^T B; every operand is symmetric.
//   workspace: wct_layout(C, Nc, 0) | S [Nc][C][C] (S_c, then B^1/2) | Q [Nc][C][C] (C_s S_c, then B^1/2 W_c)
//              | B [Nc][C][C] | Gb [Nc][C][C] (Q, rotated in place by the eigensolver) | ok_b [Nc] | sweeps_b [Nc]
// ---------------------------------------------------------------------------
// B^1/2 from the one-sided Jacobi solver run on the columns of P = S_c C_s (B = P P^T) instead of on B: the solver rotates
// them into g_i = sigma_i u_i with P P^T = sum sigma_i^2 u_i u_i^T, so  B^1/2 = sum sigma_i u_i u_i^T = G diag(1 / |g_i|) G^T.
// The singular values come out with an absolute error of ~the solver's tolerance times sigma_max; B's eigenvalues would carry
// that error squared relative to mu_max, and their roots ~1e-4 sqrt(mu_max) on every null direction, which W_c then
// amplifies by up to 1 / (lambda_min + eps_eig).  A column whose squared norm is below 1e-11 of the largest is one the solver
// treats as null (k_jacobi's null2: below what fp32 resolves) and gets d = 0: sigma_i = 0, sqrt(max(mu, 0)) of the oracle.
__global__ void __launch_bounds__(256)
k_root_post(const float* __restrict__ Gall, int C, float* __restrict__ dvec, const int* __restrict__ skip) {
    const int prob = blockIdx.x;
    if (skip && skip[prob]) return;
    __shared__ float ss_col[512];
    __shared__ float red[8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float m = 0.f;
    for (int col = warp; col < C; col += 8) {
        const float* g = Gall + ((long long)prob * C + col) * C;
        float ss = 0.f;
        for (int i = lane; i < C; i += 32) ss = fmaf(g[i], g[i], ss);
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
        if (lane == 0) ss_col[col] = ss;
        m = fmaxf(m, ss);
    }
    if (lane == 0) red[warp] = m;
    __syncthreads();
    float smax = 0.f;
    for (int i = 0; i < 8; ++i) smax = fmaxf(smax, red[i]);
    const float floor_ss = 1e-11f * smax;
    for (int col = threadIdx.x; col < C; col += blockDim.x) {
        const float ss = ss_col[col];
        dvec[(long long)prob * C + col] = (ss > floor_ss && ss > 0.f) ? rsqrtf(ss) : 0.f;
    }
}

__global__ void k_add_scaled(float* __restrict__ dst, const float* __restrict__ src, float a, long long n) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        dst[i] = fmaf(a, src[i], dst[i]);
}

struct OstWs {
    WctWs L;
    size_t S, Q, B, Gb, okb, swb, total;
};
static OstWs ost_layout(int C, int Nc) {
    OstWs o;
    o.L = wct_layout(C, Nc, 0);
    size_t p = o.L.total;
    auto take = [&](size_t bytes) { size_t r = p; p = align_up(p + bytes, 256); return r; };
    const size_t mat = (size_t)Nc * C * C * 4;
    o.S = take(mat);
    o.Q = take(mat);
    o.B = take(mat);
    o.Gb = take(mat);
    o.okb = take((size_t)Nc * 4);
    o.swb = take((size_t)Nc * 4);
    o.total = p;
    return o;
}
size_t ost_workspace_bytes(int C, int Nc) { return ost_layout(C, Nc).total; }

// after wct_content_side / wct_whiten: M into L.T, then the split operand and bias of k_finalize_transform
static int ost_transform(int Nc, int C, const float* Cs, const float* mean_s, int Ns, float alpha, int readd, float eps_eig,
                         uint8_t* w, const OstWs& O, __half* Msplit, int* Mexp, float* bias, cudaStream_t st) {
    const WctWs& L = O.L;
    const long long CC = (long long)C * C;
    const float* mean = reinterpret_cast<const float*>(w + L.mean);
    const float* A0 = reinterpret_cast<const float*>(w + L.A0);
    const float* Wcm = reinterpret_cast<const float*>(w + L.Wc);
    float* T = reinterpret_cast<float*>(w + L.T);
    float* S = reinterpret_cast<float*>(w + O.S);
    float* Q = reinterpret_cast<float*>(w + O.Q);
    float* B = reinterpret_cast<float*>(w + O.B);
    float* Gb = reinterpret_cast<float*>(w + O.Gb);
    int* okb = reinterpret_cast<int*>(w + O.okb);
    int* swb = reinterpret_cast<int*>(w + O.swb);
    const dim3 gg((unsigned)(C / 64), (unsigned)(C / 64), (unsigned)Nc);
    k_outer_gemm<<<gg, 256, 0, st>>>(Wcm, CC, A0, CC, nullptr, 0, S, CC, C);                  // S_c = W_c A_c
    WCTB_CHECK_LAUNCH("k_outer_gemm(Sc)");
    if (eps_eig != 0.f) {                                                                     // + eps_eig W_c
        k_add_scaled<<<cdiv((long long)Nc * CC, 256) > 1024 ? 1024 : cdiv((long long)Nc * CC, 256), 256, 0, st>>>(S, Wcm, eps_eig,
                                                                                                              (long long)Nc * CC);
        WCTB_CHECK_LAUNCH("k_add_scaled(Sc)");
    }
    k_outer_gemm<<<gg, 256, 0, st>>>(Cs, Ns == 1 ? 0 : CC, S, CC, nullptr, 0, Q, CC, C);      // Q = C_s S_c
    WCTB_CHECK_LAUNCH("k_outer_gemm(Q)");
    k_outer_gemm<<<gg, 256, 0, st>>>(Q, CC, Q, CC, nullptr, 0, B, CC, C);                     // B = Q^T Q (bit-symmetric)
    WCTB_CHECK_LAUNCH("k_outer_gemm(B)");
    // the rows of Q are the columns of P = S_c C_s: the eigensolver's input where the fast path does not take B
    WCTB_CUDA(cudaMemcpyAsync(Gb, Q, (size_t)Nc * CC * 4, cudaMemcpyDeviceToDevice, st));
    // B^1/2 into S: Newton-Schulz where it converges, else the singular values of P by the one-sided Jacobi solver
    int rc = launch_matfun_ns(B, C, Nc, /*n_first=*/0, /*thresh=*/0.f, /*eps_eig=*/0.f, S, okb, nullptr, st);
    if (rc < 0) return rc;
    rc = launch_jacobi(Gb, C, Nc, reinterpret_cast<float*>(w + L.conv), swb, st, okb, /*thresh=*/0.f);
    if (rc) return rc;
    k_root_post<<<(unsigned)Nc, 256, 0, st>>>(Gb, C, reinterpret_cast<float*>(w + L.dvec), okb);
    WCTB_CHECK_LAUNCH("k_root_post");
    k_outer_gemm<<<gg, 256, 0, st>>>(Gb, CC, Gb, CC, reinterpret_cast<const float*>(w + L.dvec), C, S, CC, C, okb);
    WCTB_CHECK_LAUNCH("k_outer_gemm(B^1/2)");
    k_outer_gemm<<<gg, 256, 0, st>>>(S, CC, Wcm, CC, nullptr, 0, Q, CC, C);                   // B^1/2 W_c
    WCTB_CHECK_LAUNCH("k_outer_gemm(B^1/2 Wc)");
    k_outer_gemm<<<gg, 256, 0, st>>>(Wcm, CC, Q, CC, nullptr, 0, T, CC, C);                   // M = W_c B^1/2 W_c
    WCTB_CHECK_LAUNCH("k_outer_gemm(M)");
    const dim3 gf((unsigned)cdiv(C, 8), (unsigned)Nc);
    k_finalize_transform<<<gf, 256, 0, st>>>(T, C, Nc, Ns, alpha, readd, mean, mean_s, Msplit, Mexp, bias);
    WCTB_CHECK_LAUNCH("k_finalize_transform");
    return 0;
}

int launch_ost_apply(const __half* content, int Nc, int Hc, int Wc, int C, const void* state, int Ns, float alpha,
                     float eps_cov, float eps_eig, float thresh, int readd, __half* out, int32_t* k_out, void* ws,
                     size_t ws_bytes, cudaStream_t st) {
    WCTB_REQUIRE(C == 64 || C == 128 || C == 256 || C == 512, "ost_apply: C=%d not in {64,128,256,512}", C);
    WCTB_REQUIRE(Ns == 1 || Ns == Nc, "ost_apply: Ns must be 1 or Nc");
    const OstWs O = ost_layout(C, Nc);
    if (ws_bytes < O.total) {
        set_error("ost_apply: workspace %zu < %zu bytes", ws_bytes, O.total);
        return WCTB200_EWS;
    }
    uint8_t* w = static_cast<uint8_t*>(ws);
    size_t off_cs, off_k;
    style_state_offsets(C, Ns, &off_cs, &off_k);
    const uint8_t* sp = static_cast<const uint8_t*>(state);
    int rc = wct_content_side(content, Nc, Hc, Wc, C, eps_cov, eps_eig, thresh, w, O.L, st);
    if (rc) return rc;
    __half* Msplit = reinterpret_cast<__half*>(w + O.L.Msplit);
    int* Mexp = reinterpret_cast<int*>(w + O.L.Mexp);
    float* bias = reinterpret_cast<float*>(w + O.L.bias);
    rc = ost_transform(Nc, C, reinterpret_cast<const float*>(sp + off_cs), reinterpret_cast<const float*>(sp), Ns, alpha, readd,
                       eps_eig, w, O, Msplit, Mexp, bias, st);
    if (rc) return rc;
    rc = launch_conv_apply(content, Nc, Hc, Wc, C, Msplit, Nc, Mexp, bias, out, st);
    if (rc) return rc;
    if (k_out) {
        // k_out: [k_c x Nc | sweeps_c x Nc | ok_c x Nc | ok_b x Nc | sweeps_b x Nc]
        WCTB_CUDA(cudaMemcpyAsync(k_out, w + O.L.kcount, (size_t)Nc * 2 * 4, cudaMemcpyDeviceToDevice, st));
        WCTB_CUDA(cudaMemcpyAsync(k_out + 2 * Nc, w + O.L.ok, (size_t)Nc * 4, cudaMemcpyDeviceToDevice, st));
        WCTB_CUDA(cudaMemcpyAsync(k_out + 3 * Nc, w + O.okb, (size_t)Nc * 4, cudaMemcpyDeviceToDevice, st));
        WCTB_CUDA(cudaMemcpyAsync(k_out + 4 * Nc, w + O.swb, (size_t)Nc * 4, cudaMemcpyDeviceToDevice, st));
    }
    return 0;
}

int launch_ost_transform_from_stats(const void* record, int Nc, int C, const void* state, int Ns, float alpha, float eps_cov,
                                    float eps_eig, float thresh, int readd, void* transform, void* ws, size_t ws_bytes,
                                    cudaStream_t st) {
    WCTB_REQUIRE(C == 64 || C == 128 || C == 256 || C == 512, "ost_transform_from_stats: C=%d not in {64,128,256,512}", C);
    WCTB_REQUIRE(Ns == 1 || Ns == Nc, "ost_transform_from_stats: Ns must be 1 or Nc");
    const OstWs O = ost_layout(C, Nc);
    if (ws_bytes < O.total) {
        set_error("ost_transform_from_stats: workspace %zu < %zu bytes", ws_bytes, O.total);
        return WCTB200_EWS;
    }
    uint8_t* w = static_cast<uint8_t*>(ws);
    size_t off_cs, off_k;
    style_state_offsets(C, Ns, &off_cs, &off_k);
    const uint8_t* sp = static_cast<const uint8_t*>(state);
    int* kc = reinterpret_cast<int*>(w + O.L.kcount);
    WCTB_CUDA(cudaMemsetAsync(kc, 0, (size_t)Nc * 2 * 4, st));
    int rc = launch_record_cov_finalize(stats_record_at(record, C, Nc, 0), C, Nc, eps_cov, reinterpret_cast<float*>(w + O.L.mean),
                                        reinterpret_cast<float*>(w + O.L.G), reinterpret_cast<float*>(w + O.L.A0), st);
    if (rc) return rc;
    rc = wct_whiten(Nc, C, eps_eig, thresh, w, O.L, st);
    if (rc) return rc;
    size_t om, ob, ok, oexp;
    wct_transform_layout(C, Nc, &om, &ob, &ok, &oexp);
    uint8_t* tp = static_cast<uint8_t*>(transform);
    rc = ost_transform(Nc, C, reinterpret_cast<const float*>(sp + off_cs), reinterpret_cast<const float*>(sp), Ns, alpha, readd,
                       eps_eig, w, O, reinterpret_cast<__half*>(tp + om), reinterpret_cast<int*>(tp + oexp),
                       reinterpret_cast<float*>(tp + ob), st);
    if (rc) return rc;
    k_transform_kout<<<(unsigned)cdiv(Nc, 256), 256, 0, st>>>(kc, stats_record_at(record, C, Nc, 0).n,
                                                            reinterpret_cast<const int*>(sp + off_k), Nc, Ns,
                                                            reinterpret_cast<int*>(tp + ok));
    WCTB_CHECK_LAUNCH("k_transform_kout");
    return 0;
}

static size_t adain_state_offsets(int C, int Ns, size_t* off_var);
int launch_adain_transform_from_stats(const void* record, int Nc, int C, const void* state, int Ns, float eps, void* transform,
                                      cudaStream_t st) {
    WCTB_REQUIRE(C % 8 == 0 && C <= 2048, "adain_transform_from_stats: C=%d must be a multiple of 8 (<= 2048)", C);
    WCTB_REQUIRE(Ns == 1 || Ns == Nc, "adain_transform_from_stats: Ns must be 1 or Nc");
    size_t off_var, a, b, c, d;
    adain_state_offsets(C, Ns, &off_var);
    adain_transform_layout(C, Nc, &a, &b, &c, &d);
    const uint8_t* sp = static_cast<const uint8_t*>(state);
    uint8_t* tp = static_cast<uint8_t*>(transform);
    float* mean = reinterpret_cast<float*>(tp + a);
    float* var = reinterpret_cast<float*>(tp + b);
    k_record_moments_finalize<<<cdiv((long long)Nc * C, 256), 256, 0, st>>>(stats_record_at(record, C, Nc, 1), C, Nc * C, mean, var);
    WCTB_CHECK_LAUNCH("k_record_moments_finalize");
    k_adain_coeffs<<<cdiv((long long)Nc * C, 256), 256, 0, st>>>(var, reinterpret_cast<const float*>(sp), reinterpret_cast<const float*>(sp + off_var),
                                                              C, Nc, Ns, eps, reinterpret_cast<float*>(tp + c), reinterpret_cast<float*>(tp + d));
    WCTB_CHECK_LAUNCH("k_adain_coeffs");
    return 0;
}
int launch_adain_transform_apply(const __half* act, int N, int H, int W, int C, const void* transform, float alpha, __half* out,
                                 cudaStream_t st) {
    WCTB_REQUIRE(C % 8 == 0 && C <= 2048, "adain_transform_apply: C=%d must be a multiple of 8 (<= 2048)", C);
    size_t a, c, d;
    adain_transform_layout(C, N, &a, nullptr, &c, &d);
    const uint8_t* tp = static_cast<const uint8_t*>(transform);
    const long long total = (long long)N * H * W * (C / 8);
    long long blocks = (total + 255) / 256;
    if (blocks > device_sm_count() * 16) blocks = device_sm_count() * 16;
    k_affine_apply<<<(unsigned)blocks, 256, 0, st>>>(act, ActGeom(N, H, W, C), reinterpret_cast<const float*>(tp + a),
                                                     reinterpret_cast<const float*>(tp + c), reinterpret_cast<const float*>(tp + d),
                                                     alpha, out);
    WCTB_CHECK_LAUNCH("k_affine_apply");
    return 0;
}
int launch_adain_transform_apply_strength(const __half* act, int N, int H, int W, int C, const void* transform, float alpha,
                                          const float* strength, __half* out, cudaStream_t st) {
    WCTB_REQUIRE(C % 8 == 0 && C <= 2048, "adain_transform_apply_strength: C=%d must be a multiple of 8 (<= 2048)", C);
    size_t a, c, d;
    adain_transform_layout(C, N, &a, nullptr, &c, &d);
    const uint8_t* tp = static_cast<const uint8_t*>(transform);
    const long long total = (long long)N * H * W * (C / 8);
    long long blocks = (total + 255) / 256;
    if (blocks > device_sm_count() * 16) blocks = device_sm_count() * 16;
    k_affine_apply_strength<<<(unsigned)blocks, 256, 0, st>>>(act, ActGeom(N, H, W, C), reinterpret_cast<const float*>(tp + a),
                                                              reinterpret_cast<const float*>(tp + c), reinterpret_cast<const float*>(tp + d),
                                                              alpha, strength, out);
    WCTB_CHECK_LAUNCH("k_affine_apply_strength");
    return 0;
}

// ---------------------------------------------------------------------------
// Style interpolation (WCT paper, section 4): a weighted blend of K styles.  Both transforms are affine in the style
// statistics, so for weights that sum to 1 the blend of the K outputs is the transform of the blended statistics:
//   WCT    sum_k w_k (a (C_sk W_c (x - m_c) + m_sk) + (1 - a) base) = a (C_w W_c (x - m_c) + m_w) + (1 - a) base,
//          C_w = sum_k w_k C_sk, m_w = sum_k w_k m_sk;
//   AdaIN  the same with sigma_w = sum_k w_k sqrt(v_sk) and mu_w = sum_k w_k mu_sk.
// The blend runs on the small per-style state; the content side and the tensor-core apply run once.
// ---------------------------------------------------------------------------
struct BlendSrc {
    const float* Cs[8];
    const float* ms[8];
};

// For every weight row (blockIdx.y of Nw rows of K): Cs_w = sum_k w[k] Cs_k and ms_w = sum_k w[k] ms_k, an fp32 fmaf chain
// in k order that starts from the product w[0] S_0.  A one-hot row reproduces its style bit for bit.
__global__ void __launch_bounds__(256)
k_blend_styles(BlendSrc src, int K, const float* __restrict__ weights, int C, float* __restrict__ Cs, float* __restrict__ ms) {
    const int row = blockIdx.y;
    const long long CC4 = (long long)C * C / 4, n4 = CC4 + C / 4;
    float wk[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) wk[k] = k < K ? weights[(long long)row * K + k] : 0.f;
    float4* cs_out = reinterpret_cast<float4*>(Cs + (long long)row * C * C);
    float4* ms_out = reinterpret_cast<float4*>(ms + (long long)row * C);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const bool is_cs = i < CC4;
        const long long j = is_cs ? i : i - CC4;
        float4 s = is_cs ? reinterpret_cast<const float4*>(src.Cs[0])[j] : reinterpret_cast<const float4*>(src.ms[0])[j];
        float4 a = make_float4(__fmul_rn(wk[0], s.x), __fmul_rn(wk[0], s.y), __fmul_rn(wk[0], s.z), __fmul_rn(wk[0], s.w));
#pragma unroll
        for (int k = 1; k < 8; ++k) {
            if (k < K) {
                s = is_cs ? reinterpret_cast<const float4*>(src.Cs[k])[j] : reinterpret_cast<const float4*>(src.ms[k])[j];
                a = make_float4(fmaf(wk[k], s.x, a.x), fmaf(wk[k], s.y, a.y), fmaf(wk[k], s.z, a.z), fmaf(wk[k], s.w, a.w));
            }
        }
        if (is_cs) cs_out[j] = a;
        else ms_out[j] = a;
    }
}

struct BlendWs {
    size_t base, Cs, ms, total;
};
static BlendWs blend_layout(int C, int Nc, int Nw) {
    BlendWs L;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o = align_up(o + bytes, 256); return r; };
    L.base = take(wct_layout(C, Nc, 0).total);   // the content side and apply, as wct_apply's
    L.Cs = take((size_t)Nw * C * C * 4);         // the blended style states, one per weight row
    L.ms = take((size_t)Nw * C * 4);
    L.total = o;
    return L;
}
size_t wct_blend_workspace_bytes(int C, int Nc, int K, int Nw) {
    (void)K;
    return blend_layout(C, Nc, Nw).total;
}

int launch_wct_apply_blend(const __half* content, int Nc, int Hc, int Wc, int C, const void* const* states, int K,
                           const float* weights, int Nw, float alpha, float eps_cov, float eps_eig, float thresh, int readd,
                           __half* out, int32_t* k_out, void* ws, size_t ws_bytes, cudaStream_t st) {
    WCTB_REQUIRE(C == 64 || C == 128 || C == 256 || C == 512, "wct_apply_blend: C=%d not in {64,128,256,512}", C);
    WCTB_REQUIRE(K >= 1 && K <= 8, "wct_apply_blend: K=%d not in 1..8", K);
    WCTB_REQUIRE(Nw == 1 || Nw == Nc, "wct_apply_blend: Nw=%d must be 1 or Nc=%d", Nw, Nc);
    const BlendWs BL = blend_layout(C, Nc, Nw);
    if (ws_bytes < BL.total) {
        set_error("wct_apply_blend: workspace %zu < %zu bytes", ws_bytes, BL.total);
        return WCTB200_EWS;
    }
    // each state from wct_style_prepare with Ns = 1: [C] mean_s | [C][C] C_s | k_s, sweeps
    size_t off_cs, off_k;
    style_state_offsets(C, 1, &off_cs, &off_k);
    BlendSrc src = {};
    for (int k = 0; k < K; ++k) {
        WCTB_REQUIRE(states[k], "wct_apply_blend: style state %d is null", k);
        const uint8_t* sp = static_cast<const uint8_t*>(states[k]);
        src.ms[k] = reinterpret_cast<const float*>(sp);
        src.Cs[k] = reinterpret_cast<const float*>(sp + off_cs);
    }
    const WctWs L = wct_layout(C, Nc, 0);
    uint8_t* w = static_cast<uint8_t*>(ws) + BL.base;
    float* Cs = reinterpret_cast<float*>(static_cast<uint8_t*>(ws) + BL.Cs);
    float* ms = reinterpret_cast<float*>(static_cast<uint8_t*>(ws) + BL.ms);
    int rc = wct_content_side(content, Nc, Hc, Wc, C, eps_cov, eps_eig, thresh, w, L, st);
    if (rc) return rc;
    const long long n4 = ((long long)C * C + C) / 4;
    long long blocks = cdiv(n4, 256);
    if (blocks > device_sm_count() * 4ll) blocks = device_sm_count() * 4ll;
    k_blend_styles<<<dim3((unsigned)blocks, (unsigned)Nw), 256, 0, st>>>(src, K, weights, C, Cs, ms);
    WCTB_CHECK_LAUNCH("k_blend_styles");
    rc = wct_colour_apply(content, Nc, Hc, Wc, C, Cs, ms, Nw, alpha, readd, w, L, out, st);
    if (rc) return rc;
    if (k_out) {
        // k_out: [k_c x Nc | k_s x K | sweeps_c x Nc | sweeps_s x K]
        const int* kc = reinterpret_cast<const int*>(w + L.kcount);
        WCTB_CUDA(cudaMemcpyAsync(k_out, kc, (size_t)Nc * 4, cudaMemcpyDeviceToDevice, st));
        WCTB_CUDA(cudaMemcpyAsync(k_out + Nc + K, kc + Nc, (size_t)Nc * 4, cudaMemcpyDeviceToDevice, st));
        for (int k = 0; k < K; ++k) {
            const int* ks = reinterpret_cast<const int*>(static_cast<const uint8_t*>(states[k]) + off_k);
            WCTB_CUDA(cudaMemcpyAsync(k_out + Nc + k, ks, 4, cudaMemcpyDeviceToDevice, st));
            WCTB_CUDA(cudaMemcpyAsync(k_out + 2 * Nc + K + k, ks + 1, 4, cudaMemcpyDeviceToDevice, st));
        }
    }
    return 0;
}

// test / profiling hook: means and covariance of a feature batch (stage A of the transform)
int launch_covariance(const __half* act, int N, int H, int W, int C, float eps_cov, float* mean_out, float* cov_out,
                      cudaStream_t st) {
    WCTB_REQUIRE(C == 64 || (C % 128 == 0 && C >= 128), "covariance: C=%d must be 64 or a multiple of 128", C);
    double* dsum = nullptr;
    { int rc0 = scratch_alloc(reinterpret_cast<void**>(&dsum), (size_t)N * C * sizeof(double), st, 1); if (rc0) return rc0; }
    return launch_mean_cov(act, ActGeom(N, H, W, C), eps_cov, mean_out, cov_out, nullptr, dsum, st);
}

// ---------------------------------------------------------------------------
// AdaIN in split form: the style side is the per-channel moments of the style, which depend on the style features only.
//   state layout: [Ns][C] mean | [Ns][C] var (fp32, biased; what k_moments_finalize writes), 256-byte aligned blocks
// The apply computes the content moments, the coefficients and the affine map in the workspace of
// wct_layout(C, Nc, 0) (fields shift, mean, var, inv, ms).  adain_level and adain_blend are prepare followed by apply.
// ---------------------------------------------------------------------------
static size_t adain_state_offsets(int C, int Ns, size_t* off_var) {
    *off_var = align_up((size_t)Ns * C * 4, 256);
    return align_up(*off_var + (size_t)Ns * C * 4, 256);
}
size_t adain_style_state_layout(int C, int Ns, size_t* off_mean, size_t* off_var) {
    size_t ov;
    const size_t total = adain_state_offsets(C, Ns, &ov);
    if (off_mean) *off_mean = 0;
    if (off_var) *off_var = ov;
    return total;
}

int launch_adain_style_prepare(const __half* style, int Ns, int Hs, int Ws, int C, void* state, cudaStream_t st) {
    WCTB_REQUIRE(C % 8 == 0 && C <= 2048, "adain_style_prepare: C=%d must be a multiple of 8 (<= 2048)", C);
    size_t off_var;
    adain_state_offsets(C, Ns, &off_var);
    // centring shift and slot partials in the per-stream scratch
    const size_t nshift = align_up((size_t)Ns * C, 64);
    const size_t part = (size_t)Ns * cdiv((long long)Hs * Ws, moments_slice(C)) * 2 * C;
    float* scratch = nullptr;
    { int rc0 = scratch_alloc(reinterpret_cast<void**>(&scratch), (nshift + part) * sizeof(float), st, 5); if (rc0) return rc0; }
    uint8_t* sp = static_cast<uint8_t*>(state);
    return launch_moments(style, ActGeom(Ns, Hs, Ws, C), scratch, scratch + nshift, reinterpret_cast<float*>(sp),
                          reinterpret_cast<float*>(sp + off_var), st);
}

// content moments of the apply calls into the workspace of wct_layout(C, Nc, 0)
static int adain_content_moments(const __half* content, int Nc, int Hc, int Wc, int C, uint8_t* w, const WctWs& L, cudaStream_t st) {
    const size_t part_c = (size_t)Nc * cdiv((long long)Hc * Wc, moments_slice(C)) * 2 * C;
    float* part = nullptr;
    { int rc0 = scratch_alloc(reinterpret_cast<void**>(&part), part_c * sizeof(float), st, 5); if (rc0) return rc0; }
    return launch_moments(content, ActGeom(Nc, Hc, Wc, C), reinterpret_cast<float*>(w + L.shift), part, reinterpret_cast<float*>(w + L.mean),
                          reinterpret_cast<float*>(w + L.var), st);
}
static int adain_affine(const __half* content, int Nc, int Hc, int Wc, int C, float alpha, uint8_t* w, const WctWs& L, __half* out,
                        cudaStream_t st) {
    const long long total = (long long)Nc * Hc * Wc * (C / 8);
    long long blocks = (total + 255) / 256;
    if (blocks > device_sm_count() * 16) blocks = device_sm_count() * 16;
    k_affine_apply<<<(unsigned)blocks, 256, 0, st>>>(content, ActGeom(Nc, Hc, Wc, C), reinterpret_cast<const float*>(w + L.mean),
                                                     reinterpret_cast<const float*>(w + L.inv), reinterpret_cast<const float*>(w + L.ms),
                                                     alpha, out);
    WCTB_CHECK_LAUNCH("k_affine_apply");
    return 0;
}

int launch_adain_apply(const __half* content, int Nc, int Hc, int Wc, int C, const void* state, int Ns, float alpha, float eps,
                       __half* out, void* ws, size_t ws_bytes, cudaStream_t st) {
    WCTB_REQUIRE(C % 8 == 0 && C <= 2048, "adain_apply: C=%d must be a multiple of 8 (<= 2048)", C);
    WCTB_REQUIRE(Ns == 1 || Ns == Nc, "adain_apply: Ns must be 1 or Nc");
    const WctWs L = wct_layout(C, Nc, 0);
    if (ws_bytes < L.total) {
        set_error("adain_apply: workspace %zu < %zu bytes", ws_bytes, L.total);
        return WCTB200_EWS;
    }
    uint8_t* w = static_cast<uint8_t*>(ws);
    size_t off_var;
    adain_state_offsets(C, Ns, &off_var);
    const uint8_t* sp = static_cast<const uint8_t*>(state);
    int rc = adain_content_moments(content, Nc, Hc, Wc, C, w, L, st);
    if (rc) return rc;
    k_adain_coeffs<<<cdiv((long long)Nc * C, 256), 256, 0, st>>>(reinterpret_cast<const float*>(w + L.var), reinterpret_cast<const float*>(sp),
                                                              reinterpret_cast<const float*>(sp + off_var), C, Nc, Ns, eps,
                                                              reinterpret_cast<float*>(w + L.inv), reinterpret_cast<float*>(w + L.ms));
    WCTB_CHECK_LAUNCH("k_adain_coeffs");
    return adain_affine(content, Nc, Hc, Wc, C, alpha, w, L, out, st);
}

int launch_adain_level(const __half* content, int Nc, int Hc, int Wc, const __half* style, int Ns, int Hs, int Ws, int C,
                       float alpha, float eps, __half* out, void* ws, size_t ws_bytes, cudaStream_t st) {
    WCTB_REQUIRE(C % 8 == 0 && C <= 2048, "adain_level: C=%d must be a multiple of 8 (<= 2048)", C);
    WCTB_REQUIRE(Ns == 1 || Ns == Nc, "adain_level: Ns must be 1 or Nc");
    const size_t need = wct_layout(C, Nc, Ns).total;
    if (ws_bytes < need) {
        set_error("adain_level: workspace %zu < %zu bytes", ws_bytes, need);
        return WCTB200_EWS;
    }
    // the apply's workspace, then the style state (wct_layout(C, Nc, Ns) holds both)
    const size_t base = wct_layout(C, Nc, 0).total;
    size_t off_var;
    const size_t sbytes = adain_state_offsets(C, Ns, &off_var);
    WCTB_REQUIRE(base + sbytes <= need, "adain_level: workspace layout");
    uint8_t* state = static_cast<uint8_t*>(ws) + base;
    int rc = launch_adain_style_prepare(style, Ns, Hs, Ws, C, state, st);
    if (rc) return rc;
    return launch_adain_apply(content, Nc, Hc, Wc, C, state, Ns, alpha, eps, out, ws, base, st);
}

// AdaIN of a style blend: inv = rsqrt(vc + eps) * sum_k w_k sqrt(v_sk) and ms = sum_k w_k m_sk per (frame, channel), in k
// order from the product w_0 S_0 (K = 1 with weight 1 gives k_adain_coeffs' values bit for bit).  Weight row z, or 0 if Nw == 1.
struct AdainSrc {
    const float* mean[8];
    const float* var[8];
};
__global__ void k_adain_blend_coeffs(const float* __restrict__ var_c, AdainSrc src, int C, int Nc, int K,
                                     const float* __restrict__ weights, int Nw, float eps, float* __restrict__ inv,
                                     float* __restrict__ ms) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Nc * C) return;
    const int z = i / C, c = i % C;
    const float* wr = weights + (long long)(Nw == 1 ? 0 : z) * K;
    float s = __fmul_rn(wr[0], sqrtf(src.var[0][c])), m = __fmul_rn(wr[0], src.mean[0][c]);
#pragma unroll
    for (int k = 1; k < 8; ++k) {              // unrolled: the state pointers stay in the parameter space
        if (k < K) {
            s = fmaf(wr[k], sqrtf(src.var[k][c]), s);
            m = fmaf(wr[k], src.mean[k][c], m);
        }
    }
    inv[i] = rsqrtf(var_c[i] + eps) * s;
    ms[i] = m;
}

int launch_adain_apply_blend(const __half* content, int Nc, int Hc, int Wc, int C, const void* const* states, int K,
                             const float* weights, int Nw, float alpha, float eps, __half* out, void* ws, size_t ws_bytes,
                             cudaStream_t st) {
    WCTB_REQUIRE(C % 8 == 0 && C <= 2048, "adain_apply_blend: C=%d must be a multiple of 8 (<= 2048)", C);
    WCTB_REQUIRE(K >= 1 && K <= 8, "adain_apply_blend: K=%d not in 1..8", K);
    WCTB_REQUIRE(Nw == 1 || Nw == Nc, "adain_apply_blend: Nw=%d must be 1 or Nc=%d", Nw, Nc);
    const WctWs L = wct_layout(C, Nc, 0);
    if (ws_bytes < L.total) {
        set_error("adain_apply_blend: workspace %zu < %zu bytes", ws_bytes, L.total);
        return WCTB200_EWS;
    }
    // each state from adain_style_prepare with Ns = 1: [C] mean | [C] var
    size_t off_var;
    adain_state_offsets(C, 1, &off_var);
    AdainSrc src = {};
    for (int k = 0; k < K; ++k) {
        WCTB_REQUIRE(states[k], "adain_apply_blend: style state %d is null", k);
        src.mean[k] = static_cast<const float*>(states[k]);
        src.var[k] = reinterpret_cast<const float*>(static_cast<const uint8_t*>(states[k]) + off_var);
    }
    uint8_t* w = static_cast<uint8_t*>(ws);
    int rc = adain_content_moments(content, Nc, Hc, Wc, C, w, L, st);
    if (rc) return rc;
    k_adain_blend_coeffs<<<cdiv((long long)Nc * C, 256), 256, 0, st>>>(reinterpret_cast<const float*>(w + L.var), src, C, Nc, K, weights,
                                                                    Nw, eps, reinterpret_cast<float*>(w + L.inv),
                                                                    reinterpret_cast<float*>(w + L.ms));
    WCTB_CHECK_LAUNCH("k_adain_blend_coeffs");
    return adain_affine(content, Nc, Hc, Wc, C, alpha, w, L, out, st);
}

// adain_blend: the K style states after the apply's workspace
static size_t adain_blend_layout(int C, int Nc, int K, size_t* state_bytes) {
    *state_bytes = adain_style_state_layout(C, 1, nullptr, nullptr);
    return wct_layout(C, Nc, 0).total + (size_t)K * *state_bytes;
}
size_t adain_blend_workspace_bytes(int C, int Nc, int K) {
    size_t sb;
    return adain_blend_layout(C, Nc, K, &sb);
}

int launch_adain_blend(const __half* content, int Nc, int Hc, int Wc, int C, const void* const* styles, const int* Hs, const int* Ws,
                       int K, const float* weights, int Nw, float alpha, float eps, __half* out, void* ws, size_t ws_bytes,
                       cudaStream_t st) {
    WCTB_REQUIRE(C % 8 == 0 && C <= 2048, "adain_blend: C=%d must be a multiple of 8 (<= 2048)", C);
    WCTB_REQUIRE(K >= 1 && K <= 8, "adain_blend: K=%d not in 1..8", K);
    WCTB_REQUIRE(Nw == 1 || Nw == Nc, "adain_blend: Nw=%d must be 1 or Nc=%d", Nw, Nc);
    size_t sbytes;
    const size_t need = adain_blend_layout(C, Nc, K, &sbytes);
    if (ws_bytes < need) {
        set_error("adain_blend: workspace %zu < %zu bytes", ws_bytes, need);
        return WCTB200_EWS;
    }
    const size_t base = wct_layout(C, Nc, 0).total;
    const void* states[8];
    for (int k = 0; k < K; ++k) {
        WCTB_REQUIRE(styles[k], "adain_blend: style %d is null", k);
        WCTB_REQUIRE(Hs[k] >= 2 && Ws[k] >= 2, "adain_blend: style %d is %dx%d", k, Hs[k], Ws[k]);
        void* state = static_cast<uint8_t*>(ws) + base + (size_t)k * sbytes;
        int rc = launch_adain_style_prepare(static_cast<const __half*>(styles[k]), 1, Hs[k], Ws[k], C, state, st);
        if (rc) return rc;
        states[k] = state;
    }
    return launch_adain_apply_blend(content, Nc, Hc, Wc, C, states, K, weights, Nw, alpha, eps, out, ws, base, st);
}

// ---------------------------------------------------------------------------
// Spatial control (WCT paper, section 4): a label map splits every frame into regions and region r takes style r.  Per
// (frame, region) the transform is the reference's own, restricted to the region's pixels; labels >= R, and regions with
// fewer than 2 pixels at a level, keep the content feature.
// ---------------------------------------------------------------------------
// proportional nearest sampling of an Hm x Wm label map onto an Hf x Wf grid, integer arithmetic (no divisibility needed):
//   dst[y][x] = src[((2y+1) Hm) / (2 Hf)][((2x+1) Wm) / (2 Wf)]
__global__ void k_labels_resize(const uint8_t* __restrict__ src, int N, int Hm, int Wm, int Hf, int Wf, uint8_t* __restrict__ dst) {
    const long long total = (long long)N * Hf * Wf;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % Wf);
        const long long t = i / Wf;
        const int y = (int)(t % Hf);
        const int n = (int)(t / Hf);
        const int sy = (int)(((2ll * y + 1) * Hm) / (2ll * Hf)), sx = (int)(((2ll * x + 1) * Wm) / (2ll * Wf));
        dst[i] = src[((long long)n * Hm + sy) * Wm + sx];
    }
}
int launch_labels_resize(const uint8_t* src, int N, int Hm, int Wm, int Hf, int Wf, uint8_t* dst, cudaStream_t st) {
    const long long total = (long long)N * Hf * Wf;
    long long blocks = (total + 255) / 256;
    if (blocks > device_sm_count() * 16ll) blocks = device_sm_count() * 16ll;
    k_labels_resize<<<(unsigned)blocks, 256, 0, st>>>(src, N, Hm, Wm, Hf, Wf, dst);
    WCTB_CHECK_LAUNCH("k_labels_resize");
    return 0;
}

// one warp per 32 x 2 covariance tile (cov_tc.cu): tmask[n][tile] = regions present (bit r, r < R), counts[n*R + r] += pixels
// (integer counts: order-independent).  grid (cdiv(tiles, 8), N), 256 threads.  counts must be zeroed.
__global__ void __launch_bounds__(256)
k_region_scan(const uint8_t* __restrict__ labels, int H, int W, int R, int tiles_x, int tiles, int* __restrict__ counts,
              uint16_t* __restrict__ tmask) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int t = blockIdx.x * 8 + warp, n = blockIdx.y;
    if (t >= tiles) return;
    const int ty = t / tiles_x, tx = t - ty * tiles_x;
    const int x = tx * 32 + lane;
    int l[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const int y = ty * 2 + k;
        l[k] = (x < W && y < H) ? labels[((long long)n * H + y) * W + x] : 255;
    }
    unsigned bits = 0;
    for (int r = 0; r < R; ++r) {
        const int c = __popc(__ballot_sync(0xffffffffu, l[0] == r)) + __popc(__ballot_sync(0xffffffffu, l[1] == r));
        if (c) {
            bits |= 1u << r;
            if (lane == 0) atomicAdd(&counts[n * R + r], c);
        }
    }
    if (lane == 0) tmask[(long long)n * tiles + t] = (uint16_t)bits;
}

// per 128-position tile of the regions apply (conv_tc.cu, per-image tiling over the padded plane): bit r for every region
// whose pixels the tile transforms, bit R when it holds a pixel that keeps its input.  One warp per tile.
__global__ void __launch_bounds__(256)
k_region_apply_tiles(const uint8_t* __restrict__ labels, const int* __restrict__ counts, int N, int H, int W, int R,
                     int tiles_per_image, uint16_t* __restrict__ amask) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long t = (long long)blockIdx.x * 8 + warp;
    if (t >= (long long)N * tiles_per_image) return;
    const int n = (int)(t / tiles_per_image), mt = (int)(t - (long long)n * tiles_per_image);
    const int Wp = W + 2;
    const long long HpWp = (long long)(H + 2) * Wp;
    unsigned bits = 0;
    for (int k = lane; k < 128; k += 32) {
        const long long r = (long long)mt * 128 + k;
        if (r >= HpWp) break;
        const int yy = (int)(r / Wp), xx = (int)(r - (long long)yy * Wp);
        if (yy < 1 || yy > H || xx < 1 || xx > W) continue;
        const int l = labels[((long long)n * H + yy - 1) * W + xx - 1];
        bits |= 1u << ((l < R && counts[n * R + l] >= 2) ? l : R);
    }
    bits = __reduce_or_sync(0xffffffffu, bits);
    if (lane == 0) amask[t] = (uint16_t)bits;
}

// k_out of the regions apply: [k_c x Nc*R | k_s x R | sweeps_c x Nc*R | sweeps_s x R], k_c = -1 for a skipped (frame, region)
__global__ void k_regions_kout(const int* __restrict__ kc, const int* __restrict__ counts, const int* __restrict__ ks, int np, int R,
                               int32_t* __restrict__ k_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < np) {
        k_out[i] = counts[i] < 2 ? -1 : kc[i];
        k_out[np + R + i] = counts[i] < 2 ? 0 : kc[np + i];
    }
    if (i < R) {
        k_out[np + i] = ks[2 * i];
        k_out[2 * np + R + i] = ks[2 * i + 1];
    }
}

struct RegionWs {
    size_t base, mean_s, Cs, ks, counts, tmask, amask, total;
    int tiles_x, tiles, tiles_per_image;
};
static RegionWs regions_layout(int C, int Nc, int R, int Hc, int Wc) {
    RegionWs L;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o = align_up(o + bytes, 256); return r; };
    L.tiles_x = (Wc + 31) / 32;
    L.tiles = L.tiles_x * ((Hc + 1) / 2);
    L.tiles_per_image = cdiv((long long)(Hc + 2) * (Wc + 2), 128);
    L.base = take(wct_layout(C, Nc * R, 0).total);   // the per-(frame, region) transform, as wct_apply's for Nc*R frames
    L.mean_s = take((size_t)R * C * 4);                // the R style states, gathered
    L.Cs = take((size_t)R * C * C * 4);
    L.ks = take((size_t)R * 2 * 4);
    L.counts = take((size_t)Nc * R * 4);
    L.tmask = take((size_t)Nc * L.tiles * 2);
    L.amask = take((size_t)Nc * L.tiles_per_image * 2);
    L.total = o;
    return L;
}
size_t wct_regions_workspace_bytes(int C, int Nc, int R, int Hc, int Wc) { return regions_layout(C, Nc, R, Hc, Wc).total; }

int launch_mean_cov_regions(const __half* act, ActGeom g, const uint8_t* labels, int R, const int* counts, const uint16_t* tmask,
                            float eps_cov, float* mean, float* G, float* A0, double* dsum, cudaStream_t st);
int launch_conv_apply_regions(const __half* in, int N, int H, int W, int C, const __half* w_split, const int* rexp, const float* bias,
                              const uint8_t* labels, const int* counts, const uint16_t* amask, int R, __half* out, cudaStream_t st);

static int region_scan(const uint8_t* labels, int N, int H, int W, int R, int* counts, uint16_t* tmask, cudaStream_t st) {
    const int tiles_x = (W + 31) / 32, tiles = tiles_x * ((H + 1) / 2);
    WCTB_CUDA(cudaMemsetAsync(counts, 0, (size_t)N * R * 4, st));
    k_region_scan<<<dim3((unsigned)cdiv(tiles, 8), (unsigned)N), 256, 0, st>>>(labels, H, W, R, tiles_x, tiles, counts, tmask);
    WCTB_CHECK_LAUNCH("k_region_scan");
    return 0;
}

// a style state entry with k_s = -1 (a style mask region of < 2 pixels, wct_style_prepare_regions) keeps region r of every
// frame: its pixel counts drop to 0, and every consumer skips a (frame, region) with counts < 2
__global__ void k_regions_drop_empty_styles(const int* __restrict__ ks, int np, int R, int* __restrict__ counts) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < np && ks[2 * (i % R)] == -1) counts[i] = 0;
}

int launch_wct_apply_regions(const __half* content, int Nc, int Hc, int Wc, int C, const uint8_t* labels, int R,
                             const void* const* states, float alpha, float eps_cov, float eps_eig, float thresh, int readd,
                             __half* out, int32_t* k_out, void* ws, size_t ws_bytes, cudaStream_t st) {
    WCTB_REQUIRE(C == 64 || C == 128 || C == 256 || C == 512, "wct_apply_regions: C=%d not in {64,128,256,512}", C);
    WCTB_REQUIRE(R >= 1 && R <= 8, "wct_apply_regions: R=%d not in 1..8", R);
    const RegionWs RL = regions_layout(C, Nc, R, Hc, Wc);
    if (ws_bytes < RL.total) {
        set_error("wct_apply_regions: workspace %zu < %zu bytes", ws_bytes, RL.total);
        return WCTB200_EWS;
    }
    const int np = Nc * R;
    const WctWs L = wct_layout(C, np, 0);
    uint8_t* w = static_cast<uint8_t*>(ws) + RL.base;
    uint8_t* rw = static_cast<uint8_t*>(ws);
    float* mean_s = reinterpret_cast<float*>(rw + RL.mean_s);
    float* Cs = reinterpret_cast<float*>(rw + RL.Cs);
    int* ks = reinterpret_cast<int*>(rw + RL.ks);
    int* counts = reinterpret_cast<int*>(rw + RL.counts);
    uint16_t* tmask = reinterpret_cast<uint16_t*>(rw + RL.tmask);
    uint16_t* amask = reinterpret_cast<uint16_t*>(rw + RL.amask);
    double* dsum = reinterpret_cast<double*>(w + L.dsum);
    float* mean = reinterpret_cast<float*>(w + L.mean);
    float* G = reinterpret_cast<float*>(w + L.G);
    float* sigma = reinterpret_cast<float*>(w + L.sigma);
    float* dvec = reinterpret_cast<float*>(w + L.dvec);
    float* Wcm = reinterpret_cast<float*>(w + L.Wc);
    float* T = reinterpret_cast<float*>(w + L.T);
    __half* Msplit = reinterpret_cast<__half*>(w + L.Msplit);
    float* bias = reinterpret_cast<float*>(w + L.bias);
    float* conv = reinterpret_cast<float*>(w + L.conv);
    int* kc = reinterpret_cast<int*>(w + L.kcount);
    float* A0 = reinterpret_cast<float*>(w + L.A0);
    float* lam = reinterpret_cast<float*>(w + L.lam);
    int* ok = reinterpret_cast<int*>(w + L.ok);
    const long long CC = (long long)C * C;
    // gather the R style states (each from wct_style_prepare with Ns = 1: [C] mean_s | [C][C] C_s | k_s, sweeps)
    size_t off_cs, off_k;
    style_state_offsets(C, 1, &off_cs, &off_k);
    for (int r = 0; r < R; ++r) {
        WCTB_REQUIRE(states[r], "wct_apply_regions: style state %d is null", r);
        const uint8_t* sp = static_cast<const uint8_t*>(states[r]);
        WCTB_CUDA(cudaMemcpyAsync(mean_s + (long long)r * C, sp, (size_t)C * 4, cudaMemcpyDeviceToDevice, st));
        WCTB_CUDA(cudaMemcpyAsync(Cs + r * CC, sp + off_cs, (size_t)CC * 4, cudaMemcpyDeviceToDevice, st));
        WCTB_CUDA(cudaMemcpyAsync(ks + 2 * r, sp + off_k, 2 * 4, cudaMemcpyDeviceToDevice, st));
    }
    WCTB_CUDA(cudaMemsetAsync(kc, 0, (size_t)np * 2 * 4, st));
    int rc = region_scan(labels, Nc, Hc, Wc, R, counts, tmask, st);
    if (rc) return rc;
    k_regions_drop_empty_styles<<<(unsigned)cdiv(np, 256), 256, 0, st>>>(ks, np, R, counts);
    WCTB_CHECK_LAUNCH("k_regions_drop_empty_styles");
    // per (frame, region): masked covariance; then the content side of wct_apply over Nc*R matrices, style z % R
    rc = launch_mean_cov_regions(content, ActGeom(Nc, Hc, Wc, C), labels, R, counts, tmask, eps_cov, mean, G, A0, dsum, st);
    if (rc) return rc;
    rc = launch_matfun_ns(A0, C, np, /*n_first=*/np, thresh, eps_eig, Wcm, ok, kc, st);
    if (rc < 0) return rc;
    rc = launch_jacobi(G, C, np, conv, kc + np, st, ok, thresh);
    if (rc) return rc;
    rc = launch_eig_post(G, A0, lam, C, np, thresh, eps_eig, np, sigma, dvec, kc, st, ok);
    if (rc) return rc;
    dim3 gg((unsigned)(C / 64), (unsigned)(C / 64), (unsigned)np);
    k_outer_gemm<<<gg, 256, 0, st>>>(G, CC, G, CC, dvec, C, Wcm, CC, C, ok);
    WCTB_CHECK_LAUNCH("k_outer_gemm(Wc)");
    k_outer_gemm<<<gg, 256, 0, st>>>(Cs, CC, Wcm, CC, nullptr, 0, T, CC, C, nullptr, R);   // T = C_s(z % R) W_c(z)
    WCTB_CHECK_LAUNCH("k_outer_gemm(T)");
    dim3 gf((unsigned)cdiv(C, 8), (unsigned)np);
    int* Mexp = reinterpret_cast<int*>(w + L.Mexp);
    k_finalize_transform<<<gf, 256, 0, st>>>(T, C, np, R, alpha, readd, mean, mean_s, Msplit, Mexp, bias);
    WCTB_CHECK_LAUNCH("k_finalize_transform");
    // out = M_{n,r} x + bias_{n,r} per pixel of region r; every other pixel keeps its input bytes
    const long long napply = (long long)Nc * RL.tiles_per_image;
    k_region_apply_tiles<<<(unsigned)cdiv(napply, 8), 256, 0, st>>>(labels, counts, Nc, Hc, Wc, R, RL.tiles_per_image, amask);
    WCTB_CHECK_LAUNCH("k_region_apply_tiles");
    rc = launch_conv_apply_regions(content, Nc, Hc, Wc, C, Msplit, Mexp, bias, labels, counts, amask, R, out, st);
    if (rc) return rc;
    if (k_out) {
        k_regions_kout<<<(unsigned)cdiv(np > R ? np : R, 256), 256, 0, st>>>(kc, counts, ks, np, R, k_out);
        WCTB_CHECK_LAUNCH("k_regions_kout");
    }
    return 0;
}

// test hook: means, covariances (+ eps_cov I) and pixel counts per (image, region): mean [N*R][C], cov [N*R][C][C],
// counts [N*R]; a region with fewer than 2 pixels gets cov = I
int launch_covariance_regions(const __half* act, int N, int H, int W, int C, const uint8_t* labels, int R, float eps_cov,
                              float* mean_out, float* cov_out, int* counts, cudaStream_t st) {
    WCTB_REQUIRE(C == 64 || (C % 128 == 0 && C >= 128), "covariance_regions: C=%d must be 64 or a multiple of 128", C);
    WCTB_REQUIRE(R >= 1 && R <= 8, "covariance_regions: R=%d not in 1..8", R);
    const int tiles = ((W + 31) / 32) * ((H + 1) / 2);
    uint8_t* scratch = nullptr;
    const size_t dsum_bytes = align_up((size_t)N * R * C * sizeof(double), 256);
    { int rc0 = scratch_alloc(reinterpret_cast<void**>(&scratch), dsum_bytes + (size_t)N * tiles * 2, st, 1); if (rc0) return rc0; }
    double* dsum = reinterpret_cast<double*>(scratch);
    uint16_t* tmask = reinterpret_cast<uint16_t*>(scratch + dsum_bytes);
    int rc = region_scan(labels, N, H, W, R, counts, tmask, st);
    if (rc) return rc;
    return launch_mean_cov_regions(act, ActGeom(N, H, W, C), labels, R, counts, tmask, eps_cov, mean_out, cov_out, nullptr, dsum, st);
}

// ---------------------------------------------------------------------------
// Soft spatial control (DESIGN.md §3.3.11): K weight planes per frame and a strength map.  Region k's statistics are
// weighted by w_k (a Kish-normalised record, cov_tc.cu), and the apply blends the K transforms per pixel:
//   out(p) = sum_k v_k(p) (M_{n,k} x_p + b_{n,k}) + (1 - sum_k v_k(p)) x_p,   v_k = s(p) w_k(p).
// ---------------------------------------------------------------------------
// feathering: one-hot plane r of a label map (r < R), blurred by a separable Gaussian of sigma mask pixels, truncated at
// rad = ceil(3 sigma), taps exp(-d^2 / 2 sigma^2) normalised in fp64, clamp-to-edge borders.  Pass 1 (rows) writes fp64
// [N][R][Hm][Wm] partial sums, pass 2 (columns) the fp32 planes.  Every block makes the taps in shared memory.
__device__ __forceinline__ void feather_taps(double* taps, int rad, double sigma) {
    for (int d = threadIdx.x; d <= rad; d += blockDim.x) taps[d] = exp(-(double)d * d / (2.0 * sigma * sigma));
    __syncthreads();
    __shared__ double norm;
    if (threadIdx.x == 0) {
        double a = taps[0];
        for (int d = 1; d <= rad; ++d) a += 2.0 * taps[d];
        norm = a;
    }
    __syncthreads();
    for (int d = threadIdx.x; d <= rad; d += blockDim.x) taps[d] /= norm;
    __syncthreads();
}
__global__ void __launch_bounds__(256)
k_feather_rows(const uint8_t* __restrict__ labels, int N, int Hm, int Wm, int R, double sigma, int rad, double* __restrict__ tmp) {
    extern __shared__ double taps[];
    feather_taps(taps, rad, sigma);
    const long long total = (long long)N * R * Hm * Wm;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % Wm);
        const long long t = i / Wm;
        const int y = (int)(t % Hm);
        const long long nr = t / Hm;
        const int r = (int)(nr % R), n = (int)(nr / R);
        const uint8_t* row = labels + ((long long)n * Hm + y) * Wm;
        double a = 0.0;
        for (int d = -rad; d <= rad; ++d) {
            const int xx = min(max(x + d, 0), Wm - 1);
            if (row[xx] == r) a += taps[d < 0 ? -d : d];
        }
        tmp[i] = a;
    }
}
__global__ void __launch_bounds__(256)
k_feather_cols(const double* __restrict__ tmp, int N, int Hm, int Wm, int R, double sigma, int rad, float* __restrict__ out) {
    extern __shared__ double taps[];
    feather_taps(taps, rad, sigma);
    const long long total = (long long)N * R * Hm * Wm;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % Wm);
        const long long t = i / Wm;
        const int y = (int)(t % Hm);
        const double* plane = tmp + (t / Hm) * Hm * Wm;
        double a = 0.0;
        for (int d = -rad; d <= rad; ++d) {
            const int yy = min(max(y + d, 0), Hm - 1);
            a += taps[d < 0 ? -d : d] * plane[(long long)yy * Wm + x];
        }
        out[i] = (float)a;
    }
}
int launch_mask_feather(const uint8_t* labels, int N, int Hm, int Wm, int R, float sigma, float* out, cudaStream_t st) {
    WCTB_REQUIRE(R >= 1 && R <= 8, "mask_feather: R=%d not in 1..8", R);
    WCTB_REQUIRE(sigma > 0.f && sigma <= 1024.f, "mask_feather: sigma=%g not in (0, 1024]", (double)sigma);
    const int rad = (int)ceil(3.0 * (double)sigma);
    const long long total = (long long)N * R * Hm * Wm;
    double* tmp = nullptr;
    { int rc0 = scratch_alloc(reinterpret_cast<void**>(&tmp), (size_t)total * sizeof(double), st, 6); if (rc0) return rc0; }
    long long blocks = (total + 255) / 256;
    if (blocks > device_sm_count() * 16ll) blocks = device_sm_count() * 16ll;
    const size_t smem = (size_t)(rad + 1) * sizeof(double);
    if (smem > 48 * 1024) {
        WCTB_CUDA(cudaFuncSetAttribute(k_feather_rows, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        WCTB_CUDA(cudaFuncSetAttribute(k_feather_cols, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    k_feather_rows<<<(unsigned)blocks, 256, smem, st>>>(labels, N, Hm, Wm, R, (double)sigma, rad, tmp);
    WCTB_CHECK_LAUNCH("k_feather_rows");
    k_feather_cols<<<(unsigned)blocks, 256, smem, st>>>(tmp, N, Hm, Wm, R, (double)sigma, rad, out);
    WCTB_CHECK_LAUNCH("k_feather_cols");
    return 0;
}

// exact area average of P planes Hm x Wm onto Hf x Wf: in units of 1 / (Hf Hm), output row y covers [y Hm, (y+1) Hm) and
// source row i covers [i Hf, (i+1) Hf); the integer overlaps weigh the sources, the fp64 sum is divided by Hm Wm and rounded
// once.  The identity at equal size; preserves a constant.
__global__ void k_weights_resize_area(const float* __restrict__ src, long long P, int Hm, int Wm, int Hf, int Wf, float* __restrict__ dst) {
    const long long total = P * Hf * Wf;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % Wf);
        const long long t = i / Wf;
        const int y = (int)(t % Hf);
        const float* plane = src + (t / Hf) * Hm * Wm;
        const long long ya = (long long)y * Hm, yb = ya + Hm, xa = (long long)x * Wm, xb = xa + Wm;
        double a = 0.0;
        for (long long si = ya / Hf; si * Hf < yb; ++si) {
            const long long oy = min(yb, (si + 1) * Hf) - max(ya, si * Hf);
            double r = 0.0;
            for (long long sj = xa / Wf; sj * Wf < xb; ++sj) {
                const long long ox = min(xb, (sj + 1) * Wf) - max(xa, sj * Wf);
                r += (double)ox * (double)plane[si * Wm + sj];
            }
            a += (double)oy * r;
        }
        dst[i] = (float)(a / ((double)Hm * (double)Wm));
    }
}
int launch_weights_resize_area(const float* src, int N, int K, int Hm, int Wm, int Hf, int Wf, float* dst, cudaStream_t st) {
    const long long total = (long long)N * K * Hf * Wf;
    long long blocks = (total + 255) / 256;
    if (blocks > device_sm_count() * 16ll) blocks = device_sm_count() * 16ll;
    k_weights_resize_area<<<(unsigned)blocks, 256, 0, st>>>(src, (long long)N * K, Hm, Wm, Hf, Wf, dst);
    WCTB_CHECK_LAUNCH("k_weights_resize_area");
    return 0;
}

// one warp per 32 x 2 covariance tile: tmask[n][tile] bit k when a pixel of the tile has w_k > 0.  grid (cdiv(tiles, 8), N)
__global__ void __launch_bounds__(256)
k_weights_scan(const float* __restrict__ wts, int H, int W, int K, int tiles_x, int tiles, uint16_t* __restrict__ tmask) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int t = blockIdx.x * 8 + warp, n = blockIdx.y;
    if (t >= tiles) return;
    const int ty = t / tiles_x, tx = t - ty * tiles_x;
    const int x = tx * 32 + lane;
    const long long HW = (long long)H * W;
    unsigned bits = 0;
    for (int k = 0; k < K; ++k) {
        bool any = false;
        for (int j = 0; j < 2; ++j) {
            const int y = ty * 2 + j;
            if (x < W && y < H && wts[((long long)n * K + k) * HW + (long long)y * W + x] > 0.f) any = true;
        }
        if (__any_sync(0xffffffffu, any)) bits |= 1u << k;
    }
    if (lane == 0) tmask[(long long)n * tiles + t] = (uint16_t)bits;
}
// wq[z] = (W, Q) = (sum w, sum w^2) of weight plane z, fp64 in a fixed order (256 strided partial sums, then a fixed tree):
// a function of the plane alone.  grid N*K.
__global__ void __launch_bounds__(256) k_weights_wq(const float* __restrict__ wts, long long HW, double* __restrict__ wq) {
    __shared__ double sw[256], sq[256];
    const float* w = wts + (long long)blockIdx.x * HW;
    double a = 0.0, b = 0.0;
    for (long long i = threadIdx.x; i < HW; i += 256) {
        const double v = (double)w[i];
        a += v;
        b += v * v;
    }
    sw[threadIdx.x] = a;
    sq[threadIdx.x] = b;
    __syncthreads();
    for (int o = 128; o >= 1; o >>= 1) {
        if (threadIdx.x < o) {
            sw[threadIdx.x] += sw[threadIdx.x + o];
            sq[threadIdx.x] += sq[threadIdx.x + o];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        wq[2 * blockIdx.x] = sw[0];
        wq[2 * blockIdx.x + 1] = sq[0];
    }
}

int launch_cov_record_weighted(const __half* act, int N, int H, int W, int C, const float* wts, int K, const uint16_t* tmask,
                               const double* wq, const StatsRecord& rec, cudaStream_t st);   // cov_tc.cu

int launch_wct_stats_weighted(const __half* act, int N, int H, int W, int C, const float* wts, int K, void* record, cudaStream_t st) {
    WCTB_REQUIRE(C == 64 || C == 128 || C == 256 || C == 512, "wct_stats_weighted: C=%d not in {64,128,256,512}", C);
    WCTB_REQUIRE(K >= 1 && K <= 8, "wct_stats_weighted: K=%d not in 1..8", K);
    const int tiles_x = (W + 31) / 32, tiles = tiles_x * ((H + 1) / 2);
    const size_t wq_bytes = align_up((size_t)N * K * 2 * sizeof(double), 256);
    uint8_t* scratch = nullptr;
    { int rc0 = scratch_alloc(reinterpret_cast<void**>(&scratch), wq_bytes + (size_t)N * tiles * 2, st, 6); if (rc0) return rc0; }
    double* wq = reinterpret_cast<double*>(scratch);
    uint16_t* tmask = reinterpret_cast<uint16_t*>(scratch + wq_bytes);
    k_weights_scan<<<dim3((unsigned)cdiv(tiles, 8), (unsigned)N), 256, 0, st>>>(wts, H, W, K, tiles_x, tiles, tmask);
    WCTB_CHECK_LAUNCH("k_weights_scan");
    k_weights_wq<<<(unsigned)(N * K), 256, 0, st>>>(wts, (long long)H * W, wq);
    WCTB_CHECK_LAUNCH("k_weights_wq");
    return launch_cov_record_weighted(act, N, H, W, C, wts, K, tmask, wq, stats_record_at(record, C, N * K, 0), st);
}

// per 128-position tile of the weighted apply (per-image tiling over the padded plane): bit k when a pixel has v_k > 0,
// bit K when a pixel has every v_k = 0 (it keeps its input).  One warp per tile.
__global__ void __launch_bounds__(256)
k_weighted_apply_tiles(const float* __restrict__ wts, const float* __restrict__ str, const int* __restrict__ kc, int N, int H, int W,
                       int K, int tiles_per_image, uint16_t* __restrict__ amask) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long t = (long long)blockIdx.x * 8 + warp;
    if (t >= (long long)N * tiles_per_image) return;
    const int n = (int)(t / tiles_per_image), mt = (int)(t - (long long)n * tiles_per_image);
    const int Wp = W + 2;
    const long long HpWp = (long long)(H + 2) * Wp, HW = (long long)H * W;
    unsigned bits = 0;
    for (int j = lane; j < 128; j += 32) {
        const long long r = (long long)mt * 128 + j;
        if (r >= HpWp) break;
        const int yy = (int)(r / Wp), xx = (int)(r - (long long)yy * Wp);
        if (yy < 1 || yy > H || xx < 1 || xx > W) continue;
        const long long pix = (long long)(yy - 1) * W + xx - 1;
        unsigned b = 0;
        for (int k = 0; k < K; ++k)
            if (soft_weight(wts, str, kc, K, n, k, HW, pix) > 0.f) b |= 1u << k;
        bits |= b ? b : 1u << K;
    }
    bits = __reduce_or_sync(0xffffffffu, bits);
    if (lane == 0) amask[t] = (uint16_t)bits;
}

int launch_conv_apply_weighted(const __half* in, int N, int H, int W, int C, const __half* w_split, const int* rexp, const float* bias,
                               const float* wts, const float* str, const int* kc, const uint16_t* amask, int K, __half* out,
                               cudaStream_t st);

int launch_wct_transform_apply_weighted(const __half* act, int N, int H, int W, int C, const void* transform, int K, const float* wts,
                                        const float* str, __half* out, cudaStream_t st) {
    WCTB_REQUIRE(C == 64 || C == 128 || C == 256 || C == 512, "wct_transform_apply_weighted: C=%d not in {64,128,256,512}", C);
    WCTB_REQUIRE(K >= 1 && K <= 8 && (wts || K == 1), "wct_transform_apply_weighted: K=%d not in 1..8 (1 without weights)", K);
    size_t om, ob, ok, oexp;
    wct_transform_layout(C, N * K, &om, &ob, &ok, &oexp);
    const uint8_t* tp = static_cast<const uint8_t*>(transform);
    const int* kc = reinterpret_cast<const int*>(tp + ok);
    const int tpi = cdiv((long long)(H + 2) * (W + 2), 128);
    uint16_t* amask = nullptr;
    { int rc0 = scratch_alloc(reinterpret_cast<void**>(&amask), (size_t)N * tpi * 2, st, 7); if (rc0) return rc0; }
    k_weighted_apply_tiles<<<(unsigned)cdiv((long long)N * tpi, 8), 256, 0, st>>>(wts, str, kc, N, H, W, K, tpi, amask);
    WCTB_CHECK_LAUNCH("k_weighted_apply_tiles");
    return launch_conv_apply_weighted(act, N, H, W, C, reinterpret_cast<const __half*>(tp + om), reinterpret_cast<const int*>(tp + oexp),
                                      reinterpret_cast<const float*>(tp + ob), wts, str, kc, amask, K, out, st);
}

// ---------------------------------------------------------------------------
// Style masks: the style side of spatial control over the labelled parts of ONE style.  Entry r of the state of R styles
// is wct_style_prepare restricted to the style pixels labelled r (the masked covariance of the content side, N = 1 and R
// problems).  With every label equal to r the covariance kernel adds in the unmasked order, so entry r is then
// byte-identical to wct_style_prepare.  An entry of < 2 pixels is the sentinel k_s = -1, 0 sweeps, mean 0, C_s 0, and
// wct_apply_regions keeps the content of that region.
// ---------------------------------------------------------------------------
struct StyleRegionWs {
    size_t base, counts, tmask, total;
};
static StyleRegionWs style_regions_layout(int C, int R, int Hs, int Ws) {
    StyleRegionWs L;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o = align_up(o + bytes, 256); return r; };
    L.base = take(wct_layout(C, 0, R).total);        // the eigensolver's, as wct_style_prepare's for R styles
    L.counts = take((size_t)R * 4);
    L.tmask = take((size_t)((Ws + 31) / 32) * ((Hs + 1) / 2) * 2);
    L.total = o;
    return L;
}
size_t wct_style_prepare_regions_workspace_bytes(int C, int R, int Hs, int Ws) { return style_regions_layout(C, R, Hs, Ws).total; }

// entries whose region has < 2 pixels -> the sentinel.  grid (blocks, R)
__global__ void k_style_regions_empty(const int* __restrict__ counts, int C, int R, float* __restrict__ mean, float* __restrict__ Cs,
                                      int* __restrict__ ks) {
    const int r = blockIdx.y;
    if (counts[r] >= 2) return;
    const long long CC = (long long)C * C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < CC; i += (long long)gridDim.x * blockDim.x) {
        Cs[r * CC + i] = 0.f;
        if (i < C) mean[(long long)r * C + i] = 0.f;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        ks[r] = -1;
        ks[R + r] = 0;
    }
}

int launch_wct_style_prepare_regions(const __half* style, int Hs, int Ws, int C, const uint8_t* labels, int R, float eps_cov,
                                     float eps_eig, float thresh, void* state, int32_t* k_out, void* ws, size_t ws_bytes,
                                     cudaStream_t st) {
    WCTB_REQUIRE(C == 64 || C == 128 || C == 256 || C == 512, "wct_style_prepare_regions: C=%d not in {64,128,256,512}", C);
    WCTB_REQUIRE(R >= 1 && R <= 8, "wct_style_prepare_regions: R=%d not in 1..8", R);
    const StyleRegionWs SL = style_regions_layout(C, R, Hs, Ws);
    if (ws_bytes < SL.total) {
        set_error("wct_style_prepare_regions: workspace %zu < %zu bytes", ws_bytes, SL.total);
        return WCTB200_EWS;
    }
    const WctWs L = wct_layout(C, 0, R);
    uint8_t* w = static_cast<uint8_t*>(ws) + SL.base;
    int* counts = reinterpret_cast<int*>(static_cast<uint8_t*>(ws) + SL.counts);
    uint16_t* tmask = reinterpret_cast<uint16_t*>(static_cast<uint8_t*>(ws) + SL.tmask);
    size_t off_cs, off_k;
    style_state_offsets(C, R, &off_cs, &off_k);
    uint8_t* sp = static_cast<uint8_t*>(state);
    float* mean_s = reinterpret_cast<float*>(sp);
    float* Cs = reinterpret_cast<float*>(sp + off_cs);
    int* kc = reinterpret_cast<int*>(sp + off_k);
    double* dsum = reinterpret_cast<double*>(w + L.dsum);
    float* G = reinterpret_cast<float*>(w + L.G);
    float* A0 = reinterpret_cast<float*>(w + L.A0);
    float* lam = reinterpret_cast<float*>(w + L.lam);
    float* sigma = reinterpret_cast<float*>(w + L.sigma);
    float* dvec = reinterpret_cast<float*>(w + L.dvec);
    float* conv = reinterpret_cast<float*>(w + L.conv);
    int* ok = reinterpret_cast<int*>(w + L.ok);
    const long long CC = (long long)C * C;
    WCTB_CUDA(cudaMemsetAsync(kc, 0, (size_t)R * 2 * 4, st));
    int rc = region_scan(labels, 1, Hs, Ws, R, counts, tmask, st);
    if (rc) return rc;
    rc = launch_mean_cov_regions(style, ActGeom(1, Hs, Ws, C), labels, R, counts, tmask, eps_cov, mean_s, G, A0, dsum, st);
    if (rc) return rc;
    // from here on wct_style_prepare's steps over the R matrices (an empty region's placeholder G = I is harmless)
    rc = launch_matfun_ns(A0, C, R, /*n_first=*/0, thresh, eps_eig, Cs, ok, kc, st);
    if (rc < 0) return rc;
    rc = launch_jacobi(G, C, R, conv, kc + R, st, ok, thresh);
    if (rc) return rc;
    rc = launch_eig_post(G, A0, lam, C, R, thresh, eps_eig, /*n_content=*/0, sigma, dvec, kc, st, ok);
    if (rc) return rc;
    dim3 gg((unsigned)(C / 64), (unsigned)(C / 64), (unsigned)R);
    k_outer_gemm<<<gg, 256, 0, st>>>(G, CC, G, CC, dvec, C, Cs, CC, C, ok);
    WCTB_CHECK_LAUNCH("k_outer_gemm(Cs)");
    k_style_regions_empty<<<dim3((unsigned)cdiv(CC, 256 * 8), (unsigned)R), 256, 0, st>>>(counts, C, R, mean_s, Cs, kc);
    WCTB_CHECK_LAUNCH("k_style_regions_empty");
    if (k_out) WCTB_CUDA(cudaMemcpyAsync(k_out, kc, (size_t)R * 2 * 4, cudaMemcpyDeviceToDevice, st));
    return 0;
}

// ---------------------------------------------------------------------------
// Style swap at one level (ops.py:145-278: wct_style_swap + style_swap), ONE content/style pair, 3x3 patches, stride 1.
//   whiten content and style (same eigensolver as the WCT level; whitening on BOTH sides, ops.py:187-196)
//   -> every 3x3 patch of the whitened style becomes a conv filter, normalised per filter TAP across patches
//      (tf.nn.l2_normalize(style_patches, dim=3), ops.py:233) -> cross-correlation with the whitened content on the
//      tensor cores (the patches are just a weight tensor for the 3x3 conv kernel; VALID = the interior of the SAME conv)
//   -> first arg-max per position (ops.py:242) -> paste the un-normalised patch back and average the overlaps
//      (conv2d_transpose / counting, ops.py:255-276 = a gather of <= 9 style pixels per output pixel)
//   -> colour with the style (S^+1/2), add the style mean, blend with the content (ops.py:203-210).
// ---------------------------------------------------------------------------
static inline int swap_grid(long long total, int block) {
    long long b = (total + block - 1) / block;
    return (int)(b < 1 ? 1 : (b > device_sm_count() * 32ll ? device_sm_count() * 32ll : b));
}

// The style swap in split form.  The style side -- whitening of the style, its patch filters and the colouring operand --
// depends only on the style features, so it is prepared once into a state and applied to any number of content frames.
//   state layout (256-byte aligned blocks): [C] mean_s | int32 [2] (k_s, sweeps_s) | whitened style SPF16 [1,Hs,Ws,C]
//   (gathered from) | [P*P][C] 1/||tap|| | split-fp16 patch filters [2][cout_pad][P*P*C] | colouring operand [2][C][C] (C_s
//   split, row i times 2^e_i) | int32 [C] e | [C] its bias (m_s)
struct SwapState {
    size_t mean, k, feat, norms, wsplit, cmsplit, cmexp, cbias, total;
    int cout_pad, n_patches, prow, pcol;           // style patch grid prow x pcol
};
static SwapState swap_state_layout(int C, int Hs, int Ws, int P, int S) {
    SwapState L;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o = align_up(o + bytes, 256); return r; };
    L.prow = (Hs - P) / S + 1;                                    // tf.extract_image_patches, VALID (ops.py:226)
    L.pcol = (Ws - P) / S + 1;
    L.n_patches = L.prow * L.pcol;
    L.cout_pad = (L.n_patches + 63) / 64 * 64;
    L.mean = take((size_t)C * 4);
    L.k = take(2 * 4);
    L.feat = take((size_t)ActGeom(1, Hs, Ws, C).plane * 2 * sizeof(__half));
    L.norms = take((size_t)P * P * C * 4);
    L.wsplit = take((size_t)2 * P * P * C * L.cout_pad * sizeof(__half));
    L.cmsplit = take((size_t)2 * C * C * 2);
    L.cmexp = take((size_t)C * 4);
    L.cbias = take((size_t)C * 4);
    L.total = o;
    return L;
}
// workspace of the prepare: the eigensolver's (wct_layout(C, 0, 1)) and the style's whitening / colouring matrices
struct SwapPrepWs {
    size_t base, zeros, dvec2, sigma2, Wm, Cm, msplit, mexp, bias, total;
};
static SwapPrepWs swap_prep_layout(int C) {
    SwapPrepWs L;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o = align_up(o + bytes, 256); return r; };
    L.base = take(wct_layout(C, 0, 1).total);
    L.zeros = take((size_t)C * 4);
    L.dvec2 = take((size_t)C * 4);
    L.sigma2 = take((size_t)C * 4);
    L.Wm = take((size_t)C * C * 4);                               // W_s (whitening)
    L.Cm = take((size_t)C * C * 4);                               // C_s (colouring)
    L.msplit = take((size_t)2 * C * C * 2);
    L.mexp = take((size_t)C * 4);
    L.bias = take((size_t)C * 4);
    L.total = o;
    return L;
}
// workspace of the apply over Nc frames: the content side (wct_layout(C, Nc, 0): per-frame whitening operands), the
// whitened, swapped and coloured features, the correlation scores of `cols` patches (all cout_pad of them in one chunk, or
// one chunk of them) and the arg-max per VALID position.  The running best score of a chunked arg-max lives in `tmp`,
// which only the colouring after the gather writes.
struct SwapApplyWs {
    size_t base, zeros, idx, wc_feat, ss_feat, tmp, scores, total;
    int ho, wo;                                     // content score grid ho x wo
};
static SwapApplyWs swap_apply_layout(int C, int Nc, int Hc, int Wc, int P, int S, int cols) {
    SwapApplyWs L;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o = align_up(o + bytes, 256); return r; };
    L.ho = (Hc - P) / S + 1;                                      // tf.nn.conv2d VALID with the same stride (ops.py:236-239)
    L.wo = (Wc - P) / S + 1;
    L.base = take(wct_layout(C, Nc, 0).total);
    L.zeros = take((size_t)C * 4);
    L.idx = take((size_t)Nc * L.ho * L.wo * 4);
    const size_t fc = (size_t)ActGeom(Nc, Hc, Wc, C).plane * 2 * sizeof(__half);
    L.wc_feat = take(fc);
    L.ss_feat = take(fc);
    L.tmp = take(fc);
    L.scores = take((size_t)ActGeom(Nc, Hc, Wc, cols).plane * 2 * sizeof(__half));
    L.total = o;
    return L;
}
// where the stages of one prepare + apply leave their results (wctb200_debug_style_swap_layout: tests read them back)
void style_swap_debug_layout(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int P, int S, long long* out) {
    const SwapState SL = swap_state_layout(C, Hs, Ws, P, S);
    const SwapApplyWs AL = swap_apply_layout(C, Nc, Hc, Wc, P, S, SL.cout_pad);
    const long long v[11] = {SL.n_patches, SL.cout_pad, AL.ho, AL.wo, (long long)SL.feat, (long long)SL.norms,
                             (long long)SL.wsplit, (long long)AL.wc_feat, (long long)AL.scores, (long long)AL.idx,
                             (long long)AL.ss_feat};
    for (int i = 0; i < 11; ++i) out[i] = v[i];
}
size_t style_swap_state_bytes(int C, int Hs, int Ws, int P, int S) { return swap_state_layout(C, Hs, Ws, P, S).total; }
size_t style_swap_prepare_workspace_bytes(int C) { return swap_prep_layout(C).total; }
size_t style_swap_apply_workspace_bytes(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int P, int S) {
    return swap_apply_layout(C, Nc, Hc, Wc, P, S, swap_state_layout(C, Hs, Ws, P, S).cout_pad).total;
}
// the chunked apply's least workspace: a score buffer one N tile of the whole correlation wide
size_t style_swap_apply_min_workspace_bytes(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int P, int S) {
    return swap_apply_layout(C, Nc, Hc, Wc, P, S, conv_tc_bn(swap_state_layout(C, Hs, Ws, P, S).cout_pad)).total;
}
// style_swap_level: the state, then the prepare's or the apply's workspace
size_t style_swap_workspace_bytes(int C, int Hc, int Wc, int Hs, int Ws, int P, int S) {
    const size_t a = style_swap_prepare_workspace_bytes(C), b = style_swap_apply_workspace_bytes(C, 1, Hc, Wc, Hs, Ws, P, S);
    return style_swap_state_bytes(C, Hs, Ws, P, S) + (a > b ? a : b);
}

// patch geometry of the swap: P x P patches taken every S pixels (ops.py:219-278: --ss-patch-size, --ss-stride)
struct SwapGeom { int P, S, prow, pcol, ho, wo; };

// 1 / ||patch tap||: for every (tap, channel) the l2 norm ACROSS all patches (ops.py:233); block = (tap, 256 channels)
__global__ void k_swap_tap_norms(const __half* __restrict__ feat, ActGeom g, SwapGeom q, float* __restrict__ inv_norm) {
    const int tap = blockIdx.y, c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= g.C) return;
    const int ky = tap / q.P, kx = tap % q.P;
    float s = 0.f;
    for (int py = 0; py < q.prow; ++py)
        for (int px = 0; px < q.pcol; ++px) {
            const long long pos = ((long long)(py * q.S + ky + 1)) * g.Wp + (px * q.S + kx + 1);      // interior pixel -> padded position
            const float v = merge_f32(feat[pos * g.C + c], feat[g.plane + pos * g.C + c]);
            s = fmaf(v, v, s);
        }
    inv_norm[tap * g.C + c] = rsqrtf(fmaxf(s, 1e-12f));
}
// conv weights of the correlation: [plane][patch n][tap*C + c] = whitened_style[py*S+ky][px*S+kx][c] * inv_norm[tap][c]; rows >= n_patches zero
__global__ void k_swap_patch_weights(const __half* __restrict__ feat, ActGeom g, SwapGeom q, const float* __restrict__ inv_norm,
                                     int n_patches, int cout_pad, __half* __restrict__ wsplit) {
    const long long K = (long long)q.P * q.P * g.C, total = K * cout_pad;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int n = (int)(i / K);
        const int k = (int)(i - (long long)n * K);
        float v = 0.f;
        if (n < n_patches) {
            const int tap = k / g.C, c = k - tap * g.C;
            const int py = n / q.pcol, px = n - py * q.pcol;
            const long long pos = ((long long)(py * q.S + tap / q.P + 1)) * g.Wp + (px * q.S + tap % q.P + 1);
            v = merge_f32(feat[pos * g.C + c], feat[g.plane + pos * g.C + c]) * inv_norm[k];
        }
        __half hi, lo;
        split_f32(v, hi, lo);
        wsplit[i] = hi;
        wsplit[total + i] = lo;
    }
}
// Labels of a labelled swap (DESIGN.md §3.3.13): the content and style label maps sampled onto their feature grids
// (k_labels_resize), patch n's label l(n) = Ls'[py*S + o][px*S + o] with o = (P-1)/2, and the 256-bit set of labels some
// patch carries.  An anchor whose label no patch carries may take any patch.
struct SwapLabels {
    const uint8_t* clab;        // sampled content labels [Ncl][Hc][Wc]
    long long clab_frame;       // frame stride of clab: Hc*Wc, or 0 when every frame shares one map
    const uint8_t* plab;        // l(n) for n < n_patches
    const uint32_t* present;    // [8]: bit l of word l/32 set when some patch carries label l
};
// l(n) of every patch and the present set (order-independent atomicOr into zeroed words); one thread per patch
__global__ void k_swap_patch_labels(const uint8_t* __restrict__ slab, int Ws, SwapGeom q, int n_patches, uint8_t* __restrict__ plab,
                                    uint32_t* __restrict__ present) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_patches) return;
    const int o = (q.P - 1) / 2;
    const int py = i / q.pcol, px = i - py * q.pcol;
    const uint8_t l = slab[(long long)(py * q.S + o) * Ws + px * q.S + o];
    plab[i] = l;
    atomicOr(&present[l >> 5], 1u << (l & 31));
}
// first arg-max over the patch axis for every VALID strided position (y,x) of frame blockIdx.y: the top-left-anchored P x P
// correlation at interior pixel (y*S, x*S), which the conv kernel stored at that pixel's own padded cell.  A VALID anchor
// reads padded rows y*S+1 .. y*S+P <= H of its own frame only, so a batch of frames in one correlation keeps them apart.
// The scores hold the chunk of patches [n0, n0 + g.C) (g.C = the chunk's width); patches >= n_patches are padding.  The
// first chunk (n0 = 0) sets (best, idx); a later one replaces them only where its own first maximum is strictly greater,
// so after the last chunk idx is the first maximum over all patches, whatever the chunking.
// LABELS: only the patches of the anchor's own label are candidates (all of them when no patch carries it); a skipped
// patch's score is never loaded.  A chunk without a candidate leaves (-inf, sentinel), which the first chunk may store and
// any later candidate replaces, so idx ends as a real patch: every anchor has at least one candidate overall.
template <bool LABELS>
__global__ void k_swap_argmax(const __half* __restrict__ scores, ActGeom g, SwapGeom q, int n0, int n_patches,
                              float* __restrict__ best_run, int* __restrict__ idx, SwapLabels lab) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= q.ho * q.wo) return;
    const int n = blockIdx.y;
    const int y = warp / q.wo, x = warp - y * q.wo;
    const long long pos = ((long long)n * g.Hp + y * q.S + 1) * g.Wp + (x * q.S + 1);
    const int cols = min(g.C, n_patches - n0);
    float best = -INFINITY;
    int bi = 0x7fffffff;
    if constexpr (LABELS) {
        const int o = (q.P - 1) / 2;
        const int l = lab.clab[n * lab.clab_frame + (long long)(y * q.S + o) * g.W + x * q.S + o];
        const bool any = ((lab.present[l >> 5] >> (l & 31)) & 1u) == 0u;
        for (int j = lane; j < cols; j += 32) {
            if (!any && lab.plab[n0 + j] != l) continue;
            const float v = merge_f32(scores[pos * g.C + j], scores[g.plane + pos * g.C + j]);
            if (v > best) { best = v; bi = n0 + j; }
        }
    } else {
        for (int j = lane; j < cols; j += 32) {
            const float v = merge_f32(scores[pos * g.C + j], scores[g.plane + pos * g.C + j]);
            if (v > best) { best = v; bi = n0 + j; }              // strictly greater: keeps the first maximum of this lane
        }
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if (lane == 0) {
        const long long o = (long long)n * q.ho * q.wo + warp;
        if (n0 == 0 || best > best_run[o]) {
            best_run[o] = best;
            idx[o] = bi;
        }
    }
}
// conv2d_transpose of the one-hot map with the raw patches, divided by the overlap count (ops.py:255-276): output pixel
// (Y,X) averages, over the <= P*P patch positions (py,px) with py*S + dy = Y, px*S + dx = X that cover it, the style
// pixel (sy*S + dy, sx*S + dx) of the matched patch.  The caller guarantees (ho-1)*S + P == H (wct.py:84-90 refits).
// gc.N frames, each with its own arg-max map [ho*wo], all against the one style feature.
__global__ void k_swap_gather(const __half* __restrict__ sfeat, ActGeom gs, SwapGeom q, const int* __restrict__ idx, ActGeom gc,
                              __half* __restrict__ out) {
    const int cg = gc.C / 8;
    const long long hw = (long long)gc.H * gc.W;
    const long long total = (long long)gc.N * hw * cg;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c0 = (int)(i % cg) * 8;
        const long long fp = i / cg;
        const int n = (int)(fp / hw);
        const int pix = (int)(fp - n * hw);
        const int Y = pix / gc.W, X = pix - Y * gc.W;
        const int* fidx = idx + (long long)n * q.ho * q.wo;
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.f;
        int cnt = 0;
        for (int dy = 0; dy < q.P; ++dy) {
            const int ty = Y - dy;
            if (ty < 0 || ty % q.S != 0 || ty / q.S >= q.ho) continue;
            for (int dx = 0; dx < q.P; ++dx) {
                const int tx = X - dx;
                if (tx < 0 || tx % q.S != 0 || tx / q.S >= q.wo) continue;
                const int m = fidx[(ty / q.S) * q.wo + tx / q.S];
                const int sy = m / q.pcol, sx = m - sy * q.pcol;
                float v[8];
                load8(sfeat, gs, ((long long)(sy * q.S + dy + 1)) * gs.Wp + (sx * q.S + dx + 1), c0, v);
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[j] += v[j];
                ++cnt;
            }
        }
        const float inv = cnt > 0 ? 1.f / (float)cnt : 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] *= inv;
        Half8 hi, lo;
        split8(acc, hi, lo);
        store8_with_halo(out, gc, n, Y, X, c0, hi, lo);
    }
}
// out = a*x + b*y on SPF16 interiors (+ halos)
__global__ void k_blend2(const __half* __restrict__ x, const __half* __restrict__ y, ActGeom g, float a, float b,
                         __half* __restrict__ out) {
    const int cg = g.C / 8;
    const long long total = (long long)g.N * g.H * g.W * cg;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c0 = (int)(i % cg) * 8;
        long long pix = i / cg;
        const int X = (int)(pix % g.W); pix /= g.W;
        const int Y = (int)(pix % g.H);
        const int n = (int)(pix / g.H);
        const long long pos = ((long long)n * g.Hp + Y + 1) * g.Wp + X + 1;
        float u[8], v[8];
        load8(x, g, pos, c0, u);
        load8(y, g, pos, c0, v);
#pragma unroll
        for (int j = 0; j < 8; ++j) u[j] = fmaf(a, u[j], b * v[j]);
        Half8 hi, lo;
        split8(u, hi, lo);
        store8_with_halo(out, g, n, Y, X, c0, hi, lo);
    }
}

static int swap_check_style(int C, int Hs, int Ws, int patch, int stride) {
    WCTB_REQUIRE(C == 64 || C == 128 || C == 256 || C == 512, "style_swap: C=%d not in {64,128,256,512}", C);
    WCTB_REQUIRE(patch >= 1 && patch <= 16 && stride >= 1 && stride <= 16, "style_swap: patch %d / stride %d out of range", patch, stride);
    WCTB_REQUIRE(Hs >= patch && Ws >= patch && Hs >= 2 && Ws >= 2, "style_swap: the style map must be at least %dx%d (style %dx%d)",
                 patch, patch, Hs, Ws);
    return 0;
}

// Style side: whiten the style (S^-1/2, ops.py:193), colour operand S^+1/2 and m_s (ops.py:203-206), the whitened style
// feature, its per-tap norms and the patch filters of the correlation (ops.py:226-233).
int launch_style_swap_prepare(const __half* style, int Hs, int Ws, int C, int patch, int stride, float eps_cov, float thresh,
                              void* state, int32_t* k_out, void* ws, size_t ws_bytes, cudaStream_t st) {
    int rc = swap_check_style(C, Hs, Ws, patch, stride);
    if (rc) return rc;
    const SwapPrepWs PL = swap_prep_layout(C);
    if (ws_bytes < PL.total) {
        set_error("style_swap_prepare: workspace %zu < %zu bytes", ws_bytes, PL.total);
        return WCTB200_EWS;
    }
    const SwapState SL = swap_state_layout(C, Hs, Ws, patch, stride);
    const SwapGeom q = {patch, stride, SL.prow, SL.pcol, 0, 0};
    uint8_t* sw = static_cast<uint8_t*>(ws);
    uint8_t* sp = static_cast<uint8_t*>(state);
    const WctWs L = wct_layout(C, 0, 1);
    uint8_t* w = sw + PL.base;
    double* dsum = reinterpret_cast<double*>(w + L.dsum);
    float* G = reinterpret_cast<float*>(w + L.G);
    float* A0 = reinterpret_cast<float*>(w + L.A0);
    float* lam = reinterpret_cast<float*>(w + L.lam);
    float* sigma = reinterpret_cast<float*>(w + L.sigma);
    float* dvec = reinterpret_cast<float*>(w + L.dvec);          // whitening scaling of the style
    float* conv = reinterpret_cast<float*>(w + L.conv);
    float* zeros = reinterpret_cast<float*>(sw + PL.zeros);
    float* dvec2 = reinterpret_cast<float*>(sw + PL.dvec2);      // colouring scaling of the style
    float* sigma2 = reinterpret_cast<float*>(sw + PL.sigma2);
    float* Wm = reinterpret_cast<float*>(sw + PL.Wm);
    float* Cm = reinterpret_cast<float*>(sw + PL.Cm);
    __half* msplit = reinterpret_cast<__half*>(sw + PL.msplit);
    int* mexp = reinterpret_cast<int*>(sw + PL.mexp);
    float* bias = reinterpret_cast<float*>(sw + PL.bias);
    float* mean_s = reinterpret_cast<float*>(sp + SL.mean);
    int* ks = reinterpret_cast<int*>(sp + SL.k);
    __half* feat = reinterpret_cast<__half*>(sp + SL.feat);
    float* norms = reinterpret_cast<float*>(sp + SL.norms);
    __half* wsplit = reinterpret_cast<__half*>(sp + SL.wsplit);
    const long long CC = (long long)C * C;

    WCTB_CUDA(cudaMemsetAsync(ks, 0, 2 * 4, st));
    WCTB_CUDA(cudaMemsetAsync(zeros, 0, (size_t)C * 4, st));
    ActGeom gs(1, Hs, Ws, C);
    rc = launch_mean_cov(style, gs, eps_cov, mean_s, G, A0, dsum, st);
    if (rc) return rc;
    rc = launch_jacobi(G, C, 1, conv, ks + 1, st, nullptr, thresh);
    if (rc) return rc;
    rc = launch_eig_post(G, A0, lam, C, 1, thresh, 0.f, 1, sigma, dvec, ks, st);                // S^-1/2 (ops.py:193)
    if (rc) return rc;
    k_eig_post<<<dim3((unsigned)cdiv(C, 8), 1), 256, 0, st>>>(G, lam, C, thresh, 0.f, 0, sigma2, dvec2, nullptr, nullptr);   // S^+1/2 (ops.py:203)
    WCTB_CHECK_LAUNCH("k_eig_post(colour)");
    dim3 g1((unsigned)(C / 64), (unsigned)(C / 64), 1);
    k_outer_gemm<<<g1, 256, 0, st>>>(G, CC, G, CC, dvec, C, Wm, CC, C);                        // W_s
    WCTB_CHECK_LAUNCH("k_outer_gemm(whiten)");
    k_outer_gemm<<<g1, 256, 0, st>>>(G, CC, G, CC, dvec2, C, Cm, CC, C);                       // C_s
    WCTB_CHECK_LAUNCH("k_outer_gemm(colour)");
    // whitening operand: x -> W_s (x - m_s) (alpha = 1, "style mean" = 0); colouring operand: x -> C_s x + m_s ("content mean" = 0)
    k_finalize_transform<<<dim3((unsigned)cdiv(C, 8), 1), 256, 0, st>>>(Wm, C, 1, 1, 1.f, 0, mean_s, zeros, msplit, mexp, bias);
    WCTB_CHECK_LAUNCH("k_finalize_transform(whiten)");
    k_finalize_transform<<<dim3((unsigned)cdiv(C, 8), 1), 256, 0, st>>>(Cm, C, 1, 1, 1.f, 0, zeros, mean_s,
                                                                         reinterpret_cast<__half*>(sp + SL.cmsplit),
                                                                         reinterpret_cast<int*>(sp + SL.cmexp),
                                                                         reinterpret_cast<float*>(sp + SL.cbias));
    WCTB_CHECK_LAUNCH("k_finalize_transform(colour)");
    rc = launch_conv_apply(style, 1, Hs, Ws, C, msplit, 1, mexp, bias, feat, st);
    if (rc) return rc;
    k_swap_tap_norms<<<dim3((unsigned)cdiv(C, 256), (unsigned)(patch * patch)), 256, 0, st>>>(feat, gs, q, norms);
    WCTB_CHECK_LAUNCH("k_swap_tap_norms");
    k_swap_patch_weights<<<swap_grid((long long)patch * patch * C * SL.cout_pad, 256), 256, 0, st>>>(feat, gs, q, norms, SL.n_patches,
                                                                                                   SL.cout_pad, wsplit);
    WCTB_CHECK_LAUNCH("k_swap_patch_weights");
    if (k_out) WCTB_CUDA(cudaMemcpyAsync(k_out, ks, 4, cudaMemcpyDeviceToDevice, st));
    return 0;
}

// the label buffer of a labelled apply (256-byte aligned blocks): sampled content labels [Ncl][Hc][Wc] | sampled style labels
// [Hs][Ws] | l(n) [n_patches] | present set uint32 [8].  Separate from the apply's workspace, whose layout and chunk policy
// it leaves as they are.
struct SwapLabelWs {
    size_t clab, slab, plab, present, total;
};
static SwapLabelWs swap_labels_layout(int Ncl, int Hc, int Wc, int Hs, int Ws, int n_patches) {
    SwapLabelWs L;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o = align_up(o + bytes, 256); return r; };
    L.clab = take((size_t)Ncl * Hc * Wc);
    L.slab = take((size_t)Hs * Ws);
    L.plab = take((size_t)n_patches);
    L.present = take(8 * sizeof(uint32_t));
    L.total = o;
    return L;
}
size_t style_swap_labels_workspace_bytes(int Ncl, int Hc, int Wc, int Hs, int Ws, int P, int S) {
    return swap_labels_layout(Ncl, Hc, Wc, Hs, Ws, swap_state_layout(64, Hs, Ws, P, S).n_patches).total;
}
// the label maps of a labelled apply as given: content [Ncl][Hm][Wm] (Ncl in {1, Nc}), style [Hms][Wms]
struct SwapLabelMaps {
    const uint8_t* content;
    int Ncl, Hm, Wm;
    const uint8_t* style;
    int Hms, Wms;
    void* buf;
    size_t buf_bytes;
};

// checks shared by every apply: the style geometry, the content frames, the tiling of the content encoding and, for a
// labelled call, its maps and label buffer (*LL gets the buffer's layout)
static int swap_apply_check(int Nc, int Hc, int Wc, int C, int Hs, int Ws, int patch, int stride, const SwapLabelMaps* maps,
                            SwapLabelWs* LL) {
    int rc = swap_check_style(C, Hs, Ws, patch, stride);
    if (rc) return rc;
    WCTB_REQUIRE(Nc >= 1 && Hc >= patch && Wc >= patch && Hc >= 2 && Wc >= 2,
                 "style_swap_apply: %d content maps of %dx%d (patch %d)", Nc, Hc, Wc, patch);
    // the swapped encoding must have the content's size (ops.py:199 reshapes it to [Hc*Wc, C]); wct.py:84-90 crops the content
    // image beforehand when the stride makes the filter not fit (utils.swap_filter_fit)
    const int ho = (Hc - patch) / stride + 1, wo = (Wc - patch) / stride + 1;
    WCTB_REQUIRE((ho - 1) * stride + patch == Hc && (wo - 1) * stride + patch == Wc,
                 "style_swap: patch %d / stride %d does not tile a %dx%d encoding (refit the content: swap_filter_fit, wct.py:84-90)",
                 patch, stride, Hc, Wc);
    if (maps) {
        WCTB_REQUIRE(maps->content && maps->style && maps->buf, "style_swap_apply_labels: null pointer");
        WCTB_REQUIRE((maps->Ncl == 1 || maps->Ncl == Nc) && maps->Hm >= 1 && maps->Wm >= 1 && maps->Hms >= 1 && maps->Wms >= 1,
                     "style_swap_apply_labels: %d content label maps of %dx%d for %d frames, style labels %dx%d", maps->Ncl,
                     maps->Hm, maps->Wm, Nc, maps->Hms, maps->Wms);
        *LL = swap_labels_layout(maps->Ncl, Hc, Wc, Hs, Ws, swap_state_layout(C, Hs, Ws, patch, stride).n_patches);
        if (maps->buf_bytes < LL->total) {
            set_error("style_swap_apply_labels: label buffer %zu < %zu bytes", maps->buf_bytes, LL->total);
            return WCTB200_EWS;
        }
    }
    return 0;
}

// the content side's whitening over Nc frames (ops.py:187): per-frame mean / covariance, eigensolver, W_c, and the whitened
// content into wc_feat.  `w` is the apply workspace's wct_layout(C, Nc, 0) block; `zeros` [C] is zeroed here.
static int swap_apply_whiten(const __half* content, int Nc, int Hc, int Wc, int C, uint8_t* w, float* zeros, float eps_cov,
                             float thresh, __half* wc_feat, cudaStream_t st) {
    const WctWs L = wct_layout(C, Nc, 0);
    double* dsum = reinterpret_cast<double*>(w + L.dsum);
    float* mean = reinterpret_cast<float*>(w + L.mean);
    float* G = reinterpret_cast<float*>(w + L.G);
    float* A0 = reinterpret_cast<float*>(w + L.A0);
    float* lam = reinterpret_cast<float*>(w + L.lam);
    float* sigma = reinterpret_cast<float*>(w + L.sigma);
    float* dvec = reinterpret_cast<float*>(w + L.dvec);
    float* Wcm = reinterpret_cast<float*>(w + L.Wc);
    __half* msplit = reinterpret_cast<__half*>(w + L.Msplit);
    int* mexp = reinterpret_cast<int*>(w + L.Mexp);
    float* bias = reinterpret_cast<float*>(w + L.bias);
    float* conv = reinterpret_cast<float*>(w + L.conv);
    int* kc = reinterpret_cast<int*>(w + L.kcount);
    const long long CC = (long long)C * C;

    WCTB_CUDA(cudaMemsetAsync(kc, 0, (size_t)Nc * 2 * 4, st));
    WCTB_CUDA(cudaMemsetAsync(zeros, 0, (size_t)C * 4, st));
    ActGeom gc(Nc, Hc, Wc, C);
    int rc = launch_mean_cov(content, gc, eps_cov, mean, G, A0, dsum, st);
    if (rc) return rc;
    rc = launch_jacobi(G, C, Nc, conv, kc + Nc, st, nullptr, thresh);
    if (rc) return rc;
    rc = launch_eig_post(G, A0, lam, C, Nc, thresh, 0.f, Nc, sigma, dvec, kc, st);             // S^-1/2 per frame (ops.py:187)
    if (rc) return rc;
    k_outer_gemm<<<dim3((unsigned)(C / 64), (unsigned)(C / 64), (unsigned)Nc), 256, 0, st>>>(G, CC, G, CC, dvec, C, Wcm, CC, C);   // W_c
    WCTB_CHECK_LAUNCH("k_outer_gemm(whiten)");
    k_finalize_transform<<<dim3((unsigned)cdiv(C, 8), (unsigned)Nc), 256, 0, st>>>(Wcm, C, Nc, 1, 1.f, 0, mean, zeros, msplit, mexp, bias);
    WCTB_CHECK_LAUNCH("k_finalize_transform(whiten)");
    return launch_conv_apply(content, Nc, Hc, Wc, C, msplit, Nc, mexp, bias, wc_feat, st);
}

// the sampled label maps, the patch labels and the present set of a labelled apply
static int swap_labels_setup(const SwapLabelMaps* maps, const SwapLabelWs& LL, int Hc, int Wc, int Hs, int Ws, const SwapGeom& q,
                             int n_patches, SwapLabels* lab, cudaStream_t st) {
    uint8_t* lb = static_cast<uint8_t*>(maps->buf);
    int rc = launch_labels_resize(maps->content, maps->Ncl, maps->Hm, maps->Wm, Hc, Wc, lb + LL.clab, st);
    if (rc) return rc;
    rc = launch_labels_resize(maps->style, 1, maps->Hms, maps->Wms, Hs, Ws, lb + LL.slab, st);
    if (rc) return rc;
    uint32_t* present = reinterpret_cast<uint32_t*>(lb + LL.present);
    WCTB_CUDA(cudaMemsetAsync(present, 0, 8 * sizeof(uint32_t), st));
    k_swap_patch_labels<<<(unsigned)cdiv(n_patches, 256), 256, 0, st>>>(lb + LL.slab, Ws, q, n_patches, lb + LL.plab, present);
    WCTB_CHECK_LAUNCH("k_swap_patch_labels");
    *lab = {lb + LL.clab, maps->Ncl == 1 ? 0ll : (long long)Hc * Wc, lb + LL.plab, present};
    return 0;
}

// colour the swapped feature with the style (ops.py:203-206), blend with the content (ops.py:210), report k
static int swap_apply_finish(const __half* ss_feat, const __half* content, int Nc, int Hc, int Wc, int C, const uint8_t* sp,
                             const SwapState& SL, const int* kc, float alpha, __half* tmp, __half* out, int32_t* k_out,
                             cudaStream_t st) {
    int rc = launch_conv_apply(ss_feat, Nc, Hc, Wc, C, reinterpret_cast<const __half*>(sp + SL.cmsplit), 1,
                               reinterpret_cast<const int*>(sp + SL.cmexp), reinterpret_cast<const float*>(sp + SL.cbias), tmp, st);
    if (rc) return rc;
    const ActGeom gc(Nc, Hc, Wc, C);
    k_blend2<<<swap_grid((long long)Nc * Hc * Wc * (C / 8), 256), 256, 0, st>>>(tmp, content, gc, alpha, 1.f - alpha, out);   // ops.py:210
    WCTB_CHECK_LAUNCH("k_blend2");
    if (k_out) {
        // k_out: [k_c x Nc | k_s]
        WCTB_CUDA(cudaMemcpyAsync(k_out, kc, (size_t)Nc * 4, cudaMemcpyDeviceToDevice, st));
        WCTB_CUDA(cudaMemcpyAsync(k_out + Nc, sp + SL.k, 4, cudaMemcpyDeviceToDevice, st));
    }
    return 0;
}

// Content side over Nc frames against one prepared style: whiten every frame with its own W_c (ops.py:187), correlate all
// frames with the shared patch filters in one launch, arg-max and gather per frame, colour with the style, blend.  With
// `maps` the arg-max is the labelled one (DESIGN.md §3.3.13); everything else is the same launch for launch.
static int style_swap_apply_impl(const __half* content, int Nc, int Hc, int Wc, int C, const void* state, int Hs, int Ws, int patch,
                                 int stride, float alpha, float eps_cov, float thresh, __half* out, int32_t* k_out, void* ws,
                                 size_t ws_bytes, const SwapLabelMaps* maps, cudaStream_t st) {
    SwapLabels lab = {nullptr, 0, nullptr, nullptr};
    SwapLabelWs LL = {};
    int rc = swap_apply_check(Nc, Hc, Wc, C, Hs, Ws, patch, stride, maps, &LL);
    if (rc) return rc;
    const SwapState SL = swap_state_layout(C, Hs, Ws, patch, stride);
    const SwapApplyWs AL = swap_apply_layout(C, Nc, Hc, Wc, patch, stride, SL.cout_pad);
    // chunk width: all cout_pad patches when the workspace holds their scores, else the largest multiple of the whole
    // correlation's N tile that fits (the same tile, hence the same kernel variant and k order, for every chunk)
    const int BN = conv_tc_bn(SL.cout_pad);
    int cols = SL.cout_pad;
    if (ws_bytes < AL.total) {
        const size_t col_bytes = (size_t)ActGeom(Nc, Hc, Wc, 1).plane * 2 * sizeof(__half);
        const size_t avail = ws_bytes > AL.scores ? ws_bytes - AL.scores : 0;
        const size_t fit = avail / col_bytes / BN * BN;
        cols = (int)(fit < (size_t)SL.cout_pad ? fit : (size_t)SL.cout_pad);
        while (cols >= BN && swap_apply_layout(C, Nc, Hc, Wc, patch, stride, cols).total > ws_bytes) cols -= BN;
        if (cols < BN) {
            set_error("style_swap_apply: workspace %zu < %zu bytes", ws_bytes,
                      swap_apply_layout(C, Nc, Hc, Wc, patch, stride, BN).total);
            return WCTB200_EWS;
        }
    }
    const SwapGeom q = {patch, stride, SL.prow, SL.pcol, AL.ho, AL.wo};
    uint8_t* sw = static_cast<uint8_t*>(ws);
    const uint8_t* sp = static_cast<const uint8_t*>(state);
    const int* kc = reinterpret_cast<const int*>(sw + AL.base + wct_layout(C, Nc, 0).kcount);
    int* idx = reinterpret_cast<int*>(sw + AL.idx);
    __half* wc_feat = reinterpret_cast<__half*>(sw + AL.wc_feat);
    __half* ss_feat = reinterpret_cast<__half*>(sw + AL.ss_feat);
    __half* tmp = reinterpret_cast<__half*>(sw + AL.tmp);
    __half* scores = reinterpret_cast<__half*>(sw + AL.scores);
    ActGeom gc(Nc, Hc, Wc, C), gs(1, Hs, Ws, C);
    rc = swap_apply_whiten(content, Nc, Hc, Wc, C, sw + AL.base, reinterpret_cast<float*>(sw + AL.zeros), eps_cov, thresh, wc_feat,
                           st);
    if (rc) return rc;
    // every style patch is a filter: the P x P correlation of all frames (top-left anchored, all positions; the strided VALID
    // subset is read by the arg-max) runs on the tensor-core conv kernel, `cols` filters (rows n0.. of the state's filter
    // planes, read in place) per chunk
    const long long K = (long long)patch * patch * C;
    const __half* wsplit = reinterpret_cast<const __half*>(sp + SL.wsplit);
    float* best_run = reinterpret_cast<float*>(tmp);
    const int npos = AL.ho * AL.wo;
    if (maps) {
        rc = swap_labels_setup(maps, LL, Hc, Wc, Hs, Ws, q, SL.n_patches, &lab, st);
        if (rc) return rc;
    }
    for (int n0 = 0; n0 < SL.cout_pad; n0 += cols) {
        const int m = SL.cout_pad - n0 < cols ? SL.cout_pad - n0 : cols;
        rc = launch_conv_taps_rows(wc_feat, Nc, Hc, Wc, C, wsplit + (long long)n0 * K, (long long)SL.cout_pad * K, m, BN, scores, st,
                                   patch);
        if (rc) return rc;
        const dim3 grid((unsigned)cdiv((long long)npos * 32, 256), (unsigned)Nc);
        if (maps)
            k_swap_argmax<true><<<grid, 256, 0, st>>>(scores, ActGeom(Nc, Hc, Wc, m), q, n0, SL.n_patches, best_run, idx, lab);
        else
            k_swap_argmax<false><<<grid, 256, 0, st>>>(scores, ActGeom(Nc, Hc, Wc, m), q, n0, SL.n_patches, best_run, idx, lab);
        WCTB_CHECK_LAUNCH("k_swap_argmax");
    }
    k_swap_gather<<<swap_grid((long long)Nc * Hc * Wc * (C / 8), 256), 256, 0, st>>>(reinterpret_cast<const __half*>(sp + SL.feat), gs, q,
                                                                                     idx, gc, ss_feat);
    WCTB_CHECK_LAUNCH("k_swap_gather");
    return swap_apply_finish(ss_feat, content, Nc, Hc, Wc, C, sp, SL, kc, alpha, tmp, out, k_out, st);
}
int launch_style_swap_apply(const __half* content, int Nc, int Hc, int Wc, int C, const void* state, int Hs, int Ws, int patch,
                            int stride, float alpha, float eps_cov, float thresh, __half* out, int32_t* k_out, void* ws, size_t ws_bytes,
                            cudaStream_t st) {
    return style_swap_apply_impl(content, Nc, Hc, Wc, C, state, Hs, Ws, patch, stride, alpha, eps_cov, thresh, out, k_out, ws,
                                 ws_bytes, nullptr, st);
}
int launch_style_swap_apply_labels(const __half* content, int Nc, int Hc, int Wc, int C, const void* state, int Hs, int Ws,
                                   int patch, int stride, float alpha, float eps_cov, float thresh, const uint8_t* content_labels,
                                   int Ncl, int Hm, int Wm, const uint8_t* style_labels, int Hms, int Wms, __half* out,
                                   int32_t* k_out, void* ws, size_t ws_bytes, void* label_buf, size_t label_bytes, cudaStream_t st) {
    const SwapLabelMaps maps = {content_labels, Ncl, Hm, Wm, style_labels, Hms, Wms, label_buf, label_bytes};
    return style_swap_apply_impl(content, Nc, Hc, Wc, C, state, Hs, Ws, patch, stride, alpha, eps_cov, thresh, out, k_out, ws,
                                 ws_bytes, &maps, st);
}

// ---------------------------------------------------------------------------
// Softmax style swap (DESIGN.md §3.3.17).  The hard swap's scores s(a,n), from the same correlation launches, become the
// weights of a softmax over patches:
//   z(a,n) = s(a,n) r_a,  r_a = 1 / (||c_a|| sqrt(K / n_p))  (0 where ||c_a|| = 0),  ||c_a||^2 = sum of wc^2 over the window
//   w(a,n) = exp((z - M_a) / tau) / sum_{m in A(a)} exp((z(a,m) - M_a) / tau) on the allowed set A(a), 0 elsewhere
// and every anchor pastes the w-weighted blend of the raw patches instead of its arg-max; the overlaps are averaged as in
// k_swap_gather.  The padded patch axis is split into blocks of SOFTMAX_SWAP_BLOCK patches (all of cout_pad when that is
// smaller).  Pass 1 reduces every (anchor, block) to (max, sum of exp) with a fixed tree and combines the blocks in block
// order into (M_a, 1/Z_a); pass 2 writes each block's weights into a map and folds them with the patches on the tensor
// cores.  A chunk is a union of whole blocks, so every workspace size -- hence every batch size -- gives the same bytes.
// ---------------------------------------------------------------------------
// B: a multiple of 128 (so every chunk is a multiple of the correlation's N tile); the fold's K = P*P*B stays at 2304 for
// 3x3 patches, inside the cross-product accumulator bound of DESIGN.md §3.1
constexpr int SOFTMAX_SWAP_BLOCK = 256;
// the weights are split to fp16 times 2^15: unscaled, weights below 6e-8 would flush to zero (there are 64 516 patches at
// relu2_1); the fold's epilogue multiplies by 2^-15, exactly
constexpr float SOFTMAX_SWAP_WSCALE = 32768.f;
// the most Sinkhorn iterations of a balanced apply (DESIGN.md §3.3.18)
constexpr int BALANCED_SWAP_MAX_ITERS = 256;

// workspace of a softmax apply: the hard apply's layout with `cols` score columns (wc_feat, ss_feat, tmp -- tmp holds the
// fold's fp32 sum -- and the scores), then r_a [Nc*ho*wo] | (max, sum) per (anchor, block) | (M_a, 1/Z_a) per anchor | the
// fold's unscale factor | one block's fold filters [2][C][P*P][B] | the weight map SPF16 [Nc, Hc+P-1, Wc+P-1, B] | the fold
// of one block SPF16 [Nc, Hc+P-1, Wc+P-1, C].  A balanced apply (DESIGN.md §3.3.18) adds the potentials h [Nc][cout_pad] |
// the log column targets [Nc][cout_pad] | (max, sum) per (frame, anchor block, chunk column) [Nc][nablk_a][cols].
struct SwapSoftmaxWs {
    SwapApplyWs A;
    size_t ascale, bstat, mz, wscale, filt, wmap, fold, hpot, logc, cstat, total;
    int B, nblk, nablk_a;
};
// anchors per block of the balanced swap's column statistics (per frame; the last block of a frame may be short)
constexpr int BALANCED_SWAP_ABLK = 256;
static SwapSoftmaxWs swap_softmax_layout(int C, int Nc, int Hc, int Wc, int P, int S, int cout_pad, int cols,
                                         bool balanced = false) {
    SwapSoftmaxWs L;
    L.A = swap_apply_layout(C, Nc, Hc, Wc, P, S, cols);
    L.B = cout_pad < SOFTMAX_SWAP_BLOCK ? cout_pad : SOFTMAX_SWAP_BLOCK;
    L.nblk = cdiv(cout_pad, L.B);
    size_t o = L.A.total;
    auto take = [&](size_t bytes) { size_t r = o; o = align_up(o + bytes, 256); return r; };
    const size_t na = (size_t)Nc * L.A.ho * L.A.wo;
    L.ascale = take(na * 4);
    L.bstat = take(na * L.nblk * sizeof(float2));
    L.mz = take(na * sizeof(float2));
    L.wscale = take(4);
    L.filt = take((size_t)2 * C * P * P * L.B * sizeof(__half));
    L.wmap = take((size_t)ActGeom(Nc, Hc + P - 1, Wc + P - 1, L.B).plane * 2 * sizeof(__half));
    L.fold = take((size_t)ActGeom(Nc, Hc + P - 1, Wc + P - 1, C).plane * 2 * sizeof(__half));
    L.nablk_a = cdiv(L.A.ho * L.A.wo, BALANCED_SWAP_ABLK);
    L.hpot = L.logc = L.cstat = 0;
    if (balanced) {
        L.hpot = take((size_t)Nc * cout_pad * 4);
        L.logc = take((size_t)Nc * cout_pad * 4);
        L.cstat = take((size_t)Nc * L.nablk_a * cols * sizeof(float2));
    }
    L.total = o;
    return L;
}
// one chunk (all cout_pad scores), and the least: one block of scores
size_t style_swap_softmax_workspace_bytes(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int P, int S) {
    const int cp = swap_state_layout(C, Hs, Ws, P, S).cout_pad;
    return swap_softmax_layout(C, Nc, Hc, Wc, P, S, cp, cp).total;
}
size_t style_swap_softmax_min_workspace_bytes(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int P, int S) {
    const int cp = swap_state_layout(C, Hs, Ws, P, S).cout_pad;
    return swap_softmax_layout(C, Nc, Hc, Wc, P, S, cp, cp < SOFTMAX_SWAP_BLOCK ? cp : SOFTMAX_SWAP_BLOCK).total;
}

// chunk width of a softmax apply in ws_bytes: all cout_pad patches when the workspace holds their scores, else the largest
// whole number of blocks that fits; 0 when not even one block does
static int softmax_swap_cols(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int P, int S, size_t ws_bytes, bool balanced = false) {
    const int cp = swap_state_layout(C, Hs, Ws, P, S).cout_pad;
    const SwapSoftmaxWs full = swap_softmax_layout(C, Nc, Hc, Wc, P, S, cp, cp, balanced);
    if (ws_bytes >= full.total) return cp;
    int cols = (cp - 1) / full.B * full.B;
    while (cols >= full.B && swap_softmax_layout(C, Nc, Hc, Wc, P, S, cp, cols, balanced).total > ws_bytes) cols -= full.B;
    return cols >= full.B ? cols : 0;
}
// kernels one softmax apply in ws_bytes launches, counted as the hard apply's 11 are (memsets and copies not counted): the
// whitening and colouring suffix (8), the anchor factors and the unscale factor (2), per chunk the correlation and the
// statistics, the combine, the second correlation per chunk when there are several, per block the weights, the filters,
// the fold and the sum; a labelled apply adds the two label resizes and the patch labels.  0 when ws_bytes is too small.
int style_swap_softmax_launches(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int P, int S, size_t ws_bytes, int labelled) {
    const int cols = softmax_swap_cols(C, Nc, Hc, Wc, Hs, Ws, P, S, ws_bytes);
    if (cols == 0) return 0;
    const int cp = swap_state_layout(C, Hs, Ws, P, S).cout_pad;
    const SwapSoftmaxWs L = swap_softmax_layout(C, Nc, Hc, Wc, P, S, cp, cols);
    const int chunks = cdiv(cp, cols);
    return 8 + 2 + 2 * chunks + 1 + (chunks > 1 ? chunks : 0) + 4 * L.nblk + (labelled ? 3 : 0);
}

// the balanced swap's workspaces (the softmax layout plus its buffers; one chunk, and one block of scores) and launches:
// the softmax apply's, plus the targets when iters > 0, per iteration and chunk the column statistics, the column update,
// the row statistics and -- with several chunks -- the correlation, one combine per iteration, and per chunk the column
// statistics and their output when `want_cols`.  0 when ws_bytes is too small.
size_t style_swap_balanced_workspace_bytes(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int P, int S) {
    const int cp = swap_state_layout(C, Hs, Ws, P, S).cout_pad;
    return swap_softmax_layout(C, Nc, Hc, Wc, P, S, cp, cp, true).total;
}
size_t style_swap_balanced_min_workspace_bytes(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int P, int S) {
    const int cp = swap_state_layout(C, Hs, Ws, P, S).cout_pad;
    return swap_softmax_layout(C, Nc, Hc, Wc, P, S, cp, cp < SOFTMAX_SWAP_BLOCK ? cp : SOFTMAX_SWAP_BLOCK, true).total;
}
int style_swap_balanced_launches(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int P, int S, size_t ws_bytes, int labelled,
                                 int iters, int want_cols) {
    if (iters < 0 || iters > BALANCED_SWAP_MAX_ITERS) return 0;
    const int cols = softmax_swap_cols(C, Nc, Hc, Wc, Hs, Ws, P, S, ws_bytes, true);
    if (cols == 0) return 0;
    const int cp = swap_state_layout(C, Hs, Ws, P, S).cout_pad;
    const SwapSoftmaxWs L = swap_softmax_layout(C, Nc, Hc, Wc, P, S, cp, cols, true);
    const int chunks = cdiv(cp, cols);
    const int base = 8 + 2 + 2 * chunks + 1 + (chunks > 1 ? chunks : 0) + 4 * L.nblk + (labelled ? 3 : 0);
    return base + (iters > 0 ? 1 : 0) + iters * (chunks * (chunks > 1 ? 4 : 3) + 1) + (want_cols ? 2 * chunks : 0);
}

// r_a of every anchor of frame blockIdx.y, one warp each: lane l sums wc^2 over the channels l, l+32, .. of every tap in
// tap order, then a fixed butterfly.  rms_f = sqrt(K / n_p).
__global__ void k_softmax_swap_anchor_scale(const __half* __restrict__ wc, ActGeom g, SwapGeom q, float rms_f,
                                            float* __restrict__ ascale) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= q.ho * q.wo) return;
    const int n = blockIdx.y;
    const int y = warp / q.wo, x = warp - y * q.wo;
    float s = 0.f;
    for (int ky = 0; ky < q.P; ++ky)
        for (int kx = 0; kx < q.P; ++kx) {
            const long long pos = ((long long)n * g.Hp + y * q.S + ky + 1) * g.Wp + (x * q.S + kx + 1);
            for (int c = lane; c < g.C; c += 32) {
                const float v = merge_f32(wc[pos * g.C + c], wc[g.plane + pos * g.C + c]);
                s = fmaf(v, v, s);
            }
        }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) ascale[(long long)n * q.ho * q.wo + warp] = s > 0.f ? 1.f / (sqrtf(s) * rms_f) : 0.f;
}
__global__ void k_softmax_swap_set(float* __restrict__ p, float v) { *p = v; }

// whether patch n (< n_patches) is in the allowed set of an anchor with label l (`any`: no patch carries l)
template <bool LABELS>
__device__ __forceinline__ bool softmax_swap_allowed(const SwapLabels& lab, bool any, int l, int n) {
    if constexpr (LABELS) return any || lab.plab[n] == l;
    return true;
}
// the label of anchor (y, x) of frame n, and whether no patch carries it
template <bool LABELS>
__device__ __forceinline__ int softmax_swap_label(const SwapLabels& lab, const ActGeom& g, const SwapGeom& q, int n, int y, int x,
                                                  bool& any) {
    any = true;
    if constexpr (LABELS) {
        const int o = (q.P - 1) / 2;
        const int l = lab.clab[n * lab.clab_frame + (long long)(y * q.S + o) * g.W + x * q.S + o];
        any = ((lab.present[l >> 5] >> (l & 31)) & 1u) == 0u;
        return l;
    }
    return 0;
}

// z(a,n) = s(a,n) r_a, rounded once.  Pass 1 and pass 2 must form the same z bit for bit, so that z - M_a is exactly 0 at
// the maximum (w <= 1/Z_a <= 1): with a plain `merge * r - M` the compiler may contract the product into the subtraction
// (one FFMA, the unrounded product), and at small tau that difference of half an ulp of z becomes a factor exp(delta/tau)
__device__ __forceinline__ float softmax_swap_z(const __half* __restrict__ scores, const ActGeom& g, long long pos, int j, float r) {
    return __fmul_rn(merge_f32(scores[pos * g.C + j], scores[g.plane + pos * g.C + j]), r);
}
// exp((x - m) / tau), formed the same way wherever it is used
__device__ __forceinline__ float softmax_swap_exp(float x, float m, float inv_t) { return expf(__fmul_rn(__fsub_rn(x, m), inv_t)); }

constexpr int SOFTMAX_SWAP_PER_LANE = SOFTMAX_SWAP_BLOCK / 32;
// pass 1: (max_b, sum_b exp((z - max_b) / tau)) over the allowed real patches of each of the `nb` blocks of this chunk
// (scores of patches [n0, n0 + g.C)), one warp per anchor; lane l takes the block's patches l, l+32, .., then fixed
// butterflies.  A block without an allowed patch gives (-inf, 0).  POT (the balanced swap's row step, DESIGN.md §3.3.18)
// takes x = z + h_n, rounded once, in place of z; hpot points at h of patch n0 of frame 0, frames `hstride` apart.
template <bool LABELS, bool POT = false>
__global__ void k_softmax_swap_stats(const __half* __restrict__ scores, ActGeom g, SwapGeom q, int n0, int nb, int B, int n_patches,
                                     const float* __restrict__ ascale, float inv_t, int nblk, float2* __restrict__ bstat,
                                     SwapLabels lab, const float* __restrict__ hpot = nullptr, int hstride = 0) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= q.ho * q.wo) return;
    const int n = blockIdx.y;
    const int y = warp / q.wo, x = warp - y * q.wo;
    const long long a = (long long)n * q.ho * q.wo + warp;
    const long long pos = ((long long)n * g.Hp + y * q.S + 1) * g.Wp + (x * q.S + 1);
    const float r = ascale[a];
    bool any;
    const int l = softmax_swap_label<LABELS>(lab, g, q, n, y, x, any);
    for (int bi = 0; bi < nb; ++bi) {
        float z[SOFTMAX_SWAP_PER_LANE];
        float mx = -INFINITY;
#pragma unroll
        for (int i = 0; i < SOFTMAX_SWAP_PER_LANE; ++i) {
            const int jj = lane + 32 * i, j = bi * B + jj;
            z[i] = -INFINITY;
            if (jj < B && n0 + j < n_patches && softmax_swap_allowed<LABELS>(lab, any, l, n0 + j)) {
                z[i] = softmax_swap_z(scores, g, pos, j, r);
                if constexpr (POT) z[i] = __fadd_rn(z[i], hpot[(long long)n * hstride + j]);
                mx = fmaxf(mx, z[i]);
            }
        }
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        float sum = 0.f;
        if (mx > -INFINITY) {
#pragma unroll
            for (int i = 0; i < SOFTMAX_SWAP_PER_LANE; ++i)
                if (z[i] > -INFINITY) sum += softmax_swap_exp(z[i], mx, inv_t);
        }
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        if (lane == 0) bstat[a * nblk + n0 / B + bi] = make_float2(mx, sum);
    }
}
// (M_a, 1/Z_a) from the blocks' (max, sum), in block order
__global__ void k_softmax_swap_combine(const float2* __restrict__ bstat, long long na, int nblk, float inv_t, float2* __restrict__ mz) {
    for (long long a = (long long)blockIdx.x * blockDim.x + threadIdx.x; a < na; a += (long long)gridDim.x * blockDim.x) {
        const float2* t = bstat + a * nblk;
        float M = -INFINITY;
        for (int b = 0; b < nblk; ++b) M = fmaxf(M, t[b].x);
        float Z = 0.f;
        for (int b = 0; b < nblk; ++b)
            if (t[b].y > 0.f) Z += t[b].y * softmax_swap_exp(t[b].x, M, inv_t);
        mz[a] = make_float2(M, 1.f / Z);
    }
}
// pass 2: the weights of block [n0 + c0, n0 + c0 + gm.C) times 2^15, split, at map pixel (y*S + P-1, x*S + P-1) of every
// anchor; padding, foreign-label and non-patch channels get 0.  One warp per anchor.  POT: x = z + h_n as in the statistics.
template <bool LABELS, bool POT = false>
__global__ void k_softmax_swap_weights(const __half* __restrict__ scores, ActGeom g, SwapGeom q, int n0, int c0, int n_patches,
                                       const float* __restrict__ ascale, const float2* __restrict__ mz, float inv_t, ActGeom gm,
                                       __half* __restrict__ wmap, SwapLabels lab, const float* __restrict__ hpot = nullptr,
                                       int hstride = 0) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= q.ho * q.wo) return;
    const int n = blockIdx.y;
    const int y = warp / q.wo, x = warp - y * q.wo;
    const long long a = (long long)n * q.ho * q.wo + warp;
    const long long pos = ((long long)n * g.Hp + y * q.S + 1) * g.Wp + (x * q.S + 1);
    const long long mpos = ((long long)n * gm.Hp + y * q.S + q.P) * gm.Wp + (x * q.S + q.P);
    const float r = ascale[a];
    const float2 t = mz[a];
    bool any;
    const int l = softmax_swap_label<LABELS>(lab, g, q, n, y, x, any);
    for (int jj = lane; jj < gm.C; jj += 32) {
        const int j = c0 + jj;
        float w = 0.f;
        if (n0 + j < n_patches && softmax_swap_allowed<LABELS>(lab, any, l, n0 + j)) {
            float x = softmax_swap_z(scores, g, pos, j, r);
            if constexpr (POT) x = __fadd_rn(x, hpot[(long long)n * hstride + j]);
            w = softmax_swap_exp(x, t.x, inv_t) * t.y * SOFTMAX_SWAP_WSCALE;
        }
        __half hi, lo;
        split_f32(w, hi, lo);
        wmap[mpos * gm.C + jj] = hi;
        wmap[gm.plane + mpos * gm.C + jj] = lo;
    }
}
// the fold's filters of the patch block [b0, b0 + B): [plane][c][tap = ky*P + kx][j] = the whitened style (hi, lo as stored)
// of patch b0 + j at its pixel (P-1-ky, P-1-kx) -- the raw patches, taps flipped; 0 for padding patches
__global__ void k_softmax_swap_fold_filters(const __half* __restrict__ feat, ActGeom gs, SwapGeom q, int b0, int B, int n_patches,
                                            __half* __restrict__ filt) {
    const int PP = q.P * q.P;
    const long long per = (long long)PP * B, total = per * gs.C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i / per);
        const int rem = (int)(i - c * per);
        const int tap = rem / B, j = rem - tap * B;
        const int nn = b0 + j;
        __half hi = __float2half_rn(0.f), lo = hi;
        if (nn < n_patches) {
            const int dy = q.P - 1 - tap / q.P, dx = q.P - 1 - tap % q.P;
            const int py = nn / q.pcol, px = nn - py * q.pcol;
            const long long pos = ((long long)(py * q.S + dy + 1)) * gs.Wp + (px * q.S + dx + 1);
            hi = feat[pos * gs.C + c];
            lo = feat[gs.plane + pos * gs.C + c];
        }
        filt[i] = hi;
        filt[total + i] = lo;
    }
}
// acc (fp32 [Nc][Hc][Wc][C], in the apply's tmp) = / += the fold of one block, read at interior pixel (Y, X) of
// gf = [Nc, Hc+P-1, Wc+P-1, C]; after the last block the average over the anchors covering (Y, X), split and stored with the
// halo as k_swap_gather does
__global__ void k_softmax_swap_accum(const __half* __restrict__ fold, ActGeom gf, SwapGeom q, ActGeom gc, int first, int last,
                                     float* __restrict__ acc, __half* __restrict__ out) {
    const int cg = gc.C / 8;
    const long long hw = (long long)gc.H * gc.W;
    const long long total = (long long)gc.N * hw * cg;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c0 = (int)(i % cg) * 8;
        const long long fp = i / cg;
        const int n = (int)(fp / hw);
        const int pix = (int)(fp - n * hw);
        const int Y = pix / gc.W, X = pix - Y * gc.W;
        float v[8];
        load8(fold, gf, ((long long)n * gf.Hp + Y + 1) * gf.Wp + X + 1, c0, v);
        float4* ap = reinterpret_cast<float4*>(acc + fp * gc.C + c0);
        if (!first) {
            const float4 u0 = ap[0], u1 = ap[1];
            v[0] = u0.x + v[0]; v[1] = u0.y + v[1]; v[2] = u0.z + v[2]; v[3] = u0.w + v[3];
            v[4] = u1.x + v[4]; v[5] = u1.y + v[5]; v[6] = u1.z + v[6]; v[7] = u1.w + v[7];
        }
        if (!last) {
            ap[0] = make_float4(v[0], v[1], v[2], v[3]);
            ap[1] = make_float4(v[4], v[5], v[6], v[7]);
            continue;
        }
        int cy = 0, cx = 0;
        for (int d = 0; d < q.P; ++d) {
            const int ty = Y - d, tx = X - d;
            if (ty >= 0 && ty % q.S == 0 && ty / q.S < q.ho) ++cy;
            if (tx >= 0 && tx % q.S == 0 && tx / q.S < q.wo) ++cx;
        }
        const int cnt = cy * cx;
        const float inv = cnt > 0 ? 1.f / (float)cnt : 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] *= inv;
        Half8 hi, lo;
        split8(v, hi, lo);
        store8_with_halo(out, gc, n, Y, X, c0, hi, lo);
    }
}

// ---------------------------------------------------------------------------
// Balanced style swap (DESIGN.md §3.3.18): Sinkhorn iterations on the softmax swap's plan.  Potentials h_n (units of z,
// one per frame and patch) enter as x(a,n) = z(a,n) + h_n; the row step is the softmax swap's statistics of x, and the
// column step moves h_n by tau (log c_n - log S_n), S_n = sum_a exp((x - M_a) / tau) / Z_a over the anchors that may take n.
// ---------------------------------------------------------------------------
// log c_n of every patch of frame blockIdx.x: c_n = cnt(l(n)) / np(l(n)) + F / n_p from exact integer histograms (anchors
// per present label, patches per label, F the anchors whose label the style lacks); without labels cnt = 0, np = 1 and
// F = Na, so c_n = Na / n_p.  Padding patches and c_n = 0 (no anchor may take n) get -inf.
template <bool LABELS>
__global__ void k_balanced_swap_targets(ActGeom g, SwapGeom q, int n_patches, int cp, SwapLabels lab, float* __restrict__ logc) {
    __shared__ int ha[256], hp[256], fallback;
    const int n = blockIdx.x, npos = q.ho * q.wo;
    for (int i = threadIdx.x; i < 256; i += blockDim.x) ha[i] = hp[i] = 0;
    if (threadIdx.x == 0) fallback = LABELS ? 0 : npos;
    __syncthreads();
    if constexpr (LABELS) {
        for (int a = threadIdx.x; a < npos; a += blockDim.x) {
            const int y = a / q.wo, x = a - y * q.wo;
            bool any;
            const int l = softmax_swap_label<true>(lab, g, q, n, y, x, any);
            atomicAdd(any ? &fallback : &ha[l], 1);
        }
        for (int p = threadIdx.x; p < n_patches; p += blockDim.x) atomicAdd(&hp[lab.plab[p]], 1);
    }
    __syncthreads();
    const float f = __fdiv_rn((float)fallback, (float)n_patches);
    for (int p = threadIdx.x; p < cp; p += blockDim.x) {
        float c = 0.f;
        if (p < n_patches) {
            const int l = LABELS ? lab.plab[p] : 0;
            c = __fadd_rn(__fdiv_rn((float)ha[l], (float)(LABELS ? hp[l] : 1)), f);
        }
        logc[(long long)n * cp + p] = c > 0.f ? logf(c) : -INFINITY;
    }
}

// the column statistics of the chunk's patches [n0, n0 + g.C) over anchor block blockIdx.y of frame blockIdx.z: one thread
// per patch (the contiguous axis of the scores), the block's anchors in order, an online (max, sum of exp) of
// e(a,n) = (x(a,n) - M_a) / tau + log(1 / Z_a) over the anchors that may take n.  (-inf, 0) when none may.
// cstat [Nc][nablk][g.C]; (M_a, 1/Z_a) and r_a of the block's anchors are staged in shared memory.
template <bool LABELS>
__global__ void __launch_bounds__(BALANCED_SWAP_ABLK) k_balanced_swap_col_stats(
    const __half* __restrict__ scores, ActGeom g, SwapGeom q, int n0, int n_patches, const float* __restrict__ ascale,
    const float2* __restrict__ mz, const float* __restrict__ hpot, int cp, float inv_t, int nablk, float2* __restrict__ cstat,
    SwapLabels lab) {
    __shared__ float s_r[BALANCED_SWAP_ABLK], s_m[BALANCED_SWAP_ABLK], s_lz[BALANCED_SWAP_ABLK];
    __shared__ int s_l[BALANCED_SWAP_ABLK];
    const int n = blockIdx.z, ab = blockIdx.y, npos = q.ho * q.wo;
    const int a0 = ab * BALANCED_SWAP_ABLK;
    const int na = npos - a0 < BALANCED_SWAP_ABLK ? npos - a0 : BALANCED_SWAP_ABLK;
    for (int i = threadIdx.x; i < na; i += blockDim.x) {
        const long long a = (long long)n * npos + a0 + i;
        const float2 t = mz[a];
        s_r[i] = ascale[a];
        s_m[i] = t.x;
        s_lz[i] = logf(t.y);
        s_l[i] = -1;
        if constexpr (LABELS) {
            const int y = (a0 + i) / q.wo, x = (a0 + i) - y * q.wo;
            bool any;
            const int l = softmax_swap_label<true>(lab, g, q, n, y, x, any);
            s_l[i] = any ? -1 : l;
        }
    }
    __syncthreads();
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= g.C || n0 + j >= n_patches) return;
    const float h = hpot[(long long)n * cp + n0 + j];
    const int pl = LABELS ? (int)lab.plab[n0 + j] : 0;
    float mx = -INFINITY, sum = 0.f;
    for (int i = 0; i < na; ++i) {
        if (LABELS && s_l[i] >= 0 && s_l[i] != pl) continue;
        const int y = (a0 + i) / q.wo, x = (a0 + i) - y * q.wo;
        const long long pos = ((long long)n * g.Hp + y * q.S + 1) * g.Wp + (x * q.S + 1);
        const float xv = __fadd_rn(softmax_swap_z(scores, g, pos, j, s_r[i]), h);
        const float e = __fadd_rn(__fmul_rn(__fsub_rn(xv, s_m[i]), inv_t), s_lz[i]);
        if (e > mx) {
            sum = sum * expf(mx - e) + 1.f;
            mx = e;
        } else {
            sum += expf(e - mx);
        }
    }
    cstat[((long long)n * nablk + ab) * g.C + j] = make_float2(mx, sum);
}

// log S_n of the chunk's patches from the anchor blocks' (max, sum), in block order; then either the column step
// h_n += tau (log c_n - log S_n) (col_sums == nullptr; patches with c_n = 0 are left alone) or S_n into col_sums [Nc][n_p].
// Grid (patches of the chunk, Nc).
__global__ void k_balanced_swap_col_update(const float2* __restrict__ cstat, int m, int n0, int n_patches, int cp, int nablk,
                                           const float* __restrict__ logc, float tau, float* __restrict__ hpot,
                                           float* __restrict__ col_sums) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x, n = blockIdx.y;
    if (j >= m || n0 + j >= n_patches) return;
    const float2* t = cstat + (long long)n * nablk * m + j;
    float M = -INFINITY;
    for (int b = 0; b < nablk; ++b) M = fmaxf(M, t[(long long)b * m].x);
    float S = 0.f;
    for (int b = 0; b < nablk; ++b) {
        const float2 v = t[(long long)b * m];
        if (v.y > 0.f) S += v.y * expf(__fsub_rn(v.x, M));
    }
    const float log_s = S > 0.f ? __fadd_rn(M, logf(S)) : -INFINITY;
    const long long k = (long long)n * cp + n0 + j;
    if (col_sums) {
        col_sums[(long long)n * n_patches + n0 + j] = expf(log_s);
        return;
    }
    const float lc = logc[k];
    if (lc == -INFINITY || log_s == -INFINITY) return;
    hpot[k] = __fadd_rn(hpot[k], __fmul_rn(tau, __fsub_rn(lc, log_s)));
}

// The softmax apply and, with `balanced`, the balanced one (DESIGN.md §3.3.18): `iters` Sinkhorn iterations between pass 1
// and pass 2, each a column step then a row step, and the final plan's column sums into `col_sums` when it is given.  A
// balanced apply uses the balanced workspace layout; at iters = 0 it runs the softmax apply's launches, and its bytes.
static int style_swap_apply_softmax_impl(const __half* content, int Nc, int Hc, int Wc, int C, const void* state, int Hs, int Ws,
                                         int patch, int stride, float alpha, float eps_cov, float thresh, float temperature,
                                         __half* out, int32_t* k_out, void* ws, size_t ws_bytes, const SwapLabelMaps* maps,
                                         cudaStream_t st, bool balanced = false, int iters = 0, float* col_sums = nullptr) {
    const char* fn = balanced ? "style_swap_apply_balanced" : "style_swap_apply_softmax";
    // a normal float: a subnormal tau has no finite 1/tau, and (z - M) * inf would be NaN at every maximum
    WCTB_REQUIRE(std::isfinite(temperature) && temperature >= FLT_MIN && std::isfinite(1.f / temperature),
                 "%s: temperature %g must be a finite, normal float32 > 0", fn, (double)temperature);
    WCTB_REQUIRE(iters >= 0 && iters <= BALANCED_SWAP_MAX_ITERS, "%s: iters %d not in 0..%d", fn, iters, BALANCED_SWAP_MAX_ITERS);
    SwapLabels lab = {nullptr, 0, nullptr, nullptr};
    SwapLabelWs LL = {};
    int rc = swap_apply_check(Nc, Hc, Wc, C, Hs, Ws, patch, stride, maps, &LL);
    if (rc) return rc;
    const SwapState SL = swap_state_layout(C, Hs, Ws, patch, stride);
    const int cp = SL.cout_pad;
    const int cols = softmax_swap_cols(C, Nc, Hc, Wc, Hs, Ws, patch, stride, ws_bytes, balanced);
    if (cols == 0) {
        set_error("%s: workspace %zu < %zu bytes", fn, ws_bytes,
                  balanced ? style_swap_balanced_min_workspace_bytes(C, Nc, Hc, Wc, Hs, Ws, patch, stride)
                           : style_swap_softmax_min_workspace_bytes(C, Nc, Hc, Wc, Hs, Ws, patch, stride));
        return WCTB200_EWS;
    }
    const SwapSoftmaxWs L = swap_softmax_layout(C, Nc, Hc, Wc, patch, stride, cp, cols, balanced);
    const SwapApplyWs& AL = L.A;
    const int B = L.B;
    const SwapGeom q = {patch, stride, SL.prow, SL.pcol, AL.ho, AL.wo};
    uint8_t* sw = static_cast<uint8_t*>(ws);
    const uint8_t* sp = static_cast<const uint8_t*>(state);
    const int* kc = reinterpret_cast<const int*>(sw + AL.base + wct_layout(C, Nc, 0).kcount);
    __half* wc_feat = reinterpret_cast<__half*>(sw + AL.wc_feat);
    __half* ss_feat = reinterpret_cast<__half*>(sw + AL.ss_feat);
    __half* tmp = reinterpret_cast<__half*>(sw + AL.tmp);
    __half* scores = reinterpret_cast<__half*>(sw + AL.scores);
    float* ascale = reinterpret_cast<float*>(sw + L.ascale);
    float2* bstat = reinterpret_cast<float2*>(sw + L.bstat);
    float2* mz = reinterpret_cast<float2*>(sw + L.mz);
    float* wscale = reinterpret_cast<float*>(sw + L.wscale);
    __half* filt = reinterpret_cast<__half*>(sw + L.filt);
    __half* wmap = reinterpret_cast<__half*>(sw + L.wmap);
    __half* fold = reinterpret_cast<__half*>(sw + L.fold);
    const ActGeom gc(Nc, Hc, Wc, C), gs(1, Hs, Ws, C);
    const ActGeom gm(Nc, Hc + patch - 1, Wc + patch - 1, B), gf(Nc, Hc + patch - 1, Wc + patch - 1, C);
    rc = swap_apply_whiten(content, Nc, Hc, Wc, C, sw + AL.base, reinterpret_cast<float*>(sw + AL.zeros), eps_cov, thresh, wc_feat,
                           st);
    if (rc) return rc;
    if (maps) {
        rc = swap_labels_setup(maps, LL, Hc, Wc, Hs, Ws, q, SL.n_patches, &lab, st);
        if (rc) return rc;
    }
    const long long K = (long long)patch * patch * C;
    const __half* wsplit = reinterpret_cast<const __half*>(sp + SL.wsplit);
    const int BN = conv_tc_bn(cp);
    const int npos = AL.ho * AL.wo;
    const float inv_t = 1.f / temperature;
    const dim3 agrid((unsigned)cdiv((long long)npos * 32, 256), (unsigned)Nc);
    k_softmax_swap_anchor_scale<<<agrid, 256, 0, st>>>(wc_feat, gc, q, (float)std::sqrt((double)K / SL.n_patches), ascale);
    WCTB_CHECK_LAUNCH("k_softmax_swap_anchor_scale");
    k_softmax_swap_set<<<1, 1, 0, st>>>(wscale, 1.f / SOFTMAX_SWAP_WSCALE);
    WCTB_CHECK_LAUNCH("k_softmax_swap_set");
    // pass 1: the correlation (the hard swap's launches and bits) and the statistics of every block
    for (int n0 = 0; n0 < cp; n0 += cols) {
        const int m = cp - n0 < cols ? cp - n0 : cols;
        rc = launch_conv_taps_rows(wc_feat, Nc, Hc, Wc, C, wsplit + (long long)n0 * K, (long long)cp * K, m, BN, scores, st, patch);
        if (rc) return rc;
        if (maps)
            k_softmax_swap_stats<true><<<agrid, 256, 0, st>>>(scores, ActGeom(Nc, Hc, Wc, m), q, n0, cdiv(m, B), B, SL.n_patches,
                                                              ascale, inv_t, L.nblk, bstat, lab);
        else
            k_softmax_swap_stats<false><<<agrid, 256, 0, st>>>(scores, ActGeom(Nc, Hc, Wc, m), q, n0, cdiv(m, B), B, SL.n_patches,
                                                               ascale, inv_t, L.nblk, bstat, lab);
        WCTB_CHECK_LAUNCH("k_softmax_swap_stats");
    }
    const long long na = (long long)Nc * npos;
    k_softmax_swap_combine<<<swap_grid(na, 256), 256, 0, st>>>(bstat, na, L.nblk, inv_t, mz);
    WCTB_CHECK_LAUNCH("k_softmax_swap_combine");
    // the balanced swap's iterations: per chunk (the correlation again when there are several) the column step of its
    // patches from the previous (M_a, Z_a), then its row statistics with the new h; the rows are combined after the last
    // chunk.  h = 0 until the first column step, where z + 0 = z: pass 1 is the row step of h = 0.
    float* hpot = reinterpret_cast<float*>(sw + L.hpot);
    float* logc = reinterpret_cast<float*>(sw + L.logc);
    float2* cstat = reinterpret_cast<float2*>(sw + L.cstat);
    if (iters > 0 || col_sums) WCTB_CUDA(cudaMemsetAsync(hpot, 0, (size_t)Nc * cp * 4, st));
    if (iters > 0) {
        if (maps)
            k_balanced_swap_targets<true><<<(unsigned)Nc, 1024, 0, st>>>(gc, q, SL.n_patches, cp, lab, logc);
        else
            k_balanced_swap_targets<false><<<(unsigned)Nc, 1024, 0, st>>>(gc, q, SL.n_patches, cp, lab, logc);
        WCTB_CHECK_LAUNCH("k_balanced_swap_targets");
    }
    // the column statistics of one chunk's patches, then the column step (col_out == nullptr) or the column sums
    auto column_pass = [&](int n0, int m, float* col_out) {
        const dim3 cgrid((unsigned)cdiv(m, BALANCED_SWAP_ABLK), (unsigned)L.nablk_a, (unsigned)Nc);
        if (maps)
            k_balanced_swap_col_stats<true><<<cgrid, BALANCED_SWAP_ABLK, 0, st>>>(scores, ActGeom(Nc, Hc, Wc, m), q, n0, SL.n_patches,
                                                                                 ascale, mz, hpot, cp, inv_t, L.nablk_a, cstat, lab);
        else
            k_balanced_swap_col_stats<false><<<cgrid, BALANCED_SWAP_ABLK, 0, st>>>(scores, ActGeom(Nc, Hc, Wc, m), q, n0, SL.n_patches,
                                                                                  ascale, mz, hpot, cp, inv_t, L.nablk_a, cstat, lab);
        WCTB_CHECK_LAUNCH("k_balanced_swap_col_stats");
        k_balanced_swap_col_update<<<dim3((unsigned)cdiv(m, 256), (unsigned)Nc), 256, 0, st>>>(cstat, m, n0, SL.n_patches, cp, L.nablk_a,
                                                                                             logc, temperature, hpot, col_out);
        WCTB_CHECK_LAUNCH("k_balanced_swap_col_update");
    };
    for (int it = 0; it < iters; ++it) {
        for (int n0 = 0; n0 < cp; n0 += cols) {
            const int m = cp - n0 < cols ? cp - n0 : cols;
            if (cols < cp) {
                rc = launch_conv_taps_rows(wc_feat, Nc, Hc, Wc, C, wsplit + (long long)n0 * K, (long long)cp * K, m, BN, scores, st, patch);
                if (rc) return rc;
            }
            column_pass(n0, m, nullptr);
            if (maps)
                k_softmax_swap_stats<true, true><<<agrid, 256, 0, st>>>(scores, ActGeom(Nc, Hc, Wc, m), q, n0, cdiv(m, B), B,
                                                                        SL.n_patches, ascale, inv_t, L.nblk, bstat, lab, hpot + n0, cp);
            else
                k_softmax_swap_stats<false, true><<<agrid, 256, 0, st>>>(scores, ActGeom(Nc, Hc, Wc, m), q, n0, cdiv(m, B), B,
                                                                         SL.n_patches, ascale, inv_t, L.nblk, bstat, lab, hpot + n0, cp);
            WCTB_CHECK_LAUNCH("k_softmax_swap_stats");
        }
        k_softmax_swap_combine<<<swap_grid(na, 256), 256, 0, st>>>(bstat, na, L.nblk, inv_t, mz);
        WCTB_CHECK_LAUNCH("k_softmax_swap_combine");
    }
    // pass 2: the correlation again when it ran in more than one chunk (the scores are the same bits), then per block the
    // weight map, the block's filters, the fold on the tensor cores and its sum in block order
    WCTB_CUDA(cudaMemsetAsync(wmap, 0, (size_t)gm.plane * 2 * sizeof(__half), st));
    const long long PPCB = (long long)patch * patch * C * B;
    for (int n0 = 0; n0 < cp; n0 += cols) {
        const int m = cp - n0 < cols ? cp - n0 : cols;
        if (cols < cp) {
            rc = launch_conv_taps_rows(wc_feat, Nc, Hc, Wc, C, wsplit + (long long)n0 * K, (long long)cp * K, m, BN, scores, st, patch);
            if (rc) return rc;
        }
        if (col_sums) column_pass(n0, m, col_sums);
        for (int c0 = 0; c0 < m; c0 += B) {
            const int b = (n0 + c0) / B;
            if (iters > 0 && maps)
                k_softmax_swap_weights<true, true><<<agrid, 256, 0, st>>>(scores, ActGeom(Nc, Hc, Wc, m), q, n0, c0, SL.n_patches,
                                                                          ascale, mz, inv_t, gm, wmap, lab, hpot + n0, cp);
            else if (iters > 0)
                k_softmax_swap_weights<false, true><<<agrid, 256, 0, st>>>(scores, ActGeom(Nc, Hc, Wc, m), q, n0, c0, SL.n_patches,
                                                                           ascale, mz, inv_t, gm, wmap, lab, hpot + n0, cp);
            else if (maps)
                k_softmax_swap_weights<true><<<agrid, 256, 0, st>>>(scores, ActGeom(Nc, Hc, Wc, m), q, n0, c0, SL.n_patches, ascale,
                                                                    mz, inv_t, gm, wmap, lab);
            else
                k_softmax_swap_weights<false><<<agrid, 256, 0, st>>>(scores, ActGeom(Nc, Hc, Wc, m), q, n0, c0, SL.n_patches, ascale,
                                                                     mz, inv_t, gm, wmap, lab);
            WCTB_CHECK_LAUNCH("k_softmax_swap_weights");
            k_softmax_swap_fold_filters<<<swap_grid(PPCB, 256), 256, 0, st>>>(reinterpret_cast<const __half*>(sp + SL.feat), gs, q,
                                                                              n0 + c0, B, SL.n_patches, filt);
            WCTB_CHECK_LAUNCH("k_softmax_swap_fold_filters");
            rc = launch_conv_tc(CONV_TAPS, wmap, Nc, gm.H, gm.W, B, filt, 1, wscale, nullptr, C, 0, fold, st, patch);
            if (rc) return rc;
            k_softmax_swap_accum<<<swap_grid((long long)Nc * Hc * Wc * (C / 8), 256), 256, 0, st>>>(
                fold, gf, q, gc, b == 0, b == L.nblk - 1, reinterpret_cast<float*>(tmp), ss_feat);
            WCTB_CHECK_LAUNCH("k_softmax_swap_accum");
        }
    }
    return swap_apply_finish(ss_feat, content, Nc, Hc, Wc, C, sp, SL, kc, alpha, tmp, out, k_out, st);
}
int launch_style_swap_apply_softmax(const __half* content, int Nc, int Hc, int Wc, int C, const void* state, int Hs, int Ws,
                                    int patch, int stride, float alpha, float eps_cov, float thresh, float temperature,
                                    const uint8_t* content_labels, int Ncl, int Hm, int Wm, const uint8_t* style_labels, int Hms,
                                    int Wms, __half* out, int32_t* k_out, void* ws, size_t ws_bytes, void* label_buf,
                                    size_t label_bytes, cudaStream_t st) {
    WCTB_REQUIRE((content_labels == nullptr) == (style_labels == nullptr),
                 "style_swap_apply_softmax: give both label maps or neither");
    const SwapLabelMaps maps = {content_labels, Ncl, Hm, Wm, style_labels, Hms, Wms, label_buf, label_bytes};
    return style_swap_apply_softmax_impl(content, Nc, Hc, Wc, C, state, Hs, Ws, patch, stride, alpha, eps_cov, thresh, temperature,
                                         out, k_out, ws, ws_bytes, content_labels ? &maps : nullptr, st);
}
int launch_style_swap_apply_balanced(const __half* content, int Nc, int Hc, int Wc, int C, const void* state, int Hs, int Ws,
                                     int patch, int stride, float alpha, float eps_cov, float thresh, float temperature, int iters,
                                     const uint8_t* content_labels, int Ncl, int Hm, int Wm, const uint8_t* style_labels, int Hms,
                                     int Wms, __half* out, int32_t* k_out, float* col_sums, void* ws, size_t ws_bytes,
                                     void* label_buf, size_t label_bytes, cudaStream_t st) {
    WCTB_REQUIRE((content_labels == nullptr) == (style_labels == nullptr),
                 "style_swap_apply_balanced: give both label maps or neither");
    const SwapLabelMaps maps = {content_labels, Ncl, Hm, Wm, style_labels, Hms, Wms, label_buf, label_bytes};
    return style_swap_apply_softmax_impl(content, Nc, Hc, Wc, C, state, Hs, Ws, patch, stride, alpha, eps_cov, thresh, temperature,
                                         out, k_out, ws, ws_bytes, content_labels ? &maps : nullptr, st, true, iters, col_sums);
}

int launch_style_swap_level(const __half* content, int Hc, int Wc, const __half* style, int Hs, int Ws, int C, int patch, int stride,
                            float alpha, float eps_cov, float thresh, __half* out, int32_t* k_out, void* ws, size_t ws_bytes,
                            cudaStream_t st) {
    int rc = swap_check_style(C, Hs, Ws, patch, stride);
    if (rc) return rc;
    WCTB_REQUIRE(Hc >= patch && Wc >= patch && Hc >= 2 && Wc >= 2,
                 "style_swap: maps must be at least %dx%d (content %dx%d, style %dx%d)", patch, patch, Hc, Wc, Hs, Ws);
    WCTB_REQUIRE(((Hc - patch) / stride) * stride + patch == Hc && ((Wc - patch) / stride) * stride + patch == Wc,
                 "style_swap: patch %d / stride %d does not tile a %dx%d encoding (refit the content: swap_filter_fit, wct.py:84-90)",
                 patch, stride, Hc, Wc);
    const size_t need = style_swap_workspace_bytes(C, Hc, Wc, Hs, Ws, patch, stride);
    if (ws_bytes < need) {
        set_error("style_swap: workspace %zu < %zu bytes", ws_bytes, need);
        return WCTB200_EWS;
    }
    const size_t sbytes = style_swap_state_bytes(C, Hs, Ws, patch, stride);
    uint8_t* state = static_cast<uint8_t*>(ws);
    rc = launch_style_swap_prepare(style, Hs, Ws, C, patch, stride, eps_cov, thresh, state, nullptr, state + sbytes, ws_bytes - sbytes,
                                   st);
    if (rc) return rc;
    return launch_style_swap_apply(content, 1, Hc, Wc, C, state, Hs, Ws, patch, stride, alpha, eps_cov, thresh, out, k_out,
                                   state + sbytes, ws_bytes - sbytes, st);
}

}  // namespace wctb
