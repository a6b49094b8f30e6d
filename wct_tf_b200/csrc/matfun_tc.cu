// Whitening / colouring matrices WITHOUT an eigendecomposition when every eigenvalue is kept.
//
//   reference: ops.py:53-77 (wct_tf) / ops.py:110-128 (wct_np):  U S V^T = svd(cov);  k = #{S > 1e-5};
//              W_c = E_k S_k^-1/2 E_k^T   (content),   C_s = E_k S_k^+1/2 E_k^T   (style).
//
// When k = C (no eigenvalue at or below the threshold) these are the matrix functions  A^-1/2  and  A^+1/2  of
// A = cov (+ eps_eig I), and both come out of ONE coupled Newton-Schulz iteration (Denman-Beavers in Higham's stable
// product form) that consists of nothing but C x C x C products -- tensor-core work instead of ~1.7 M plane rotations:
//       Y_0 = A / s,  Z_0 = I                  (s = ||A||_F >= lambda_max)
//       T   = (3 I - Z Y) / 2 ;   Y <- Y T ;   Z <- T Z          ->   Y -> (A/s)^1/2 ,  Z -> (A/s)^-1/2
// The products are TRUE products (A operand K-major, B operand MN-major through the wgmma descriptors): although every
// iterate is symmetric in exact arithmetic, using rows for columns destabilises the iteration.  All operands live in HBM/L2 as split-fp16 planes [matrix][hi|lo][C][C]; a product is one launch of
// `ns_gemm_kernel` (the TMA / wgmma pipeline of conv_tc.cu: a_hi b_hi + a_hi b_lo + a_lo b_hi, chunks of 4 k-iterations
// summed in fp32 registers), batched over the matrices of a level.  The residual max|I - Z Y| falls out of the first product of an
// iteration; a matrix that reaches `tol` is skipped by every later launch (`conv_iter`), so the launch count is fixed and
// nothing synchronises with the host.
//
// Guard (all on the device, per matrix).  The fast path is taken only if (i) the iteration converged within the budget
// (cond(A) up to ~1e4) and (ii) the threshold provably keeps every eigenvalue:  1 / lambda_min <= sum_i 1 / lambda_i =
// ||A^-1/2||_F^2 = ||Z||_F^2 / s, so  s / ||Z||_F^2 - eps_eig > thresh * 1.01  implies  lambda_min(cov) > thresh, i.e. k = C.
// Everything else -- rank-deficient or ill-conditioned covariances, eigenvalues near the threshold -- is left to the Jacobi
// eigensolver, whose kernels skip the matrices flagged here (`ok`).  Measured accuracy of the products (split-fp16 x3):
// tests/test_gpu_transform.py holds the transformed features to 1e-3 of the eigendecomposition in float64.
#include <math.h>

#include "common.cuh"

namespace wctb {

int make_tensor_map_3d(CUtensorMap* m, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1_bytes,
                       uint64_t stride2_bytes, uint32_t box1);

struct NsCfg {
    static constexpr int BM = 128, BN = 128, BK = 64;
    static constexpr int A_BYTES = BM * BK * 2;
    static constexpr int B_BYTES = BN * BK * 2;
    static constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * B_BYTES;      // 64 KB
    static constexpr int STAGES = 2;
    static constexpr int CH = 4;                                       // k-iterations per accumulation chunk
    static constexpr int CONSUMERS = 256;                              // two wgmma warpgroups (64 rows each)
    static constexpr int THREADS = CONSUMERS + 128;                    // + producer warpgroup
    static constexpr int AUX_BYTES = 512;
    static constexpr int PITCH = BN + 4;
    static constexpr int TILE_BYTES = BM * PITCH * 4;                  // fp32 tile, aliased with the store staging buffers
    static constexpr int STG_BYTES = 8 * 8192;                         // per-warp transposition buffer (coalesced row stores)
    static constexpr int EPI_BYTES = TILE_BYTES > STG_BYTES ? TILE_BYTES : STG_BYTES;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + AUX_BYTES + EPI_BYTES + 1024;
};

struct NsState {                 // per matrix
    float s;                     // ||A||_F
    float f32_scale;             // factor of the fp32 output: s^-1/2 (whitening) or s^+1/2 (colouring)
    int conv_iter;               // iteration whose residual was below tol (INT_MAX: not yet)
    unsigned int resid_bits;     // max |I - Z Y| of the running iteration (float bits, >= 0)
    int tiles_done;
    int ok;                      // set by k_ns_finish
    float last_resid;
    int pad;
};

struct NsGemmParams {
    int n, batch, tiles_m, it, mode;          // mode 1: T = 1.5 I - 0.5 A B (+ residual); mode 2: A B
    int f32_rule;                             // 0: no fp32 output; 1: matrices b < n_first; 2: matrices b >= n_first
    int n_first;
    int want_zz;                              // per-tile sums of squares of the output (the guard's ||Z||_F^2)
    float tol;
    NsState* state;
    __half* out_split;                        // [batch][2][n][n]
    float* out_f32;                           // [batch][n][n]
    float* zz_slots;                          // [batch][tiles_m * tiles_m]
    unsigned int* err;
};

__global__ void __launch_bounds__(NsCfg::THREADS, 1)
ns_gemm_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, const NsGemmParams p) {
    using Cfg = NsCfg;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* aux = smem + Cfg::STAGES * Cfg::STAGE_BYTES;
    uint64_t* full = reinterpret_cast<uint64_t*>(aux);
    uint64_t* empty = full + Cfg::STAGES;
    volatile int* abort_flag = reinterpret_cast<volatile int*>(empty + Cfg::STAGES);
    float* red = reinterpret_cast<float*>(aux + 256);          // [8] epilogue partials
    uint8_t* epi = aux + Cfg::AUX_BYTES;
    float* ctile = reinterpret_cast<float*>(epi);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    {
        __shared__ unsigned int s_prev_err;
        if (threadIdx.x == 0) s_prev_err = *reinterpret_cast<volatile unsigned int*>(p.err);
        __syncthreads();
        if (s_prev_err != 0u) return;
    }
    if (threadIdx.x == 0) {
        for (int s = 0; s < Cfg::STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], Cfg::CONSUMERS / 32);
        }
        *abort_flag = 0;
        fence_barrier_init();
        tma_prefetch_desc(&mapA);
        tma_prefetch_desc(&mapB);
    }
    __syncthreads();

    const int kiters = p.n / Cfg::BK;
    const int nchunks = (kiters + Cfg::CH - 1) / Cfg::CH;
    const int tpm = p.tiles_m * p.tiles_m;
    const int total_tiles = p.batch * tpm;
    // a matrix that has converged is skipped from the NEXT iteration on (conv_iter is written by the last tile of the
    // mode-1 product of iteration `it` itself: `it > conv_iter` is false for every reader of this launch either way)
    auto skipped = [&](int b) { return p.it > *reinterpret_cast<volatile int*>(&p.state[b].conv_iter); };

    if (warp >= Cfg::CONSUMERS / 32) {
        setmaxnreg_dec<40>();
        if (warp == Cfg::CONSUMERS / 32 && lane == 0) {
            uint32_t itg = 0;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const int b = tile / tpm, r = tile - b * tpm;
                if (skipped(b)) continue;
                const int mi = r / p.tiles_m, ni = r - mi * p.tiles_m;
                const int rowA = (b * 2) * p.n + mi * Cfg::BM;           // plane 0; plane 1 is n rows further
                const int rowB = (b * 2) * p.n;                          // B: k-rows of plane 0 start here
                const int colB = ni * Cfg::BN;
                for (int ki = 0; ki < kiters; ++ki, ++itg) {
                    const int s = itg % Cfg::STAGES;
                    mbar_wait(&empty[s], ((itg / Cfg::STAGES) & 1) ^ 1u, abort_flag, p.err, 0x150u + s);
                    uint8_t* st = smem + s * Cfg::STAGE_BYTES;
                    mbar_arrive_expect_tx(&full[s], Cfg::STAGE_BYTES);
                    tma_load_3d(st, &mapA, &full[s], ki * Cfg::BK, rowA, 0);
                    tma_load_3d(st + Cfg::A_BYTES, &mapA, &full[s], ki * Cfg::BK, rowA + p.n, 0);
                    // B is read as it stands -- rows k, columns j -- i.e. MN-major: four [64 k][64 j] boxes (hi j-groups, lo j-groups)
                    uint8_t* sb = st + 2 * Cfg::A_BYTES;
                    tma_load_3d(sb, &mapB, &full[s], colB, rowB + ki * Cfg::BK, 0);
                    tma_load_3d(sb + 8192, &mapB, &full[s], colB + 64, rowB + ki * Cfg::BK, 0);
                    tma_load_3d(sb + 16384, &mapB, &full[s], colB, rowB + p.n + ki * Cfg::BK, 0);
                    tma_load_3d(sb + 24576, &mapB, &full[s], colB + 64, rowB + p.n + ki * Cfg::BK, 0);
                }
            }
        }
        return;
    }

    // ---- consumer warpgroups: rows [64 wg, 64 wg + 64) of the tile; then the epilogue, one row and 64 columns per thread ----
    setmaxnreg_inc<232>();
    const int wg = warp >> 2;
    const int t = threadIdx.x & 127;
    const int e = warp;
    const int g = e & 3;
    const int colbase = (e >> 2) * 64;
    uint32_t itg = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int b = tile / tpm, r = tile - b * tpm;
        if (skipped(b)) continue;
        const int mi = r / p.tiles_m, ni = r - mi * p.tiles_m;
        float sum[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) sum[i] = 0.f;
        int ki = 0;
        for (int c = 0; c < nchunks; ++c) {
            float ch[64];
#pragma unroll
            for (int i = 0; i < 64; ++i) ch[i] = 0.f;
            const int it_end = min(kiters, (c + 1) * Cfg::CH);
            for (; ki < it_end; ++ki, ++itg) {
                const int s = itg % Cfg::STAGES;
                mbar_wait(&full[s], (itg / Cfg::STAGES) & 1, abort_flag, p.err, 0x250u + s);
                // A K-major (rows of A), B MN-major (rows of B are the contraction index): TRUE products A B.  (Using B's rows
                // as columns -- legitimate for exactly symmetric B -- makes the iteration unstable: the iterates only commute
                // up to rounding, and the transposed products diverge after reaching ~1e-4; tools/ns_emulation.py.)
                const uint32_t st = smem_u32(smem + s * Cfg::STAGE_BYTES);
                const uint64_t a_hi = gmma_desc_sw128(st + wg * (Cfg::A_BYTES / 2));
                const uint64_t a_lo = gmma_desc_sw128(st + Cfg::A_BYTES + wg * (Cfg::A_BYTES / 2));
                const bool first = (ki == c * Cfg::CH);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < Cfg::BK / 16; ++k) {
                    const uint64_t ko = (uint64_t)(k * 32 >> 4);
                    const uint64_t b_hi = gmma_desc_mn_sw128(st + 2 * Cfg::A_BYTES + k * 2048);          // 16 k-rows of 128 B per step
                    const uint64_t b_lo = gmma_desc_mn_sw128(st + 2 * Cfg::A_BYTES + 16384 + k * 2048);
                    wgmma_m64n128k16<0, 1>(ch, a_hi + ko, b_hi, (first && k == 0) ? 0u : 1u);
                    wgmma_m64n128k16<0, 1>(ch, a_hi + ko, b_lo, 1u);
                    wgmma_m64n128k16<0, 1>(ch, a_lo + ko, b_hi, 1u);
                }
                wgmma_commit();
                wgmma_wait<0>();
                acc_fence(ch);
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[s]);
            }
#pragma unroll
            for (int i = 0; i < 64; ++i) sum[i] += ch[i];
        }
        asm volatile("bar.sync 1, %0;" ::"r"(Cfg::CONSUMERS) : "memory");   // staging buffers of the previous tile are free
        frag_to_tile(sum, ctile, Cfg::PITCH, 64 * wg, t);
        asm volatile("bar.sync 1, %0;" ::"r"(Cfg::CONSUMERS) : "memory");
        float acc[64];
        {
            const float4* src = reinterpret_cast<const float4*>(ctile + (g * 32 + lane) * Cfg::PITCH + colbase);
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const float4 v = src[j];
                acc[4 * j] = v.x; acc[4 * j + 1] = v.y; acc[4 * j + 2] = v.z; acc[4 * j + 3] = v.w;
            }
        }
        asm volatile("bar.sync 1, %0;" ::"r"(Cfg::CONSUMERS) : "memory");   // tile read: the staging buffers may be written

        // ---- epilogue: this thread owns row `row`, columns [col0, col0 + 64) ----
        const int row = mi * Cfg::BM + g * 32 + lane;
        const int col0 = ni * Cfg::BN + colbase;
        const int dj = row - col0;                               // diagonal element sits at acc[dj] when 0 <= dj < 64
        float rmax = 0.f, zz = 0.f;
        if (p.mode == 1) {
#pragma unroll
            for (int j = 0; j < 64; ++j) {
                const float d = (j == dj) ? 1.f : 0.f;
                rmax = fmaxf(rmax, fabsf(acc[j] - d));           // |I - Z Y|
                acc[j] = fmaf(-0.5f, acc[j], 1.5f * d);          // T = (3 I - Z Y) / 2
            }
        }
        // the fp32 result and ||Z||_F^2 are only needed from the FINAL iterate: the mode-1 product of this very iteration
        // (earlier in stream order) has set conv_iter = it for a matrix whose residual passed
        const bool final_it = *reinterpret_cast<volatile int*>(&p.state[b].conv_iter) == p.it;
        const bool f32 = final_it && p.f32_rule != 0 && ((p.f32_rule == 1) == (b < p.n_first));
        const float fs = f32 ? p.state[b].f32_scale : 0.f;
        // Row-major stores through a per-warp transposition buffer: a thread owns a ROW of the tile, so direct stores
        // would put 32 lanes on 32 different rows.  The 64 columns go through 8 KB of shared memory (XOR-swizzled 16-byte
        // chunks) and leave as full 128 / 256-byte row segments.
        uint8_t* stg = epi + e * 8192;
        const int rowbase = mi * Cfg::BM + g * 32;
        if (!*abort_flag) {
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                Half8 hi, lo;
                split8(acc + q * 8, hi, lo);
                const int slot = q ^ (lane & 7);
                *reinterpret_cast<Half8*>(stg + (lane * 8 + slot) * 16) = hi;
                *reinterpret_cast<Half8*>(stg + 4096 + (lane * 8 + slot) * 16) = lo;
            }
            __syncwarp();
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int rr = j * 4 + (lane >> 3), c = lane & 7;
                const int slot = c ^ (rr & 7);
                const Half8 hi = *reinterpret_cast<const Half8*>(stg + (rr * 8 + slot) * 16);
                const Half8 lo = *reinterpret_cast<const Half8*>(stg + 4096 + (rr * 8 + slot) * 16);
                __half* o = p.out_split + ((long long)(b * 2) * p.n + rowbase + rr) * p.n + col0 + c * 8;
                *reinterpret_cast<Half8*>(o) = hi;
                *reinterpret_cast<Half8*>(o + (long long)p.n * p.n) = lo;
            }
            __syncwarp();
            if (f32) {                                   // warp-uniform (one matrix per tile)
#pragma unroll
                for (int q = 0; q < 16; ++q) {
                    const float* a4 = acc + q * 4;
                    const int slot = q ^ (lane & 15);
                    *reinterpret_cast<float4*>(stg + (lane * 16 + slot) * 16) = make_float4(a4[0] * fs, a4[1] * fs, a4[2] * fs, a4[3] * fs);
                }
                __syncwarp();
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int rr = j * 2 + (lane >> 4), c = lane & 15;
                    const int slot = c ^ (rr & 15);
                    const float4 v = *reinterpret_cast<const float4*>(stg + (rr * 16 + slot) * 16);
                    *reinterpret_cast<float4*>(p.out_f32 + ((long long)b * p.n + rowbase + rr) * p.n + col0 + c * 4) = v;
                }
                __syncwarp();
            }
        }
        if (p.want_zz && final_it) {
#pragma unroll
            for (int j = 0; j < 64; ++j) zz = fmaf(acc[j], acc[j], zz);
#pragma unroll
            for (int o = 16; o >= 1; o >>= 1) zz += __shfl_xor_sync(0xffffffffu, zz, o);
            if (lane == 0) red[e] = zz;
        }
        if (p.mode == 1) {
#pragma unroll
            for (int o = 16; o >= 1; o >>= 1) rmax = fmaxf(rmax, __shfl_xor_sync(0xffffffffu, rmax, o));
            if (lane == 0) atomicMax(&p.state[b].resid_bits, __float_as_uint(rmax));     // order independent
        }
        __threadfence();
        asm volatile("bar.sync 1, %0;" ::"r"(Cfg::CONSUMERS) : "memory");
        if (e == 0 && lane == 0) {
            if (p.want_zz && final_it)                                                   // fixed order
                p.zz_slots[(long long)b * tpm + r] = ((red[0] + red[1]) + (red[2] + red[3])) + ((red[4] + red[5]) + (red[6] + red[7]));
            if (p.mode == 1) {
                const int done = atomicAdd(&p.state[b].tiles_done, 1);
                if (done == tpm - 1) {                           // last tile of this matrix in this launch
                    __threadfence();
                    const float res = __uint_as_float(atomicAdd(&p.state[b].resid_bits, 0u));
                    p.state[b].last_resid = res;
                    p.state[b].resid_bits = 0u;
                    p.state[b].tiles_done = 0;
                    if (res < p.tol) p.state[b].conv_iter = p.it;
                }
            }
        }
        // (red[] is rewritten only after the next tile's three consumer barriers)
    }
}

// s = ||A + eps I||_F, Y0 = (A + eps I)/s and Z0 = I as split planes, state reset.  Two launches of NS_INIT_BLOCKS blocks per
// matrix (the first version used ONE block per matrix: 119 us, 12 % of a C = 512 call): partial sums of squares in fixed
// slots, then every block adds the slots in the same order (deterministic) and converts its slice.
constexpr int NS_INIT_BLOCKS = 32;

__global__ void __launch_bounds__(256)
k_ns_norm(const float* __restrict__ A, int n, float eps_eig, float* __restrict__ partial) {
    const int b = blockIdx.y;
    const float* a = A + (long long)b * n * n;
    const int per = n * n / NS_INIT_BLOCKS;
    const int i0 = blockIdx.x * per;
    __shared__ float red[8];
    float ss = 0.f;
    for (int i = i0 + threadIdx.x; i < i0 + per; i += blockDim.x) {
        float v = a[i];
        if (i / n == i % n) v += eps_eig;
        ss = fmaf(v, v, ss);
    }
    for (int o = 16; o >= 1; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int i = 0; i < 8; ++i) t += red[i];
        partial[b * NS_INIT_BLOCKS + blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(256)
k_ns_init(const float* __restrict__ A, int n, float eps_eig, int n_first, const float* __restrict__ partial, __half* __restrict__ Y,
          __half* __restrict__ Z, NsState* __restrict__ state) {
    const int b = blockIdx.y;
    const float* a = A + (long long)b * n * n;
    float t = 0.f;
    for (int i = 0; i < NS_INIT_BLOCKS; ++i) t += partial[b * NS_INIT_BLOCKS + i];        // same order in every thread
    const float s0 = sqrtf(t);
    const bool good = isfinite(s0) && s0 > 0.f;
    const float s = good ? s0 : 1.f;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        NsState st;
        st.s = s;
        st.f32_scale = (b < n_first) ? rsqrtf(s) : sqrtf(s);
        st.conv_iter = good ? 0x7fffffff : -1;          // a degenerate matrix never enters the iteration
        st.resid_bits = 0u;
        st.tiles_done = 0;
        st.ok = 0;
        st.last_resid = good ? 1.f : 1e30f;
        st.pad = 0;
        state[b] = st;
    }
    const float inv = 1.f / s;
    __half* y_hi = Y + (long long)(b * 2) * n * n;
    __half* y_lo = y_hi + (long long)n * n;
    __half* z_hi = Z + (long long)(b * 2) * n * n;
    __half* z_lo = z_hi + (long long)n * n;
    const int per = n * n / NS_INIT_BLOCKS;
    const int i0 = blockIdx.x * per;
    for (int i = i0 + threadIdx.x; i < i0 + per; i += blockDim.x) {
        const bool diag = (i / n == i % n);
        float v = a[i];
        if (diag) v += eps_eig;
        __half hi, lo;
        split_f32(v * inv, hi, lo);
        y_hi[i] = hi;
        y_lo[i] = lo;
        z_hi[i] = __float2half(diag ? 1.f : 0.f);
        z_lo[i] = __float2half(0.f);
    }
}

// the guard: converged within the budget AND the threshold provably keeps every eigenvalue
__global__ void k_ns_finish(NsState* __restrict__ state, const float* __restrict__ zz_slots, int tpm, int batch, int max_it,
                            float thresh, float eps_eig, int* __restrict__ ok, int* __restrict__ kcount, int C, float* __restrict__ info) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= batch) return;
    NsState st = state[b];
    float zz = 0.f;
    for (int i = 0; i < tpm; ++i) zz += zz_slots[(long long)b * tpm + i];
    // sum_i 1/lambda_i(A) = ||Z||_F^2 / s  >=  1 / lambda_min(A);  lambda_min(cov) = lambda_min(A) - eps_eig
    const float lmin_bound = st.s / zz - eps_eig;
    const bool good = st.conv_iter >= 0 && st.conv_iter < max_it && isfinite(zz) && zz > 0.f && lmin_bound > thresh * 1.01f;
    ok[b] = good ? 1 : 0;
    state[b].ok = good ? 1 : 0;
    if (good && kcount) kcount[b] = C;                  // every eigenvalue kept (ops.py:57-64)
    if (info) {                                         // probe: iteration of convergence, last residual, eigenvalue bound
        info[4 * b] = (float)(st.conv_iter == 0x7fffffff ? -1 : st.conv_iter);
        info[4 * b + 1] = st.last_resid;
        info[4 * b + 2] = lmin_bound;
        info[4 * b + 3] = st.s;
    }
}

int g_matfun = 1;                 // 0: never (always the Jacobi eigensolver), 1: auto  (wctb200_debug_set_matfun)
int g_matfun_max_it = 16;          // matrices that need more (cond > ~5e3) fail the eigenvalue guard anyway

static int ns_gemm(const __half* A, const __half* B, int n, int batch, int it, int mode, int f32_rule, int n_first, int want_zz,
                   float tol, NsState* state, __half* out_split, float* out_f32, float* zz_slots, cudaStream_t st) {
    using Cfg = NsCfg;
    CUtensorMap mA, mB;
    const uint64_t rows = (uint64_t)batch * 2 * n;
    int rc = make_tensor_map_3d(&mA, A, (uint64_t)n, rows, 1, (uint64_t)n * 2, rows * n * 2, Cfg::BM);
    if (rc) return rc;
    rc = make_tensor_map_3d(&mB, B, (uint64_t)n, rows, 1, (uint64_t)n * 2, rows * n * 2, 64);
    if (rc) return rc;
    NsGemmParams p;
    p.n = n; p.batch = batch; p.tiles_m = n / Cfg::BM; p.it = it; p.mode = mode;
    p.f32_rule = out_f32 ? f32_rule : 0;
    p.n_first = n_first;
    p.want_zz = want_zz;
    p.tol = tol;
    p.state = state;
    p.out_split = out_split;
    p.out_f32 = out_f32;
    p.zz_slots = zz_slots;
    p.err = device_error_word();
    WCTB_ENSURE_SMEM(ns_gemm_kernel, Cfg::SMEM_BYTES);
    int grid = device_sm_count();
    const int total = batch * p.tiles_m * p.tiles_m;
    if (grid > total) grid = total;
    ns_gemm_kernel<<<grid, Cfg::THREADS, Cfg::SMEM_BYTES, st>>>(mA, mB, p);
    WCTB_CHECK_LAUNCH("ns_gemm_kernel");
    return 0;
}

size_t matfun_scratch_bytes(int C, int count) {
    const size_t plane2 = (size_t)2 * C * C * 2;                     // one split matrix
    return (size_t)count * (5 * plane2 + 64 * 4) + (size_t)count * sizeof(NsState) + 4096;
}

// A: `count` covariances (fp32, [count][C][C]); the first n_first want A^-1/2 (whitening), the rest A^+1/2 (colouring).
// out: [count][C][C] fp32, written for every matrix the iteration touches; ok[b] = 1 where `out` is valid (guard passed),
// kcount[b] = C there.  Returns 1 when the fast path is not attempted at all (ok[] is zeroed then).
int launch_matfun_ns(const float* A, int C, int count, int n_first, float thresh, float eps_eig, float* out, int* ok, int* kcount,
                     cudaStream_t st, float* info) {
    WCTB_CUDA(cudaMemsetAsync(ok, 0, (size_t)count * sizeof(int), st));
    if (!g_matfun || C < 128 || C % 128 != 0 || count < 1) return 1;
    uint8_t* scratch = nullptr;
    { int rc0 = scratch_alloc(reinterpret_cast<void**>(&scratch), matfun_scratch_bytes(C, count), st, 4); if (rc0) return rc0; }
    const size_t msz = (size_t)count * 2 * C * C;                    // halves per operand buffer
    __half* Y[2] = {reinterpret_cast<__half*>(scratch), reinterpret_cast<__half*>(scratch) + msz};
    __half* Z[2] = {Y[1] + msz, Y[1] + 2 * msz};
    __half* T = Z[1] + msz;
    float* zz = reinterpret_cast<float*>(T + msz);
    NsState* state = reinterpret_cast<NsState*>(zz + (size_t)count * 64);
    const int tpm = (C / 128) * (C / 128);
    WCTB_CUDA(cudaMemsetAsync(zz, 0, (size_t)count * 64 * 4, st));
    float* partial = zz + (size_t)count * 32;            // the upper half of each matrix's 64 slots (the guard uses <= 16)
    k_ns_norm<<<dim3(NS_INIT_BLOCKS, (unsigned)count), 256, 0, st>>>(A, C, eps_eig, partial);
    WCTB_CHECK_LAUNCH("k_ns_norm");
    k_ns_init<<<dim3(NS_INIT_BLOCKS, (unsigned)count), 256, 0, st>>>(A, C, eps_eig, n_first, partial, Y[0], Z[0], state);
    WCTB_CHECK_LAUNCH("k_ns_init");
    // the tensor core adds into its fp32 accumulator with truncation (conv_tc.cu): (Z Y)_ii settles ~3e-6 below 1, which is the
    // floor of the measured residual; tol sits above it and one more (quadratically convergent) iteration always follows
    const float tol = 2e-5f;
    int cur = 0;
    for (int it = 0; it < g_matfun_max_it; ++it) {
        int rc = ns_gemm(Z[cur], Y[cur], C, count, it, 1, 0, n_first, 0, tol, state, T, nullptr, nullptr, st);        // T = (3I - ZY)/2
        if (rc) return rc;
        rc = ns_gemm(Y[cur], T, C, count, it, 2, 2, n_first, 0, tol, state, Y[cur ^ 1], out, nullptr, st);            // Y' = Y T  (fp32: colouring)
        if (rc) return rc;
        rc = ns_gemm(T, Z[cur], C, count, it, 2, 1, n_first, 1, tol, state, Z[cur ^ 1], out, zz, st);                 // Z' = T Z  (fp32: whitening; ||Z||_F^2)
        if (rc) return rc;
        cur ^= 1;
    }
    k_ns_finish<<<cdiv(count, 128), 128, 0, st>>>(state, zz, tpm, count, g_matfun_max_it, thresh, eps_eig, ok, kcount, C, info);
    WCTB_CHECK_LAUNCH("k_ns_finish");
    return 0;
}

}  // namespace wctb
