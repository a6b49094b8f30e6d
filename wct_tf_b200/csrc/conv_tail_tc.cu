// Decoder tail  Conv2DReflect(3, activation=None)  (model.py:297-298; + the inter-level clip of model.py:17,86) for the
// 64-channel last block, as a TRANSPOSED tensor-core product.
//
// A 3x3 conv with 3 output channels has N = 3: useless as a GEMM.  Turn it round.  For every padded input position p compute
// ONCE the 27 partial products
//       P[p][(ky*3+kx)*3 + co] = sum_c x[p][c] * w[ky][kx][c][co]          (one 128 x 32 x 64 GEMM tile per 128 positions)
// and let the epilogue gather   out(y, x)[co] = bias[co] + sum_{ky,kx} P[(y+ky-1, x+kx-1)][(ky*3+kx)*3 + co].
// The activations are read from HBM/L2 exactly once (the implicit-GEMM form reads them 9 times, the SIMT kernel 3 times and
// spends 1728 FMAs per pixel); what is left per pixel is 27 shared-memory loads and adds.
//
// Tiling.  A CTA owns a vertical strip of <= 126 output columns (a row tile is 128 consecutive padded positions: the strip
// plus one neighbour column on either side) and walks DOWN a chunk of 32 output rows; the P rows live in a 3-row ring in
// shared memory, so no partial product is computed twice vertically (2 extra rows per 32) and 2 of 128 columns horizontally.
//   warp 4   : TMA producer (one 128 x 64 fp16 box per plane per row, 128B swizzle)
//   warps 0-3: one warpgroup: wgmma (a_hi + a_lo) * [b_hi | b_lo] (N = 64, two m64 halves) into registers -> P ring (fp32)
//              -> gather / scale / bias / clip -> fp32 stores
// Two CTAs per SM (100 KB of shared memory each): the gather of one overlaps the MMAs of the other.
// Precision: split-fp16 products like the big convs (weights scaled by a power of two so their lo plane stays out of the fp16
// subnormals; the a_lo b_lo term rides along); the K = 64 partial sums are accumulated by the tensor core, the 9-term
// gather in fp32 registers.
#include "common.cuh"

namespace wctb {

int make_tensor_map_3d(CUtensorMap* m, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1_bytes,
                       uint64_t stride2_bytes, uint32_t box1);

struct TailCfg {
    static constexpr int STAGES = 3;
    static constexpr int STAGE_BYTES = 128 * 64 * 2;       // one plane of one row tile
    static constexpr int B_BYTES = 2 * 32 * 64 * 2;        // [b_hi (32 rows) | b_lo (32 rows)], K-major, 128 B rows
    static constexpr int NJ = 27;
    static constexpr int RING_ROW = NJ * 128;              // floats per ring slot: [j][position]
    static constexpr int RING_BYTES = 3 * RING_ROW * 4;
    static constexpr int AUX_BYTES = 256;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + B_BYTES + RING_BYTES + AUX_BYTES + 1024;
    static constexpr int ROWS = 32;                        // output rows per work item
    static constexpr int THREADS = 160;
};

struct TailParams {
    int N, H, W, Hp, Wp;
    int nstrips, ow, chunks, items;
    int flags;
    const float* bias;
    const float* inv_scale;
    float* img;
    unsigned int* err;
};

// w fp32 [9*64][3] (k = tap*64 + c)  ->  bop fp16 [2 planes][32 rows j = tap*3 + co][64 c], scaled by a power of two
__global__ void k_prep_tail_weights(const float* __restrict__ w, __half* __restrict__ bop, float* __restrict__ inv_scale) {
    __shared__ float red[8];
    __shared__ float s_scale;
    float m = 0.f;
    for (int i = threadIdx.x; i < 9 * 64 * 3; i += blockDim.x) m = fmaxf(m, fabsf(w[i]));
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        float mm = 0.f;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) mm = fmaxf(mm, red[i]);
        int e = 0;
        float sc = 1.f;
        if (mm > 0.f && isfinite(mm)) {
            frexpf(mm, &e);                               // mm = f * 2^e, f in [0.5, 1)
            sc = ldexpf(1.f, 10 - e);                     // mm * sc in [512, 1024)
        }
        s_scale = sc;
        inv_scale[0] = 1.f / sc;
    }
    __syncthreads();
    const float sc = s_scale;
    for (int i = threadIdx.x; i < 32 * 64; i += blockDim.x) {
        const int j = i >> 6, c = i & 63;
        float v = 0.f;
        if (j < 27) v = w[((j / 3) * 64 + c) * 3 + (j % 3)] * sc;
        __half hi, lo;
        split_f32(v, hi, lo);
        bop[i] = hi;
        bop[32 * 64 + i] = lo;
    }
}

__global__ void __launch_bounds__(TailCfg::THREADS, 2)
conv_tail_tc_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, const TailParams p) {
    using Cfg = TailCfg;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* bsm = smem + Cfg::STAGES * Cfg::STAGE_BYTES;
    float* ring = reinterpret_cast<float*>(bsm + Cfg::B_BYTES);
    uint8_t* aux = reinterpret_cast<uint8_t*>(ring) + Cfg::RING_BYTES;
    uint64_t* full = reinterpret_cast<uint64_t*>(aux);
    uint64_t* empty = full + Cfg::STAGES;
    uint64_t* bfull = empty + Cfg::STAGES;
    volatile int* abort_flag = reinterpret_cast<volatile int*>(bfull + 1);

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
            mbar_init(&empty[s], 4);         // one arrival per consumer warp
        }
        mbar_init(bfull, 1);
        *abort_flag = 0;
        fence_barrier_init();
        tma_prefetch_desc(&mapA);
        tma_prefetch_desc(&mapB);
    }
    __syncthreads();
    const long long HpWp = (long long)p.Hp * p.Wp;

    // work item -> (image n, strip s, row chunk): chunk fastest so CTAs running together read neighbouring rows
    auto item_rows = [&](int item, int& n, int& px0, int& py0) {
        const int c = item % p.chunks;
        const int r = item / p.chunks;
        const int s = r % p.nstrips;
        n = r / p.nstrips;
        px0 = s * p.ow;
        py0 = c * Cfg::ROWS;
        return min(Cfg::ROWS, p.H - py0) + 2;             // P rows: padded rows py0 .. py0 + nrows - 1
    };

    if (warp == 4) {
        if (lane == 0) {
            mbar_arrive_expect_tx(bfull, Cfg::B_BYTES);
            tma_load_3d(bsm, &mapB, bfull, 0, 0, 0);
            tma_load_3d(bsm + Cfg::B_BYTES / 2, &mapB, bfull, 0, 0, 1);
            uint32_t sg = 0;
            for (int item = blockIdx.x; item < p.items; item += gridDim.x) {
                int n, px0, py0;
                const int nrows = item_rows(item, n, px0, py0);
                for (int r = 0; r < nrows; ++r) {
                    const int row = (int)(n * HpWp + (long long)(py0 + r) * p.Wp + px0);
#pragma unroll
                    for (int plane = 0; plane < 2; ++plane, ++sg) {
                        const int s = sg % Cfg::STAGES;
                        mbar_wait(&empty[s], ((sg / Cfg::STAGES) & 1) ^ 1u, abort_flag, p.err, 0x110u + s);
                        mbar_arrive_expect_tx(&full[s], Cfg::STAGE_BYTES);
                        tma_load_3d(smem + s * Cfg::STAGE_BYTES, &mapA, &full[s], 0, row, plane);
                    }
                }
            }
        }
        return;
    }

    // ---- consumer warpgroup (warps 0-3): wgmma, P rows into the ring, gather ----
    const int t = threadIdx.x;                             // 0..127
    const int pos = t;                                     // position inside the row tile (gather)
    const float isc = __ldg(p.inv_scale);
    const float b0 = __ldg(p.bias), b1 = __ldg(p.bias + 1), b2 = __ldg(p.bias + 2);
    const bool clip = (p.flags & WCTB200_CLIP01) != 0;
    // fragment coordinates: rows fr, fr + 8 (+64 for the second half), columns 8j + fc (+1)
    const int fr = 16 * (t >> 5) + ((t & 31) >> 2);
    const int fc = 2 * (t & 3);
    mbar_wait(bfull, 0u, abort_flag, p.err, 0x210u);
    const uint64_t b_desc = gmma_desc_sw128(smem_u32(bsm));       // 64 rows: b_hi then b_lo
    uint32_t sg = 0;
    for (int item = blockIdx.x; item < p.items; item += gridDim.x) {
        int n, px0, py0;
        const int nrows = item_rows(item, n, px0, py0);
        const int x = px0 + pos - 1;                       // output column of this thread (interior coordinates)
        const bool col_ok = pos >= 1 && pos <= p.ow && x < p.W;
        for (int r = 0; r < nrows; ++r) {
            // (a_hi + a_lo) x [b_hi | b_lo]: columns [0,32) = a b_hi, [32,64) = a b_lo (this includes the a_lo b_lo term)
            float acc[2][32];
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int i = 0; i < 32; ++i) acc[h][i] = 0.f;
            const int s0 = sg % Cfg::STAGES, s1 = (sg + 1) % Cfg::STAGES;
            mbar_wait(&full[s0], (sg / Cfg::STAGES) & 1, abort_flag, p.err, 0x220u + s0);
            mbar_wait(&full[s1], ((sg + 1) / Cfg::STAGES) & 1, abort_flag, p.err, 0x220u + s1);
            const uint32_t a_hi = smem_u32(smem + s0 * Cfg::STAGE_BYTES);
            const uint32_t a_lo = smem_u32(smem + s1 * Cfg::STAGE_BYTES);
            wgmma_fence();
#pragma unroll
            for (int h = 0; h < 2; ++h) {
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const uint64_t ko = (uint64_t)(k * 32 >> 4);
                    wgmma_m64n64k16<0, 0>(acc[h], gmma_desc_sw128(a_hi + h * 8192) + ko, b_desc + ko, k == 0 ? 0u : 1u);
                    wgmma_m64n64k16<0, 0>(acc[h], gmma_desc_sw128(a_lo + h * 8192) + ko, b_desc + ko, 1u);
                }
            }
            wgmma_commit();
            wgmma_wait<0>();
            acc_fence(acc[0]);
            acc_fence(acc[1]);
            __syncwarp();
            if (lane == 0) {
                mbar_arrive(&empty[s0]);
                mbar_arrive(&empty[s1]);
            }
            sg += 2;
            float* slot = ring + (r % 3) * Cfg::RING_ROW;
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int j = 0; j < 4; ++j)
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const int col = 8 * j + fc + (q & 1);                  // P column (tap*3 + co)
                        const int prow = 64 * h + fr + 8 * (q >> 1);           // position
                        if (col < Cfg::NJ) slot[col * 128 + prow] = acc[h][4 * j + q] + acc[h][4 * (j + 4) + q];
                    }
            asm volatile("bar.sync 1, 128;" ::: "memory");           // P row r complete
            if (r >= 2) {
                if (col_ok && !*abort_flag) {
                    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
#pragma unroll
                    for (int ky = 0; ky < 3; ++ky) {
                        const float* row = ring + ((r - 2 + ky) % 3) * Cfg::RING_ROW + pos - 1;
#pragma unroll
                        for (int kx = 0; kx < 3; ++kx) {
                            const float* q = row + ((ky * 3 + kx) * 3) * 128 + kx;
                            a0 += q[0];
                            a1 += q[128];
                            a2 += q[256];
                        }
                    }
                    a0 = fmaf(a0, isc, b0);
                    a1 = fmaf(a1, isc, b1);
                    a2 = fmaf(a2, isc, b2);
                    if (clip) {
                        a0 = fminf(fmaxf(a0, 0.f), 1.f);
                        a1 = fminf(fmaxf(a1, 0.f), 1.f);
                        a2 = fminf(fmaxf(a2, 0.f), 1.f);
                    }
                    float* d = p.img + (((long long)n * p.H + (py0 + r - 2)) * p.W + x) * 3;
                    d[0] = a0;
                    d[1] = a1;
                    d[2] = a2;
                }
                asm volatile("bar.sync 1, 128;" ::: "memory");       // ring slot (r+1)%3 may be overwritten
            }
        }
    }
}

int g_conv_tail_tc = 1;          // 0: always the SIMT kernels of layers.cu (wctb200_debug_set_conv_tail_tc)

// returns 1 when the shape is not handled here (the caller falls through to the SIMT kernels), 0 on success, < 0 on error
int launch_conv_tail_tc(const __half* in, ActGeom gi, const float* w, const float* b, int flags, float* img, cudaStream_t st) {
    using Cfg = TailCfg;
    if (!g_conv_tail_tc || gi.C != 64 || gi.P >= (1ll << 31) - 4096) return 1;
    uint8_t* scratch = nullptr;
    { int rc0 = scratch_alloc(reinterpret_cast<void**>(&scratch), Cfg::B_BYTES + 256, st, 3); if (rc0) return rc0; }
    __half* bop = reinterpret_cast<__half*>(scratch);
    float* inv_scale = reinterpret_cast<float*>(scratch + Cfg::B_BYTES);
    k_prep_tail_weights<<<1, 256, 0, st>>>(w, bop, inv_scale);
    WCTB_CHECK_LAUNCH("k_prep_tail_weights");

    CUtensorMap mA, mB;
    int rc = make_tensor_map_3d(&mA, in, 64, (uint64_t)gi.P, 2, 128, (uint64_t)gi.plane * 2, 128);
    if (rc) return rc;
    rc = make_tensor_map_3d(&mB, bop, 64, 32, 2, 128, 32 * 128, 32);
    if (rc) return rc;

    TailParams p;
    p.N = gi.N; p.H = gi.H; p.W = gi.W; p.Hp = gi.Hp; p.Wp = gi.Wp;
    p.nstrips = cdiv(gi.W, 126);
    p.ow = cdiv(gi.W, p.nstrips);
    p.chunks = cdiv(gi.H, Cfg::ROWS);
    p.items = gi.N * p.nstrips * p.chunks;
    p.flags = flags;
    p.bias = b;
    p.inv_scale = inv_scale;
    p.img = img;
    p.err = device_error_word();
    WCTB_ENSURE_SMEM(conv_tail_tc_kernel, Cfg::SMEM_BYTES);
    int grid = device_sm_count() * 2;
    if (grid > p.items) grid = p.items;
    conv_tail_tc_kernel<<<grid, Cfg::THREADS, Cfg::SMEM_BYTES, st>>>(mA, mB, p);
    WCTB_CHECK_LAUNCH("conv_tail_tc_kernel");
    return 0;
}

}  // namespace wctb
