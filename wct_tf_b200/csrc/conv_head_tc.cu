// Encoder head on the tensor cores: (1x1 preprocess conv folded into) conv1_1 3 -> 64 + ReLU  (vgg_normalised.py:25-40),
// fp32 image in, SPF16 activation (interior + reflect halo) out.
//
// K = 27 is too short for a TMA-fed implicit GEMM (the operand would be 9 boxes of 6 bytes), so the A operand is BUILT in
// shared memory by four producer warps: thread = pixel, its 3x3x3 reflect- (or wrap-) indexed neighbourhood (27 fp32, L1 hits) is scaled
// by 256 (the [0,1] image would put the lo halves into the fp16 subnormals), split into fp16 hi/lo and written as ONE
// 128-byte K-major row  [hi k=0..31 | lo k=0..31]  in the 128B-swizzled layout the MMA expects.  With
//     B rows  0..63  = [w_hi | w_hi]        ->  D[:,  0:64 ) = x_hi w_hi + x_lo w_hi
//     B rows 64..127 = [w_lo |  0  ]        ->  D[:, 64:128) = x_hi w_lo
// one wgmma (M = 64, N = 128) per 16-wide k-step and 64-pixel half -- 8 per 128-pixel tile -- computes all three split products.
//   warps 0-3 : producers (global -> split fp16 -> swizzled smem, fence.proxy.async, mbarrier)
//   warps 4-7 : one warpgroup: wgmma, the two column halves summed into an fp32 tile in shared memory, then the epilogue
//               (undo the scales, bias, ReLU, split, coalesced stores incl. the halo cells)
// Two CTAs per SM.  The SIMT kernel (layers.cu k_conv_head) spends 1728 FMAs per pixel; this one is bound by its
// 258 B/pixel of output.
#include "common.cuh"

namespace wctb {

struct HeadCfg {
    static constexpr int A_BYTES = 128 * 128;              // one tile: 128 pixels x 128 B
    static constexpr int STAGES = 2;
    static constexpr int B_BYTES = 128 * 128;              // 128 rows (n) x 64 fp16 (k)
    static constexpr int PITCH = 68;                       // fp32 tile [128 pixels][64 channels] (+4: conflict-free row reads)
    static constexpr int TILE_BYTES = 128 * PITCH * 4;
    static constexpr int STG_BYTES = 4 * 8192;             // per-epilogue-warp store staging, aliased with the fp32 tile
    static constexpr int EPI_BYTES = TILE_BYTES > STG_BYTES ? TILE_BYTES : STG_BYTES;
    static constexpr int AUX_BYTES = 512;                  // barriers + bias[64]
    static constexpr int SMEM_BYTES = STAGES * A_BYTES + B_BYTES + EPI_BYTES + AUX_BYTES + 1024;
    static constexpr int THREADS = 256;
};

struct HeadParams {
    int N, H, W;
    long long total_px;
    int tiles;
    const float* img;
    const float* w;        // [27][64], k = (ky*3 + kx)*3 + ci
    const float* bias;     // [64]
    int flags;             // WCTB200_HALO_WRAP_X / _Y: circular padding of the image and a wrapped halo on those axes
    __half* out;
    unsigned int* err;
};

__global__ void __launch_bounds__(HeadCfg::THREADS, 2)
conv_head_tc_kernel(const HeadParams p) {
    using Cfg = HeadCfg;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* bsm = smem + Cfg::STAGES * Cfg::A_BYTES;
    uint8_t* epi = bsm + Cfg::B_BYTES;
    float* ctile = reinterpret_cast<float*>(epi);
    uint8_t* aux = epi + Cfg::EPI_BYTES;
    uint64_t* full = reinterpret_cast<uint64_t*>(aux);
    uint64_t* empty = full + Cfg::STAGES;
    volatile int* abort_flag = reinterpret_cast<volatile int*>(empty + Cfg::STAGES);
    float* s_oscale = reinterpret_cast<float*>(empty + Cfg::STAGES) + 1;
    float* sbias = reinterpret_cast<float*>(aux + 256);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    __shared__ unsigned int s_prev_err;
    __shared__ float s_red[16];
    if (threadIdx.x == 0) s_prev_err = *reinterpret_cast<volatile unsigned int*>(p.err);
    __syncthreads();
    if (s_prev_err != 0u) return;

    if (threadIdx.x == 0) {
        for (int s = 0; s < Cfg::STAGES; ++s) {
            mbar_init(&full[s], 4);          // one arrival per producer warp
            mbar_init(&empty[s], 4);         // one arrival per consumer warp
        }
        *abort_flag = 0;
        fence_barrier_init();
    }

    // ---- B operand (all threads): power-of-two weight scale, split, swizzled K-major rows ----
    float m = 0.f;
    for (int i = threadIdx.x; i < 27 * 64; i += Cfg::THREADS) m = fmaxf(m, fabsf(p.w[i]));
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) s_red[warp] = m;
    if (threadIdx.x < 64) sbias[threadIdx.x] = p.bias[threadIdx.x];
    __syncthreads();
    float wsc = 1.f;
    {
        float mm = 0.f;
        for (int i = 0; i < Cfg::THREADS / 32; ++i) mm = fmaxf(mm, s_red[i]);
        if (mm > 0.f && isfinite(mm)) {
            int e = 0;
            frexpf(mm, &e);
            wsc = ldexpf(1.f, 10 - e);                     // max |w| * wsc in [512, 1024)
        }
    }
    if (threadIdx.x == 0) *s_oscale = 1.f / (wsc * 256.f);  // undoes the weight scale and the x256 of the image
    for (int i = threadIdx.x; i < 128 * 8; i += Cfg::THREADS) {
        const int row = i >> 3, c = i & 7;                 // 16-byte chunk c of B row `row`
        const int n = row & 63;
        const bool lo_row = row >= 64;
        Half8 v;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            __half h2[2];
#pragma unroll
            for (int t = 0; t < 2; ++t) {
                const int k = (c & 3) * 8 + j * 2 + t;
                float x = k < 27 ? p.w[k * 64 + n] * wsc : 0.f;
                __half hi, lo;
                split_f32(x, hi, lo);
                h2[t] = lo_row ? (c < 4 ? lo : __float2half(0.f)) : hi;
            }
            v.v[j] = __halves2half2(h2[0], h2[1]);
        }
        *reinterpret_cast<Half8*>(bsm + row * 128 + ((c ^ (row & 7)) * 16)) = v;
    }
    fence_proxy_async();
    __syncthreads();
    const unsigned int HW = (unsigned int)p.H * (unsigned int)p.W;

    if (warp < 4) {
        // ---- producers: one pixel per thread ----
        const int i = warp * 32 + lane;                    // row of the A tile
        const bool wrap_x = (p.flags & WCTB200_HALO_WRAP_X) != 0, wrap_y = (p.flags & WCTB200_HALO_WRAP_Y) != 0;
        uint32_t tg = 0;
        for (int tile = blockIdx.x; tile < p.tiles; tile += gridDim.x, ++tg) {
            const int s = tg % Cfg::STAGES;
            mbar_wait(&empty[s], ((tg / Cfg::STAGES) & 1) ^ 1u, abort_flag, p.err, 0x120u + s);
            const long long q = (long long)tile * 128 + i;
            float v[32];
#pragma unroll
            for (int k = 27; k < 32; ++k) v[k] = 0.f;
            if (q < p.total_px) {
                const unsigned int n = (unsigned int)(q / HW);
                const unsigned int r = (unsigned int)(q - (long long)n * HW);
                const int y = (int)(r / (unsigned int)p.W);
                const int x = (int)(r - (unsigned int)y * (unsigned int)p.W);
                const float* base = p.img + (long long)n * HW * 3;
#pragma unroll
                for (int ky = 0; ky < 3; ++ky) {
                    const float* row = base + (long long)pad_index(y + ky - 1, p.H, wrap_y) * p.W * 3;
#pragma unroll
                    for (int kx = 0; kx < 3; ++kx) {
                        const float* px = row + pad_index(x + kx - 1, p.W, wrap_x) * 3;
#pragma unroll
                        for (int ci = 0; ci < 3; ++ci) v[(ky * 3 + kx) * 3 + ci] = __ldg(px + ci) * 256.f;
                    }
                }
            } else {
#pragma unroll
                for (int k = 0; k < 27; ++k) v[k] = 0.f;
            }
            uint8_t* rowp = smem + s * Cfg::A_BYTES + i * 128;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                Half8 hi, lo;
                split8(v + c * 8, hi, lo);
                *reinterpret_cast<Half8*>(rowp + ((c ^ (i & 7)) * 16)) = hi;
                *reinterpret_cast<Half8*>(rowp + (((c + 4) ^ (i & 7)) * 16)) = lo;
            }
            fence_proxy_async();
            __syncwarp();
            if (lane == 0) mbar_arrive(&full[s]);
        }
        return;
    }

    // ---- consumer warpgroup (warps 4-7): wgmma per 64-row half, D[:, 0:64) + D[:, 64:128) -> fp32 tile -> epilogue ----
    const int t = threadIdx.x - 128;
    const int fr = 16 * (t >> 5) + ((t & 31) >> 2), fc = 2 * (t & 3);
    ActGeom go(p.N, p.H, p.W, 64);
    go.set_halo(p.flags);
    const float osc = *s_oscale;
    uint8_t* wstg = epi + (warp - 4) * 8192;
    const uint64_t b_desc = gmma_desc_sw128(smem_u32(bsm));
    uint32_t tg = 0;
    for (int tile = blockIdx.x; tile < p.tiles; tile += gridDim.x, ++tg) {
        const int s = tg % Cfg::STAGES;
        mbar_wait(&full[s], (tg / Cfg::STAGES) & 1, abort_flag, p.err, 0x230u + s);
        asm volatile("bar.sync 1, 128;" ::: "memory");             // previous tile's staging buffers are free
#pragma unroll 1
        for (int h = 0; h < 2; ++h) {
            float d[64];
#pragma unroll
            for (int i = 0; i < 64; ++i) d[i] = 0.f;
            const uint64_t a_desc = gmma_desc_sw128(smem_u32(smem + s * Cfg::A_BYTES + h * 8192));
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint64_t ko = (uint64_t)(k * 32 >> 4);
                wgmma_m64n128k16<0, 0>(d, a_desc + ko, b_desc + ko, k == 0 ? 0u : 1u);
            }
            wgmma_commit();
            wgmma_wait<0>();
            acc_fence(d);
            // columns [0,64) = x_hi w_hi + x_lo w_hi, [64,128) = x_hi w_lo of the same channels
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int r = 64 * h + fr;
                *reinterpret_cast<float2*>(ctile + r * Cfg::PITCH + 8 * j + fc) =
                    make_float2(d[4 * j] + d[4 * (j + 8)], d[4 * j + 1] + d[4 * (j + 8) + 1]);
                *reinterpret_cast<float2*>(ctile + (r + 8) * Cfg::PITCH + 8 * j + fc) =
                    make_float2(d[4 * j + 2] + d[4 * (j + 8) + 2], d[4 * j + 3] + d[4 * (j + 8) + 3]);
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
        asm volatile("bar.sync 1, 128;" ::: "memory");             // fp32 tile complete
        float acc[64];
        {
            const float4* src4 = reinterpret_cast<const float4*>(ctile + t * Cfg::PITCH);
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const float4 v = src4[j];
                acc[4 * j] = v.x; acc[4 * j + 1] = v.y; acc[4 * j + 2] = v.z; acc[4 * j + 3] = v.w;
            }
        }
        asm volatile("bar.sync 1, 128;" ::: "memory");             // tile read: the staging buffers may be written
        const long long q = (long long)tile * 128 + t;
        int flags = -1;
        unsigned int ppos = 0;
        if (q < p.total_px && !*abort_flag) {
            const unsigned int n = (unsigned int)(q / HW);
            const unsigned int r = (unsigned int)(q - (long long)n * HW);
            const int y = (int)(r / (unsigned int)p.W);
            const int x = (int)(r - (unsigned int)y * (unsigned int)p.W);
            flags = halo_flags(go, y, x);
            ppos = (n * (unsigned int)go.Hp + (unsigned int)(y + 1)) * (unsigned int)go.Wp + (unsigned int)(x + 1);
        }
        store_tile_rows<64>(acc, osc, sbias, true, wstg, lane, ppos, flags, p.out, go, 0);
    }
}

int g_conv_head_tc = 1;          // 0: the SIMT kernel of layers.cu (wctb200_debug_set_conv_head_tc)

// returns 1 when not handled here (caller falls through to the SIMT kernel), 0 on success, < 0 on error
int launch_conv_head_tc(const float* img, int N, int H, int W, const float* w, const float* b, int flags, __half* out,
                        cudaStream_t st) {
    using Cfg = HeadCfg;
    const ActGeom go(N, H, W, 64);
    if (!g_conv_head_tc || H < 2 || W < 2 || go.P >= (1ll << 31)) return 1;
    HeadParams p;
    p.N = N; p.H = H; p.W = W;
    p.total_px = (long long)N * H * W;
    p.tiles = cdiv(p.total_px, 128);
    p.img = img;
    p.w = w;
    p.bias = b;
    p.flags = flags;
    p.out = out;
    p.err = device_error_word();
    WCTB_ENSURE_SMEM(conv_head_tc_kernel, Cfg::SMEM_BYTES);
    int grid = device_sm_count() * 2;
    if (grid > p.tiles) grid = p.tiles;
    conv_head_tc_kernel<<<grid, Cfg::THREADS, Cfg::SMEM_BYTES, st>>>(p);
    WCTB_CHECK_LAUNCH("conv_head_tc_kernel");
    return 0;
}

}  // namespace wctb
