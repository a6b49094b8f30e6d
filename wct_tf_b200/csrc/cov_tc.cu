// Covariance GEMM  S = sum_p (x_p - t)(x_p - t)^T  (C x HW . HW x C, ops.py:43-45,48-50,105-108) on the tensor cores,
// with the centring and the per-channel sums fused in: ONE pass over the features.
//
// The features are SPF16 [pixel][channel]: for the product X^T X the contraction index K is the
// PIXEL, so both operands are "MN-major" (for a fixed k the 64 channels of a slice are the 128
// contiguous bytes of a row).  A TMA box of 64 pixels x 64 channels lands as the canonical
// MN-major SWIZZLE_128B tile (8-pixel groups of 1024 B), and wgmma reads A and B from the
// same staged tiles with both operands transposed (MN-major).  The tensor map is built over the INTERIOR of the
// reflect-padded plane (base pointer at pixel (0,0), padded strides, dims W x H): boxes that stick
// out at a ragged edge are zero-filled by TMA and add nothing to the sums, halo cells are never read.
//
// Centring (ops.py:44,49,106: fc = f - mean BEFORE the product).  Round 1 ran three extra passes for it (channel sums,
// a centred SPF16 copy written to HBM, the product over the copy).  Now a tiny pre-kernel estimates a per-channel SHIFT t
// (the mean of <= 1024 strided pixels; the exact mean when HW <= 1024), the two consumer warpgroups subtract t from every
// staged tile IN SHARED MEMORY (hi+lo -> fp32 -> minus t -> re-split, zero-filled out-of-range pixels stay zero) before
// their wgmma read it, and accumulate s = sum_p (x_p - t) on the way.  The finalize kernel forms
//     cov = (S - s s^T / HW) / (HW - 1),   mean = t + s / HW
// in fp64: exact algebra for ANY t, and with t within sigma/32 of the mean the subtracted term is ~1e-3 of S, so nothing
// cancels (the fully uncentred form, t = 0, was measured in round 1: it produced a spurious eigenvalue above the 1e-5 cut).
//
// Determinism.  Products in fp32 (split-fp16 x3), a fresh register accumulator every 128 pixels added into the running sum
// (the tensor core accumulates with truncation and the diagonals are all-positive sums).  Every CTA writes its partial block and partial sums
// to its OWN slot; the finalize kernel adds the slots in a fixed order.  The split of an image into CTAs depends on (C, H, W)
// only -- not on the batch size or the SM count -- so a frame's covariance is bit-identical whatever batch or GPU it is in
// (tests: 2-GPU shards == 1 GPU, batch == single frames).
//
// One CTA = one 128 x 128 block pair (bi <= bj) of the C x C matrix x one range of pixel tiles.
#include "common.cuh"

namespace wctb {

struct CovParams {
    int C, W, H, N;
    int tiles_x, tiles_y;        // 32 x 2 pixel tiles per image
    int ksplit, tiles_per_split;
    int nb;                      // 128-channel blocks (C=64: 1 block, rows duplicated)
    int nslots;                  // partial slots per image: ksplit (C=64: 4*ksplit)
    int max_stages;              // cap on the ring depth (probe knob; 12 = no cap)
    const float* shift;          // [N][C]   (regions: [N*R][C])
    float* part;                 // [N][nslots][C][C] fp32 partial products (upper block triangle)   (regions: [N*R]...)
    float* psum;                 // [N][ksplit][C] fp32 partial sums of (x - shift)
    unsigned int* err;
    // spatial control (cov_tc_kernel<true>): problem z = image * R + region covers the pixels labelled `region` only
    const uint8_t* labels;       // [N][H][W] region label per pixel
    const uint16_t* tmask;       // [N][tiles_y * tiles_x]: bit r set when the 32 x 2 tile holds a pixel labelled r
    int R;
    // soft spatial control (cov_tc_kernel<true, true>): problem z = image * R + k weighs pixel p by wts[z][p] >= 0
    const float* wts;            // [N][R][H][W]; tmask bit k: the tile holds a pixel of nonzero weight k
};

struct CovCfg {
    static constexpr int SLICE = 64 * 128;                  // 64 pixels x 64 channels fp16 = 8 KB
    static constexpr int OPER = 4 * SLICE;                  // 2 channel slices x 2 planes
    static constexpr int STAGE = 2 * OPER;                  // A + B (off-diagonal block pair); a diagonal pair uses OPER, C = 64 two SLICEs
    static constexpr int RING_BYTES = 3 * STAGE;            // 192 KB of tiles in flight whatever the stage size: 3 / 6 / 12 stages
    static constexpr int STAGES = 12;                       // barrier slots (the deepest ring)
    static constexpr int CH = 2;                            // 64-pixel tiles per register accumulation chunk (24 truncating adds)
    static constexpr int CONSUMERS = 256;                   // two warpgroups: centring + wgmma
    static constexpr int THREADS = CONSUMERS + 128;         // + producer warpgroup
    static constexpr int RED_BYTES = 32 * 128 * 4;          // consumers: [32 row groups][128 channels] partial sums
    static constexpr int SMEM_BYTES = RING_BYTES + 512 + RED_BYTES + 1024;
};

__device__ __forceinline__ void tma_load_5d_cov(void* smem_dst, const void* map, uint64_t* bar, int c0, int c1, int c2,
                                                int c3, int c4) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
        "r"(c3), "r"(c4)
        : "memory");
}

// MASK = false: one problem per image (blockIdx.y = image).  MASK = true (spatial control): blockIdx.y = image * R + region;
// producer and consumers skip the tiles without a pixel of the region (each tile is read once per region present in it),
// and the centring step writes zeros for the staged pixels of other regions, exactly as for out-of-range pixels.
// WGT (with MASK, soft spatial control, DESIGN.md §3.3.11): region r is weight plane r; the centring step scales the staged
// x - t by sqrt(w) (zeros where w = 0, as MASK writes them), so the product sums w (x - t)(x - t)^T, and s sums w (x - t).
// With 0/1 weights every value, and so every sum, is that of MASK.
template <bool MASK, bool WGT = false>
__global__ void __launch_bounds__(CovCfg::THREADS, 1)
cov_tc_kernel(const __grid_constant__ CUtensorMap mapX, const CovParams p) {
    using Cfg = CovCfg;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* aux = smem + Cfg::RING_BYTES;
    uint64_t* full = reinterpret_cast<uint64_t*>(aux);
    uint64_t* empty = full + Cfg::STAGES;
    volatile int* abort_flag = reinterpret_cast<volatile int*>(empty + Cfg::STAGES);
    float* red = reinterpret_cast<float*>(aux + 512);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // block pair / k-split / image of this CTA
    const int npairs = p.nb * (p.nb + 1) / 2;
    const int pair = blockIdx.x % npairs;
    const int split = blockIdx.x / npairs;
    int bi = 0, rem = pair;
    while (rem >= p.nb - bi) { rem -= p.nb - bi; ++bi; }
    const int bj = bi + rem;
    const bool diag = (bi == bj);
    const int prob = blockIdx.y;                     // output slot: image (MASK: image * R + region)
    const int img = MASK ? prob / p.R : prob;
    const int reg = MASK ? prob - img * p.R : 0;
    const uint16_t* tmask = MASK ? p.tmask + (long long)img * p.tiles_x * p.tiles_y : nullptr;
    const int tiles_img = p.tiles_x * p.tiles_y;
    const int t0 = split * p.tiles_per_split;
    const int t1 = min(t0 + p.tiles_per_split, tiles_img);
    const int ntiles = max(t1 - t0, 0);
    // C = 64: a single 64-channel slice.  The 128-row operand is [hi plane | lo plane] of that slice and is used as BOTH
    // A and B: ONE MMA per 16 pixels yields hi.hi, hi.lo, lo.hi (and lo.lo) as the four 64x64 quadrants of the 128x128
    // accumulator; the epilogue adds the quadrants.
    const bool dup = (p.C == 64);

    if (threadIdx.x == 0) {
        for (int s = 0; s < Cfg::STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], Cfg::CONSUMERS / 32); }
        *abort_flag = 0;
        fence_barrier_init();
        tma_prefetch_desc(&mapX);
    }
    __syncthreads();
    const int nchunks = (ntiles + Cfg::CH - 1) / Cfg::CH;
    // One stage holds exactly what one tile needs, so the ring is 3 (off-diagonal pair), 6 (diagonal pair) or 12 (C = 64)
    // stages deep: the C <= 128 levels are HBM-latency bound and want many tiles in flight
    const uint32_t stage_bytes = dup ? 2 * Cfg::SLICE : (diag ? Cfg::OPER : Cfg::STAGE);
    const int nst = min(Cfg::RING_BYTES / (int)stage_bytes, p.max_stages);

    if (warp >= Cfg::CONSUMERS / 32) {
        setmaxnreg_dec<40>();
        if (warp == Cfg::CONSUMERS / 32 && lane == 0) {
            // (stage index, barrier phase and tile coordinates advance incrementally: runtime div/mod cost ~40 instructions each)
            int s = 0, ty = t0 / p.tiles_x, tx = t0 - ty * p.tiles_x;
            uint32_t ph = 0;
            for (int it = 0; it < ntiles; ++it, ++tx) {
                if (tx == p.tiles_x) { tx = 0; ++ty; }
                if (MASK && !((tmask[t0 + it] >> reg) & 1u)) continue;
                if (s == nst) { s = 0; ph ^= 1u; }
                mbar_wait(&empty[s], ph ^ 1u, abort_flag, p.err, 0x510u + s);
                uint8_t* st = smem + s * stage_bytes;
                mbar_arrive_expect_tx(&full[s], stage_bytes);
                if (dup) {
                    tma_load_5d_cov(st, &mapX, &full[s], 0, tx * 32, ty * 2, img, 0);                  // rows 0..63   : hi
                    tma_load_5d_cov(st + Cfg::SLICE, &mapX, &full[s], 0, tx * 32, ty * 2, img, 1);     // rows 64..127 : lo
                    ++s;
                    continue;
                }
                for (int op = 0; op < (diag ? 1 : 2); ++op) {
                    const int blk = op == 0 ? bi : bj;
                    for (int sl = 0; sl < 2; ++sl) {
                        const int ch = blk * 128 + sl * 64;
                        for (int pl = 0; pl < 2; ++pl)
                            tma_load_5d_cov(st + op * Cfg::OPER + (pl * 2 + sl) * Cfg::SLICE, &mapX, &full[s], ch, tx * 32,
                                            ty * 2, img, pl);
                    }
                }
                ++s;
            }
        }
        return;
    }

    // ---- two consumer warpgroups (warps 0-7).  All 256 threads centre each staged tile (x -> x - shift in place, sums of
    // the shifted values); then warpgroup w multiplies accumulator rows [64w, 64w + 64) (channels of block bi) with all 128
    // columns (block bj) by wgmma with both operands MN-major.
    setmaxnreg_inc<232>();
    const int wg = warp >> 2;
    const int ct = threadIdx.x;           // 0..255
    const int chunk = ct & 7;             // logical 16-byte chunk of a 128-byte row = channels chunk*8 .. +7 of the slice
    const int rg = ct >> 3;               // rows rg and rg+32 of every 64-pixel slice
    const int pchunk = (chunk ^ (rg & 7)) << 4;      // SWIZZLE_128B: physical chunk = logical ^ (row & 7); row & 7 == rg & 7
    const int nops = dup ? 1 : (diag ? 1 : 2);
    const int nsl = dup ? 1 : 2;
    const bool want_sums = dup || diag;   // every channel block has exactly one diagonal pair
    float sh[2][2][8], sums[2][8], acc[64];
#pragma unroll
    for (int op = 0; op < 2; ++op)
#pragma unroll
        for (int sl = 0; sl < 2; ++sl) {
            const int blk = op == 0 ? bi : bj;
            const int c0 = dup ? chunk * 8 : blk * 128 + sl * 64 + chunk * 8;
#pragma unroll
            for (int j = 0; j < 8; ++j) sh[op][sl][j] = (op < nops && sl < nsl) ? __ldg(p.shift + (long long)prob * p.C + c0 + j) : 0.f;
        }
#pragma unroll
    for (int sl = 0; sl < 2; ++sl)
#pragma unroll
        for (int j = 0; j < 8; ++j) sums[sl][j] = 0.f;
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    int s = 0, ty = t0 / p.tiles_x, tx = t0 - ty * p.tiles_x;
    uint32_t ph = 0;
    // one staged tile: centre it in shared memory, then multiply it into `chk` (first: the chunk starts from zero)
    auto tile = [&](float (&chk)[64], bool first) {
        mbar_wait(&full[s], ph, abort_flag, p.err, 0x550u + s);
        uint8_t* st = smem + s * stage_bytes;
        bool keep[2] = {true, true};                 // MASK: the pixel carries this CTA's region label
        float wv[2] = {1.f, 1.f};                    // WGT: the pixel's weight
        if (MASK) {
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const int r = rg + 32 * k;
                const int x = tx * 32 + (r & 31), y = ty * 2 + (r >> 5);
                if (WGT) {
                    wv[k] = (x < p.W && y < p.H) ? __ldg(p.wts + ((long long)prob * p.H + y) * p.W + x) : 0.f;
                    keep[k] = wv[k] > 0.f;
                } else {
                    keep[k] = x < p.W && y < p.H && p.labels[((long long)img * p.H + y) * p.W + x] == reg;
                }
            }
        }
#pragma unroll
        for (int op = 0; op < 2; ++op) {
            if (op >= nops) break;
#pragma unroll
            for (int sl = 0; sl < 2; ++sl) {
                if (sl >= nsl) break;
                uint8_t* hi_base = dup ? st : st + op * Cfg::OPER + sl * Cfg::SLICE;
                uint8_t* lo_base = dup ? st + Cfg::SLICE : st + op * Cfg::OPER + (2 + sl) * Cfg::SLICE;
#pragma unroll
                for (int k = 0; k < 2; ++k) {
                    const int r = rg + 32 * k;
                    const int x = tx * 32 + (r & 31), y = ty * 2 + (r >> 5);
                    if (x < p.W && y < p.H) {           // out-of-range pixels were zero-filled by TMA and must stay zero
                        const int off = r * 128 + pchunk;
                        if (MASK && !keep[k]) {         // another region's pixel: TMA loaded it, overwrite with zeros
                            const Half8 z = {};
                            *reinterpret_cast<Half8*>(hi_base + off) = z;
                            *reinterpret_cast<Half8*>(lo_base + off) = z;
                            continue;
                        }
                        const Half8 h = *reinterpret_cast<const Half8*>(hi_base + off);
                        const Half8 l = *reinterpret_cast<const Half8*>(lo_base + off);
                        float v[8];
                        merge8(h, l, v);
#pragma unroll
                        for (int j = 0; j < 8; ++j) v[j] -= sh[op][sl][j];
                        if (op == 0) {
#pragma unroll
                            for (int j = 0; j < 8; ++j) sums[sl][j] += WGT ? wv[k] * v[j] : v[j];
                        }
                        if (WGT) {
                            const float sq = sqrtf(wv[k]);
#pragma unroll
                            for (int j = 0; j < 8; ++j) v[j] *= sq;
                        }
                        Half8 nh, nl;
                        split8(v, nh, nl);
                        *reinterpret_cast<Half8*>(hi_base + off) = nh;
                        *reinterpret_cast<Half8*>(lo_base + off) = nl;
                    }
                }
            }
        }
        fence_proxy_async();                                   // generic-proxy writes -> visible to the tensor core
        asm volatile("bar.sync 1, %0;" ::"r"(Cfg::CONSUMERS) : "memory");   // the whole tile is centred
        const uint32_t a0 = smem_u32(st);
        const uint32_t b0 = diag ? a0 : a0 + Cfg::OPER;
        wgmma_fence();
        if (dup) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {            // 64 pixels = 4 x k16: 16 rows of 128 B = 2048 B per step
                const uint32_t ko = k * 2048;
                // [hi | lo] x [hi | lo]^T: warpgroup w takes the rows of plane w
                wgmma_m64n128k16<1, 1>(chk, gmma_desc_mn_sw128(a0 + wg * Cfg::SLICE + ko), gmma_desc_mn_sw128(a0 + ko),
                                       (first && k == 0) ? 0u : 1u);
            }
        } else {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint32_t ko = k * 2048;
                const uint64_t a_hi = gmma_desc_mn_sw128(a0 + wg * Cfg::SLICE + ko);
                const uint64_t a_lo = gmma_desc_mn_sw128(a0 + 2 * Cfg::SLICE + wg * Cfg::SLICE + ko);
                const uint64_t b_hi = gmma_desc_mn_sw128(b0 + ko);
                const uint64_t b_lo = gmma_desc_mn_sw128(b0 + 2 * Cfg::SLICE + ko);
                wgmma_m64n128k16<1, 1>(chk, a_hi, b_lo, (first && k == 0) ? 0u : 1u);
                wgmma_m64n128k16<1, 1>(chk, a_lo, b_hi, 1u);
                wgmma_m64n128k16<1, 1>(chk, a_hi, b_hi, 1u);
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
        acc_fence(chk);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
        if (++s == nst) { s = 0; ph ^= 1u; }
    };
    if constexpr (!MASK) {
        int it = 0;
        for (int c = 0; c < nchunks; ++c) {
            float chk[64];
#pragma unroll
            for (int i = 0; i < 64; ++i) chk[i] = 0.f;
            const int it_end = min(ntiles, (c + 1) * Cfg::CH);
            for (; it < it_end; ++it, ++tx) {
                if (tx == p.tiles_x) { tx = 0; ++ty; }
                tile(chk, it == c * Cfg::CH);
            }
#pragma unroll
            for (int i = 0; i < 64; ++i) acc[i] += chk[i];
        }
    } else {
        // chunks of CH tiles of THIS region (the tiles without it are skipped): with every label equal to the region the
        // chunks, and so the rounding, are those of the unmasked kernel
        float chk[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) chk[i] = 0.f;
        int done = 0;
        for (int it = 0; it < ntiles; ++it, ++tx) {
            if (tx == p.tiles_x) { tx = 0; ++ty; }
            if (!((tmask[t0 + it] >> reg) & 1u)) continue;
            tile(chk, done == 0);
            if (++done == Cfg::CH) {
#pragma unroll
                for (int i = 0; i < 64; ++i) acc[i] += chk[i];
                done = 0;
            }
        }
        if (done) {
#pragma unroll
            for (int i = 0; i < 64; ++i) acc[i] += chk[i];
        }
    }
    // ---- this CTA's partial block -> its own slot.  Fragment: rows m, m + 8; columns 8j + 2 (lane & 3) (+1) ----
    const int m = 64 * wg + 16 * (warp & 3) + (lane >> 2);
    const int cl = 2 * (lane & 3);
    if (!*abort_flag) {
#pragma unroll
        for (int j = 0; j < 16; ++j) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int mm = m + 8 * h, col = 8 * j + cl;
                float* dst;
                if (dup)   // rows m and m+64 both belong to channel m & 63, columns j and 64+j to channel j: quadrant -> slot
                    dst = p.part + (((long long)prob * p.nslots + split * 4 + (mm >> 6) * 2 + (col >> 6)) * p.C + (mm & 63)) * p.C + (col & 63);
                else
                    dst = p.part + (((long long)prob * p.nslots + split) * p.C + bi * 128 + mm) * p.C + bj * 128 + col;
                *reinterpret_cast<float2*>(dst) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            }
        }
    }
    if (want_sums) {
        // fixed-order reduction over the 32 row groups, then one partial per (image, split, channel)
#pragma unroll
        for (int sl = 0; sl < 2; ++sl)
#pragma unroll
            for (int j = 0; j < 8; ++j) red[rg * 128 + sl * 64 + chunk * 8 + j] = sums[sl][j];
    }
    asm volatile("bar.sync 2, 256;" ::: "memory");
    if (want_sums) {
        const int nch = dup ? 64 : 128;
        if (ct < nch && !*abort_flag) {
            float a = 0.f;
#pragma unroll
            for (int r = 0; r < 32; ++r) a += red[r * 128 + ct];
            p.psum[((long long)prob * p.ksplit + split) * p.C + (dup ? 0 : bi * 128) + ct] = a;
        }
    }
}

// shift[n][c] = mean of <= ~1024 strided interior pixels (all pixels when HW <= 1024): fixed-order reduction.
// grid (cdiv(C, 64), N): one CTA per 64 channels of an image (a single CTA per image took 180 us at C = 512);
// 256 threads = 8 channel groups x 32 pixel lanes (groups past C idle: AdaIN takes any multiple of 8 channels).
// MASK (spatial control): grid (C/64, N*R); problem z = n*R + r takes the mean of the sampled pixels labelled r, or of the
// whole sample when it holds none of them.  A frame-wide shift alone is not enough: a region mean far from t cancels in
// S - s s^T / n.  With every label equal to r the additions are those of the unmasked kernel.
// WGT (soft spatial control): the weighted mean of the sampled pixels under weight plane z (wts [N*R][H][W]), or the
// frame's shift when they carry no weight; 0/1 weights give MASK's additions.
template <bool MASK, bool WGT = false>
__global__ void __launch_bounds__(256)
k_sample_shift(const __half* __restrict__ act, ActGeom g, int stride, float* __restrict__ shift, const uint8_t* __restrict__ labels,
               int R, const float* __restrict__ wts = nullptr) {
    __shared__ float red[32][64];
    __shared__ float red_all[MASK ? 32 : 1][64];
    __shared__ int red_n[MASK ? 32 : 1];
    __shared__ float red_w[WGT ? 32 : 1];
    const int grp = threadIdx.x & 7, rl = threadIdx.x >> 3;
    const int c0 = blockIdx.x * 64 + grp * 8;
    const int n = MASK ? blockIdx.y / R : blockIdx.y;
    const int reg = MASK ? blockIdx.y - n * R : 0;
    const long long HW = (long long)g.H * g.W;
    const long long ns = (HW + stride - 1) / stride;
    const long long nk = c0 < g.C ? ns : 0;
    float s[8], sa[8];
    int cnt = 0;
    float sw = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) { s[j] = 0.f; sa[j] = 0.f; }
#pragma unroll 4
    for (long long k = rl; k < nk; k += 32) {
        const long long q = k * stride;
        const int y = (int)(q / g.W), x = (int)(q - (long long)y * g.W);
        float v[8];
        load8(act, g, ((long long)n * g.Hp + y + 1) * g.Wp + x + 1, c0, v);
        if (MASK) {
#pragma unroll
            for (int j = 0; j < 8; ++j) sa[j] += v[j];
            if (WGT) {
                const float w = wts[(long long)blockIdx.y * HW + q];
                if (!(w > 0.f)) continue;
                sw += w;
#pragma unroll
                for (int j = 0; j < 8; ++j) s[j] = fmaf(w, v[j], s[j]);
                continue;
            }
            if (labels[(long long)n * HW + q] != reg) continue;
            ++cnt;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) s[j] += v[j];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        red[rl][grp * 8 + j] = s[j];
        if (MASK) red_all[rl][grp * 8 + j] = sa[j];
    }
    if (MASK && grp == 0) red_n[rl] = cnt;
    if (WGT && grp == 0) red_w[rl] = sw;
    __syncthreads();
    if (threadIdx.x < 64 && blockIdx.x * 64 + threadIdx.x < g.C) {
        float a = 0.f, aa = 0.f, ww = 0.f;
        int m = 0;
#pragma unroll
        for (int r = 0; r < 32; ++r) {
            a += red[r][threadIdx.x];
            if (MASK) { aa += red_all[r][threadIdx.x]; m += red_n[r]; }
            if (WGT) ww += red_w[r];
        }
        float t = a / (float)ns;
        if (MASK) t = m > 0 ? a / (float)m : aa / (float)ns;
        if (WGT) t = ww > 0.f ? a / ww : aa / (float)ns;
        shift[(long long)blockIdx.y * g.C + blockIdx.x * 64 + threadIdx.x] = t;
    }
}

// The fixed-order fp64 reductions of the slots and the finalize expressions, shared by the whole-frame path (k_cov_sums,
// k_cov_finalize) and the statistics record of a rectangle (k_cov_record, k_record_cov_finalize): a record of the whole
// frame gives the same bits.
__device__ __forceinline__ double psum_total(const float* __restrict__ psum, int ksplit, int C, int n, int c) {
    double a = 0.0;
    for (int s = 0; s < ksplit; ++s) a += (double)psum[((long long)n * ksplit + s) * C + c];
    return a;
}
// four interleaved partial sums (a fixed order all the same): the serial fp64 chain over up to 256 slots took 73-85 us
__device__ __forceinline__ double part_total(const float* __restrict__ pp, int nslots, long long cc) {
    double v0 = 0.0, v1 = 0.0, v2 = 0.0, v3 = 0.0;
    int s = 0;
    for (; s + 4 <= nslots; s += 4) {
        v0 += (double)pp[(long long)s * cc];
        v1 += (double)pp[(long long)(s + 1) * cc];
        v2 += (double)pp[(long long)(s + 2) * cc];
        v3 += (double)pp[(long long)(s + 3) * cc];
    }
    for (; s < nslots; ++s) v0 += (double)pp[(long long)s * cc];
    return (v0 + v1) + (v2 + v3);
}
__device__ __forceinline__ float mean_from_sums(float shift, double s, long long cnt) {
    return cnt > 0 ? (float)((double)shift + s / (double)cnt) : shift;
}
// (a record's n is a real number: Kish's effective count of a weighted record; an integer n gives the integer form's bits)
__device__ __forceinline__ float mean_from_sums(float shift, double s, double cnt) {
    return cnt > 0.0 ? (float)((double)shift + s / cnt) : shift;
}
// (S - si sj / cnt) / (cnt - 1) (+ eps_cov on the diagonal)
__device__ __forceinline__ float cov_from_sums(double S, double si, double sj, long long cnt, bool diag, float eps_cov) {
    double v = S;
    v -= si * sj / (double)cnt;
    float r = (float)(v / (double)(cnt - 1));
    if (diag) r += eps_cov;
    return r;
}
__device__ __forceinline__ float cov_from_sums(double S, double si, double sj, double cnt, bool diag, float eps_cov) {
    double v = S;
    v -= si * sj / cnt;
    float r = (float)(v / (cnt - 1.0));
    if (diag) r += eps_cov;
    return r;
}

// dsum[n][c] = sum over splits of psum (fp64, fixed order); mean = shift + dsum / HW
// (spatial control: `counts` [problems] replaces HW; a problem without pixels keeps its shift as the mean)
__global__ void k_cov_sums(const float* __restrict__ psum, const float* __restrict__ shift, int C, int ksplit, long long HW,
                           int total, double* __restrict__ dsum, float* __restrict__ mean, const int* __restrict__ counts = nullptr) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int n = i / C, c = i - n * C;
    const long long cnt = counts ? (long long)counts[n] : HW;
    const double a = psum_total(psum, ksplit, C, n, c);
    dsum[i] = a;
    mean[i] = mean_from_sums(shift[i], a, cnt);
}

// G = (sum_slots part - s s^T / HW) / (HW - 1) + eps_cov * I   (ops.py:45,50,108,121), exactly symmetric
// (spatial control: `counts` [problems] replaces HW; a problem with fewer than 2 pixels gets G = I, a well-posed
//  placeholder whose transform is never applied)
__global__ void k_cov_finalize(const float* __restrict__ part, const double* __restrict__ dsum, int C, int nslots, long long HW,
                               float eps_cov, int count, float* __restrict__ G, float* __restrict__ A0,
                               const int* __restrict__ counts = nullptr) {
    const long long total = (long long)count * C * C;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int j = (int)(t % C);
        const int i = (int)((t / C) % C);
        const long long n = t / ((long long)C * C);
        if (counts && counts[n] < 2) {
            G[t] = i == j ? 1.f : 0.f;
            if (A0) A0[t] = G[t];
            continue;
        }
        const long long cnt = counts ? (long long)counts[n] : HW;
        // every (min,max) entry lies in a stored upper block: reading it for both (i,j) and (j,i) makes G exactly symmetric
        const long long e = (i <= j) ? (long long)i * C + j : (long long)j * C + i;
        const float* pp = part + n * nslots * (long long)C * C + e;
        const double v = part_total(pp, nslots, (long long)C * C);
        const float r = cov_from_sums(v, dsum[n * C + i], dsum[n * C + j], cnt, i == j, eps_cov);
        G[t] = r;
        if (A0) A0[t] = r;          // pristine copy: the Jacobi kernel overwrites G, the Rayleigh quotients need A
    }
}

// ---------------------------------------------------------------------------
// Statistics records (tiled stylisation, DESIGN.md §3.3.7).  A record of N frames holds, per frame, the pixel count n,
// the centring shift t, s = sum (x - t) and S = sum (x - t)(x - t)^T (the diagonal only for AdaIN's moments), all fp64
// (layout: stats_record_layout, wct.cu).  k_cov_record turns the slots of cov_tc_kernel into a record with the reductions
// of k_cov_sums / k_cov_finalize; S is written in full, symmetric.
// Weighted (wq: W = sum w, Q = sum w^2 per problem): the record of Kish's effective count n_eff = W^2 / Q, with s and S
// scaled by n_eff / W, so that the record's finalize gives mean t + s / W and cov (S - s s^T / W) / (W - Q / W); 0/1
// weights give n_eff = W and the scale 1 exactly.  A problem without weight gets n = 0.
// ---------------------------------------------------------------------------
__global__ void k_cov_record(const float* __restrict__ part, const float* __restrict__ psum, const float* __restrict__ shift, int C,
                             int nslots, int ksplit, long long HW, int count, double* __restrict__ rn, double* __restrict__ rt,
                             double* __restrict__ rs, double* __restrict__ rS, const double* __restrict__ wq = nullptr) {
    const long long total = (long long)count * C * C;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int j = (int)(t % C);
        const int i = (int)((t / C) % C);
        const long long n = t / ((long long)C * C);
        const long long e = (i <= j) ? (long long)i * C + j : (long long)j * C + i;
        double cnt = (double)HW, sc = 1.0;
        if (wq) {
            const double W = wq[2 * n], Q = wq[2 * n + 1];
            cnt = W > 0.0 ? W * W / Q : 0.0;
            sc = W > 0.0 ? cnt / W : 0.0;
        }
        double v = part_total(part + n * nslots * (long long)C * C + e, nslots, (long long)C * C);
        if (wq) v *= sc;
        rS[t] = v;
        if (j == 0) {
            double a = psum_total(psum, ksplit, C, (int)n, i);
            if (wq) a *= sc;
            rs[n * C + i] = a;
            rt[n * C + i] = (double)shift[n * C + i];
            if (i == 0) rn[n] = cnt;
        }
    }
}

// record -> mean [N][C], G (+ eps_cov I) and its copy A0, [N][C][C]: the expressions of k_cov_sums / k_cov_finalize.
// n is read as a real number (a weighted record's n_eff); a record of n < 2 gets G = I, k_cov_finalize's placeholder for a
// problem that is skipped (its k_c is -1: k_transform_kout).
__global__ void k_record_cov_finalize(const double* __restrict__ rn, const double* __restrict__ rt, const double* __restrict__ rs,
                                      const double* __restrict__ rS, int C, int count, float eps_cov, float* __restrict__ mean,
                                      float* __restrict__ G, float* __restrict__ A0) {
    const long long total = (long long)count * C * C;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int j = (int)(t % C);
        const int i = (int)((t / C) % C);
        const long long n = t / ((long long)C * C);
        const double cnt = rn[n];
        const long long e = (i <= j) ? (long long)i * C + j : (long long)j * C + i;
        const float r = cnt < 2.0 ? (i == j ? 1.f : 0.f)
                                  : cov_from_sums(rS[n * C * C + e], rs[n * C + i], rs[n * C + j], cnt, i == j, eps_cov);
        G[t] = r;
        A0[t] = r;
        if (j == 0) mean[n * C + i] = mean_from_sums((float)rt[n * C + i], rs[n * C + i], cnt);
    }
}

// ---------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiledC)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                     const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                     CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int g_cov_max_stages = 12;   // probe knob (wctb200_debug_set_cov_stages)

static inline int shift_stride(long long HW) { return HW <= 1024 ? 1 : (int)(HW / 1024); }

// shift [N][C] of a feature batch (k_sample_shift): the centring point of the covariance and of AdaIN's moments (wct.cu).
// A function of the frame alone.
int launch_sample_shift(const __half* act, ActGeom g, float* shift, cudaStream_t st) {
    k_sample_shift<false><<<dim3((unsigned)cdiv(g.C, 64), (unsigned)g.N), 256, 0, st>>>(act, g, shift_stride((long long)g.H * g.W),
                                                                                        shift, nullptr, 1);
    WCTB_CHECK_LAUNCH("k_sample_shift");
    return 0;
}

// Means and covariance (+ eps_cov I) of a feature batch: mean [N][C], G [N][C][C] (and a copy A0 if not null), fp32.
// dsum: [N][C] fp64 scratch (caller's workspace); partial products live in the per-stream scratch cache.
// Spatial control (labels != nullptr): one problem per (image, region), z = n * R + r, over the pixels labelled r:
// outputs [N*R][...]; counts [N*R] = pixels per problem and tmask [N][tiles] = regions present per 32 x 2 tile
// (k_region_scan, wct.cu).
// With `rec` the sums go to a statistics record instead (mean, G, A0, dsum unused).
// With `wts` (soft spatial control, [N][R][H][W] fp32 weights, tmask of nonzero weights, wq = W, Q per problem) the
// problems are weighted and the sums go to the Kish-normalised record `rec` (k_cov_record).
static int mean_cov_impl(const __half* act, ActGeom g, float eps_cov, float* mean, float* G, float* A0, double* dsum,
                         const uint8_t* labels, int R, const int* counts, const uint16_t* tmask, cudaStream_t st,
                         const StatsRecord* rec = nullptr, const float* wts = nullptr, const double* wq = nullptr) {
    static PFN_encodeTiledC enc = nullptr;
    if (!enc) {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess) {
            set_error("cuTensorMapEncodeTiled entry point not available");
            return WCTB200_ECUDA;
        }
        enc = reinterpret_cast<PFN_encodeTiledC>(ptr);
    }
    WCTB_REQUIRE(g.C == 64 || (g.C % 128 == 0 && g.C <= 2048), "covariance: C=%d must be 64 or a multiple of 128 (<= 2048)", g.C);
    const long long HW = (long long)g.H * g.W;
    const bool weighted = wts != nullptr;
    const bool masked = labels != nullptr || weighted;
    const int nprob = masked ? g.N * R : g.N;
    CovParams p;
    p.C = g.C; p.W = g.W; p.H = g.H; p.N = g.N;
    p.tiles_x = (g.W + 31) / 32;
    p.tiles_y = (g.H + 1) / 2;
    p.nb = g.C == 64 ? 1 : g.C / 128;
    const int npairs = p.nb * (p.nb + 1) / 2;
    const int tiles_img = p.tiles_x * p.tiles_y;
    // Split of one image into CTAs: a function of (C, H, W) ONLY (batch- and device-invariant results).  Up to 64 tiles
    // (4096 pixels) per CTA keeps the per-CTA set-up small and still gives a single 512x512 frame 64 CTAs per block pair.
    int tps = 64;
    if (tiles_img < 64 * 8) tps = (tiles_img + 7) / 8;        // small maps: 8 splits
    if (tps < 8) tps = 8;
    p.tiles_per_split = tps;
    p.ksplit = (tiles_img + tps - 1) / tps;
    p.nslots = g.C == 64 ? 4 * p.ksplit : p.ksplit;
    // scratch: shift [P][C] | psum [P][ksplit][C] | part [P][nslots][C][C]   (P problems)
    const size_t n_shift = (size_t)nprob * g.C, n_psum = (size_t)nprob * p.ksplit * g.C;
    const size_t n_part = (size_t)nprob * p.nslots * g.C * g.C;
    float* scratch = nullptr;
    { int rc0 = scratch_alloc(reinterpret_cast<void**>(&scratch), (n_shift + n_psum + n_part + 64) * sizeof(float), st, 0); if (rc0) return rc0; }
    float* shift = scratch;
    float* psum = shift + ((n_shift + 3) & ~(size_t)3);
    float* part = psum + ((n_psum + 3) & ~(size_t)3);
    p.shift = shift; p.psum = psum; p.part = part;
    p.err = device_error_word();
    p.max_stages = g_cov_max_stages;
    p.labels = labels;
    p.tmask = tmask;
    p.R = masked ? R : 1;
    p.wts = wts;
    // (blocks below the diagonal are never written -- and never read: k_cov_finalize only touches (min,max) entries)

    if (weighted) {
        k_sample_shift<true, true><<<dim3((unsigned)(g.C / 64), (unsigned)nprob), 256, 0, st>>>(act, g, shift_stride(HW), shift,
                                                                                                 nullptr, R, wts);
        WCTB_CHECK_LAUNCH("k_sample_shift");
    } else if (masked) {
        k_sample_shift<true><<<dim3((unsigned)(g.C / 64), (unsigned)nprob), 256, 0, st>>>(act, g, shift_stride(HW), shift, labels, R);
        WCTB_CHECK_LAUNCH("k_sample_shift");
    } else {
        int rc = launch_sample_shift(act, g, shift, st);
        if (rc) return rc;
    }

    // tensor map over the interior pixels only (see header comment)
    CUtensorMap mX;
    const __half* base = act + ((long long)g.Wp + 1) * g.C;
    cuuint64_t dims[5] = {(cuuint64_t)g.C, (cuuint64_t)g.W, (cuuint64_t)g.H, (cuuint64_t)g.N, 2};
    cuuint64_t strides[4] = {(cuuint64_t)g.C * 2, (cuuint64_t)g.Wp * g.C * 2, (cuuint64_t)g.Hp * g.Wp * g.C * 2,
                             (cuuint64_t)g.plane * 2};
    cuuint32_t box[5] = {64, 32, 2, 1, 1};
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = enc(&mX, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, const_cast<__half*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cov_tc: cuTensorMapEncodeTiled failed (%d)", (int)r);
        return WCTB200_ECUDA;
    }
    dim3 grid((unsigned)(npairs * p.ksplit), (unsigned)nprob);
    if (weighted) {
        WCTB_ENSURE_SMEM((cov_tc_kernel<true, true>), CovCfg::SMEM_BYTES);
        cov_tc_kernel<true, true><<<grid, CovCfg::THREADS, CovCfg::SMEM_BYTES, st>>>(mX, p);
    } else if (masked) {
        WCTB_ENSURE_SMEM(cov_tc_kernel<true>, CovCfg::SMEM_BYTES);
        cov_tc_kernel<true><<<grid, CovCfg::THREADS, CovCfg::SMEM_BYTES, st>>>(mX, p);
    } else {
        WCTB_ENSURE_SMEM(cov_tc_kernel<false>, CovCfg::SMEM_BYTES);
        cov_tc_kernel<false><<<grid, CovCfg::THREADS, CovCfg::SMEM_BYTES, st>>>(mX, p);
    }
    WCTB_CHECK_LAUNCH("cov_tc_kernel");
    if (rec) {
        const long long tot = (long long)nprob * g.C * g.C;
        k_cov_record<<<(unsigned)(cdiv(tot, 256) > 4096 ? 4096 : cdiv(tot, 256)), 256, 0, st>>>(
            part, psum, shift, g.C, p.nslots, p.ksplit, HW, nprob, rec->n, rec->t, rec->s, rec->S, wq);
        WCTB_CHECK_LAUNCH("k_cov_record");
        return 0;
    }
    k_cov_sums<<<cdiv((long long)nprob * g.C, 256), 256, 0, st>>>(psum, shift, g.C, p.ksplit, HW, nprob * g.C, dsum, mean, counts);
    WCTB_CHECK_LAUNCH("k_cov_sums");
    const long long tot = (long long)nprob * g.C * g.C;
    k_cov_finalize<<<(unsigned)(cdiv(tot, 256) > 4096 ? 4096 : cdiv(tot, 256)), 256, 0, st>>>(part, dsum, g.C, p.nslots, HW,
                                                                                               eps_cov, nprob, G, A0, counts);
    WCTB_CHECK_LAUNCH("k_cov_finalize");
    return 0;
}

int launch_mean_cov(const __half* act, ActGeom g, float eps_cov, float* mean, float* G, float* A0, double* dsum, cudaStream_t st) {
    return mean_cov_impl(act, g, eps_cov, mean, G, A0, dsum, nullptr, 1, nullptr, nullptr, st);
}
int launch_mean_cov_regions(const __half* act, ActGeom g, const uint8_t* labels, int R, const int* counts, const uint16_t* tmask,
                            float eps_cov, float* mean, float* G, float* A0, double* dsum, cudaStream_t st) {
    return mean_cov_impl(act, g, eps_cov, mean, G, A0, dsum, labels, R, counts, tmask, st);
}
// The record of the rectangle [y0, y0+h) x [x0, x0+w) of a feature batch [N][H][W][C]: the rectangle is a view of the
// padded planes (base at its first pixel, the planes' strides, dims h x w), so the TMA boxes that stick out of it are
// zero-filled and every kernel sees a frame of h x w pixels.  The split into CTAs and the sampled shift are those of an
// h x w frame: the whole-frame rectangle takes today's split, samples and sums.
int launch_cov_record(const __half* act, int N, int H, int W, int C, int y0, int x0, int h, int w, const StatsRecord& rec,
                      cudaStream_t st) {
    ActGeom v(N, H, W, C);
    v.H = h;
    v.W = w;
    const __half* base = act + ((long long)y0 * v.Wp + x0) * C;
    return mean_cov_impl(base, v, 0.f, nullptr, nullptr, nullptr, nullptr, nullptr, 1, nullptr, nullptr, st, &rec);
}
// The weighted record of N*K problems (soft spatial control): weights [N][K][H][W], tmask [N][tiles] of nonzero weights,
// wq [N*K][2] = (W, Q) (wct.cu: launch_wct_stats_weighted)
int launch_cov_record_weighted(const __half* act, int N, int H, int W, int C, const float* wts, int K, const uint16_t* tmask,
                               const double* wq, const StatsRecord& rec, cudaStream_t st) {
    return mean_cov_impl(act, ActGeom(N, H, W, C), 0.f, nullptr, nullptr, nullptr, nullptr, nullptr, K, nullptr, tmask, st, &rec,
                         wts, wq);
}
int launch_record_cov_finalize(const StatsRecord& rec, int C, int N, float eps_cov, float* mean, float* G, float* A0, cudaStream_t st) {
    const long long tot = (long long)N * C * C;
    k_record_cov_finalize<<<(unsigned)(cdiv(tot, 256) > 4096 ? 4096 : cdiv(tot, 256)), 256, 0, st>>>(rec.n, rec.t, rec.s, rec.S, C, N,
                                                                                                      eps_cov, mean, G, A0);
    WCTB_CHECK_LAUNCH("k_record_cov_finalize");
    return 0;
}

}  // namespace wctb
