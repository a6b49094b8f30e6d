// Memory-bound layers of the encoder/decoder and the SPF16 conversion helpers.
// All kernels are HBM-bound streaming kernels: 16-byte vector loads/stores, one
// 8-channel group per thread, grid sized from the element count.
#include "common.cuh"

namespace wctb {

// ---------------------------------------------------------------------------
// image pre/post   (wct.py:60-68)
// ---------------------------------------------------------------------------
__global__ void k_u8_to_f32(const uint8_t* __restrict__ in, size_t n, float* __restrict__ out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) out[i] = (float)in[i] / 255.f;   // image / 255.  (wct.py:64)
}
__global__ void k_f32_to_u8(const float* __restrict__ in, size_t n, uint8_t* __restrict__ out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        float v = fminf(fmaxf(in[i], 0.f), 1.f) * 255.f;        // np.clip(x,0,1)*255 (wct.py:68)
        out[i] = (uint8_t)v;                                     // np.uint8 truncates
    }
}

// ---------------------------------------------------------------------------
// fp32 NHWC <-> SPF16
// ---------------------------------------------------------------------------
__global__ void k_act_from_f32(const float* __restrict__ in, ActGeom g, __half* __restrict__ act) {
    const int cg = g.C / 8;
    const long long total = (long long)g.N * g.H * g.W * cg;
    // 32-bit index arithmetic (launcher guarantees total < 2^32): 64-bit div/mod costs ~100 instructions each
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < (unsigned)total; i += gridDim.x * blockDim.x) {
        const int c0 = (int)(i % (unsigned)cg) * 8;
        unsigned pix = i / (unsigned)cg;
        const int x = (int)(pix % (unsigned)g.W); pix /= (unsigned)g.W;
        const int y = (int)(pix % (unsigned)g.H);
        const int n = (int)(pix / (unsigned)g.H);
        const float* src = in + (((long long)n * g.H + y) * g.W + x) * g.C + c0;
        float v[8];
        *reinterpret_cast<float4*>(v) = *reinterpret_cast<const float4*>(src);
        *reinterpret_cast<float4*>(v + 4) = *reinterpret_cast<const float4*>(src + 4);
        Half8 hi, lo;
        split8(v, hi, lo);
        store8_with_halo(act, g, n, y, x, c0, hi, lo);
    }
}
__global__ void k_act_to_f32(const __half* __restrict__ act, ActGeom g, float* __restrict__ out) {
    const int cg = g.C / 8;
    const long long total = (long long)g.N * g.H * g.W * cg;
    // 32-bit index arithmetic (launcher guarantees total < 2^32): 64-bit div/mod costs ~100 instructions each
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < (unsigned)total; i += gridDim.x * blockDim.x) {
        const int c0 = (int)(i % (unsigned)cg) * 8;
        unsigned pix = i / (unsigned)cg;
        const int x = (int)(pix % (unsigned)g.W); pix /= (unsigned)g.W;
        const int y = (int)(pix % (unsigned)g.H);
        const int n = (int)(pix / (unsigned)g.H);
        const long long pos = ((long long)n * g.Hp + y + 1) * g.Wp + x + 1;
        float v[8];
        load8(act, g, pos, c0, v);
        float* dst = out + (((long long)n * g.H + y) * g.W + x) * g.C + c0;
        *reinterpret_cast<float4*>(dst) = *reinterpret_cast<float4*>(v);
        *reinterpret_cast<float4*>(dst + 4) = *reinterpret_cast<float4*>(v + 4);
    }
}

// Rewrites every halo cell of an SPF16 activation from the interior, in the halo mode of g (ActGeom::set_halo): one thread
// per (halo cell, 8-channel group).  A cell reads only interior cells, so the order of the stores does not matter.  The
// 2 (W+2) + 2 H halo cells of a frame are numbered top row, bottom row, then the left and right cells of each interior row.
__global__ void k_act_halo(__half* __restrict__ act, ActGeom g) {
    const int cg = g.C / 8;
    const unsigned cells = 2u * (unsigned)g.Wp + 2u * (unsigned)g.H;
    const long long total = (long long)g.N * cells * cg;
    // 32-bit index arithmetic (launcher guarantees total < 2^32)
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < (unsigned)total; i += gridDim.x * blockDim.x) {
        const int c0 = (int)(i % (unsigned)cg) * 8;
        const unsigned t = i / (unsigned)cg;
        const unsigned k = t % cells;
        const int n = (int)(t / cells);
        int py, px;                                   // padded coordinates of the halo cell
        if (k < 2u * (unsigned)g.Wp) {
            py = k < (unsigned)g.Wp ? 0 : g.H + 1;
            px = (int)(k % (unsigned)g.Wp);
        } else {
            const unsigned r = k - 2u * (unsigned)g.Wp;
            py = (int)(r >> 1) + 1;
            px = (r & 1u) ? g.W + 1 : 0;
        }
        const int sy = py == 0 ? g.ht : (py == g.H + 1 ? g.hb : py - 1);
        const int sx = px == 0 ? g.wl : (px == g.W + 1 ? g.wr : px - 1);
        const long long src = (((long long)n * g.Hp + sy + 1) * g.Wp + sx + 1) * g.C + c0;
        const long long dst = (((long long)n * g.Hp + py) * g.Wp + px) * g.C + c0;
        *reinterpret_cast<Half8*>(act + dst) = *reinterpret_cast<const Half8*>(act + src);
        *reinterpret_cast<Half8*>(act + g.plane + dst) = *reinterpret_cast<const Half8*>(act + g.plane + src);
    }
}

// ---------------------------------------------------------------------------
// weights: fp32 [taps][Cin][Cout] -> split fp16 [2][Cout][taps*Cin], stored scaled by a power of two
//   trailer (after the planes): float[0] = 1/scale (undone in the conv epilogue), uint[1] = max|w| bits (scratch).
//   Why: conv weights are ~1e-2 (He-normal std sqrt(2/(9 Cin)), trained VGG alike): hi = fp16(w) keeps 11 bits, but
//   lo = w - hi ~ 5e-6 is an fp16 SUBNORMAL (spacing 6e-8), so hi+lo kept only ~16 bits of the weight.  With max|w|
//   scaled into [512,1024) every lo that matters is a normal fp16 number and hi+lo carries 22 bits.
// ---------------------------------------------------------------------------
__global__ void k_absmax(const float* __restrict__ w, long long n, unsigned int* __restrict__ out_bits) {
    float m = 0.f;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float v = fabsf(w[i]);
        if (v < 3.0e38f) m = fmaxf(m, v);          // ignores inf / NaN
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(out_bits, __float_as_uint(m));    // non-negative floats order like their bits
}
__global__ void k_prep_weights(const float* __restrict__ w, int taps, int Cin, int Cout, __half* __restrict__ ws,
                               float* __restrict__ trailer) {
    const long long K = (long long)taps * Cin;
    const long long total = K * Cout;
    const float sc = weight_scale(reinterpret_cast<const unsigned int*>(trailer)[1]);
    if (blockIdx.x == 0 && threadIdx.x == 0) trailer[0] = 1.f / sc;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int co = (int)(i / K);
        const long long k = i - (long long)co * K;      // k = tap*Cin + cin
        const float v = w[k * Cout + co] * sc;
        __half hi, lo;
        split_f32(v, hi, lo);
        ws[i] = hi;
        ws[total + i] = lo;
    }
}
// UpSampling2D -> Conv2DReflect as four 2x2-tap convs over the low-resolution input (conv_tc.cu, mode UP2):
// [class a*2+b][plane][Cout][4*Cin], k = (ty*2+tx)*Cin + cin; the weight of class (a,b), tap (ty,tx) is the sum of the
// 3x3 taps that land on low-resolution row i-1+a+ty / column j-1+b+tx:  a=0: ty=0 <- {ky=0}, ty=1 <- {1,2};
// a=1: ty=0 <- {0,1}, ty=1 <- {2} (same for columns).  Sums in fp64, rounded once.
__global__ void k_prep_weights_up2(const float* __restrict__ w, int Cin, int Cout, __half* __restrict__ ws,
                                   float* __restrict__ trailer) {
    const long long K = 4ll * Cin;
    const long long per_plane = K * Cout;
    const long long total = 4 * per_plane;
    const float sc = weight_scale(reinterpret_cast<const unsigned int*>(trailer)[1]);
    if (blockIdx.x == 0 && threadIdx.x == 0) trailer[0] = 1.f / sc;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int cls = (int)(i / per_plane);
        const long long r = i - cls * per_plane;
        const int co = (int)(r / K);
        const int k = (int)(r - (long long)co * K);
        const int tap = k / Cin, cin = k - tap * Cin;
        const int a = cls >> 1, b = cls & 1, ty = tap >> 1, tx = tap & 1;
        const int ky0 = a == 0 ? (ty == 0 ? 0 : 1) : (ty == 0 ? 0 : 2), ky1 = a == 0 ? (ty == 0 ? 0 : 2) : (ty == 0 ? 1 : 2);
        const int kx0 = b == 0 ? (tx == 0 ? 0 : 1) : (tx == 0 ? 0 : 2), kx1 = b == 0 ? (tx == 0 ? 0 : 2) : (tx == 0 ? 1 : 2);
        double v = 0.0;
        for (int ky = ky0; ky <= ky1; ++ky)
            for (int kx = kx0; kx <= kx1; ++kx) v += (double)w[((long long)(ky * 3 + kx) * Cin + cin) * Cout + co];
        __half hi, lo;
        split_f32((float)(v * (double)sc), hi, lo);
        ws[(long long)(cls * 2) * per_plane + r] = hi;
        ws[(long long)(cls * 2 + 1) * per_plane + r] = lo;
    }
}

// ---------------------------------------------------------------------------
// validation conv: plain fp32 FFMA, one thread per (pixel, cout)
// ---------------------------------------------------------------------------
__global__ void k_conv3x3_ref(const __half* __restrict__ in, ActGeom gi, const float* __restrict__ w,
                              const float* __restrict__ bias, int Cout, int flags, __half* __restrict__ out) {
    const ActGeom go(gi.N, gi.H, gi.W, Cout);
    const long long total = (long long)gi.N * gi.H * gi.W * Cout;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int co = (int)(i % Cout);
        long long pix = i / Cout;
        const int x = (int)(pix % gi.W); pix /= gi.W;
        const int y = (int)(pix % gi.H);
        const int n = (int)(pix / gi.H);
        float acc = bias ? bias[co] : 0.f;
        for (int ky = 0; ky < 3; ++ky)
            for (int kx = 0; kx < 3; ++kx) {
                const long long pos = ((long long)n * gi.Hp + y + ky) * gi.Wp + x + kx;
                const __half* ph = in + pos * gi.C;
                const __half* pl = ph + gi.plane;
                const float* wp = w + (long long)(ky * 3 + kx) * gi.C * Cout + co;
                for (int ci = 0; ci < gi.C; ++ci) acc = fmaf(merge_f32(ph[ci], pl[ci]), wp[(long long)ci * Cout], acc);
            }
        if (flags & WCTB200_RELU) acc = fmaxf(acc, 0.f);
        __half hi, lo;
        split_f32(acc, hi, lo);
        int rows[3], cols[3];
        const int nr = halo_rows(y, go.H, rows), nc = halo_rows(x, go.W, cols);
        for (int a = 0; a < nr; ++a)
            for (int b = 0; b < nc; ++b) {
                const long long off = (((long long)n * go.Hp + rows[a]) * go.Wp + cols[b]) * Cout + co;
                out[off] = hi;
                out[go.plane + off] = lo;
            }
    }
}

// ---------------------------------------------------------------------------
// encoder head: (1x1 preprocess conv folded into) conv1_1 3->64 + ReLU
//   vgg_normalised.py:25-40.  One thread = one pixel x 8 output channels.
// ---------------------------------------------------------------------------
// one thread = 4 horizontally adjacent pixels x 8 output channels: each conflict-free LDS.128
// pair of weights feeds 32 FMAs (the first version, 1 pixel per thread, was shared-memory bound:
// ncu short_scoreboard + mio_throttle, 2-way bank conflicts on the 32-byte-strided weight reads)
__global__ void __launch_bounds__(256)
k_conv_head(const float* __restrict__ img, int N, int H, int W, const float* __restrict__ w,
            const float* __restrict__ b, int flags, __half* __restrict__ out) {
    // weights re-laid out [k][half][group][4] (channel c = 8*group + 4*half + j): the 8 lanes of a
    // quarter-warp read 8 consecutive 16-byte words
    __shared__ __align__(16) float sw[27 * 64];
    __shared__ float sb[64];
    for (int i = threadIdx.x; i < 27 * 64; i += blockDim.x) {
        const int k = i >> 6, c = i & 63;
        sw[(k * 2 + ((c >> 2) & 1)) * 32 + (c >> 3) * 4 + (c & 3)] = w[i];
    }
    if (threadIdx.x < 64) sb[threadIdx.x] = b[threadIdx.x];
    __syncthreads();
    ActGeom go(N, H, W, 64);
    go.set_halo(flags);
    const bool wrap_x = (flags & WCTB200_HALO_WRAP_X) != 0, wrap_y = (flags & WCTB200_HALO_WRAP_Y) != 0;
    const unsigned segs = (unsigned)(W + 3) / 4u;
    const unsigned total = (unsigned)N * (unsigned)H * segs * 8u;
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int g = (int)(i & 7u);
        unsigned t = i >> 3;
        const int xs = (int)(t % segs) * 4; t /= segs;
        const int y = (int)(t % (unsigned)H);
        const int n = (int)(t / (unsigned)H);
        // accumulators as fp32 pairs (two channels each)
        f32x2 acc[4][4];
#pragma unroll
        for (int p = 0; p < 4; ++p)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[p][j] = pack2(sb[g * 8 + 2 * j], sb[g * 8 + 2 * j + 1]);
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
            const int yy = pad_index(y + ky - 1, H, wrap_y);
            const float* row = img + ((long long)n * H + yy) * W * 3;
            f32x2 in[6][3];
#pragma unroll
            for (int j = 0; j < 6; ++j) {
                int xx = pad_index(xs + j - 1, W, wrap_x);
                xx = min(max(xx, 0), W - 1);                 // columns past the ragged right edge: any valid address
#pragma unroll
                for (int ci = 0; ci < 3; ++ci) {
                    const float v = __ldg(row + xx * 3 + ci);
                    in[j][ci] = pack2(v, v);
                }
            }
#pragma unroll
            for (int kx = 0; kx < 3; ++kx)
#pragma unroll
                for (int ci = 0; ci < 3; ++ci) {
                    const int k = (ky * 3 + kx) * 3 + ci;
                    const f32x2x2 w0 = *reinterpret_cast<const f32x2x2*>(sw + (k * 2) * 32 + g * 4);       // channels 0..3 as two pairs
                    const f32x2x2 w1 = *reinterpret_cast<const f32x2x2*>(sw + (k * 2 + 1) * 32 + g * 4);   // channels 4..7
#pragma unroll
                    for (int p = 0; p < 4; ++p) {
                        const f32x2 v = in[p + kx][ci];
                        acc[p][0] = fma2(v, w0.x, acc[p][0]);
                        acc[p][1] = fma2(v, w0.y, acc[p][1]);
                        acc[p][2] = fma2(v, w1.x, acc[p][2]);
                        acc[p][3] = fma2(v, w1.y, acc[p][3]);
                    }
                }
        }
#pragma unroll
        for (int p = 0; p < 4; ++p) {
            if (xs + p < W) {
                float v[8];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    unpack2(acc[p][j], v[2 * j], v[2 * j + 1]);
                    v[2 * j] = fmaxf(v[2 * j], 0.f);
                    v[2 * j + 1] = fmaxf(v[2 * j + 1], 0.f);
                }
                Half8 hi, lo;
                split8(v, hi, lo);
                store8_with_halo(out, go, n, y, xs + p, g * 8, hi, lo);
            }
        }
    }
}

// ---------------------------------------------------------------------------
// decoder tail: Conv2DReflect Cin->3, no activation (model.py:297-298) [+ clip, model.py:86]
//   8 lanes cooperate on 4 horizontally adjacent pixels (lane = 8-channel group, looped for
//   Cin > 64): each activation vector is loaded/merged once and used by 3 horizontal taps,
//   each weight LDS.128 (conflict-free layout) feeds 16 FMAs; 3-step shuffle reduction.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_conv_tail(const __half* __restrict__ in, ActGeom gi, const float* __restrict__ w, const float* __restrict__ b,
            int flags, float* __restrict__ img) {
    extern __shared__ __align__(16) float swt[];   // [tap][out][half][group][4], channel c = 8*group + 4*half + j
    const int K = 9 * gi.C;
    const int cgs = gi.C / 8;
    for (int i = threadIdx.x; i < K * 3; i += blockDim.x) {
        const int o = i % 3, k = i / 3;            // w is [9*Cin][3], k = tap*Cin + c
        const int tap = k / gi.C, c = k - tap * gi.C;
        swt[((((tap * 3 + o) * 2 + ((c >> 2) & 1)) * cgs) + (c >> 3)) * 4 + (c & 3)] = w[i];
    }
    __syncthreads();
    const unsigned segs = (unsigned)(gi.W + 3) / 4u;
    const unsigned nseg = (unsigned)gi.N * (unsigned)gi.H * segs;
    const int sub = threadIdx.x & 7;
    const int lane = threadIdx.x & 31;
    // warp-uniform loop bound (the shuffles below need the whole warp): 4 segments per warp
    for (unsigned wbase = ((blockIdx.x * blockDim.x + threadIdx.x) - lane) >> 3; wbase < nseg;
         wbase += (gridDim.x * blockDim.x) >> 3) {
        const unsigned seg = wbase + (lane >> 3);
        const bool ok = seg < nseg;
        unsigned t = ok ? seg : 0u;
        const int xs = (int)(t % segs) * 4; t /= segs;
        const int y = (int)(t % (unsigned)gi.H);
        const int n = (int)(t / (unsigned)gi.H);
        float acc[4][3];
#pragma unroll
        for (int p = 0; p < 4; ++p) acc[p][0] = acc[p][1] = acc[p][2] = 0.f;
        if (ok) {
            for (int cgi = sub; cgi < cgs; cgi += 8) {
#pragma unroll
                for (int ky = 0; ky < 3; ++ky) {
                    float v[6][8];
                    const long long rowpos = ((long long)n * gi.Hp + y + ky) * gi.Wp + xs;
#pragma unroll
                    for (int j = 0; j < 6; ++j) {
                        if (xs + j <= gi.W + 1) load8(in, gi, rowpos + j, cgi * 8, v[j]);
                        else {
#pragma unroll
                            for (int e = 0; e < 8; ++e) v[j][e] = 0.f;
                        }
                    }
#pragma unroll
                    for (int kx = 0; kx < 3; ++kx)
#pragma unroll
                        for (int o = 0; o < 3; ++o) {
                            const int base = (((ky * 3 + kx) * 3 + o) * 2) * cgs;
                            const float4 w0 = *reinterpret_cast<const float4*>(swt + (base + cgi) * 4);
                            const float4 w1 = *reinterpret_cast<const float4*>(swt + (base + cgs + cgi) * 4);
#pragma unroll
                            for (int p = 0; p < 4; ++p) {
                                const float* vv = v[p + kx];
                                float a = acc[p][o];
                                a = fmaf(vv[0], w0.x, a); a = fmaf(vv[1], w0.y, a); a = fmaf(vv[2], w0.z, a); a = fmaf(vv[3], w0.w, a);
                                a = fmaf(vv[4], w1.x, a); a = fmaf(vv[5], w1.y, a); a = fmaf(vv[6], w1.z, a); a = fmaf(vv[7], w1.w, a);
                                acc[p][o] = a;
                            }
                        }
                }
            }
        }
#pragma unroll
        for (int p = 0; p < 4; ++p)
#pragma unroll
            for (int o = 0; o < 3; ++o) {
                float a = acc[p][o];
                a += __shfl_xor_sync(0xffffffffu, a, 4);
                a += __shfl_xor_sync(0xffffffffu, a, 2);
                a += __shfl_xor_sync(0xffffffffu, a, 1);
                acc[p][o] = a;
            }
        if (ok && sub == 0) {
#pragma unroll
            for (int p = 0; p < 4; ++p) {
                if (xs + p < gi.W) {
                    float* d = img + (((long long)n * gi.H + y) * gi.W + xs + p) * 3;
#pragma unroll
                    for (int o = 0; o < 3; ++o) {
                        float a = acc[p][o] + b[o];
                        if (flags & WCTB200_CLIP01) a = fminf(fmaxf(a, 0.f), 1.f);
                        d[o] = a;
                    }
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------
// decoder tail, tiled: the version above re-reads and re-merges every activation vector for each of the three
// vertical taps and keeps only 8 lanes on a pixel (measured 0.95 TB/s of input, 12 TFLOP/s).  Here a CTA of
// 128 threads owns a 32x32 output tile and walks the input in 8-channel slices:
//   * the raw split-fp16 patch (34x34 pixels x 16 B per plane) of slice s+1 is fetched with cp.async into a
//     staging buffer WHILE slice s is being multiplied (a first version that loaded synchronously spent 70 % of
//     its cycles on long-scoreboard stalls: only 8 warps per SM);
//   * a short pass merges the staged slice to fp32 into [4-channel group][row][col] float4 (lanes = consecutive
//     columns, conflict free);
//   * each thread accumulates an 8-row column strip x 3 outputs: per (group, kx) 10 activation LDS.128 + 9
//     broadcast weight LDS.128 feed 288 FMAs.
// ---------------------------------------------------------------------------
constexpr int TT_W = 32, TT_H = 32, TT_PW = TT_W + 2, TT_PH = TT_H + 2, TT_CH = 8;
constexpr int TT_PIX = TT_PH * TT_PW;                                           // 1156 patch pixels
constexpr int TT_ACT_F4 = (TT_CH / 4) * TT_PIX;                                 // merged slice: float4 slots
constexpr int TT_STAGE_F4 = 2 * TT_PIX;                                         // raw slice: 16 B per plane per pixel

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}

__global__ void __launch_bounds__(128, 2)
k_conv_tail_tiled(const __half* __restrict__ in, ActGeom gi, const float* __restrict__ w, const float* __restrict__ b,
                  int flags, float* __restrict__ img, int tiles_x, int tiles_y) {
    extern __shared__ __align__(16) float4 tsm[];
    float4* sact = tsm;                               // [TT_CH/4][TT_PH][TT_PW]
    float4* stage = tsm + TT_ACT_F4;                  // [plane][TT_PIX] raw Half8
    float4* swt = stage + TT_STAGE_F4;                // [tap][c4 of all Cin][out]
    const int C4 = gi.C / 4;
    int t = blockIdx.x;
    const int tx = t % tiles_x; t /= tiles_x;
    const int ty = t % tiles_y;
    const int n = t / tiles_y;
    const int x0 = tx * TT_W, y0 = ty * TT_H;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    auto prefetch = [&](int c0) {
        for (int i = threadIdx.x; i < 2 * TT_PIX; i += 128) {
            const int plane = i >= TT_PIX ? 1 : 0, pp = i - plane * TT_PIX;
            const int pr = pp / TT_PW, pc = pp - pr * TT_PW;
            const int yy = min(y0 + pr, gi.Hp - 1), xx = min(x0 + pc, gi.Wp - 1);   // padded coordinates; ragged tiles clamp
            const long long off = (((long long)n * gi.Hp + yy) * gi.Wp + xx) * gi.C + c0;
            cp_async16(stage + i, in + (plane ? gi.plane : 0) + off);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    prefetch(0);
    for (int i = threadIdx.x; i < 9 * C4 * 3; i += 128) {
        const int o = i % 3, c4 = (i / 3) % C4, tap = i / (3 * C4);
        const float* src = w + ((size_t)(tap * gi.C + c4 * 4)) * 3 + o;          // w is [9*Cin][3], k = tap*Cin + c
        swt[i] = make_float4(src[0], src[3], src[6], src[9]);
    }
    f32x2 acc[8][3];                                  // packed pairs: (even, odd) channel partial sums, added at the end
#pragma unroll
    for (int p = 0; p < 8; ++p) acc[p][0] = acc[p][1] = acc[p][2] = pack2(0.f, 0.f);

    for (int c0 = 0; c0 < gi.C; c0 += TT_CH) {
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();                              // staged slice visible; previous slice's FMAs are done with sact
        for (int pp = threadIdx.x; pp < TT_PIX; pp += 128) {
            const Half8 hi = *reinterpret_cast<const Half8*>(stage + pp);
            const Half8 lo = *reinterpret_cast<const Half8*>(stage + TT_PIX + pp);
            float v[8];
            merge8(hi, lo, v);
            sact[pp] = make_float4(v[0], v[1], v[2], v[3]);
            sact[TT_PIX + pp] = make_float4(v[4], v[5], v[6], v[7]);
        }
        __syncthreads();                              // merged slice ready, staging buffer free
        if (c0 + TT_CH < gi.C) prefetch(c0 + TT_CH);
#pragma unroll 1
        for (int g = 0; g < TT_CH / 4; ++g) {
            const float4* wg = swt + (c0 / 4 + g) * 3;
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                f32x2x2 a[10];                     // float4 viewed as two packed fp32 pairs
                const f32x2x2* col = reinterpret_cast<const f32x2x2*>(sact) + (g * TT_PH + warp * 8) * TT_PW + lane + kx;
#pragma unroll
                for (int r = 0; r < 10; ++r) a[r] = col[r * TT_PW];
#pragma unroll
                for (int ky = 0; ky < 3; ++ky) {
#pragma unroll
                    for (int o = 0; o < 3; ++o) {
                        const f32x2x2 wv = *reinterpret_cast<const f32x2x2*>(wg + (ky * 3 + kx) * C4 * 3 + o);
#pragma unroll
                        for (int p = 0; p < 8; ++p) acc[p][o] = fma2(a[p + ky].y, wv.y, fma2(a[p + ky].x, wv.x, acc[p][o]));
                    }
                }
            }
        }
    }
    const int x = x0 + lane;
    if (x < gi.W) {
#pragma unroll
        for (int p = 0; p < 8; ++p) {
            const int y = y0 + warp * 8 + p;
            if (y < gi.H) {
                float* d = img + (((long long)n * gi.H + y) * gi.W + x) * 3;
#pragma unroll
                for (int o = 0; o < 3; ++o) {
                    float e0, e1;
                    unpack2(acc[p][o], e0, e1);
                    float v = (e0 + e1) + b[o];
                    if (flags & WCTB200_CLIP01) v = fminf(fmaxf(v, 0.f), 1.f);
                    d[o] = v;
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------
// MaxPooling2D 2x2/2 'same' (vgg_normalised.py:41-42) and UpSampling2D x2 (model.py:293)
// ---------------------------------------------------------------------------
__global__ void k_maxpool2(const __half* __restrict__ in, ActGeom gi, __half* __restrict__ out) {
    const ActGeom go(gi.N, (gi.H + 1) / 2, (gi.W + 1) / 2, gi.C);
    const int cg = gi.C / 8;
    const long long total = (long long)go.N * go.H * go.W * cg;
    // 32-bit index arithmetic (launcher guarantees total < 2^32): 64-bit div/mod costs ~100 instructions each
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < (unsigned)total; i += gridDim.x * blockDim.x) {
        const int c0 = (int)(i % (unsigned)cg) * 8;
        unsigned pix = i / (unsigned)cg;
        const int x = (int)(pix % (unsigned)go.W); pix /= (unsigned)go.W;
        const int y = (int)(pix % (unsigned)go.H);
        const int n = (int)(pix / (unsigned)go.H);
        float m[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) m[j] = -3.0e38f;
        for (int dy = 0; dy < 2; ++dy) {
            const int yy = 2 * y + dy;
            if (yy >= gi.H) continue;               // 'same': window clipped at the bottom/right edge
            for (int dx = 0; dx < 2; ++dx) {
                const int xx = 2 * x + dx;
                if (xx >= gi.W) continue;
                float v[8];
                load8(in, gi, ((long long)n * gi.Hp + yy + 1) * gi.Wp + xx + 1, c0, v);
#pragma unroll
                for (int j = 0; j < 8; ++j) m[j] = fmaxf(m[j], v[j]);
            }
        }
        Half8 hi, lo;
        split8(m, hi, lo);
        store8_with_halo(out, go, n, y, x, c0, hi, lo);
    }
}

__global__ void k_upsample2(const __half* __restrict__ in, ActGeom gi, __half* __restrict__ out) {
    const ActGeom go(gi.N, gi.H * 2, gi.W * 2, gi.C);
    const int cg = gi.C / 8;
    const long long total = (long long)go.N * go.H * go.W * cg;
    // 32-bit index arithmetic (launcher guarantees total < 2^32): 64-bit div/mod costs ~100 instructions each
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < (unsigned)total; i += gridDim.x * blockDim.x) {
        const int c0 = (int)(i % (unsigned)cg) * 8;
        unsigned pix = i / (unsigned)cg;
        const int x = (int)(pix % (unsigned)go.W); pix /= (unsigned)go.W;
        const int y = (int)(pix % (unsigned)go.H);
        const int n = (int)(pix / (unsigned)go.H);
        const long long off = (((long long)n * gi.Hp + (y >> 1) + 1) * gi.Wp + (x >> 1) + 1) * gi.C + c0;
        const Half8 hi = *reinterpret_cast<const Half8*>(in + off);
        const Half8 lo = *reinterpret_cast<const Half8*>(in + gi.plane + off);
        store8_with_halo(out, go, n, y, x, c0, hi, lo);
    }
}

// ---------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------
static inline int grid_for(long long total, int block) {
    long long b = (total + block - 1) / block;
    const long long cap = (long long)device_sm_count() * 16;
    return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

int launch_u8_to_f32(const uint8_t* in, size_t n, float* out, cudaStream_t st) {
    k_u8_to_f32<<<grid_for((long long)n, 256), 256, 0, st>>>(in, n, out);
    WCTB_CHECK_LAUNCH("k_u8_to_f32");
    return 0;
}
int launch_f32_to_u8(const float* in, size_t n, uint8_t* out, cudaStream_t st) {
    k_f32_to_u8<<<grid_for((long long)n, 256), 256, 0, st>>>(in, n, out);
    WCTB_CHECK_LAUNCH("k_f32_to_u8");
    return 0;
}
int launch_act_from_f32(const float* in, ActGeom g, __half* act, cudaStream_t st) {
    k_act_from_f32<<<grid_for((long long)g.N * g.H * g.W * (g.C / 8), 256), 256, 0, st>>>(in, g, act);
    WCTB_CHECK_LAUNCH("k_act_from_f32");
    return 0;
}
int launch_act_halo(__half* act, ActGeom g, cudaStream_t st) {
    k_act_halo<<<grid_for((long long)g.N * (2ll * g.Wp + 2ll * g.H) * (g.C / 8), 256), 256, 0, st>>>(act, g);
    WCTB_CHECK_LAUNCH("k_act_halo");
    return 0;
}
int launch_act_to_f32(const __half* act, ActGeom g, float* out, cudaStream_t st) {
    k_act_to_f32<<<grid_for((long long)g.N * g.H * g.W * (g.C / 8), 256), 256, 0, st>>>(act, g, out);
    WCTB_CHECK_LAUNCH("k_act_to_f32");
    return 0;
}
int launch_prep_weights(const float* w, int taps, int Cin, int Cout, __half* ws, cudaStream_t st) {
    float* trailer = const_cast<float*>(weight_scale_ptr(ws, taps, Cin, Cout));
    WCTB_CUDA(cudaMemsetAsync(trailer, 0, 256, st));
    const long long n = (long long)taps * Cin * Cout;
    k_absmax<<<grid_for(n, 256), 256, 0, st>>>(w, n, reinterpret_cast<unsigned int*>(trailer) + 1);
    WCTB_CHECK_LAUNCH("k_absmax");
    k_prep_weights<<<grid_for(n, 256), 256, 0, st>>>(w, taps, Cin, Cout, ws, trailer);
    WCTB_CHECK_LAUNCH("k_prep_weights");
    return 0;
}
int launch_prep_weights_up2(const float* w, int Cin, int Cout, __half* ws, cudaStream_t st) {
    float* trailer = const_cast<float*>(weight_scale_ptr(ws, 16, Cin, Cout));
    WCTB_CUDA(cudaMemsetAsync(trailer, 0, 256, st));
    const long long n = 9ll * Cin * Cout;
    k_absmax<<<grid_for(n, 256), 256, 0, st>>>(w, n, reinterpret_cast<unsigned int*>(trailer) + 1);
    WCTB_CHECK_LAUNCH("k_absmax");
    k_prep_weights_up2<<<grid_for(16ll * Cin * Cout, 256), 256, 0, st>>>(w, Cin, Cout, ws, trailer);
    WCTB_CHECK_LAUNCH("k_prep_weights_up2");
    return 0;
}
int launch_conv3x3_ref(const __half* in, ActGeom gi, const float* w, const float* bias, int Cout, int flags,
                       __half* out, cudaStream_t st) {
    k_conv3x3_ref<<<grid_for((long long)gi.N * gi.H * gi.W * Cout, 256), 256, 0, st>>>(in, gi, w, bias, Cout, flags, out);
    WCTB_CHECK_LAUNCH("k_conv3x3_ref");
    return 0;
}
int launch_conv_head_tc(const float* img, int N, int H, int W, const float* w, const float* b, int flags, __half* out,
                        cudaStream_t st);
int launch_conv_head(const float* img, int N, int H, int W, const float* w, const float* b, int flags, __half* out,
                     cudaStream_t st) {
    {
        const int rc = launch_conv_head_tc(img, N, H, W, w, b, flags, out, st);      // tensor-core head (conv_head_tc.cu)
        if (rc <= 0) return rc;
    }
    k_conv_head<<<grid_for((long long)N * H * ((W + 3) / 4) * 8, 256), 256, 0, st>>>(img, N, H, W, w, b, flags, out);
    WCTB_CHECK_LAUNCH("k_conv_head");
    return 0;
}
int g_conv_tail_impl = 2;      // 1 = per-pixel kernel, 2 = shared-memory tiles (default for images >= 32x32)
int launch_conv_tail_tc(const __half* in, ActGeom gi, const float* w, const float* b, int flags, float* img, cudaStream_t st);
int launch_conv_tail(const __half* in, ActGeom gi, const float* w, const float* b, int flags, float* img, cudaStream_t st) {
    {
        const int rc = launch_conv_tail_tc(in, gi, w, b, flags, img, st);     // 64-channel tail on the tensor cores (conv_tail_tc.cu)
        if (rc <= 0) return rc;
    }
    if (g_conv_tail_impl == 2 && gi.C % TT_CH == 0 && gi.H >= TT_H && gi.W >= TT_W && gi.C <= 128) {
        const size_t tsmem = ((size_t)TT_ACT_F4 + TT_STAGE_F4 + (size_t)9 * (gi.C / 4) * 3) * sizeof(float4);
        constexpr size_t tsmem_max = ((size_t)TT_ACT_F4 + TT_STAGE_F4 + (size_t)9 * (128 / 4) * 3) * sizeof(float4);   // C = 128
        WCTB_ENSURE_SMEM(k_conv_tail_tiled, tsmem_max);
        const int tiles_x = (gi.W + TT_W - 1) / TT_W, tiles_y = (gi.H + TT_H - 1) / TT_H;
        k_conv_tail_tiled<<<(unsigned)(gi.N * tiles_x * tiles_y), 128, tsmem, st>>>(in, gi, w, b, flags, img, tiles_x, tiles_y);
        WCTB_CHECK_LAUNCH("k_conv_tail_tiled");
        return 0;
    }
    const size_t smem = (size_t)9 * gi.C * 3 * sizeof(float);
    k_conv_tail<<<grid_for((long long)gi.N * gi.H * ((gi.W + 3) / 4) * 8, 256), 256, smem, st>>>(in, gi, w, b, flags, img);
    WCTB_CHECK_LAUNCH("k_conv_tail");
    return 0;
}
int launch_maxpool2(const __half* in, ActGeom gi, __half* out, cudaStream_t st) {
    const long long total = (long long)gi.N * ((gi.H + 1) / 2) * ((gi.W + 1) / 2) * (gi.C / 8);
    k_maxpool2<<<grid_for(total, 256), 256, 0, st>>>(in, gi, out);
    WCTB_CHECK_LAUNCH("k_maxpool2");
    return 0;
}
int launch_upsample2(const __half* in, ActGeom gi, __half* out, cudaStream_t st) {
    const long long total = (long long)gi.N * gi.H * 2 * gi.W * 2 * (gi.C / 8);
    k_upsample2<<<grid_for(total, 256), 256, 0, st>>>(in, gi, out);
    WCTB_CHECK_LAUNCH("k_upsample2");
    return 0;
}

}  // namespace wctb
