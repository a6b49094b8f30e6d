// Image pre/post steps of the CLI on the device (scope row 8f-3): short-side / arbitrary bilinear resize with an optional
// crop window, and the pixel-sized parts of --keep-colors (CORAL).
//
//   reference: utils.resize_to / center_crop / center_crop_to (utils.py:29-67) -> scipy.misc.imresize(interp='bilinear')
//              = Pillow's ImagingResample on the uint8 image; utils.preserve_colors_np (utils.py:87-90) ->
//              coral.coral_numpy (coral.py:13-39).
//
// Resize.  Bit-exact with Pillow's 8-bit path (src/libImaging/Resample.c): a separable triangle filter whose support is
// max(1, in/out) input pixels, coefficients computed in double precision, normalised by their sum, converted to 22-bit fixed
// point; the HORIZONTAL pass runs first and rounds to uint8, the vertical pass follows.  The double-precision coefficient
// arithmetic uses the explicit round-to-nearest intrinsics so that ptxas cannot contract it into FMAs (x86 Pillow builds do
// not).  This is byte/integer work bound by HBM: one thread per output pixel, the (<= ksize) taps of a pixel are contiguous
// in the input row (horizontal) or a strided column walk that neighbouring threads coalesce (vertical).
//
// Luminance-only transfer.  The same nine sums per frame give each frame's exact luminance moments on the host; two
// per-pixel maps (match: RGB -> a grey of given mean and scale; merge: add a luminance difference to all three channels)
// run before and after the stylisation.
//
// CORAL.  The pixel-sized work is (i) nine integer sums per image (sum x_c, sum x_c x_d -- exact in uint64) and (ii) the
// per-pixel affine map out = (A ((x/255 - m_s) / s_s)) * s_t + m_t in double precision followed by the reference's
// clip / *255 / truncation.  The 3x3 algebra in between (matSqrt through numpy's SVD, whose sign conventions the
// reference's non-symmetric U sqrt(D) U depends on) stays on the host in wct_tf_b200/device_image.py.
//
// Noise (texture synthesis; reference: webcam.py:191-192 np.random.randint(0, 256, shape, np.uint8)).  Counter-based:
// 16-byte block b of absolute frame f is Philox4x32-10(counter (b_lo, b_hi, f_lo, f_hi), key (seed_lo, seed_hi)), so every
// byte is a pure function of (seed, f, position) whatever the launch shape or batch split.  Bound by its writes.
#include "common.cuh"

namespace wctb {

static constexpr int RS_PRECISION_BITS = 32 - 8 - 2;
static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

__device__ __forceinline__ double tri_filter(double x) {
    if (x < 0.0) x = -x;
    return x < 1.0 ? __dsub_rn(1.0, x) : 0.0;
}

// precompute_coeffs + normalize_coeffs_8bpc (Resample.c) for the box [0, in_size): bounds[xx] = (xmin, count),
// kk[xx][ksize] fixed-point weights.
__global__ void k_resample_coeffs(int in_size, int out_size, int ksize, int* __restrict__ bounds, int* __restrict__ kk) {
    const int xx = blockIdx.x * blockDim.x + threadIdx.x;
    if (xx >= out_size) return;
    const double scale = __ddiv_rn((double)in_size, (double)out_size);
    const double filterscale = scale < 1.0 ? 1.0 : scale;
    const double support = filterscale;                     // BILINEAR.support = 1.0
    const double ss = __ddiv_rn(1.0, filterscale);
    const double center = __dmul_rn(__dadd_rn((double)xx, 0.5), scale);
    int xmin = (int)__dadd_rn(__dsub_rn(center, support), 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)__dadd_rn(__dadd_rn(center, support), 0.5);
    if (xmax > in_size) xmax = in_size;
    xmax -= xmin;
    if (xmax > ksize) xmax = ksize;                         // cannot happen (ksize = 2 ceil(support) + 1); keeps the table in bounds
    double ww = 0.0;
    for (int x = 0; x < xmax; ++x) {
        const double w = tri_filter(__dmul_rn(__dadd_rn(__dsub_rn((double)(x + xmin), center), 0.5), ss));
        ww = __dadd_rn(ww, w);
    }
    int* k = kk + (long long)xx * ksize;
    for (int x = 0; x < xmax; ++x) {
        double w = tri_filter(__dmul_rn(__dadd_rn(__dsub_rn((double)(x + xmin), center), 0.5), ss));
        if (ww != 0.0) w = __ddiv_rn(w, ww);
        const double kf = __dmul_rn(w, (double)(1 << RS_PRECISION_BITS));
        k[x] = (int)(kf < 0.0 ? __dadd_rn(-0.5, kf) : __dadd_rn(0.5, kf));
    }
    for (int x = xmax; x < ksize; ++x) k[x] = 0;
    bounds[2 * xx] = xmin;
    bounds[2 * xx + 1] = xmax;
}

__device__ __forceinline__ uint8_t clip8(int v) {
    v >>= RS_PRECISION_BITS;
    return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// One pass along `axis_stride`: out[n][o][i] = sum_t in[n][(xmin_o + t)][i] * k_o[t] for the output window
// o in [o0, o0 + n_out); the other axis is walked as-is.  in: [N][in_len][row] (horizontal: a row is C bytes and the lines
// are the image rows; vertical: a "row" is Wout*C bytes).
//   horizontal: thread = (line y, output column xx, channel c):  in index  (y*Win + x)*C + c
//   vertical  : thread = (output row yy, byte j of the row)    :  in index  y*rowbytes + j
template <bool HORIZONTAL>
__global__ void k_resample_pass(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, const int* __restrict__ bounds,
                                const int* __restrict__ kk, int ksize, int N, int lines, int in_len, int o0, int n_out, int C) {
    // horizontal: lines = image rows, in_len = input width, output [N][lines][n_out][C]
    // vertical  : lines = bytes per row (W*C),  in_len = input height, output [N][n_out][lines]
    const long long total = (long long)N * lines * n_out * (HORIZONTAL ? C : 1);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        int o, c = 0;
        long long base;                                        // byte offset of tap 0 in `in`
        int step;
        if (HORIZONTAL) {
            c = (int)(i % C);
            const long long r = i / C;
            o = (int)(r % n_out);
            const long long ln = r / n_out;                    // n*lines + y
            const int xmin = bounds[2 * (o0 + o)];
            base = (ln * in_len + xmin) * C + c;
            step = C;
        } else {
            const int j = (int)(i % lines);
            const long long r = i / lines;
            o = (int)(r % n_out);
            const long long n = r / n_out;
            const int ymin = bounds[2 * (o0 + o)];
            base = (n * in_len + ymin) * lines + j;
            step = lines;
        }
        const int cnt = bounds[2 * (o0 + o) + 1];
        const int* k = kk + (long long)(o0 + o) * ksize;
        int acc = 1 << (RS_PRECISION_BITS - 1);
        for (int t = 0; t < cnt; ++t) acc += (int)in[base + (long long)t * step] * __ldg(k + t);
        out[i] = clip8(acc);
    }
}

__global__ void k_crop_u8(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int N, int H, int W, int C, int y0, int x0,
                          int Ho, int Wo) {
    const long long total = (long long)N * Ho * Wo * C;
    const int rowb = Wo * C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int j = (int)(i % rowb);
        const long long r = i / rowb;
        const int y = (int)(r % Ho);
        const long long n = r / Ho;
        out[i] = in[((n * H + y0 + y) * W + x0) * C + j];
    }
}

static int grid_for(long long total, int block) {
    long long g = (total + block - 1) / block;
    const long long cap = (long long)device_sm_count() * 16;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

static int resample_ksize(int in_size, int out_size) {
    double scale = (double)in_size / (double)out_size;
    if (scale < 1.0) scale = 1.0;
    return (int)ceil(scale) * 2 + 1;
}

struct ResizeWs {
    size_t bx, kx, by, ky, tmp, total;
    int ksx, ksy;
};
static ResizeWs resize_layout(int N, int Hs, int Ws, int C, int Hd, int Wd, int Wout) {
    ResizeWs L;
    L.ksx = resample_ksize(Ws, Wd);
    L.ksy = resample_ksize(Hs, Hd);
    size_t o = 0;
    L.bx = o; o = align_up(o + (size_t)Wd * 2 * 4, 256);
    L.kx = o; o = align_up(o + (size_t)Wd * L.ksx * 4, 256);
    L.by = o; o = align_up(o + (size_t)Hd * 2 * 4, 256);
    L.ky = o; o = align_up(o + (size_t)Hd * L.ksy * 4, 256);
    L.tmp = o; o = align_up(o + (size_t)N * Hs * Wout * C, 256);
    L.total = o;
    return L;
}
size_t resize_workspace_bytes(int N, int Hs, int Ws, int C, int Hd, int Wd, int Wout) {
    return resize_layout(N, Hs, Ws, C, Hd, Wd, Wout).total;
}

// src [N][Hs][Ws][C] -> the window [y0, y0+Hout) x [x0, x0+Wout) of the Hd x Wd resample, dst [N][Hout][Wout][C]
int launch_resize_u8(const uint8_t* src, int N, int Hs, int Ws, int C, int Hd, int Wd, int y0, int x0, int Hout, int Wout,
                     uint8_t* dst, void* ws, size_t ws_bytes, cudaStream_t st) {
    const ResizeWs L = resize_layout(N, Hs, Ws, C, Hd, Wd, Wout);
    if (ws_bytes < L.total) {
        set_error("resize: workspace %zu < %zu bytes", ws_bytes, L.total);
        return WCTB200_EWS;
    }
    uint8_t* w = static_cast<uint8_t*>(ws);
    int* bx = reinterpret_cast<int*>(w + L.bx);
    int* kx = reinterpret_cast<int*>(w + L.kx);
    int* by = reinterpret_cast<int*>(w + L.by);
    int* ky = reinterpret_cast<int*>(w + L.ky);
    uint8_t* tmp = w + L.tmp;
    const bool need_h = Wd != Ws, need_v = Hd != Hs;      // Resample.c ImagingResampleInner: a pass runs only when its size changes
    if (!need_h && !need_v) {
        k_crop_u8<<<grid_for((long long)N * Hout * Wout * C, 256), 256, 0, st>>>(src, dst, N, Hs, Ws, C, y0, x0, Hout, Wout);
        WCTB_CHECK_LAUNCH("k_crop_u8");
        return 0;
    }
    const uint8_t* vin = src;      // input of the vertical pass: [N][Hs][vW][C]
    int vW = Ws;
    if (need_h) {
        k_resample_coeffs<<<cdiv(Wd, 128), 128, 0, st>>>(Ws, Wd, L.ksx, bx, kx);
        WCTB_CHECK_LAUNCH("k_resample_coeffs(x)");
        uint8_t* hout = need_v ? tmp : dst;
        if (!need_v && (y0 != 0 || Hout != Hs)) hout = tmp;
        k_resample_pass<true><<<grid_for((long long)N * Hs * Wout * C, 256), 256, 0, st>>>(src, hout, bx, kx, L.ksx, N, Hs, Ws, x0,
                                                                                           Wout, C);
        WCTB_CHECK_LAUNCH("k_resample_pass(h)");
        if (!need_v) {
            if (hout == tmp) {
                k_crop_u8<<<grid_for((long long)N * Hout * Wout * C, 256), 256, 0, st>>>(tmp, dst, N, Hs, Wout, C, y0, 0, Hout, Wout);
                WCTB_CHECK_LAUNCH("k_crop_u8");
            }
            return 0;
        }
        vin = tmp;
        vW = Wout;
    } else if (x0 != 0 || Wout != Ws) {
        // vertical pass only, with a column window: crop the columns first
        k_crop_u8<<<grid_for((long long)N * Hs * Wout * C, 256), 256, 0, st>>>(src, tmp, N, Hs, Ws, C, 0, x0, Hs, Wout);
        WCTB_CHECK_LAUNCH("k_crop_u8");
        vin = tmp;
        vW = Wout;
    }
    k_resample_coeffs<<<cdiv(Hd, 128), 128, 0, st>>>(Hs, Hd, L.ksy, by, ky);
    WCTB_CHECK_LAUNCH("k_resample_coeffs(y)");
    k_resample_pass<false><<<grid_for((long long)N * Hout * vW * C, 256), 256, 0, st>>>(vin, dst, by, ky, L.ksy, N, vW * C, Hs, y0,
                                                                                        Hout, 1);
    WCTB_CHECK_LAUNCH("k_resample_pass(v)");
    return 0;
}

// ---------------------------------------------------------------------------
// CORAL
// ---------------------------------------------------------------------------
// Frame n (blockIdx.y, striding by gridDim.y) of N: sums[n][0..2] = sum x_c, sums[n][3..8] = sum x_0x_0, x_0x_1, x_0x_2,
// x_1x_1, x_1x_2, x_2x_2 over its npf pixels (exact integers)
__global__ void k_rgb_moments(const uint8_t* __restrict__ img, int N, long long npf, unsigned long long* __restrict__ sums) {
    for (int n = blockIdx.y; n < N; n += gridDim.y) {
        const uint8_t* f = img + (long long)n * npf * 3;
        unsigned long long s[9];
#pragma unroll
        for (int i = 0; i < 9; ++i) s[i] = 0ull;
        for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < npf; p += (long long)gridDim.x * blockDim.x) {
            const unsigned int a = f[3 * p], b = f[3 * p + 1], c = f[3 * p + 2];
            s[0] += a; s[1] += b; s[2] += c;
            s[3] += a * a; s[4] += a * b; s[5] += a * c;
            s[6] += b * b; s[7] += b * c; s[8] += c * c;
        }
#pragma unroll
        for (int i = 0; i < 9; ++i) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s[i] += __shfl_xor_sync(0xffffffffu, s[i], o);
        }
        if ((threadIdx.x & 31) == 0) {
#pragma unroll
            for (int i = 0; i < 9; ++i) atomicAdd(sums + 9ll * n + i, s[i]);     // integer: order-independent, deterministic
        }
    }
}

struct CoralParams {
    double A[9], sm[3], ss[3], ts[3], tm[3];
};

// out = uint8(clip((A ((x/255 - sm)/ss)) * ts + tm, 0, 1) * 255)    coral.py:24,35-36 + utils.py:88-89, in double like NumPy
__global__ void k_coral_apply(const uint8_t* __restrict__ src, long long npix, const CoralParams P, uint8_t* __restrict__ dst) {
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < npix; p += (long long)gridDim.x * blockDim.x) {
        double sn[3];
#pragma unroll
        for (int j = 0; j < 3; ++j)
            sn[j] = __ddiv_rn(__dsub_rn(__ddiv_rn((double)src[3 * p + j], 255.0), P.sm[j]), P.ss[j]);
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            double v = __dmul_rn(P.A[3 * i], sn[0]);
            v = fma(P.A[3 * i + 1], sn[1], v);
            v = fma(P.A[3 * i + 2], sn[2], v);
            v = __dadd_rn(__dmul_rn(v, P.ts[i]), P.tm[i]);
            v = v < 0.0 ? 0.0 : (v > 1.0 ? 1.0 : v);
            dst[3 * p + i] = (uint8_t)(int)__dmul_rn(v, 255.0);
        }
    }
}

// Per-frame launches of the frame-axis kernels: frames on y, and the pixels of a frame on x with the grid_for budget shared
// between the frames of a batch (a 30-frame batch of 512^2 frames gets ~70 blocks per frame, not 1024).
static dim3 frames_grid(int N, long long npf, int block) {
    const int ny = N < 65535 ? N : 65535;
    long long gx = (npf + block - 1) / block;
    const long long cap = (long long)device_sm_count() * 16 / ny;
    if (gx > cap) gx = cap;
    return dim3((unsigned)(gx < 1 ? 1 : gx), (unsigned)ny);
}

int launch_rgb_moments_batch(const uint8_t* img, int N, long long npf, unsigned long long* sums, cudaStream_t st) {
    WCTB_CUDA(cudaMemsetAsync(sums, 0, 9ull * N * sizeof(unsigned long long), st));
    k_rgb_moments<<<frames_grid(N, npf, 256), 256, 0, st>>>(img, N, npf, sums);
    WCTB_CHECK_LAUNCH("k_rgb_moments");
    return 0;
}

int launch_rgb_moments(const uint8_t* img, long long npix, unsigned long long* sums, cudaStream_t st) {
    return launch_rgb_moments_batch(img, 1, npix, sums, st);
}

int launch_coral_apply(const uint8_t* src, long long npix, const double* A, const double* sm, const double* ss, const double* tm,
                       const double* ts, uint8_t* dst, cudaStream_t st) {
    CoralParams P;
    for (int i = 0; i < 9; ++i) P.A[i] = A[i];
    for (int i = 0; i < 3; ++i) {
        P.sm[i] = sm[i];
        P.ss[i] = ss[i];
        P.tm[i] = tm[i];
        P.ts[i] = ts[i];
    }
    k_coral_apply<<<grid_for(npix, 256), 256, 0, st>>>(src, npix, P, dst);
    WCTB_CHECK_LAUNCH("k_coral_apply");
    return 0;
}

// ---------------------------------------------------------------------------
// Luminance-only transfer (DESIGN.md §3.3.15)
// ---------------------------------------------------------------------------
// Y = (299 R + 587 G + 114 B) / 1000: the integer numerator is exact and below 2^24, so Y is one correctly rounded fp32
// division.  Every step below is an explicitly rounded fp32 operation in a fixed order, so a frame's bytes depend on its
// pixels and its (k, b) only, never on N or the launch shape.
__device__ __forceinline__ float luma_bt601(const uint8_t* p) {
    return __fdiv_rn((float)(299 * (int)p[0] + 587 * (int)p[1] + 114 * (int)p[2]), 1000.0f);
}

__device__ __forceinline__ uint8_t round_clip8(float v) {
    v = rintf(v);                                            // half to even, as numpy's rint
    return (uint8_t)(v < 0.0f ? 0.0f : (v > 255.0f ? 255.0f : v));
}

// dst[n][p] = replicated clip(rint(k_n Y + b_n)), kb[n] = (k_n, b_n)
__global__ void k_luma_match_u8(const uint8_t* __restrict__ src, int N, long long npf, const float2* __restrict__ kb,
                                uint8_t* __restrict__ dst) {
    for (int n = blockIdx.y; n < N; n += gridDim.y) {
        const float2 q = kb[n];
        const long long base = (long long)n * npf * 3;
        for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < npf; p += (long long)gridDim.x * blockDim.x) {
            const long long o = base + 3 * p;
            const uint8_t g = round_clip8(__fmaf_rn(q.x, luma_bt601(src + o), q.y));
            dst[o] = g; dst[o + 1] = g; dst[o + 2] = g;
        }
    }
}

// dst[n][p][c] = clip(rint(content_c + ((kinv_n Y_S + b_n) - Y_content))), kb[n] = (kinv_n, b_n)
__global__ void k_luma_merge_u8(const uint8_t* __restrict__ content, const uint8_t* __restrict__ styl, int N, long long npf,
                                const float2* __restrict__ kb, uint8_t* __restrict__ dst) {
    for (int n = blockIdx.y; n < N; n += gridDim.y) {
        const float2 q = kb[n];
        const long long base = (long long)n * npf * 3;
        for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < npf; p += (long long)gridDim.x * blockDim.x) {
            const long long o = base + 3 * p;
            const float d = __fsub_rn(__fmaf_rn(q.x, luma_bt601(styl + o), q.y), luma_bt601(content + o));
#pragma unroll
            for (int c = 0; c < 3; ++c) dst[o + c] = round_clip8(__fadd_rn((float)content[o + c], d));
        }
    }
}

int launch_luma_match(const uint8_t* src, int N, long long npf, const float* kb, uint8_t* dst, cudaStream_t st) {
    k_luma_match_u8<<<frames_grid(N, npf, 256), 256, 0, st>>>(src, N, npf, reinterpret_cast<const float2*>(kb), dst);
    WCTB_CHECK_LAUNCH("k_luma_match_u8");
    return 0;
}

int launch_luma_merge(const uint8_t* content, const uint8_t* styl, int N, long long npf, const float* kb, uint8_t* dst,
                      cudaStream_t st) {
    k_luma_merge_u8<<<frames_grid(N, npf, 256), 256, 0, st>>>(content, styl, N, npf, reinterpret_cast<const float2*>(kb), dst);
    WCTB_CHECK_LAUNCH("k_luma_merge_u8");
    return 0;
}

// ---------------------------------------------------------------------------
// Coarse-to-fine join (DESIGN.md §3.3.16)
// ---------------------------------------------------------------------------
// One bilinear axis of the join: output coordinate i of n maps to source s = (i + 0.5) sc - 0.5 clamped to [0, m - 1],
// taps i0 = floor(s) and i1 = min(i0 + 1, m - 1), weight s - i0.  Explicitly rounded fp32, as the NumPy oracle computes it.
__device__ __forceinline__ void join_taps(int i, float sc, int m, int& i0, int& i1, float& wt) {
    float s = __fsub_rn(__fmul_rn(__fadd_rn((float)i, 0.5f), sc), 0.5f);
    s = fminf(fmaxf(s, 0.0f), (float)(m - 1));
    i0 = (int)s;                                              // s >= 0: truncation is floor
    i1 = i0 + 1 < m ? i0 + 1 : m - 1;
    wt = __fsub_rn(s, (float)i0);
}

// dst = clip(rint(C + U(S - D))): the content with its low band (D, the coarse content) replaced by the stylised low band
// (S), U the bilinear upsampling from h x w to H x W.  Rows of the N H output rows on y (striding by gridDim.y), columns on
// x: a warp reads and writes 32 consecutive pixels of one row, and its low-resolution taps are a few pixels of two coarse
// rows, served by L1 / L2.  Every operation is a rounded fp32 add / sub / mul in a fixed order, so frame n's bytes depend on
// its own pixels only.
__global__ void k_coarse_join_u8(const uint8_t* __restrict__ content, const uint8_t* __restrict__ coarse,
                                 const uint8_t* __restrict__ styl, int N, int H, int W, int h, int w, uint8_t* __restrict__ dst) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= W) return;
    int x0, x1;
    float wx;
    join_taps(x, __fdiv_rn((float)w, (float)W), w, x0, x1, wx);
    const float sy = __fdiv_rn((float)h, (float)H);
    const long long rows = (long long)N * H;
    for (long long r = blockIdx.y; r < rows; r += gridDim.y) {
        const long long n = r / H;
        const int y = (int)(r - n * H);
        int y0, y1;
        float wy;
        join_taps(y, sy, h, y0, y1, wy);
        const long long q0 = (n * h + y0) * w, q1 = (n * h + y1) * w;
        const long long t00 = 3 * (q0 + x0), t01 = 3 * (q0 + x1), t10 = 3 * (q1 + x0), t11 = 3 * (q1 + x1);
        const long long o = 3 * (r * W + x);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float d00 = __fsub_rn((float)styl[t00 + c], (float)coarse[t00 + c]);
            const float d01 = __fsub_rn((float)styl[t01 + c], (float)coarse[t01 + c]);
            const float d10 = __fsub_rn((float)styl[t10 + c], (float)coarse[t10 + c]);
            const float d11 = __fsub_rn((float)styl[t11 + c], (float)coarse[t11 + c]);
            const float a = __fadd_rn(d00, __fmul_rn(wx, __fsub_rn(d01, d00)));
            const float b = __fadd_rn(d10, __fmul_rn(wx, __fsub_rn(d11, d10)));
            const float v = __fadd_rn(a, __fmul_rn(wy, __fsub_rn(b, a)));
            dst[o + c] = round_clip8(__fadd_rn((float)content[o + c], v));
        }
    }
}

int launch_coarse_join(const uint8_t* content, const uint8_t* coarse, const uint8_t* styl, int N, int H, int W, int h, int w,
                       uint8_t* dst, cudaStream_t st) {
    const int block = 128;
    const int gx = cdiv(W, block);
    const long long rows = (long long)N * H;
    long long gy = (long long)device_sm_count() * 32 / gx;   // enough resident blocks to cover HBM latency; rows loop
    if (gy > rows) gy = rows;
    if (gy > 65535) gy = 65535;
    if (gy < 1) gy = 1;
    k_coarse_join_u8<<<dim3((unsigned)gx, (unsigned)gy), block, 0, st>>>(content, coarse, styl, N, H, W, h, w, dst);
    WCTB_CHECK_LAUNCH("k_coarse_join_u8");
    return 0;
}

// ---------------------------------------------------------------------------
// Noise
// ---------------------------------------------------------------------------
// Philox4x32-10 (Salmon et al., SC'11; the Random123 constants)
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, unsigned int k0, unsigned int k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const unsigned int hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
        const unsigned int hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
        c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    return c;
}

// One thread per 16-byte block of a frame (frame_bytes = H*W*C).  A frame starts at out + n*frame_bytes, so its blocks share
// one alignment: 16-byte stores where that is 16-aligned, four 4-byte stores where it is 4-aligned, bytes otherwise and for
// the truncated last block of a frame.
__global__ void k_noise_u8(uint8_t* __restrict__ out, long long N, long long frame_bytes, long long blocks_per_frame,
                           unsigned int k0, unsigned int k1, unsigned long long first_index) {
    const long long total = N * blocks_per_frame;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long n = i / blocks_per_frame;
        const unsigned long long b = (unsigned long long)(i - n * blocks_per_frame);
        const unsigned long long f = first_index + (unsigned long long)n;
        const uint4 x = philox4x32_10(make_uint4((unsigned int)b, (unsigned int)(b >> 32), (unsigned int)f, (unsigned int)(f >> 32)),
                                      k0, k1);
        uint8_t* p = out + n * frame_bytes + (long long)b * 16;
        const long long left = frame_bytes - (long long)b * 16;
        const uintptr_t a = reinterpret_cast<uintptr_t>(p);
        if (left >= 16 && (a & 15) == 0) {
            *reinterpret_cast<uint4*>(p) = x;
        } else if (left >= 16 && (a & 3) == 0) {
            unsigned int* q = reinterpret_cast<unsigned int*>(p);
            q[0] = x.x; q[1] = x.y; q[2] = x.z; q[3] = x.w;
        } else {
            const int m = left < 16 ? (int)left : 16;
#pragma unroll
            for (int j = 0; j < 16; ++j)
                if (j < m) p[j] = (uint8_t)((j < 4 ? x.x : j < 8 ? x.y : j < 12 ? x.z : x.w) >> (8 * (j & 3)));
        }
    }
}

int launch_noise_u8(uint8_t* out, int N, long long frame_bytes, unsigned long long seed, long long first_index, cudaStream_t st) {
    const long long bpf = (frame_bytes + 15) / 16;
    k_noise_u8<<<grid_for((long long)N * bpf, 256), 256, 0, st>>>(out, N, frame_bytes, bpf, (unsigned int)seed,
                                                                   (unsigned int)(seed >> 32), (unsigned long long)first_index);
    WCTB_CHECK_LAUNCH("k_noise_u8");
    return 0;
}

}  // namespace wctb
