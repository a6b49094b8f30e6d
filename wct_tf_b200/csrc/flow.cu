// Temporal stabilisation of video (DESIGN.md §3.3.6): luminance of the content frames, coarse-to-fine Horn-Schunck optical
// flow with warping for both directions of every consecutive pair of a batch, the forward-backward / photometric
// confidence with the cut rule, and the recurrent uint8 blend O_t = round(P_t + beta c_t (O_{t-1}(x + w_b) - P_t)).
//
// Exactness.  tests/temporal_ref.py restates every kernel in float32 NumPy and the results agree bit for bit: every float
// operation is one explicitly rounded intrinsic (__fadd_rn / __fmul_rn / __fdiv_rn cannot be contracted into FMAs) issued
// in the order of the restatement.  The flow uses Jacobi iterations, so the result does not depend on the schedule.
//
// Flow layout: [P][2][H][W] (u = x displacement, v = y displacement), P = 2 (M - 1) problems for a stack of M luminance
// frames; problem 2t is the backward flow from frame t+1 to frame t (I0 = Y[t+1], I1 = Y[t]), problem 2t+1 the forward flow
// from frame t to frame t+1.  A flow w satisfies I1(x + w(x)) ~ I0(x).
//
// Hot path: the Jacobi stencil.  One launch runs JK iterations on a JT x JT output tile held in shared memory with a halo of
// JK pixels (temporal blocking): the level's flow and coefficients are read once and written once per JK iterations, and a
// warp's 30 iterations take 5 launches.
#include "common.cuh"

namespace wctb {

namespace tflow {
constexpr float HS_ALPHA2 = 0.0025f;    // alpha = 0.05 on luminance in [0, 1]
constexpr int MAX_LEVELS = 6;
constexpr int MIN_SIDE = 32;
constexpr int WARPS = 3;
constexpr int ITERS = 30;
constexpr float FB_A = 0.01f;
constexpr float FB_B = 0.25f;
constexpr float PHOTO_TAU = 0.05f;
constexpr int CUT_PERCENT = 50;
constexpr int JT = 32;                  // Jacobi output tile side
constexpr int JK = 6;                   // Jacobi iterations per launch = halo width
constexpr int JR = JT + 2 * JK;         // side of the tile with its halo
constexpr int JRR = JR * JR;
constexpr size_t JACOBI_SMEM = (size_t)8 * JRR * sizeof(float);
}  // namespace tflow
using namespace tflow;

static inline size_t flow_align(size_t v) { return (v + 255) / 256 * 256; }

__device__ __forceinline__ float lerp_rn(float a, float b, float f) { return __fadd_rn(a, __fmul_rn(f, __fsub_rn(b, a))); }

// bilinear sample of plane [h][w] (element stride `stride`) at (x, y), the coordinates clamped to the border
template <typename T>
__device__ __forceinline__ float sample_bl(const T* __restrict__ img, int stride, int h, int w, float x, float y) {
    x = fminf(fmaxf(x, 0.f), (float)(w - 1));
    y = fminf(fmaxf(y, 0.f), (float)(h - 1));
    const float x0 = floorf(x), y0 = floorf(y);
    const float fx = __fsub_rn(x, x0), fy = __fsub_rn(y, y0);
    const int ix0 = (int)x0, iy0 = (int)y0;
    const int ix1 = min(ix0 + 1, w - 1), iy1 = min(iy0 + 1, h - 1);
    const float a = (float)img[((long long)iy0 * w + ix0) * stride], b = (float)img[((long long)iy0 * w + ix1) * stride];
    const float c = (float)img[((long long)iy1 * w + ix0) * stride], d = (float)img[((long long)iy1 * w + ix1) * stride];
    return lerp_rn(lerp_rn(a, b, fx), lerp_rn(c, d, fx), fy);
}

static int flow_grid(long long total, int block) {
    long long g = (total + block - 1) / block;
    const long long cap = (long long)device_sm_count() * 16;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

// Y = (0.299 R + 0.587 G + 0.114 B) / 255
__global__ void k_luminance(const uint8_t* __restrict__ rgb, long long npix, float* __restrict__ Y) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (long long)gridDim.x * blockDim.x) {
        float t = __fmul_rn(0.299f, (float)rgb[3 * i]);
        t = __fadd_rn(t, __fmul_rn(0.587f, (float)rgb[3 * i + 1]));
        t = __fadd_rn(t, __fmul_rn(0.114f, (float)rgb[3 * i + 2]));
        Y[i] = __fdiv_rn(t, 255.f);
    }
}

// 2x2 box average, ceil sizes, edge replication: [M][h][w] -> [M][h2][w2]
__global__ void k_downsample(const float* __restrict__ in, int M, int h, int w, float* __restrict__ out, int h2, int w2) {
    const long long total = (long long)M * h2 * w2;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % w2);
        const long long r = i / w2;
        const int y = (int)(r % h2);
        const float* p = in + (r / h2) * h * w;
        const int ya = 2 * y, yb = min(2 * y + 1, h - 1), xa = 2 * x, xb = min(2 * x + 1, w - 1);
        const float s = __fadd_rn(__fadd_rn(p[ya * w + xa], p[ya * w + xb]), __fadd_rn(p[yb * w + xa], p[yb * w + xb]));
        out[i] = __fmul_rn(s, 0.25f);
    }
}

// flow planes [Q][hc][wc] -> [Q][h][w]: bilinear at the pixel centres, values x2
__global__ void k_upsample_flow(const float* __restrict__ coarse, int Q, int hc, int wc, float* __restrict__ fine, int h, int w) {
    const long long total = (long long)Q * h * w;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % w);
        const long long r = i / w;
        const int y = (int)(r % h);
        const long long q = r / h;
        const float sx = __fsub_rn(__fmul_rn(__fadd_rn((float)x, 0.5f), 0.5f), 0.5f);
        const float sy = __fsub_rn(__fmul_rn(__fadd_rn((float)y, 0.5f), 0.5f), 0.5f);
        fine[i] = __fmul_rn(sample_bl(coarse + q * hc * wc, 1, hc, wc, sx, sy), 2.f);
    }
}

// Linearisation of I1(x + w) - I0(x) around the current flow (u, v): coef [P][4][h][w] = (Ix, Iy, It - Ix u - Iy v, den)
__global__ void k_warp_coefs(const float* __restrict__ Y, int P, int h, int w, const float* __restrict__ flows,
                             float* __restrict__ coef) {
    const long long hw = (long long)h * w, total = (long long)P * hw;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long p = i / hw, j = i - p * hw;
        const int x = (int)(j % w), y = (int)(j / w);
        const long long t = p >> 1;
        const float* I0 = Y + (t + ((p & 1) ? 0 : 1)) * hw;
        const float* I1 = Y + (t + ((p & 1) ? 1 : 0)) * hw;
        const float u = flows[(2 * p) * hw + j], v = flows[(2 * p + 1) * hw + j];
        const float X = __fadd_rn((float)x, u), Yc = __fadd_rn((float)y, v);
        const float Iw = sample_bl(I1, 1, h, w, X, Yc);
        const float Ix = __fmul_rn(__fsub_rn(sample_bl(I1, 1, h, w, __fadd_rn(X, 1.f), Yc), sample_bl(I1, 1, h, w, __fsub_rn(X, 1.f), Yc)), 0.5f);
        const float Iy = __fmul_rn(__fsub_rn(sample_bl(I1, 1, h, w, X, __fadd_rn(Yc, 1.f)), sample_bl(I1, 1, h, w, X, __fsub_rn(Yc, 1.f))), 0.5f);
        const float It = __fsub_rn(__fsub_rn(__fsub_rn(Iw, I0[j]), __fmul_rn(Ix, u)), __fmul_rn(Iy, v));
        const float den = __fadd_rn(__fadd_rn(HS_ALPHA2, __fmul_rn(Ix, Ix)), __fmul_rn(Iy, Iy));
        float* c = coef + 4 * p * hw + j;
        c[0] = Ix;
        c[hw] = Iy;
        c[2 * hw] = It;
        c[3 * hw] = den;
    }
}

// `iters` (<= JK) Jacobi iterations u <- ubar - Ix (Ix ubar + Iy vbar + It) / den on one JT x JT tile of problem blockIdx.z.
// The tile and its JK-pixel halo are loaded once; iteration k updates the ring [k, JR - k) of the loaded square, whose
// neighbours iteration k - 1 produced, so after `iters` iterations the inner JT x JT values are exact.  ubar is the
// 4-neighbour mean with replicated image borders.
__global__ void __launch_bounds__(256) k_jacobi(const float* __restrict__ fin, float* __restrict__ fout,
                                                const float* __restrict__ coef, int h, int w, int iters) {
    extern __shared__ float sm[];
    // two flow buffers of 2 JRR floats (u at [0, JRR), v at [JRR, 2 JRR)), then the coefficients
    float* const six = sm + 4 * JRR;
    float* const siy = six + JRR;
    float* const sit = siy + JRR;
    float* const sden = sit + JRR;
    const long long hw = (long long)h * w;
    const long long p = blockIdx.z;
    const float* uin = fin + 2 * p * hw;
    const float* cf = coef + 4 * p * hw;
    const int gy0 = (int)blockIdx.y * JT - JK, gx0 = (int)blockIdx.x * JT - JK;
    for (int i = threadIdx.x; i < JRR; i += blockDim.x) {
        const int ry = i / JR, rx = i - ry * JR;
        const int gy = gy0 + ry, gx = gx0 + rx;
        if (gy < 0 || gy >= h || gx < 0 || gx >= w) continue;
        const long long g = (long long)gy * w + gx;
        sm[i] = uin[g];
        sm[JRR + i] = uin[hw + g];
        six[i] = cf[g];
        siy[i] = cf[hw + g];
        sit[i] = cf[2 * hw + g];
        sden[i] = cf[3 * hw + g];
    }
    __syncthreads();
    for (int k = 1; k <= iters; ++k) {
        const float* cu = sm + ((k - 1) & 1) * 2 * JRR;
        float* nu = sm + (k & 1) * 2 * JRR;
        for (int i = threadIdx.x; i < JRR; i += blockDim.x) {
            const int ry = i / JR, rx = i - ry * JR;
            if (ry < k || ry >= JR - k || rx < k || rx >= JR - k) continue;
            const int gy = gy0 + ry, gx = gx0 + rx;
            if (gy < 0 || gy >= h || gx < 0 || gx >= w) continue;
            const int up = gy > 0 ? i - JR : i, dn = gy < h - 1 ? i + JR : i;
            const int lf = gx > 0 ? i - 1 : i, rt = gx < w - 1 ? i + 1 : i;
            const float ub = __fmul_rn(__fadd_rn(__fadd_rn(cu[up], cu[dn]), __fadd_rn(cu[lf], cu[rt])), 0.25f);
            const float* cv = cu + JRR;
            const float vb = __fmul_rn(__fadd_rn(__fadd_rn(cv[up], cv[dn]), __fadd_rn(cv[lf], cv[rt])), 0.25f);
            const float ix = six[i], iy = siy[i];
            const float t = __fdiv_rn(__fadd_rn(__fadd_rn(__fmul_rn(ix, ub), __fmul_rn(iy, vb)), sit[i]), sden[i]);
            nu[i] = __fsub_rn(ub, __fmul_rn(ix, t));
            nu[JRR + i] = __fsub_rn(vb, __fmul_rn(iy, t));
        }
        __syncthreads();
    }
    const float* res = sm + (iters & 1) * 2 * JRR;
    float* uout = fout + 2 * p * hw;
    for (int i = threadIdx.x; i < JT * JT; i += blockDim.x) {
        const int ty = i / JT, tx = i - ty * JT;
        const int gy = gy0 + JK + ty, gx = gx0 + JK + tx;
        if (gy >= h || gx >= w) continue;
        const int l = (ty + JK) * JR + tx + JK;
        const long long g = (long long)gy * w + gx;
        uout[g] = res[l];
        uout[hw + g] = res[JRR + l];
    }
}

// Confidence of frame t+1 against frame t (pair t = blockIdx.y): inside the frame, forward-backward consistent, and
// photometrically consistent.  counts[t] += the confident pixels of the pair (counts zeroed by the caller).
__global__ void __launch_bounds__(256) k_confidence(const float* __restrict__ Y, int h, int w, const float* __restrict__ flows,
                                                    uint8_t* __restrict__ mask, int* __restrict__ counts) {
    const long long hw = (long long)h * w;
    const long long t = blockIdx.y;
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    int c = 0;
    if (j < hw) {
        const int x = (int)(j % w), y = (int)(j / w);
        const float* fb = flows + 4 * t * hw;                      // problem 2t
        const float* ff = fb + 2 * hw;                             // problem 2t + 1
        const float ub = fb[j], vb = fb[hw + j];
        const float px = __fadd_rn((float)x, ub), py = __fadd_rn((float)y, vb);
        const bool inside = px >= 0.f && px <= (float)(w - 1) && py >= 0.f && py <= (float)(h - 1);
        const float uf = sample_bl(ff, 1, h, w, px, py), vf = sample_bl(ff + hw, 1, h, w, px, py);
        const float dx = __fadd_rn(uf, ub), dy = __fadd_rn(vf, vb);
        const float lhs = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
        const float mag = __fadd_rn(__fadd_rn(__fmul_rn(uf, uf), __fmul_rn(vf, vf)), __fadd_rn(__fmul_rn(ub, ub), __fmul_rn(vb, vb)));
        const float rhs = __fadd_rn(__fmul_rn(FB_A, mag), FB_B);
        const float dY = fabsf(__fsub_rn(Y[(t + 1) * hw + j], sample_bl(Y + t * hw, 1, h, w, px, py)));
        c = (inside && lhs <= rhs && dY <= PHOTO_TAU) ? 1 : 0;
        mask[t * hw + j] = (uint8_t)c;
    }
    const int n = __syncthreads_count(c);
    if (threadIdx.x == 0 && n) atomicAdd(counts + t, n);
}

// the cut rule: a pair with fewer than CUT_PERCENT % confident pixels gets c = 0 everywhere
__global__ void k_cut(uint8_t* __restrict__ mask, long long pairs, long long hw, const int* __restrict__ counts) {
    const long long total = pairs * hw;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        if ((long long)counts[i / hw] * 100 < (long long)CUT_PERCENT * hw) mask[i] = 0;
    }
}

// one frame of the recurrence, in place: where c, cur = round(cur + beta (prev(x + w_b) - cur)) per channel
__global__ void k_blend(uint8_t* __restrict__ cur, const uint8_t* __restrict__ prev, const float* __restrict__ flow_b,
                        const uint8_t* __restrict__ mask, int h, int w, float beta) {
    const long long hw = (long long)h * w;
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < hw; j += (long long)gridDim.x * blockDim.x) {
        if (!mask[j]) continue;
        const int x = (int)(j % w), y = (int)(j / w);
        const float px = __fadd_rn((float)x, flow_b[j]), py = __fadd_rn((float)y, flow_b[hw + j]);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
            const float P = (float)cur[3 * j + ch];
            const float s = sample_bl(prev + ch, 3, h, w, px, py);
            const float v = floorf(__fadd_rn(__fadd_rn(P, __fmul_rn(beta, __fsub_rn(s, P))), 0.5f));
            cur[3 * j + ch] = (uint8_t)fminf(fmaxf(v, 0.f), 255.f);
        }
    }
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
struct FlowLayout {
    int L, h[MAX_LEVELS], w[MAX_LEVELS];
    size_t pyr[MAX_LEVELS], fa[MAX_LEVELS], fb[MAX_LEVELS], coef, total;
};

static FlowLayout flow_layout(int M, int H, int W) {
    FlowLayout F;
    F.L = 1;
    F.h[0] = H;
    F.w[0] = W;
    while (F.L < MAX_LEVELS) {
        const int h = (F.h[F.L - 1] + 1) / 2, w = (F.w[F.L - 1] + 1) / 2;
        if (h < MIN_SIDE || w < MIN_SIDE) break;
        F.h[F.L] = h;
        F.w[F.L] = w;
        ++F.L;
    }
    const size_t P = 2 * (size_t)(M - 1);
    size_t o = 0;
    for (int l = 0; l < F.L; ++l) {
        const size_t hw = (size_t)F.h[l] * F.w[l];
        F.pyr[l] = o;
        if (l > 0) o = flow_align(o + (size_t)M * hw * 4);
        F.fa[l] = o;
        if (l > 0) o = flow_align(o + P * 2 * hw * 4);
        F.fb[l] = o;
        o = flow_align(o + P * 2 * hw * 4);
    }
    F.coef = o;
    o = flow_align(o + P * 4 * (size_t)H * W * 4);
    F.total = o;
    return F;
}

size_t flow_pairs_workspace_bytes(int M, int H, int W) { return flow_layout(M, H, W).total; }

int launch_luminance(const uint8_t* rgb, long long npix, float* Y, cudaStream_t st) {
    k_luminance<<<flow_grid(npix, 256), 256, 0, st>>>(rgb, npix, Y);
    WCTB_CHECK_LAUNCH("k_luminance");
    return 0;
}

int launch_flow_pairs(const float* Y, int M, int H, int W, float* flows, void* ws, size_t ws_bytes, cudaStream_t st) {
    const FlowLayout F = flow_layout(M, H, W);
    if (ws_bytes < F.total) {
        set_error("flow_pairs: workspace %zu < %zu bytes", ws_bytes, F.total);
        return WCTB200_EWS;
    }
    WCTB_ENSURE_SMEM(k_jacobi, JACOBI_SMEM);
    uint8_t* base = static_cast<uint8_t*>(ws);
    const int P = 2 * (M - 1);
    const float* pyr[MAX_LEVELS];
    pyr[0] = Y;
    for (int l = 1; l < F.L; ++l) {
        float* out = reinterpret_cast<float*>(base + F.pyr[l]);
        k_downsample<<<flow_grid((long long)M * F.h[l] * F.w[l], 256), 256, 0, st>>>(pyr[l - 1], M, F.h[l - 1], F.w[l - 1], out,
                                                                                     F.h[l], F.w[l]);
        WCTB_CHECK_LAUNCH("k_downsample");
        pyr[l] = out;
    }
    float* coef = reinterpret_cast<float*>(base + F.coef);
    const float* coarse = nullptr;
    float* cur = nullptr;
    for (int l = F.L - 1; l >= 0; --l) {
        const int h = F.h[l], w = F.w[l];
        const long long hw = (long long)h * w;
        float* a = l == 0 ? flows : reinterpret_cast<float*>(base + F.fa[l]);
        float* b = reinterpret_cast<float*>(base + F.fb[l]);
        if (coarse == nullptr) {
            WCTB_CUDA(cudaMemsetAsync(a, 0, (size_t)P * 2 * hw * sizeof(float), st));
        } else {
            k_upsample_flow<<<flow_grid((long long)2 * P * hw, 256), 256, 0, st>>>(coarse, 2 * P, F.h[l + 1], F.w[l + 1], a, h, w);
            WCTB_CHECK_LAUNCH("k_upsample_flow");
        }
        cur = a;
        float* other = b;
        const dim3 jgrid(cdiv(w, JT), cdiv(h, JT), P);
        for (int wp = 0; wp < WARPS; ++wp) {
            k_warp_coefs<<<flow_grid((long long)P * hw, 256), 256, 0, st>>>(pyr[l], P, h, w, cur, coef);
            WCTB_CHECK_LAUNCH("k_warp_coefs");
            for (int it = 0; it < ITERS; it += JK) {
                const int k = ITERS - it < JK ? ITERS - it : JK;
                k_jacobi<<<jgrid, 256, JACOBI_SMEM, st>>>(cur, other, coef, h, w, k);
                WCTB_CHECK_LAUNCH("k_jacobi");
                float* s = cur;
                cur = other;
                other = s;
            }
        }
        coarse = cur;
    }
    if (cur != flows) WCTB_CUDA(cudaMemcpyAsync(flows, cur, (size_t)P * 2 * H * W * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return 0;
}

int launch_flow_confidence(const float* Y, int M, int H, int W, const float* flows, uint8_t* mask, int* counts, cudaStream_t st) {
    const long long hw = (long long)H * W;
    WCTB_CUDA(cudaMemsetAsync(counts, 0, (size_t)(M - 1) * sizeof(int), st));
    k_confidence<<<dim3(cdiv(hw, 256), M - 1), 256, 0, st>>>(Y, H, W, flows, mask, counts);
    WCTB_CHECK_LAUNCH("k_confidence");
    k_cut<<<flow_grid((long long)(M - 1) * hw, 256), 256, 0, st>>>(mask, M - 1, hw, counts);
    WCTB_CHECK_LAUNCH("k_cut");
    return 0;
}

int launch_temporal_blend(uint8_t* frames, int N, int H, int W, const uint8_t* prev, const float* flows, const uint8_t* masks,
                          float beta, cudaStream_t st) {
    const long long hw = (long long)H * W;
    const int first = prev ? 0 : 1;
    for (int i = first; i < N; ++i) {
        const int j = i - first;                                   // pair j: flows 2j (backward), mask j
        const uint8_t* pv = i == 0 ? prev : frames + (i - 1) * hw * 3;
        k_blend<<<flow_grid(hw, 256), 256, 0, st>>>(frames + i * hw * 3, pv, flows + 4 * j * hw, masks + j * hw, H, W, beta);
        WCTB_CHECK_LAUNCH("k_blend");
    }
    return 0;
}

}  // namespace wctb
