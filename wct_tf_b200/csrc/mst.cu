// Multimodal style transfer (DESIGN.md §3.3.10): the labelling half of MST.  The style side clusters the unit directions of
// a style feature into K modes (k-means++ seeding, then spherical Lloyd); the content side scores every content pixel against
// the K centres (data term) and smooths the labelling with red-black ICM on a Potts energy.  The transforms that consume the
// labels are the region kernels of spatial control (wctb200_wct_style_prepare_regions / wctb200_wct_apply_regions).
//
// Every pixel's norm and dot products are taken by a group of L = min(32, C/8) lanes, each over 8-channel slices: a slice's 8
// products are summed in fp32 and added to fp64 accumulators, which the group reduces by an xor butterfly (every lane ends
// with the same bits: an IEEE add is commutative).  The k-means sums are fp64 throughout, in a fixed order over a fixed
// number of pixels per CTA (PIX), so the centres depend on neither the GPU nor the schedule, and the Lloyd loop decides on
// the device when to stop: the host enqueues LLOYD_MAX iterations and the ones after convergence return at once.
#include <float.h>

#include "common.cuh"

namespace wctb {

namespace mstc {
constexpr int KMAX = 8;
constexpr int LLOYD_MAX = 16;
constexpr int PIX = 256;                    // pixels per CTA (assign, distance): also the k-means++ block size
constexpr int THREADS = 256;
constexpr unsigned int KEY0 = 0x3154534Du;  // Philox key of the k-means++ draws: "MST1", "KMPP" (little-endian ASCII)
constexpr unsigned int KEY1 = 0x50504D4Bu;
constexpr double NORM_EPS = 1e-12;
}  // namespace mstc
using namespace mstc;

static inline size_t mst_align(size_t v) { return (v + 255) / 256 * 256; }

// Philox4x32-10 (Random123 constants; the generator of the texture noise, image_ops.cu)
__device__ __forceinline__ uint4 mst_philox(uint4 c, unsigned int k0, unsigned int k1) {
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

// padded position of pixel i of an [N,H,W] map (row-major)
__device__ __forceinline__ long long mst_pos(long long i, int H, int W) {
    const long long hw = (long long)H * W;
    const long long n = i / hw, r = i - n * hw;
    const int y = (int)(r / W), x = (int)(r - (long long)y * W);
    return (n * (H + 2) + y + 1) * (long long)(W + 2) + x + 1;
}

// norm^2 and the K dot products of one pixel (element offset `base` = pos * C) with the centres cs [K][C] (shared), taken by
// the L lanes of a group (`sub` = lane within it); every lane of the group returns the same values.
__device__ __forceinline__ void pixel_dots(const __half* __restrict__ act, long long plane, long long base, int C, int sub, int L,
                                           bool valid, const float* __restrict__ cs, int K, double& ss, double (&dot)[KMAX]) {
    ss = 0.0;
#pragma unroll
    for (int k = 0; k < KMAX; ++k) dot[k] = 0.0;
    if (valid) {
        for (int g = sub; g < C / 8; g += L) {
            float x[8];
            const Half8 hi = *reinterpret_cast<const Half8*>(act + base + 8 * g);
            const Half8 lo = *reinterpret_cast<const Half8*>(act + plane + base + 8 * g);
            merge8(hi, lo, x);
            float q = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) q = fmaf(x[i], x[i], q);
            ss += (double)q;
#pragma unroll
            for (int k = 0; k < KMAX; ++k) {
                if (k < K) {
                    const float4 c0 = *reinterpret_cast<const float4*>(cs + k * C + 8 * g);
                    const float4 c1 = *reinterpret_cast<const float4*>(cs + k * C + 8 * g + 4);
                    float t = x[0] * c0.x;
                    t = fmaf(x[1], c0.y, t);
                    t = fmaf(x[2], c0.z, t);
                    t = fmaf(x[3], c0.w, t);
                    t = fmaf(x[4], c1.x, t);
                    t = fmaf(x[5], c1.y, t);
                    t = fmaf(x[6], c1.z, t);
                    t = fmaf(x[7], c1.w, t);
                    dot[k] += (double)t;
                }
            }
        }
    }
    for (int o = L >> 1; o; o >>= 1) {
        ss += __shfl_xor_sync(0xffffffffu, ss, o);
#pragma unroll
        for (int k = 0; k < KMAX; ++k)
            if (k < K) dot[k] += __shfl_xor_sync(0xffffffffu, dot[k], o);
    }
}

__device__ __forceinline__ double mst_norm(double ss) { return fmax(sqrt(ss), NORM_EPS); }

// lanes per pixel and the pixel slot of this thread within one step of a CTA (8 warps x 32/L groups)
struct Lanes {
    int L, sub, slot, per_step;
    __device__ Lanes(int C) {
        L = C / 8 < 32 ? C / 8 : 32;
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        sub = lane & (L - 1);
        slot = warp * (32 / L) + lane / L;
        per_step = (THREADS / 32) * (32 / L);
    }
};

// ---------------------------------------------------------------------------------------------------------------- k-means
// integer words of the workspace
struct MstCounters {
    int done;                     // set by the update of the first iteration in which no label changed
    int arrive[KMAX];             // CTAs of the update kernel that finished their channels, per cluster (last one normalises)
    int changes[LLOYD_MAX];       // labels changed by the assign of iteration t
    int counts[LLOYD_MAX][KMAX];  // pixels per cluster after the assign of iteration t
};

struct MstLayout {
    size_t best, bsum, slots, sums, ctr, total;
};
static MstLayout mst_layout(int P, int C, int K) {
    const size_t nb = (size_t)(P + PIX - 1) / PIX;
    MstLayout L;
    size_t o = 0;
    L.best = o;  o += mst_align((size_t)P * sizeof(double));
    L.bsum = o;  o += mst_align(nb * sizeof(double));
    L.slots = o; o += mst_align(nb * K * C * sizeof(double));
    L.sums = o;  o += mst_align((size_t)K * C * sizeof(double));
    L.ctr = o;   o += mst_align(sizeof(MstCounters));
    L.total = o;
    return L;
}

size_t mst_clusters_workspace_bytes(int Hs, int Ws, int C, int K) { return mst_layout(Hs * Ws, C, K).total; }

// k-means++ draw j: centre 0 is pixel floor(v P) (v = x0 / 2^32); centre j >= 1 is the first pixel whose running sum of d
// exceeds v sum(d), the sum taken over the PIX-pixel blocks of k_mst_dist in block order.  One CTA; also zeroes the counters
// (j = 0) and writes the centre c_j = u_p.
__global__ void __launch_bounds__(THREADS) k_mst_select(const __half* __restrict__ style, int Hs, int Ws, int C, int j, int level,
                                                        const double* __restrict__ best, const double* __restrict__ bsum, int nb,
                                                        float* __restrict__ centres, int32_t* __restrict__ info,
                                                        MstCounters* __restrict__ ctr) {
    __shared__ long long s_pick;
    __shared__ double s_red[THREADS];
    const int tid = threadIdx.x;
    const long long P = (long long)Hs * Ws;
    if (tid == 0) {
        const uint4 r = mst_philox(make_uint4((unsigned int)j, (unsigned int)level, 0u, 0u), KEY0, KEY1);
        long long pick;
        if (j == 0) {
            pick = (long long)(((unsigned long long)r.x * (unsigned long long)P) >> 32);
        } else {
            double total = 0.0;
            for (int b = 0; b < nb; ++b) total += bsum[b];
            pick = info[0];                                     // sum(d) = 0: every pixel sits on a centre; copy centre 0
            if (total > 0.0) {
                const double T = (double)r.x * 0x1p-32 * total;
                double S = 0.0;
                int bstar = -1;
                for (int b = 0; b < nb; ++b) {
                    if (S + bsum[b] > T) { bstar = b; break; }
                    S += bsum[b];
                }
                if (bstar < 0) {                               // unreachable (S after the last block is total > T); be safe
                    for (int b = nb - 1; b >= 0; --b) if (bsum[b] > 0.0) { bstar = b; break; }
                    S = 0.0;
                    for (int b = 0; b < bstar; ++b) S += bsum[b];
                }
                const long long p0 = (long long)bstar * PIX, p1 = p0 + PIX < P ? p0 + PIX : P;
                double rl = 0.0;
                long long last = p0;
                pick = -1;
                for (long long p = p0; p < p1; ++p) {
                    const double d = fmax(0.0, 1.0 - best[p]);
                    rl += d;
                    if (d > 0.0) last = p;
                    if (S + rl > T) { pick = p; break; }
                }
                if (pick < 0) pick = last;
            }
        }
        if (j == 0) {
            ctr->done = 0;
            for (int k = 0; k < KMAX; ++k) ctr->arrive[k] = 0;
            for (int t = 0; t < LLOYD_MAX; ++t) {
                ctr->changes[t] = 0;
                for (int k = 0; k < KMAX; ++k) ctr->counts[t][k] = 0;
            }
        }
        info[j] = (int32_t)pick;
        s_pick = pick;
    }
    __syncthreads();
    const ActGeom g(1, Hs, Ws, C);
    const long long base = mst_pos(s_pick, Hs, Ws) * C;
    double ss = 0.0;
    for (int c = tid; c < C; c += THREADS) {
        const double f = (double)merge_f32(style[base + c], style[g.plane + base + c]);
        ss += f * f;
    }
    s_red[tid] = ss;
    __syncthreads();
    for (int o = THREADS / 2; o; o >>= 1) {
        if (tid < o) s_red[tid] += s_red[tid + o];
        __syncthreads();
    }
    const double nrm = mst_norm(s_red[0]);
    for (int c = tid; c < C; c += THREADS)
        centres[(long long)j * C + c] = (float)((double)merge_f32(style[base + c], style[g.plane + base + c]) / nrm);
}

// k-means++ distances before draw j >= 1: best_p = max_{i<j} u_p . c_i (this launch adds centre j - 1), and the block sums
// bsum[b] = sum over the block's pixels, in pixel order, of d_p = max(0, 1 - best_p) (fp64)
__global__ void __launch_bounds__(THREADS) k_mst_dist(const __half* __restrict__ style, int Hs, int Ws, int C, int j,
                                                      const float* __restrict__ centres, double* __restrict__ best,
                                                      double* __restrict__ bsum) {
    __shared__ __align__(16) float s_c[512];
    __shared__ double s_d[PIX];
    const long long P = (long long)Hs * Ws;
    for (int c = threadIdx.x; c < C; c += THREADS) s_c[c] = centres[(long long)(j - 1) * C + c];
    __syncthreads();
    const ActGeom g(1, Hs, Ws, C);
    const Lanes ln(C);
    for (int j0 = 0; j0 < PIX; j0 += ln.per_step) {
        const int jj = j0 + ln.slot;
        const long long p = (long long)blockIdx.x * PIX + jj;
        const bool valid = p < P;
        double ss, dot[KMAX];
        pixel_dots(style, g.plane, valid ? mst_pos(p, Hs, Ws) * C : 0, C, ln.sub, ln.L, valid, s_c, 1, ss, dot);
        if (ln.sub == 0) {
            double d = 0.0;
            if (valid) {
                const double s = dot[0] / mst_norm(ss);
                const double b = j == 1 ? s : fmax(best[p], s);
                best[p] = b;
                d = fmax(0.0, 1.0 - b);
            }
            s_d[jj] = d;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double r = 0.0;
        for (int i = 0; i < PIX; ++i) r += s_d[i];
        bsum[blockIdx.x] = r;
    }
}

// dynamic shared memory of k_mst_assign
static size_t assign_smem(int C, int K) {
    const int S = C < THREADS ? THREADS / C : 1;
    return (size_t)K * C * sizeof(float) + (size_t)S * K * C * sizeof(double) + PIX * (sizeof(long long) + sizeof(double)) + PIX +
           16 * sizeof(int);
}

// Lloyd iteration t (1-based), first half: label_p = argmax_k u_p . c_k (ties: lowest k), the changes against iteration
// t - 1 and the cluster counts (integer atomics), and this CTA's fp64 sums of u_p per cluster, slots [block][K][C]: thread
// (s, c) adds pixels s, s + S, ... of the block in order, and the S partials are added in order of s.
__global__ void __launch_bounds__(THREADS) k_mst_assign(const __half* __restrict__ style, int Hs, int Ws, int C, int K, int t,
                                                        const float* __restrict__ centres, uint8_t* __restrict__ labels,
                                                        double* __restrict__ slots, MstCounters* __restrict__ ctr) {
    if (ctr->done) return;
    extern __shared__ __align__(16) uint8_t smem[];
    const int S = C < THREADS ? THREADS / C : 1;
    float* s_c = reinterpret_cast<float*>(smem);
    double* s_acc = reinterpret_cast<double*>(smem + (size_t)K * C * sizeof(float));
    long long* s_pos = reinterpret_cast<long long*>(s_acc + (size_t)S * K * C);
    double* s_inv = reinterpret_cast<double*>(s_pos + PIX);
    int* s_cnt = reinterpret_cast<int*>(s_inv + PIX);
    uint8_t* s_lab = reinterpret_cast<uint8_t*>(s_cnt + 16);
    const int tid = threadIdx.x;
    const long long P = (long long)Hs * Ws;
    for (int i = tid; i < K * C; i += THREADS) s_c[i] = centres[i];
    for (int i = tid; i < S * K * C; i += THREADS) s_acc[i] = 0.0;
    if (tid < 16) s_cnt[tid] = 0;
    __syncthreads();
    const ActGeom g(1, Hs, Ws, C);
    const Lanes ln(C);
    for (int j0 = 0; j0 < PIX; j0 += ln.per_step) {
        const int jj = j0 + ln.slot;
        const long long p = (long long)blockIdx.x * PIX + jj;
        const bool valid = p < P;
        const long long pos = valid ? mst_pos(p, Hs, Ws) : 0;
        double ss, dot[KMAX];
        pixel_dots(style, g.plane, pos * C, C, ln.sub, ln.L, valid, s_c, K, ss, dot);
        if (ln.sub == 0) {
            int lab = 0;
            double inv = 0.0;
            if (valid) {
                const double nrm = mst_norm(ss);
                double bs = dot[0] / nrm;
#pragma unroll
                for (int k = 1; k < KMAX; ++k) {
                    if (k < K) {
                        const double s = dot[k] / nrm;
                        if (s > bs) { bs = s; lab = k; }
                    }
                }
                inv = 1.0 / nrm;
                if (t == 1 || labels[p] != lab) atomicAdd(&s_cnt[KMAX], 1);
                atomicAdd(&s_cnt[lab], 1);
                labels[p] = (uint8_t)lab;
            }
            s_pos[jj] = pos;
            s_inv[jj] = inv;
            s_lab[jj] = (uint8_t)(valid ? lab : 255);
        }
    }
    __syncthreads();
    const int s = C < THREADS ? tid / C : 0;
    for (int c = C < THREADS ? tid % C : tid; c < C; c += THREADS) {
        for (int jj = s; jj < PIX; jj += S) {
            const int k = s_lab[jj];
            if (k == 255) continue;
            const long long off = s_pos[jj] * C + c;
            const double u = (double)merge_f32(style[off], style[g.plane + off]) * s_inv[jj];
            s_acc[((size_t)s * K + k) * C + c] += u;
        }
    }
    __syncthreads();
    for (int i = tid; i < K * C; i += THREADS) {
        double v = 0.0;
        for (int q = 0; q < S; ++q) v += s_acc[(size_t)q * K * C + i];
        slots[(size_t)blockIdx.x * K * C + i] = v;
    }
    if (tid < K && s_cnt[tid]) atomicAdd(&ctr->counts[t - 1][tid], s_cnt[tid]);
    if (tid == KMAX && s_cnt[KMAX]) atomicAdd(&ctr->changes[t - 1], s_cnt[KMAX]);
}

// Lloyd iteration t, second half: grid (ceil(C/32), K).  Stops the loop when the assign changed no label; otherwise warp w
// of a CTA adds the slots of blocks [w nb/8, (w+1) nb/8) in block order for 32 channels, the 8 warp partials are added in
// order, and the last CTA of cluster k to finish normalises c_k = sum / max(|sum|, 1e-12) (an empty cluster keeps its
// centre).  info: [K init | iterations | K counts].
__global__ void __launch_bounds__(THREADS) k_mst_update(int C, int K, int t, int nb, const double* __restrict__ slots,
                                                        double* __restrict__ sums, float* __restrict__ centres,
                                                        int32_t* __restrict__ info, MstCounters* __restrict__ ctr) {
    if (ctr->done) return;
    const int k = blockIdx.y, tid = threadIdx.x;
    const int changes = ctr->changes[t - 1];
    if (blockIdx.x == 0 && tid == 0) {
        info[K + 1 + k] = ctr->counts[t - 1][k];
        if (k == 0) info[K] = t;
    }
    if (changes == 0) {
        if (blockIdx.x == 0 && k == 0 && tid == 0) ctr->done = 1;   // every CTA of this launch returns here too
        return;
    }
    __shared__ double s_part[THREADS / 32][32];
    __shared__ bool s_last;
    const int warp = tid >> 5, lane = tid & 31;
    const int c = blockIdx.x * 32 + lane;
    const int b0 = (int)((long long)warp * nb / (THREADS / 32)), b1 = (int)((long long)(warp + 1) * nb / (THREADS / 32));
    double v = 0.0;
    if (c < C)
        for (int b = b0; b < b1; ++b) v += slots[((size_t)b * K + k) * C + c];
    s_part[warp][lane] = v;
    __syncthreads();
    if (warp == 0) {
        double r = 0.0;
        for (int w = 0; w < THREADS / 32; ++w) r += s_part[w][lane];
        if (c < C) sums[(size_t)k * C + c] = r;
        __threadfence();
    }
    __syncthreads();
    if (tid == 0) s_last = atomicAdd(&ctr->arrive[k], 1) == (int)gridDim.x - 1;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    if (tid == 0) {
        ctr->arrive[k] = 0;
        double n2 = 0.0;
        const volatile double* vs = sums + (size_t)k * C;
        for (int i = 0; i < C; ++i) n2 += vs[i] * vs[i];
        s_part[0][0] = mst_norm(n2);
    }
    __syncthreads();
    if (ctr->counts[t - 1][k] == 0) return;                         // empty: keeps its centre
    const double nrm = s_part[0][0];
    const volatile double* vs = sums + (size_t)k * C;
    for (int i = tid; i < C; i += THREADS) centres[(size_t)k * C + i] = (float)(vs[i] / nrm);
}

int launch_mst_style_clusters(const __half* style, int Hs, int Ws, int C, int K, int level, uint8_t* labels, float* centres,
                              int32_t* info, void* ws, size_t ws_bytes, cudaStream_t st) {
    const int P = Hs * Ws;
    const MstLayout L = mst_layout(P, C, K);
    if (ws_bytes < L.total) {
        set_error("mst_style_clusters: workspace %zu < %zu bytes", ws_bytes, L.total);
        return WCTB200_EWS;
    }
    uint8_t* base = static_cast<uint8_t*>(ws);
    double* best = reinterpret_cast<double*>(base + L.best);
    double* bsum = reinterpret_cast<double*>(base + L.bsum);
    double* slots = reinterpret_cast<double*>(base + L.slots);
    double* sums = reinterpret_cast<double*>(base + L.sums);
    MstCounters* ctr = reinterpret_cast<MstCounters*>(base + L.ctr);
    const int nb = (P + PIX - 1) / PIX;
    k_mst_select<<<1, THREADS, 0, st>>>(style, Hs, Ws, C, 0, level, best, bsum, nb, centres, info, ctr);
    WCTB_CHECK_LAUNCH("k_mst_select");
    for (int j = 1; j < K; ++j) {
        k_mst_dist<<<nb, THREADS, 0, st>>>(style, Hs, Ws, C, j, centres, best, bsum);
        WCTB_CHECK_LAUNCH("k_mst_dist");
        k_mst_select<<<1, THREADS, 0, st>>>(style, Hs, Ws, C, j, level, best, bsum, nb, centres, info, ctr);
        WCTB_CHECK_LAUNCH("k_mst_select");
    }
    const size_t smem = assign_smem(C, K);
    WCTB_ENSURE_SMEM(k_mst_assign, assign_smem(512, KMAX));
    for (int t = 1; t <= LLOYD_MAX; ++t) {
        k_mst_assign<<<nb, THREADS, smem, st>>>(style, Hs, Ws, C, K, t, centres, labels, slots, ctr);
        WCTB_CHECK_LAUNCH("k_mst_assign");
        k_mst_update<<<dim3((C + 31) / 32, K), THREADS, 0, st>>>(C, K, t, nb, slots, sums, centres, info, ctr);
        WCTB_CHECK_LAUNCH("k_mst_update");
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------------------ content side
// D[i][k] = 1 - u_i . c_k (fp32; +inf for a cluster of fewer than 2 style pixels), i over the N*H*W pixels
__global__ void __launch_bounds__(THREADS) k_mst_data_term(const __half* __restrict__ act, int N, int H, int W, int C, int K,
                                                           const float* __restrict__ centres, const int32_t* __restrict__ counts,
                                                           float* __restrict__ D) {
    __shared__ __align__(16) float s_c[KMAX * 512];
    __shared__ int s_ok[KMAX];
    for (int i = threadIdx.x; i < K * C; i += THREADS) s_c[i] = centres[i];
    if (threadIdx.x < K) s_ok[threadIdx.x] = counts[threadIdx.x] >= 2;
    __syncthreads();
    const ActGeom g(N, H, W, C);
    const long long total = (long long)N * H * W;
    const Lanes ln(C);
    for (long long i0 = (long long)blockIdx.x * PIX; i0 < total; i0 += (long long)gridDim.x * PIX) {
        for (int j0 = 0; j0 < PIX; j0 += ln.per_step) {
            const long long i = i0 + j0 + ln.slot;
            const bool valid = i < total;
            double ss, dot[KMAX];
            pixel_dots(act, g.plane, valid ? mst_pos(i, H, W) * C : 0, C, ln.sub, ln.L, valid, s_c, K, ss, dot);
            if (valid && ln.sub == 0) {
                const double nrm = mst_norm(ss);
#pragma unroll
                for (int k = 0; k < KMAX; ++k)
                    if (k < K) D[i * K + k] = s_ok[k] ? (float)(1.0 - dot[k] / nrm) : __int_as_float(0x7f800000);
            }
        }
    }
}

int launch_mst_data_term(const __half* act, int N, int H, int W, int C, const float* centres, const int32_t* counts, int K, float* D,
                         cudaStream_t st) {
    const long long total = (long long)N * H * W;
    long long grid = (total + PIX - 1) / PIX;
    const long long cap = (long long)device_sm_count() * 8;
    if (grid > cap) grid = cap;
    k_mst_data_term<<<(int)grid, THREADS, 0, st>>>(act, N, H, W, C, K, centres, counts, D);
    WCTB_CHECK_LAUNCH("k_mst_data_term");
    return 0;
}

// ICM start: label = argmin_k D (ties: lowest k)
__global__ void k_mst_argmin(const float* __restrict__ D, long long total, int K, uint8_t* __restrict__ labels) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const float* d = D + i * K;
        float b = d[0];
        int lab = 0;
        for (int k = 1; k < K; ++k)
            if (d[k] < b) { b = d[k]; lab = k; }
        labels[i] = (uint8_t)lab;
    }
}

// one half-sweep of red-black ICM: every pixel with (y + x) % 2 == parity takes argmin_k D[p,k] + lambda n_k(p), n_k the
// 4-neighbours inside the image whose label is not k; it keeps its label when that is among the minima, else takes the
// lowest k.  The cost is one __fmul_rn and one __fadd_rn.  The updated pixels read only pixels of the other parity, so the
// half-sweep is in place and its result does not depend on the schedule.
__global__ void k_mst_sweep(const float* __restrict__ D, int N, int H, int W, int K, float lambda, int parity,
                            uint8_t* __restrict__ labels) {
    const int Wh = (W + 1) / 2;                                   // pixels of one parity per row, at most
    const long long total = (long long)N * H * Wh;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / Wh;
        const int xi = (int)(i - r * Wh);
        const int y = (int)(r % H);
        const int x = 2 * xi + ((y + parity) & 1);
        if (x >= W) continue;
        const long long p = r * W + x;
        // a neighbour outside the image reads as label 255, which no k matches and nn does not count
        const int up = y > 0 ? labels[p - W] : 255, dn = y < H - 1 ? labels[p + W] : 255;
        const int lf = x > 0 ? labels[p - 1] : 255, rt = x < W - 1 ? labels[p + 1] : 255;
        const int nn = (y > 0) + (y < H - 1) + (x > 0) + (x < W - 1);
        const int cur = labels[p];
        const float* d = D + p * K;
        float cost[KMAX];
        float m = __int_as_float(0x7f800000);
#pragma unroll
        for (int k = 0; k < KMAX; ++k) {
            cost[k] = m;
            if (k < K) {
                const int same = (up == k) + (dn == k) + (lf == k) + (rt == k);
                cost[k] = __fadd_rn(d[k], __fmul_rn(lambda, (float)(nn - same)));
                m = fminf(m, cost[k]);
            }
        }
        int lab = cur;
        float cc = 0.f;
#pragma unroll
        for (int k = 0; k < KMAX; ++k)
            if (k == cur) cc = cost[k];
        if (!(cc == m)) {
#pragma unroll
            for (int k = KMAX - 1; k >= 0; --k)
                if (k < K && cost[k] == m) lab = k;
        }
        labels[p] = (uint8_t)lab;
    }
}

int launch_mst_smooth(const float* D, int N, int H, int W, int K, float lambda, int sweeps, uint8_t* labels, cudaStream_t st) {
    const long long total = (long long)N * H * W;
    const long long cap = (long long)device_sm_count() * 16;
    long long g0 = (total + 255) / 256;
    k_mst_argmin<<<(int)(g0 > cap ? cap : g0), 256, 0, st>>>(D, total, K, labels);
    WCTB_CHECK_LAUNCH("k_mst_argmin");
    const long long half = (long long)N * H * ((W + 1) / 2);
    long long g1 = (half + 255) / 256;
    if (g1 > cap) g1 = cap;
    for (int s = 0; s < sweeps; ++s) {
        for (int parity = 0; parity < 2; ++parity) {
            k_mst_sweep<<<(int)g1, 256, 0, st>>>(D, N, H, W, K, lambda, parity, labels);
            WCTB_CHECK_LAUNCH("k_mst_sweep");
        }
    }
    return 0;
}

}  // namespace wctb
