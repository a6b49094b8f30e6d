// Exact feature distribution matching (EFDM, DESIGN.md §3.3.12): every channel of every frame takes the value distribution
// of the same channel of its style, by rank.  A *segment* is one (frame, channel) of L = H*W values.  Both sides sort their
// segments with the same segmented LSD radix sort: 32-bit order-preserving keys of the fp32 values, four 8-bit digits, each
// pass a tile histogram, a per-segment scan over tiles and a stable tile scatter.  The style side keeps the sorted values
// (the state); the content side sorts (key, pixel index) pairs, then
//   q(r) = Q interpolated at u(r) = clamp((2r+1) Ms / (2 Nc) - 1/2, 0, Ms-1)    (fp64)
//   P(r) = sum_{j<r} q(j)                                                        (fp64, fixed tree per tile, tiles in order)
//   t    = (P(r1) - P(r0)) / (r1 - r0) over the run [r0, r1) of equal keys holding rank r
//   out  = alpha t + (1 - alpha) x
// scattered by pixel index into a channel-major fp32 buffer and transposed once into NHWC SPF16 with the reflect halo.
//
// Every segment is sorted by tiles of TILE keys whatever the batch, so a segment's bytes depend on nothing but its own values
// and its style's: the apply runs as many whole segments at a time as the workspace holds, with byte-identical results for
// every workspace size.  The sort's stability does not reach the output: all members of a run take the same value.
//
// Sliced distribution matching (DESIGN.md §3.3.14) chains steps of the same content pass with the keys built by
// k_efdm_rotate_keys (y = G v) instead of k_efdm_keys: the runs go to fp32 channel-major planes, which the next step
// rotates, and the last step stores alpha t + (1 - alpha) x0 with the original content x0 (k_efdm_store<true>).
#include <algorithm>

#include "common.cuh"

namespace wctb {

namespace efdmc {
constexpr int THREADS = 256;
constexpr int ITEMS = 8;
constexpr int TILE = THREADS * ITEMS;      // keys per sort tile
constexpr int WARPS = THREADS / 32;
constexpr int RADIX = 256;
constexpr int PASSES = 4;
constexpr int TP = 64;                     // pixels per transpose tile (key build, output)
constexpr int TS = 32;                     // segments per transpose tile
constexpr long long MAX_CHUNK = 65535;     // segments per chunk: gridDim.y
}  // namespace efdmc
using namespace efdmc;

static inline size_t efdm_align(size_t v) { return (v + 255) / 256 * 256; }

// order-preserving uint32 of an fp32 value; -0 is +0 (one run of zeros, as np.unique sees it)
__device__ __forceinline__ unsigned int efdm_key(float x) {
    unsigned int b = __float_as_uint(x + 0.0f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float efdm_value(unsigned int k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

// ---------------------------------------------------------------------------------------------------------------------
// key build: SPF16 interior of segments [s0, s0+S) (segment s = frame s / C, channel s % C) -> keys [S][L], channel-major.
// A CTA transposes TS segments x TP pixels through shared memory: reads 64 contiguous bytes per pixel and plane, writes
// 256 contiguous bytes per segment.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_efdm_keys(const __half* __restrict__ act, ActGeom g, long long s0, int S,
                                                   unsigned int* __restrict__ keys) {
    __shared__ unsigned int tile[TS][TP + 1];
    const int L = g.H * g.W;
    const int p0 = blockIdx.x * TP;
    const int sl0 = blockIdx.y * TS;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int sl = sl0 + tx;
    const long long s = s0 + sl;
    const long long n = s / g.C;
    const int c = (int)(s - n * g.C);
    for (int pi = ty; pi < TP; pi += 8) {
        const int p = p0 + pi;
        if (p < L && sl < S) {
            const int y = p / g.W, x = p - y * g.W;
            const long long off = ((n * g.Hp + y + 1) * g.Wp + x + 1) * g.C + c;
            tile[tx][pi] = efdm_key(merge_f32(act[off], act[g.plane + off]));
        }
    }
    __syncthreads();
    for (int si = ty; si < TS; si += 8) {
        if (sl0 + si >= S) break;
        for (int pj = tx; pj < TP; pj += 32) {
            const int p = p0 + pj;
            if (p < L) keys[(long long)(sl0 + si) * L + p] = tile[si][pj];
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// sliced key build (DESIGN.md §3.3.14): keys of y = G v for segments [s0, s0+S), channel-major [S][L], where v is frame n's
// C values at a pixel, read from the SPF16 NHWC interior (planes == NULL) or from fp32 channel-major planes [N][C][L].  A CTA
// computes RC output channels x RP pixels of one frame (C % RC == 0, so a channel block never straddles frames); every
// output is one fmaf chain over the input channels in index order, so its rounding does not depend on the tile, the chunk
// or the batch.  Blocks are aligned to RC segments from segment 0; only the chunk's segments are written.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int RC = 64, RP = 128, RJ = 32;   // output channels, pixels, input channels per smem stage
__global__ void __launch_bounds__(256) k_efdm_rotate_keys(const __half* __restrict__ act, const float* __restrict__ planes, ActGeom g,
                                                          const float* __restrict__ G, long long s0, int S,
                                                          unsigned int* __restrict__ keys) {
    __shared__ __align__(16) float Gs[RJ][RC + 4];
    __shared__ float Vs[RJ][RP + 1];
    const int C = g.C, L = g.H * g.W;
    const int p0 = blockIdx.x * RP;
    const long long sb = (s0 / RC + blockIdx.y) * RC;        // first segment of this block
    const long long n = sb / C;
    const int c0 = (int)(sb - n * C);
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // pixels tx + 32 i, channels ty * 8 + r
    float acc[8][4];
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[r][i] = 0.f;
    for (int j0 = 0; j0 < C; j0 += RJ) {
        for (int e = threadIdx.x; e < RJ * RC; e += 256) {
            const int c = e % RC, j = e / RC;
            Gs[j][c] = G[(long long)(c0 + c) * C + j0 + j];
        }
        if (planes) {
            for (int e = threadIdx.x; e < RJ * RP; e += 256) {
                const int pi = e % RP, j = e / RP;
                const int p = p0 + pi;
                Vs[j][pi] = p < L ? planes[(n * C + j0 + j) * (long long)L + p] : 0.f;
            }
        } else {
            for (int e = threadIdx.x; e < RJ * RP; e += 256) {
                const int j = e % RJ, pi = e / RJ;
                const int p = p0 + pi;
                float v = 0.f;
                if (p < L) {
                    const int y = p / g.W, x = p - y * g.W;
                    const long long off = ((n * g.Hp + y + 1) * g.Wp + x + 1) * C + j0 + j;
                    v = merge_f32(act[off], act[g.plane + off]);
                }
                Vs[j][pi] = v;
            }
        }
        __syncthreads();
#pragma unroll 4
        for (int j = 0; j < RJ; ++j) {
            const float4 ga = *reinterpret_cast<const float4*>(&Gs[j][ty * 8]);
            const float4 gb = *reinterpret_cast<const float4*>(&Gs[j][ty * 8 + 4]);
            const float gr[8] = {ga.x, ga.y, ga.z, ga.w, gb.x, gb.y, gb.z, gb.w};
            float v[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) v[i] = Vs[j][tx + 32 * i];
#pragma unroll
            for (int r = 0; r < 8; ++r)
#pragma unroll
                for (int i = 0; i < 4; ++i) acc[r][i] = fmaf(gr[r], v[i], acc[r][i]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        const long long s = sb + ty * 8 + r;
        if (s < s0 || s >= s0 + S) continue;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int p = p0 + tx + 32 * i;
            if (p < L) keys[(s - s0) * L + p] = efdm_key(acc[r][i]);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// radix pass, 1/3: digit histogram of each tile -> hist [S][T][RADIX]
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(THREADS) k_efdm_hist(const unsigned int* __restrict__ keys, int L, int T, int shift,
                                                       unsigned int* __restrict__ hist) {
    __shared__ unsigned int h[RADIX];
    const long long seg = blockIdx.y;
    const int t = blockIdx.x;
    h[threadIdx.x] = 0;
    __syncthreads();
    const unsigned int* kp = keys + seg * L;
    const int r0 = t * TILE, r1 = min(r0 + TILE, L);
    for (int r = r0 + threadIdx.x; r < r1; r += THREADS) atomicAdd(&h[(kp[r] >> shift) & 0xFF], 1u);
    __syncthreads();
    hist[(seg * T + t) * RADIX + threadIdx.x] = h[threadIdx.x];
}

// exclusive scan of one value per thread over the CTA (THREADS threads); returns the total through *total
template <typename V>
__device__ __forceinline__ V efdm_block_excl_scan(V v, V* warp_tot, V* total) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    V inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const V u = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += u;
    }
    if (lane == 31) warp_tot[w] = inc;
    __syncthreads();
    if (w == 0) {
        V a = lane < WARPS ? warp_tot[lane] : V(0);
        V ai = a;
#pragma unroll
        for (int o = 1; o < WARPS; o <<= 1) {
            const V u = __shfl_up_sync(0xffffffffu, ai, o);
            if (lane >= o) ai += u;
        }
        if (lane < WARPS) warp_tot[lane] = ai - a;          // exclusive warp offsets
        if (lane == WARPS - 1) warp_tot[WARPS] = ai;
    }
    __syncthreads();
    const V out = warp_tot[w] + inc - v;
    *total = warp_tot[WARPS];
    __syncthreads();                                          // warp_tot may be reused by the caller
    return out;
}

// ---------------------------------------------------------------------------------------------------------------------
// radix pass, 2/3: per segment, hist[t][d] <- (keys of digits < d in the segment) + (keys of digit d in tiles < t)
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(RADIX) k_efdm_scan(unsigned int* __restrict__ hist, int T) {
    __shared__ unsigned int wt[WARPS + 1];
    unsigned int* h = hist + (long long)blockIdx.x * T * RADIX + threadIdx.x;
    unsigned int tot = 0;
#pragma unroll 8
    for (int t = 0; t < T; ++t) tot += h[(long long)t * RADIX];
    unsigned int all;
    unsigned int run = efdm_block_excl_scan<unsigned int>(tot, wt, &all);
#pragma unroll 8
    for (int t = 0; t < T; ++t) {
        const unsigned int v = h[(long long)t * RADIX];
        h[(long long)t * RADIX] = run;
        run += v;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// radix pass, 3/3: stable scatter of one tile.  Warp w owns the tile's keys [w*256, (w+1)*256) in 8 rounds of 32; its
// ranks come from __match_any_sync and a per-warp digit counter.  The tile is first reordered by digit in shared memory so
// that consecutive threads write consecutive addresses of a bucket.  idx_in NULL: the index is the key's position.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(THREADS) k_efdm_scatter(const unsigned int* __restrict__ kin, const unsigned int* __restrict__ iin,
                                                          unsigned int* __restrict__ kout, unsigned int* __restrict__ iout, int L,
                                                          int T, int shift, const unsigned int* __restrict__ hist) {
    __shared__ unsigned int wh[WARPS][RADIX];
    __shared__ unsigned int tstart[RADIX];
    __shared__ unsigned int gbase[RADIX];
    __shared__ unsigned int wt[WARPS + 1];
    __shared__ unsigned int sk[TILE];
    __shared__ unsigned int si[TILE];
    const long long seg = blockIdx.y;
    const int t = blockIdx.x;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const long long base = seg * L;
    const int r0 = t * TILE;
    const int cnt = min(TILE, L - r0);
    for (int i = threadIdx.x; i < WARPS * RADIX; i += THREADS) (&wh[0][0])[i] = 0;
    gbase[threadIdx.x] = hist[(seg * T + t) * RADIX + threadIdx.x];
    __syncthreads();
    unsigned int key[ITEMS], idx[ITEMS], rank[ITEMS];
    const unsigned int lt = (1u << lane) - 1u;
#pragma unroll
    for (int j = 0; j < ITEMS; ++j) {
        const int i = w * (ITEMS * 32) + j * 32 + lane;
        const bool ok = i < cnt;
        key[j] = ok ? kin[base + r0 + i] : 0u;
        idx[j] = ok ? (iin ? iin[base + r0 + i] : (unsigned int)(r0 + i)) : 0u;
        const unsigned int d = ok ? ((key[j] >> shift) & 0xFF) : RADIX;
        const unsigned int peers = __match_any_sync(0xffffffffu, d);
        const unsigned int before = (d < RADIX) ? wh[w][d] : 0u;
        __syncwarp();
        rank[j] = before + __popc(peers & lt);
        if (d < RADIX && (peers & lt) == 0) wh[w][d] = before + __popc(peers);
        __syncwarp();
    }
    __syncthreads();
    {   // per digit: exclusive offsets over the warps, then the tile's digit starts
        const int d = threadIdx.x;
        unsigned int run = 0;
#pragma unroll
        for (int ww = 0; ww < WARPS; ++ww) {
            const unsigned int v = wh[ww][d];
            wh[ww][d] = run;
            run += v;
        }
        unsigned int all;
        tstart[d] = efdm_block_excl_scan<unsigned int>(run, wt, &all);
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < ITEMS; ++j) {
        const int i = w * (ITEMS * 32) + j * 32 + lane;
        if (i < cnt) {
            const unsigned int d = (key[j] >> shift) & 0xFF;
            const unsigned int pos = tstart[d] + wh[w][d] + rank[j];
            sk[pos] = key[j];
            si[pos] = idx[j];
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < cnt; i += THREADS) {
        const unsigned int k = sk[i];
        const unsigned int d = (k >> shift) & 0xFF;
        const long long dst = base + gbase[d] + (unsigned int)i - tstart[d];
        kout[dst] = k;
        if (iout) iout[dst] = si[i];
    }
}

// 4 passes over S segments of L keys (and indices when iA is not NULL): the result is back in kA / iA
static int efdm_sort(unsigned int* kA, unsigned int* kB, unsigned int* iA, unsigned int* iB, int S, int L, unsigned int* hist,
                     cudaStream_t st) {
    const int T = cdiv(L, TILE);
    const dim3 grid(T, S);
    for (int pass = 0; pass < PASSES; ++pass) {
        const int shift = 8 * pass;
        unsigned int* ki = (pass & 1) ? kB : kA;
        unsigned int* ko = (pass & 1) ? kA : kB;
        unsigned int* ii = iA ? ((pass & 1) ? iB : (pass ? iA : nullptr)) : nullptr;
        unsigned int* io = iA ? ((pass & 1) ? iA : iB) : nullptr;
        k_efdm_hist<<<grid, THREADS, 0, st>>>(ki, L, T, shift, hist);
        WCTB_CHECK_LAUNCH("k_efdm_hist");
        k_efdm_scan<<<S, RADIX, 0, st>>>(hist, T);
        WCTB_CHECK_LAUNCH("k_efdm_scan");
        k_efdm_scatter<<<grid, THREADS, 0, st>>>(ki, ii, ko, io, L, T, shift, hist);
        WCTB_CHECK_LAUNCH("k_efdm_scatter");
    }
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// style side: sorted keys -> fp32 values of the state
// ---------------------------------------------------------------------------------------------------------------------
__global__ void k_efdm_decode(const unsigned int* __restrict__ keys, long long n, float* __restrict__ out) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        out[i] = efdm_value(keys[i]);
}

// ---------------------------------------------------------------------------------------------------------------------
// content side: the prefix P of q over the ranks of each segment
// ---------------------------------------------------------------------------------------------------------------------
struct EfdmQ {
    const float* Q;        // state: sorted style values [Ns][C][Ms]
    int C, Ns, Ms, L;      // L = Nc
    long long s0;          // first segment of the chunk
    __device__ __forceinline__ const float* row(int sl) const {
        const long long s = s0 + sl;
        const long long n = s / C;
        const int c = (int)(s - n * C);
        return Q + ((Ns == 1 ? 0 : n) * C + c) * (long long)Ms;
    }
    // Q linearly interpolated at u(r) = (2r+1) Ms / (2L) - 1/2, clamped to [0, Ms-1]
    __device__ __forceinline__ double q(const float* __restrict__ Qr, int r) const {
        double u = ((2.0 * r + 1.0) * (double)Ms) / (2.0 * (double)L) - 0.5;
        u = fmin(fmax(u, 0.0), (double)(Ms - 1));
        const int i0 = (int)u;
        const int i1 = min(i0 + 1, Ms - 1);
        const double f = u - (double)i0;
        const double a = (double)__ldg(Qr + i0), b = (double)__ldg(Qr + i1);
        return a + f * (b - a);
    }
};

// fp64 sum of q over the ITEMS ranks a thread owns (blocked: ranks r0 + tid*ITEMS + j), then the tile's fixed tree
__device__ __forceinline__ double efdm_thread_q(const EfdmQ& E, const float* Qr, int r0, int cnt, double (&qv)[ITEMS]) {
    double s = 0.0;
#pragma unroll
    for (int j = 0; j < ITEMS; ++j) {
        const int i = threadIdx.x * ITEMS + j;
        qv[j] = i < cnt ? E.q(Qr, r0 + i) : 0.0;
        s += qv[j];
    }
    return s;
}

__global__ void __launch_bounds__(THREADS) k_efdm_qsum(EfdmQ E, int T, double* __restrict__ tsum) {
    __shared__ double wt[WARPS + 1];
    const int sl = blockIdx.y, t = blockIdx.x;
    const int r0 = t * TILE, cnt = min(TILE, E.L - r0);
    double qv[ITEMS];
    const double s = efdm_thread_q(E, E.row(sl), r0, cnt, qv);
    double all;
    efdm_block_excl_scan<double>(s, wt, &all);
    if (threadIdx.x == 0) tsum[(long long)sl * T + t] = all;
}

// per segment: tile sums -> exclusive tile bases, in tile order
__global__ void k_efdm_qscan(double* __restrict__ tsum, int T, int S) {
    const int sl = blockIdx.x * blockDim.x + threadIdx.x;
    if (sl >= S) return;
    double* p = tsum + (long long)sl * T;
    double run = 0.0;
    for (int t = 0; t < T; ++t) {
        const double v = p[t];
        p[t] = run;
        run += v;
    }
}

// P [S][L+1]: P(r) = base of r's tile + the tile's exclusive fp64 scan of q; P(L) = the whole sum
__global__ void __launch_bounds__(THREADS) k_efdm_prefix(EfdmQ E, int T, const double* __restrict__ tbase, double* __restrict__ P) {
    __shared__ double wt[WARPS + 1];
    const int sl = blockIdx.y, t = blockIdx.x;
    const int r0 = t * TILE, cnt = min(TILE, E.L - r0);
    double qv[ITEMS];
    const double s = efdm_thread_q(E, E.row(sl), r0, cnt, qv);
    double all;
    double run = efdm_block_excl_scan<double>(s, wt, &all) + tbase[(long long)sl * T + t];
    double* Ps = P + (long long)sl * (E.L + 1);
#pragma unroll
    for (int j = 0; j < ITEMS; ++j) {
        const int i = threadIdx.x * ITEMS + j;
        if (i < cnt) Ps[r0 + i] = run;
        run += qv[j];
    }
    if (t == T - 1 && threadIdx.x == THREADS - 1) Ps[E.L] = run;
}

// first rank of the run of key k that holds rank r (keys sorted, ks[r] == k): gallop left, then bisect
__device__ int efdm_run_begin(const unsigned int* __restrict__ ks, int r, unsigned int k) {
    int hi = r, step = 1, lo = r - 1;                 // ks[hi] == k; ks[lo] is the candidate
    while (lo >= 0 && ks[lo] == k) {
        hi = lo;
        step <<= 1;
        lo = hi - step;
    }
    if (lo < -1) lo = -1;                              // invariant: lo < run begin <= hi
    while (hi - lo > 1) {
        const int m = lo + (hi - lo) / 2;
        if (ks[m] == k) hi = m; else lo = m;
    }
    return hi;
}
// one past the last rank of that run
__device__ int efdm_run_end(const unsigned int* __restrict__ ks, int L, int r, unsigned int k) {
    int lo = r, step = 1, hi = r + 1;                 // ks[lo] == k; invariant at exit: lo < run end <= hi
    while (hi < L && ks[hi] == k) {
        lo = hi;
        step <<= 1;
        hi = (int)min((long long)lo + step, (long long)L);
    }
    while (hi - lo > 1) {
        const int m = lo + (hi - lo) / 2;
        if (ks[m] == k) lo = m; else hi = m;
    }
    return hi;
}

// ---------------------------------------------------------------------------------------------------------------------
// runs: every rank takes the mean of q over its run, blended with its own value, scattered by pixel index into
// out [S][L] fp32.  In a tile the run begin is a max-scan of the heads; the runs that cross the tile's edges are found by
// galloping search in the segment.  The mean of a run is computed by its tail (or by the tile's last rank) and shared.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(THREADS) k_efdm_runs(const unsigned int* __restrict__ keys, const unsigned int* __restrict__ idx,
                                                       const double* __restrict__ P, int L, int T, float alpha,
                                                       float* __restrict__ out) {
    __shared__ float tmean[TILE];
    __shared__ int wmax[WARPS];
    __shared__ int first_begin;
    const long long seg = blockIdx.y;
    const int t = blockIdx.x;
    const int r0 = t * TILE, cnt = min(TILE, L - r0);
    const unsigned int* ks = keys + seg * L;
    const double* Ps = P + seg * (long long)(L + 1);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (threadIdx.x == 0) first_begin = efdm_run_begin(ks, r0, ks[r0]);
    unsigned int key[ITEMS];
    int head[ITEMS];
    int hmax = -1;
#pragma unroll
    for (int j = 0; j < ITEMS; ++j) {
        const int i = threadIdx.x * ITEMS + j;
        key[j] = i < cnt ? ks[r0 + i] : 0u;
        const bool h = i < cnt && i > 0 && ks[r0 + i - 1] != key[j];
        hmax = h ? i : hmax;
        head[j] = hmax;                                // last head at or before i in this thread, -1 if none
    }
    // inclusive max-scan of the thread maxima over the CTA
    int inc = hmax;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc = max(inc, u);
    }
    if (lane == 31) wmax[w] = inc;
    int excl = __shfl_up_sync(0xffffffffu, inc, 1);
    if (lane == 0) excl = -1;
    __syncthreads();
    for (int ww = 0; ww < w; ++ww) excl = max(excl, wmax[ww]);
    const int fb = first_begin;
#pragma unroll
    for (int j = 0; j < ITEMS; ++j) {
        const int i = threadIdx.x * ITEMS + j;
        if (i >= cnt) break;
        const int hl = max(head[j], excl);             // local index of the run's head in this tile, -1: before the tile
        const bool tail_in = (r0 + i + 1 < L) && (i + 1 < cnt) && ks[r0 + i + 1] != key[j];
        const bool last = (i + 1 == cnt);
        if (tail_in || (r0 + i + 1 == L) || last) {
            const int b = hl >= 0 ? r0 + hl : fb;
            int e = r0 + i + 1;
            if (last && e < L && ks[e] == key[j]) e = efdm_run_end(ks, L, e, key[j]);
            const double m = (Ps[e] - Ps[b]) / (double)(e - b);
            tmean[hl >= 0 ? hl : 0] = (float)m;
        }
        head[j] = hl;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < ITEMS; ++j) {
        const int i = threadIdx.x * ITEMS + j;
        if (i >= cnt) break;
        const float tm = tmean[head[j] >= 0 ? head[j] : 0];
        const float x = efdm_value(key[j]);
        out[seg * L + idx[seg * L + r0 + i]] = fmaf(alpha, tm, (1.0f - alpha) * x);
    }
}

// store one channel of pixel (n, y, x) to its cell and to every reflect-halo cell that mirrors it
__device__ __forceinline__ void efdm_store(__half* __restrict__ act, const ActGeom& g, long long n, int y, int x, int c, __half hi,
                                           __half lo) {
    const long long pitch = (long long)g.Wp * g.C;
    const long long p0 = ((n * g.Hp + y + 1) * g.Wp + x + 1) * g.C + c;
    const long long dy[3] = {0, y == g.ht ? -(long long)(y + 1) * pitch : 0, y == g.hb ? (long long)(g.H - y) * pitch : 0};
    const long long dx[3] = {0, x == g.wl ? -(long long)(x + 1) * g.C : 0, x == g.wr ? (long long)(g.W - x) * g.C : 0};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        if (a && dy[a] == 0) continue;
#pragma unroll
        for (int b = 0; b < 3; ++b) {
            if (b && dx[b] == 0) continue;
            act[p0 + dy[a] + dx[b]] = hi;
            act[g.plane + p0 + dy[a] + dx[b]] = lo;
        }
    }
}

// out [S][L] fp32 of segments [s0, s0+S) -> SPF16 NHWC with the reflect halo (the transpose of k_efdm_keys).  BLEND (the
// last sliced step): the value stored is alpha t + (1 - alpha) x0, x0 the SPF16 content at the same cell.
template <bool BLEND>
__global__ void __launch_bounds__(256) k_efdm_store(const float* __restrict__ vals, ActGeom g, long long s0, int S,
                                                    __half* __restrict__ act, const __half* __restrict__ x0, float alpha) {
    __shared__ float tile[TS][TP + 1];
    const int L = g.H * g.W;
    const int p0 = blockIdx.x * TP;
    const int sl0 = blockIdx.y * TS;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int si = ty; si < TS; si += 8) {
        if (sl0 + si >= S) break;
        for (int pj = tx; pj < TP; pj += 32) {
            const int p = p0 + pj;
            if (p < L) tile[si][pj] = vals[(long long)(sl0 + si) * L + p];
        }
    }
    __syncthreads();
    const int sl = sl0 + tx;
    if (sl >= S) return;
    const long long s = s0 + sl;
    const long long n = s / g.C;
    const int c = (int)(s - n * g.C);
    for (int pi = ty; pi < TP; pi += 8) {
        const int p = p0 + pi;
        if (p < L) {
            const int y = p / g.W, x = p - y * g.W;
            float v = tile[tx][pi];
            if (BLEND) {
                const long long off = ((n * g.Hp + y + 1) * g.Wp + x + 1) * g.C + c;
                v = fmaf(alpha, v, (1.0f - alpha) * merge_f32(x0[off], x0[g.plane + off]));
            }
            __half hi, lo;
            split_f32(v, hi, lo);
            efdm_store(act, g, n, y, x, c, hi, lo);
        }
    }
}

__global__ void k_efdm_copy(const __half* __restrict__ in, ActGeom g, __half* __restrict__ out) {
    const long long total = (long long)g.N * g.H * g.W * (g.C / 8);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c8 = (int)(i % (g.C / 8));
        const long long pix = i / (g.C / 8);
        const int x = (int)(pix % g.W);
        const long long ny = pix / g.W;
        const int y = (int)(ny % g.H);
        const long long n = ny / g.H;
        const long long off = ((n * g.Hp + y + 1) * g.Wp + x + 1) * g.C + 8 * c8;
        const Half8 hi = *reinterpret_cast<const Half8*>(in + off);
        const Half8 lo = *reinterpret_cast<const Half8*>(in + g.plane + off);
        store8_with_halo(out, g, (int)n, y, x, 8 * c8, hi, lo);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------
struct EfdmWs {
    size_t kA, kB, iA, iB, hist, tsum, P, total;
};
// workspace of a chunk of S segments of L values; idx: content side (indices, P, tile sums)
static EfdmWs efdm_layout(long long S, long long L, bool idx) {
    const long long T = (L + TILE - 1) / TILE;
    EfdmWs w{};
    size_t o = 0;
    const size_t kb = efdm_align((size_t)(S * L * 4));
    w.kA = o; o += kb;
    w.kB = o; o += kb;
    if (idx) {
        w.iA = o; o += kb;
        w.iB = o; o += kb;
    }
    w.hist = o; o += efdm_align((size_t)(S * T * RADIX * 4));
    if (idx) {
        w.tsum = o; o += efdm_align((size_t)(S * T * 8));
        w.P = o; o += efdm_align((size_t)(S * (L + 1) * 8));
    }
    w.total = o;
    return w;
}

size_t efdm_style_state_bytes(int C, int Ns, int Hs, int Ws) { return efdm_align((size_t)Ns * C * Hs * Ws * sizeof(float)); }
size_t efdm_style_workspace_bytes(int C, int Ns, int Hs, int Ws, int max_segments) {
    const long long S = std::min<long long>(std::min<long long>((long long)Ns * C, max_segments), MAX_CHUNK);
    return efdm_layout(S, (long long)Hs * Ws, false).total;
}
size_t efdm_workspace_bytes(int C, int N, int H, int W, int max_segments) {
    const long long S = std::min<long long>(std::min<long long>((long long)N * C, max_segments), MAX_CHUNK);
    return efdm_layout(S, (long long)H * W, true).total;
}

// the largest chunk (whole segments, at most MAX_CHUNK) whose layout fits ws_bytes; 0 if not even one
static long long efdm_chunk(long long total_segs, long long L, bool idx, size_t ws_bytes) {
    long long lo = 0, hi = std::min(total_segs, MAX_CHUNK);
    while (lo < hi) {
        const long long m = (lo + hi + 1) / 2;
        if (efdm_layout(m, L, idx).total <= ws_bytes) lo = m; else hi = m - 1;
    }
    return lo;
}

// R NULL: the plain state.  R (fp32 C x C, C % RC == 0): the sorted values of R y, the state of a sliced step.
int launch_efdm_style_prepare(const __half* style, int Ns, int Hs, int Ws, int C, const float* R, float* state, void* ws,
                              size_t ws_bytes, cudaStream_t st) {
    const long long total = (long long)Ns * C, L = (long long)Hs * Ws;
    const long long S = efdm_chunk(total, L, false, ws_bytes);
    if (S < 1) {
        set_error("efdm_style_prepare: workspace %zu < %zu bytes (one segment)", ws_bytes, efdm_layout(1, L, false).total);
        return WCTB200_EWS;
    }
    const ActGeom g(Ns, Hs, Ws, C);
    uint8_t* b = static_cast<uint8_t*>(ws);
    for (long long s0 = 0; s0 < total; s0 += S) {
        const int n = (int)std::min(S, total - s0);
        const EfdmWs w = efdm_layout(n, L, false);
        unsigned int* kA = reinterpret_cast<unsigned int*>(b + w.kA);
        if (R) {
            k_efdm_rotate_keys<<<dim3(cdiv(L, RP), (unsigned)((s0 + n - 1) / RC - s0 / RC + 1)), 256, 0, st>>>(style, nullptr, g, R,
                                                                                                           s0, n, kA);
            WCTB_CHECK_LAUNCH("k_efdm_rotate_keys");
        } else {
            k_efdm_keys<<<dim3(cdiv(L, TP), cdiv(n, TS)), 256, 0, st>>>(style, g, s0, n, kA);
            WCTB_CHECK_LAUNCH("k_efdm_keys");
        }
        int rc = efdm_sort(kA, reinterpret_cast<unsigned int*>(b + w.kB), nullptr, nullptr, n, (int)L,
                           reinterpret_cast<unsigned int*>(b + w.hist), st);
        if (rc) return rc;
        const long long cnt = n * L;
        k_efdm_decode<<<(unsigned)std::min<long long>(cdiv(cnt, 256), (long long)device_sm_count() * 16), 256, 0, st>>>(
            kA, cnt, state + s0 * L);
        WCTB_CHECK_LAUNCH("k_efdm_decode");
    }
    return 0;
}

// alpha = 0: the content's own bytes, with the reflect halo
static int efdm_copy(const __half* content, const ActGeom& g, __half* out, cudaStream_t st) {
    const long long total = (long long)g.N * g.H * g.W * (g.C / 8);
    k_efdm_copy<<<(unsigned)std::min<long long>(cdiv(total, 256), (long long)device_sm_count() * 16), 256, 0, st>>>(content, g, out);
    WCTB_CHECK_LAUNCH("k_efdm_copy");
    return 0;
}

// The content side of one EFDM pass over the N*C segments, as many whole segments at a time as ws holds.  The keys are the
// content's own values (G NULL) or those of G v (v from the SPF16 `content`, or from fp32 planes `src` when not NULL).  The
// run values go to fp32 planes `out_planes` at alpha = 1, or to SPF16 `out` blended with the keys' values (plain EFDM) or,
// for a sliced step, with `content`.
static int efdm_content_pass(const __half* content, const float* src, const float* G, const ActGeom& g, const float* state,
                             int Ns, int Ms, float alpha, float* out_planes, __half* out, void* ws, size_t ws_bytes,
                             cudaStream_t st) {
    const int C = g.C;
    const long long total = (long long)g.N * C, L = (long long)g.H * g.W;
    const long long S = efdm_chunk(total, L, true, ws_bytes);
    if (S < 1) {
        set_error("efdm_apply: workspace %zu < %zu bytes (one segment)", ws_bytes, efdm_layout(1, L, true).total);
        return WCTB200_EWS;
    }
    const int T = cdiv(L, TILE);
    uint8_t* b = static_cast<uint8_t*>(ws);
    for (long long s0 = 0; s0 < total; s0 += S) {
        const int n = (int)std::min(S, total - s0);
        const EfdmWs w = efdm_layout(n, L, true);
        unsigned int* kA = reinterpret_cast<unsigned int*>(b + w.kA);
        unsigned int* kB = reinterpret_cast<unsigned int*>(b + w.kB);
        unsigned int* iA = reinterpret_cast<unsigned int*>(b + w.iA);
        double* tsum = reinterpret_cast<double*>(b + w.tsum);
        double* P = reinterpret_cast<double*>(b + w.P);
        if (G) {
            k_efdm_rotate_keys<<<dim3(cdiv(L, RP), (unsigned)((s0 + n - 1) / RC - s0 / RC + 1)), 256, 0, st>>>(content, src, g, G, s0,
                                                                                                           n, kA);
            WCTB_CHECK_LAUNCH("k_efdm_rotate_keys");
        } else {
            k_efdm_keys<<<dim3(cdiv(L, TP), cdiv(n, TS)), 256, 0, st>>>(content, g, s0, n, kA);
            WCTB_CHECK_LAUNCH("k_efdm_keys");
        }
        int rc = efdm_sort(kA, kB, iA, reinterpret_cast<unsigned int*>(b + w.iB), n, (int)L,
                           reinterpret_cast<unsigned int*>(b + w.hist), st);
        if (rc) return rc;
        EfdmQ E{state, C, Ns, Ms, (int)L, s0};
        k_efdm_qsum<<<dim3(T, n), THREADS, 0, st>>>(E, T, tsum);
        WCTB_CHECK_LAUNCH("k_efdm_qsum");
        k_efdm_qscan<<<cdiv(n, 128), 128, 0, st>>>(tsum, T, n);
        WCTB_CHECK_LAUNCH("k_efdm_qscan");
        k_efdm_prefix<<<dim3(T, n), THREADS, 0, st>>>(E, T, tsum, P);
        WCTB_CHECK_LAUNCH("k_efdm_prefix");
        // the run values: into the planes, or into kB, free after the sort (an even number of passes ends in kA)
        float* vals = out_planes ? out_planes + s0 * L : reinterpret_cast<float*>(kB);
        k_efdm_runs<<<dim3(T, n), THREADS, 0, st>>>(kA, iA, P, (int)L, T, G ? 1.0f : alpha, vals);
        WCTB_CHECK_LAUNCH("k_efdm_runs");
        if (out_planes) continue;
        if (G) {
            k_efdm_store<true><<<dim3(cdiv(L, TP), cdiv(n, TS)), 256, 0, st>>>(vals, g, s0, n, out, content, alpha);
        } else {
            k_efdm_store<false><<<dim3(cdiv(L, TP), cdiv(n, TS)), 256, 0, st>>>(vals, g, s0, n, out, nullptr, 0.f);
        }
        WCTB_CHECK_LAUNCH("k_efdm_store");
    }
    return 0;
}

int launch_efdm_apply(const __half* content, int N, int H, int W, int C, const float* state, int Ns, int Hs, int Ws, float alpha,
                      __half* out, void* ws, size_t ws_bytes, cudaStream_t st) {
    const ActGeom g(N, H, W, C);
    if (alpha == 0.f) return efdm_copy(content, g, out, st);
    return efdm_content_pass(content, nullptr, nullptr, g, state, Ns, Hs * Ws, alpha, nullptr, out, ws, ws_bytes, st);
}

size_t efdm_planes_bytes(int C, int N, int H, int W) { return efdm_align((size_t)N * C * H * W * sizeof(float)); }

// one step of the sliced chain: m = EFDM(G v, state) at alpha = 1, v = the SPF16 `content` (src NULL) or the planes `src`;
// m goes to `out_planes`, or (out_planes NULL) alpha m + (1 - alpha) content goes to SPF16 `out`
int launch_efdm_sliced_step(const __half* content, const float* src, int N, int H, int W, int C, const float* G, const float* state,
                            int Ns, int Hs, int Ws, float alpha, float* out_planes, __half* out, void* ws, size_t ws_bytes,
                            cudaStream_t st) {
    const ActGeom g(N, H, W, C);
    if (!out_planes && alpha == 0.f) return efdm_copy(content, g, out, st);
    return efdm_content_pass(content, src, G, g, state, Ns, Hs * Ws, alpha, out_planes, out, ws, ws_bytes, st);
}

}  // namespace wctb
