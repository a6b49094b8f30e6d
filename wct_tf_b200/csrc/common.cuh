// Shared device/host helpers for libwctb200 (sm_90a only).
#pragma once

#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>

#include "../../include/wctb200.h"

namespace wctb {

// ---------------------------------------------------------------------------
// host-side error plumbing
// ---------------------------------------------------------------------------
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);
// device error word (set by kernels on pipeline time-outs)
unsigned int* device_error_word();

#define WCTB_CUDA(call)                                        \
    do {                                                       \
        cudaError_t _e = (call);                               \
        if (_e != cudaSuccess) return ::wctb::cuda_fail(_e, #call); \
    } while (0)

#define WCTB_CHECK_LAUNCH(name)                                \
    do {                                                       \
        cudaError_t _e = cudaGetLastError();                   \
        if (_e != cudaSuccess) return ::wctb::cuda_fail(_e, name); \
    } while (0)

#define WCTB_REQUIRE(cond, ...)                                \
    do {                                                       \
        if (!(cond)) {                                         \
            ::wctb::set_error(__VA_ARGS__);                    \
            return WCTB200_EINVAL;                             \
        }                                                      \
    } while (0)

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// Per-DEVICE one-time kernel attribute: cudaFuncSetAttribute applies to the current device only, so the
// "already done" state is one bit per device ordinal (a process may drive several GPUs: WCT(device='/gpu:1')
// after '/gpu:0').  The kernel argument may contain commas: wrap it in parentheses.
#define WCTB_ENSURE_SMEM(kernel, bytes)                                                                  \
    do {                                                                                                 \
        static std::atomic<unsigned long long> _done{0ull};                                              \
        int _dev = 0;                                                                                    \
        WCTB_CUDA(cudaGetDevice(&_dev));                                                                 \
        const unsigned long long _bit = 1ull << (_dev & 63);                                             \
        if (!(_done.load(std::memory_order_acquire) & _bit)) {                                           \
            WCTB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes))); \
            _done.fetch_or(_bit, std::memory_order_release);                                             \
        }                                                                                                \
    } while (0)
// SM count of the CURRENT device (cached per device ordinal)
int device_sm_count();

// ---------------------------------------------------------------------------
// SPF16 geometry
// ---------------------------------------------------------------------------
// Halo written by a producer, per axis: the interior row that feeds padded row 0 (ht) and the one that feeds padded row
// H+1 (hb), and the interior columns that feed padded columns 0 (wl) and W+1 (wr).
//   REFLECT (ops.py:12-15, the default): 1 and H-2;  EDGE (input of an UP2 conv, WCTB200_HALO_EDGE): 0 and H-1;
//   WRAP (seamless stylisation, WCTB200_HALO_WRAP_X / _Y): H-1 and 0 -- a wrapped axis wraps whatever else is set.
// Corner cells follow from the two axes.  In every mode the cell a pixel feeds sits as many rows above it (row 0) as below
// it (row H+1): ht+1 = H-hb (reflect 2, edge 1, wrap H).
struct ActGeom {
    int N, H, W, C;
    int Hp, Wp;          // H+2, W+2
    int ht, hb, wl, wr;  // interior sources of the halo rows / columns (above)
    long long P;         // N*Hp*Wp padded positions
    long long plane;     // P*C elements per plane
    __host__ __device__ ActGeom() {}
    __host__ __device__ ActGeom(int n, int h, int w, int c)
        : N(n), H(h), W(w), C(c), Hp(h + 2), Wp(w + 2), ht(1), hb(h - 2), wl(1), wr(w - 2) {
        P = (long long)N * Hp * Wp;
        plane = P * C;
    }
    // halo mode from conv flags: WCTB200_HALO_EDGE and the wrap bits (other bits are ignored)
    __host__ __device__ void set_halo(int flags) {
        const bool edge = (flags & WCTB200_HALO_EDGE) != 0;
        if (flags & WCTB200_HALO_WRAP_Y) { ht = H - 1; hb = 0; }
        else if (edge) { ht = 0; hb = H - 1; }
        if (flags & WCTB200_HALO_WRAP_X) { wl = W - 1; wr = 0; }
        else if (edge) { wl = 0; wr = W - 1; }
    }
};

#ifdef __CUDACC__
// ---------------------------------------------------------------------------
// split-pair fp16
// ---------------------------------------------------------------------------
__device__ __forceinline__ void split_f32(float x, __half& hi, __half& lo) {
    x = fminf(fmaxf(x, -65000.f), 65000.f);   // keep hi finite
    hi = __float2half_rn(x);
    lo = __float2half_rn(x - __half2float(hi));
}
// exponent S of the power of two that puts a max |value| (as float bits) into [512, 1024), 0 for 0 / NaN: the split of the
// scaled values keeps every lo that matters a normal fp16 number (DESIGN.md §3.1).  Conv weights (layers.cu, weight_scale)
// and the rows of the apply operand (wct.cu: k_finalize_transform) are stored with it.
__device__ __forceinline__ int weight_scale_exp(unsigned int absmax_bits) {
    const float amax = __uint_as_float(absmax_bits);
    if (!(amax > 0.f)) return 0;
    int e;
    frexpf(amax, &e);                               // amax = m * 2^e, m in [0.5, 1)
    const int S = 10 - e;                           // amax * 2^S in [512, 1024)
    return S < -14 ? -14 : (S > 40 ? 40 : S);
}
// 2^e exactly, for e in [-126, 127]
__device__ __forceinline__ float pow2i(int e) { return __int_as_float((127 + e) << 23); }
__device__ __forceinline__ float weight_scale(unsigned int absmax_bits) { return exp2f((float)weight_scale_exp(absmax_bits)); }
__device__ __forceinline__ float merge_f32(__half hi, __half lo) { return __half2float(hi) + __half2float(lo); }

// 8 channels = one 16-byte vector per plane
struct alignas(16) Half8 { __half2 v[4]; };

// two fp32 -> (hi pair, lo pair).  cvt.rn.satfinite.f16x2.f32 (F2FP.SATFINITE.F16.F32.PACK_AB) converts, saturates to
// +-65504 and packs two values in ONE instruction: 6 instructions per pair instead of the 11 of two clamped scalar splits
// (the conv epilogue is instruction bound on the short-K layers)
__device__ __forceinline__ void split2(float a, float b, __half2& hi, __half2& lo) {
    unsigned int h, l;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(h) : "f"(b), "f"(a));       // a -> low half, b -> high half
    hi = *reinterpret_cast<__half2*>(&h);
    const float2 hf = __half22float2(hi);
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(l) : "f"(b - hf.y), "f"(a - hf.x));
    lo = *reinterpret_cast<__half2*>(&l);
}
__device__ __forceinline__ void split8(const float* x, Half8& hi, Half8& lo) {
#pragma unroll
    for (int i = 0; i < 4; ++i) split2(x[2 * i], x[2 * i + 1], hi.v[i], lo.v[i]);
}
__device__ __forceinline__ void merge8(const Half8& hi, const Half8& lo, float* x) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float2 a = __half22float2(hi.v[i]);
        float2 b = __half22float2(lo.v[i]);
        x[2 * i] = a.x + b.x;
        x[2 * i + 1] = a.y + b.y;
    }
}

// Destinations of interior pixel (y,x) in the reflect-padded plane (ops.py:12-15):
// the pixel itself at (y+1,x+1) plus the halo cells that mirror it.
// rows[] / cols[] receive padded coordinates; returns counts.
__device__ __forceinline__ int halo_rows(int y, int H, int* rows) {
    int n = 0;
    rows[n++] = y + 1;
    if (y == 1) rows[n++] = 0;
    if (y == H - 2) rows[n++] = H + 1;
    return n;
}

// store one 8-channel group (hi+lo) of pixel (n,y,x) to every padded cell that holds it.
// Interior pixels (the overwhelming majority) take the fast path: one address, two 16-byte stores.  (The first version
// evaluated all 9 candidate cells with predicated stores for EVERY pixel: 18 STG + ~26 IMAD per call, which made the
// epilogue of the 64-channel convs -- not their operand traffic -- the bound: 9.4k cycles per 128x64 tile, measured
// identical for 9 and for 4 k-iterations per tile.)
__device__ __forceinline__ void store8_with_halo(__half* __restrict__ act, const ActGeom& g, int n, int y, int x,
                                                 int c0, const Half8& hi, const Half8& lo) {
    // padded row 0 holds interior row g.ht, row H+1 holds row g.hb (ActGeom: reflect, edge or wrap); columns likewise
    __half* p0 = act + (((long long)n * g.Hp + y + 1) * g.Wp + x + 1) * g.C + c0;
    *reinterpret_cast<Half8*>(p0) = hi;
    *reinterpret_cast<Half8*>(p0 + g.plane) = lo;
    const bool yt = (y == g.ht), yb = (y == g.hb), xl = (x == g.wl), xr = (x == g.wr);
    if (!(yt | yb | xl | xr)) return;
    const long long pitch = (long long)g.Wp * g.C;
    // element offsets from the pixel's own cell to the halo row / column that mirrors it (0 = none)
    const long long dy[3] = {0, yt ? -(long long)(y + 1) * pitch : 0, yb ? (long long)(g.H - y) * pitch : 0};
    const long long dx[3] = {0, xl ? -(long long)(x + 1) * g.C : 0, xr ? (long long)(g.W - x) * g.C : 0};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        if (a && dy[a] == 0) continue;
#pragma unroll
        for (int b = 0; b < 3; ++b) {
            if ((b && dx[b] == 0) || (a == 0 && b == 0)) continue;
            __half* q = p0 + dy[a] + dx[b];
            *reinterpret_cast<Half8*>(q) = hi;
            *reinterpret_cast<Half8*>(q + g.plane) = lo;
        }
    }
}

// Epilogue variant: the pixel's padded position `ppos` = (n*Hp + y+1)*Wp + x+1 (fits 31 bits) and its border flags
// (bit0: the pixel feeds padded row 0, bit1: row H+1, bit2: column 0, bit3: column W+1) were computed ONCE by the thread
// that owns the pixel; the 8 lanes that store its channels only add the channel offset.
__device__ __forceinline__ int halo_flags(const ActGeom& g, int y, int x) {
    return (y == g.ht ? 1 : 0) | (y == g.hb ? 2 : 0) | (x == g.wl ? 4 : 0) | (x == g.wr ? 8 : 0);
}
__device__ __forceinline__ void store8_at(__half* __restrict__ act, const ActGeom& g, unsigned int ppos, int flags, int c0,
                                          const Half8& hi, const Half8& lo) {
    __half* p0 = act + (long long)ppos * g.C + c0;
    *reinterpret_cast<Half8*>(p0) = hi;
    *reinterpret_cast<Half8*>(p0 + g.plane) = lo;
    if (flags == 0) return;
    // the cell sits ht+1 rows above the pixel (row 0) or as many below it (row H+1; ActGeom); columns likewise
    const long long pitch = (long long)g.Wp * g.C;
    const long long ry = g.ht + 1, rx = g.wl + 1;
    const long long dy[3] = {0, (flags & 1) ? -ry * pitch : 0, (flags & 2) ? ry * pitch : 0};
    const long long dx[3] = {0, (flags & 4) ? -rx * g.C : 0, (flags & 8) ? rx * g.C : 0};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        if (a && dy[a] == 0) continue;
#pragma unroll
        for (int b = 0; b < 3; ++b) {
            if ((b && dx[b] == 0) || (a == 0 && b == 0)) continue;
            __half* q = p0 + dy[a] + dx[b];
            *reinterpret_cast<Half8*>(q) = hi;
            *reinterpret_cast<Half8*>(q + g.plane) = lo;
        }
    }
}

// index of padded image coordinate i (-1..n) on an axis of n pixels: reflect (ops.py:12-15) or, with wrap, circular
__device__ __forceinline__ int pad_index(int i, int n, bool wrap) {
    return i < 0 ? (wrap ? i + n : -i) : (i >= n ? (wrap ? i - n : 2 * n - 2 - i) : i);
}

__device__ __forceinline__ void load8(const __half* __restrict__ act, const ActGeom& g, long long pos, int c0,
                                      float* x) {
    long long off = pos * g.C + c0;
    Half8 hi = *reinterpret_cast<const Half8*>(act + off);
    Half8 lo = *reinterpret_cast<const Half8*>(act + g.plane + off);
    merge8(hi, lo, x);
}

// ---------------------------------------------------------------------------
// Coalesced tile store for the GEMM epilogues.  Each epilogue thread owns one output
// position (row) and NACC consecutive channels in registers.  Writing them directly puts
// 16-byte fragments 128+ bytes apart (ncu: 27 half-filled sectors per store request, the
// 64-channel convs were bound by L2 write requests).  Instead every warp transposes
// 64 channels at a time through an 8 KB shared-memory staging buffer (XOR-swizzled, conflict
// free) so that 8 consecutive lanes write one position's 128 contiguous bytes per plane.
//   stg: this warp's private 8 KB buffer; value = acc*oscale + sbias (oscale undoes the power-of-two weight scale);
//   sbias: bias of acc[0..NACC); cbase: channel of acc[0]
// ---------------------------------------------------------------------------
template <int NACC>
__device__ __forceinline__ void store_tile_rows(const float (&acc)[NACC], const float oscale, const float* __restrict__ sbias, bool relu,
                                                uint8_t* __restrict__ stg, int lane, unsigned int ppos, int flags,
                                                __half* __restrict__ out, const ActGeom& go, int cbase) {
    // flags < 0: this thread's position is not an interior pixel (halo / junk row of the padded tiling): nothing is stored
#pragma unroll
    for (int h = 0; h < NACC / 64; ++h) {
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            float v[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float t = fmaf(acc[h * 64 + q * 8 + j], oscale, sbias[h * 64 + q * 8 + j]);
                v[j] = relu ? fmaxf(t, 0.f) : t;
            }
            Half8 hi, lo;
            split8(v, hi, lo);
            const int slot = q ^ (lane & 7);
            *reinterpret_cast<Half8*>(stg + (lane * 8 + slot) * 16) = hi;
            *reinterpret_cast<Half8*>(stg + 4096 + (lane * 8 + slot) * 16) = lo;
        }
        __syncwarp();
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int row = j * 4 + (lane >> 3);
            const int c = lane & 7;
            const unsigned int pp = __shfl_sync(0xffffffffu, ppos, row);
            const int fl = __shfl_sync(0xffffffffu, flags, row);
            const int slot = c ^ (row & 7);
            const Half8 hi = *reinterpret_cast<const Half8*>(stg + (row * 8 + slot) * 16);
            const Half8 lo = *reinterpret_cast<const Half8*>(stg + 4096 + (row * 8 + slot) * 16);
            if (fl >= 0) store8_at(out, go, pp, fl, cbase + h * 64 + c * 8, hi, lo);
        }
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------
// fp32 pairs: sm_90 has no packed fp32 FMA, so a pair is two scalar fmaf (round-to-nearest, same result per element)
// ---------------------------------------------------------------------------
typedef float2 f32x2;
__device__ __forceinline__ f32x2 pack2(float a, float b) { return make_float2(a, b); }
__device__ __forceinline__ void unpack2(f32x2 v, float& a, float& b) { a = v.x; b = v.y; }
__device__ __forceinline__ f32x2 fma2(f32x2 a, f32x2 b, f32x2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
struct alignas(16) f32x2x2 { f32x2 x, y; };       // a float4 viewed as two pairs

// ---------------------------------------------------------------------------
// PTX wrappers: mbarrier / TMA / wgmma (sm_90a)
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
#ifdef WCTB_MBAR_TEST_WAIT
        "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
#else
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
#endif
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a pipeline bug must not hang the GPU.  After ~2 s the CTA-wide abort
// flag is raised (all later waits fall through) and the global error word is set.
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, volatile int* abort_flag,
                                          unsigned int* err_word, unsigned int code) {
    if (mbar_try_wait(bar, parity)) return;
    // The time-out clock is the SM cycle counter: reading %globaltimer costs ~0.5 us (measured: every wait that
    // missed its first poll paid it, which capped the tap-reuse conv pipelines at ~1 us per k-iteration).
    const long long t0 = clock64();
    for (unsigned int it = 1;; ++it) {
        if (mbar_try_wait(bar, parity)) return;
        if ((it & 255u) == 0u) {
            if (*abort_flag) return;
            if (*reinterpret_cast<volatile unsigned int*>(err_word)) { *abort_flag = 1; return; }
            if (clock64() - t0 > 4000000000ll) break;            // >= 2 s at <= 2 GHz
        }
    }
    *abort_flag = 1;
    atomicExch(err_word, code);
}

__device__ __forceinline__ void tma_prefetch_desc(const void* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const void* map, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}

// ---- warpgroup MMA (sm_90a): D[64 x N] (+)= A[64 x 16] * B[16 x N], fp16 inputs, fp32 accumulators in registers.
// Issued by all 128 threads of a warpgroup (4 consecutive warps starting at a multiple of 4).  Accumulator fragment of
// thread t of the warpgroup: rows 16*(t/32) + (t%32)/4 (+8), columns 8j + 2*(t%4) (+1), d[4j..4j+3] =
// (r, c), (r, c+1), (r+8, c), (r+8, c+1)  (PTX ISA, "wgmma .m64nNk16 register fragment D").
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// register budget of a warpgroup (producer warpgroups give theirs to the MMA warpgroups)
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMA window
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// K-major, 128B-swizzled shared-memory operand descriptor (tile rows are 128 bytes = 64 fp16 of K; 8-row groups
// 1024 B apart; the tile base is 1024-byte aligned).  Bit layout: sm_90 GMMA descriptor (start >> 4 at [0,14),
// LBO >> 4 at [16,30), SBO >> 4 at [32,46), layout type at [62,64): 1 = SWIZZLE_128B).  A 16-wide k-step inside the
// 128-byte row advances the start address by 32 bytes.  The swizzle follows the absolute shared-memory address, so an
// operand may also start at any 128-byte row of a swizzled tile (the conv's column taps, 0..15 rows into a strip) with
// the base-offset field [49,52) left 0.  Measured on an H100 with a wgmma m64n64k16 at row offsets 0..79 of a swizzled
// tile: base offset 0 gave the exact product at every offset; (start >> 7) & 7 there was wrong at every offset that is
// not a multiple of 8.  tests/test_gpu_conv_strip.py runs the conv at every row residue.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)1 << 16;                       // LBO (unused for swizzled K-major)
    d |= (uint64_t)(1024 >> 4) << 32;             // SBO = 1024 B
    d |= (uint64_t)1 << 62;                       // SWIZZLE_128B
    return d;
}
// MN-major SWIZZLE_128B operand (used when the contraction index is the slow one: covariance X^T X, true products A B):
// 64 MN elements (128 B) per row, rows = K; LBO = stride between 64-wide MN groups (8 KB: the next slice),
// SBO = stride between 8-row K groups (1 KB)  (canonical layout ((64,n),(8,k)) : ((1,LBO),(64,SBO)) in elements)
__device__ __forceinline__ uint64_t gmma_desc_mn_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)((8192 >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((1024 >> 4) & 0x3FFF) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

// TA / TB: 0 = K-major operand, 1 = MN-major (transposed) operand
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, %32, %33, p, 1, 1, %35, %36;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, %64, %65, p, 1, 1, %67, %68;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate), "n"(TA), "n"(TB));
}


// accumulator fragments of a 64-row warpgroup slice -> row-major fp32 tile in shared memory (tile[row * pitch + col])
template <int R>
__device__ __forceinline__ void frag_to_tile(const float (&d)[R], float* tile, int pitch, int row0, int t) {
    const int r = row0 + 16 * (t >> 5) + ((t & 31) >> 2);
    const int c = 2 * (t & 3);
#pragma unroll
    for (int j = 0; j < R / 4; ++j) {
        *reinterpret_cast<float2*>(tile + r * pitch + 8 * j + c) = make_float2(d[4 * j], d[4 * j + 1]);
        *reinterpret_cast<float2*>(tile + (r + 8) * pitch + 8 * j + c) = make_float2(d[4 * j + 2], d[4 * j + 3]);
    }
}
// Weight of transform k at pixel pix of frame n in the weighted apply (soft spatial control, DESIGN.md §3.3.11):
// v = s(p) w_k(p), with w = 1 without weight planes (K = 1) and s = 1 without a strength map; 0 for a skipped problem
// (k_c = -1).  wts [N][K][H][W], str [N][H][W], kc [N*K].
__device__ __forceinline__ float soft_weight(const float* __restrict__ wts, const float* __restrict__ str, const int* __restrict__ kc,
                                             int K, int n, int k, long long HW, long long pix) {
    if (kc[n * K + k] < 0) return 0.f;
    float v = wts ? __ldg(wts + ((long long)n * K + k) * HW + pix) : 1.f;
    if (str) v = __ldg(str + (long long)n * HW + pix) * v;
    return v;
}
#endif  // __CUDACC__

// per-(device, stream, slot) grow-only scratch buffer (capi.cu); valid until the next call with the same key
int scratch_alloc(void** ptr, size_t bytes, cudaStream_t st, int slot);

// ---------------------------------------------------------------------------
// kernel launchers implemented in the .cu files (host API used by capi.cu)
// ---------------------------------------------------------------------------
enum ConvMode { CONV_3X3 = 0, CONV_APPLY = 1, CONV_UP2 = 2, CONV_TAPS = 3 };
int launch_conv_tc(int mode, const __half* in, int N, int H, int W, int Cin, const __half* w_split, int nsets,
                   const float* wscale, const float* bias, int Cout, int flags, __half* out, cudaStream_t st, int kw = 3);
// out = M_n x + bias_n with row i of M_n stored times 2^rexp[n][i] (k_finalize_transform; rexp nullptr: all 0)
int launch_conv_apply(const __half* in, int N, int H, int W, int C, const __half* w_split, int nsets, const int* rexp,
                      const float* bias, __half* out, cudaStream_t st);
int conv_tc_bn(int Cout);
int launch_conv_taps_rows(const __half* in, int N, int H, int W, int Cin, const __half* w_split, long long wplane, int Cout, int bn,
                          __half* out, cudaStream_t st, int kw);
// statistics record of N frames (tiled stylisation; wctb200_stats_record_layout): fp64 n [N], t [N][C], s [N][C],
// S [N][C][C] (covariance) or [N][C] (AdaIN's moments: the diagonal)
struct StatsRecord { double *n, *t, *s, *S; };
// trailer of a prepared weight buffer: [0] = 1/scale (float), see wctb200_prep_conv_weights
static inline const float* weight_scale_ptr(const __half* w_split, int taps_total, int Cin, int Cout) {
    return reinterpret_cast<const float*>(w_split + (size_t)2 * taps_total * Cin * Cout);
}

}  // namespace wctb
