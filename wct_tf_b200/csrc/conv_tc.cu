// Conv2DReflect 3x3, the 1x1 "apply" of the feature transform, and UpSampling2D+Conv2DReflect as ONE conv,
// all as an implicit GEMM on the tensor cores (Hopper wgmma, TMA-fed).
//
//   reference: Lambda(pad_reflect) -> Conv2D(valid) (+ReLU)   ops.py:12-19,
//              vgg_normalised.py:28-40, model.py:291; the whitening/colouring
//              apply  M * fc  of ops.py:73,77 (mode APPLY); and
//              UpSampling2D() -> Conv2DReflect of model.py:291-293 (mode UP2).
//
// Formulation.  Activations are SPF16: two fp16 planes (hi, lo) of the padded
// NHWC tensor, viewed as a 2-D matrix [P = N*(H+2)*(W+2) padded positions][C].  For an
// output position p (padded coordinates) and filter tap (ky,kx) the input row is simply
// p + (ky-1)*(W+2) + (kx-1): each tap of a 128-position output tile is ONE dense
// 128 x 64 block of rows at a shifted row coordinate (rows outside [0,P) are zero-filled by
// TMA and only feed halo/junk outputs, which the epilogue never stores).
//
//   D[128 pos][BN cout] = sum_{tap, cin-slice}  A_tap[128][64] * W_tap[BN][64]^T
//
// Activation strips.  The column taps kx = 0, 1, 2 of filter row ky read the same rows shifted by one, so ONE TMA box of
// 128 + 2 rows per (filter row, 64-channel slice) feeds all three: column tap kx is a wgmma operand that starts kx rows
// (128*kx bytes) into the 128B-swizzled strip.  A k-iteration then loads only its tap's weights; the strip is loaded once
// per ncol k-iterations (3x3: 3, UP2: 2, TAPS: kw, APPLY: 1).  3x3 operand bytes per k-iteration: 64 KB -> 43 KB at
// BN = 128, 48 KB -> 27 KB at BN = 64.
//
// UP2 (nearest x2 upsampling folded into the conv that follows it).  Output pixel (2i+a, 2j+b) of
// conv3x3(reflect_pad(upsample2(L))) only ever reads the 2x2 low-resolution neighbourhood
// rows {i-1+a, i+a} x cols {j-1+b, j+b} of L, because two of the three filter rows (columns) land on the same
// low-resolution row (column): a = 0 -> {w[-1]} on row i-1 and {w[0]+w[1]} on row i; a = 1 -> {w[-1]+w[0]} on
// row i and {w[1]} on row i+1.  So each of the 4 output parities is a 2x2-tap conv over L with pre-summed
// weights (wctb200_prep_conv_weights_up2): 16 instead of 36 tap-products per low-resolution pixel (4/9 of the
// MACs), and the 4x larger upsampled tensor is never written or read.  At the border the reflect padding of the
// UPSAMPLED image mirrors onto the same low-resolution pixel (u[-1] = u[1] = L[0]), i.e. L needs an EDGE-replicated
// halo: its producer is launched with WCTB200_HALO_EDGE.  Under circular padding (seamless stylisation) u[-1] = u[2W-1] =
// L[W-1], the WRAPPED low-resolution halo: WCTB200_HALO_WRAP_X / _Y override the edge halo on their axis.
//
// Precision.  fp32-class accuracy from fp16 tensor-core inputs: x = x_hi + x_lo,
//   x*w ~= x_hi*w_hi + x_hi*w_lo + x_lo*w_hi     (3 x wgmma f16 x f16, fp32 accumulate in registers)
// the dropped lo*lo term is 2^-22 relative.  Weights are stored SCALED by a per-layer power of two
// (max|w| -> [512,1024), undone exactly in the epilogue): He-initialised / trained conv weights are ~1e-2, so the
// unscaled lo plane (~5e-6) fell into the fp16 subnormals and kept only ~16 bits of the weight -- measured as
// 8x the reference's own fp32 noise on the free-running 5-level image (tests/noise_split_cpu.py).
//
// Structure (persistent CTAs, 384 threads):
//   warp 8    : TMA producer   (cp.async.bulk.tensor 3-D, 128B swizzle, mbarrier complete_tx)
//   warps 0-7 : two wgmma warpgroups (64 tile rows each); each hands its finished fp32 tile rows over in shared memory and
//               goes straight on to the next tile's mainloop
//   warps 9-11: the epilogue (*scale +bias, ReLU -> split fp16 -> 16-byte stores of the interior pixel AND the halo cells
//               that mirror it), overlapped with the next tile's mainloop
#include "common.cuh"

namespace wctb {

extern int g_conv_bn_override;

struct ConvParams {
    int N, H, W, Cin, Cout, Hp, Wp;   // INPUT geometry (UP2: the low-resolution tensor)
    long long P;
    int mode;             // ConvMode
    int taps;             // 9 (3x3), 1 (apply), 4 (up2: per output parity), kw*kw (taps)
    int kw;               // CONV_TAPS: filter width (top-left anchored kw x kw correlation, style-swap patches)
    int ncol;             // column taps per filter row, all fed from one strip: 3 (3x3), 2 (up2), kw (taps), 1 (apply)
    int strip_rows;       // rows of one strip box: 127 + ncol (pool: 66 per segment)
    int products;         // 3 (default): a_hi b_hi + a_hi b_lo + a_lo b_hi; 2: without a_lo b_hi; 1: a_hi b_hi only (experiment knob)
    int per_image;        // tiles never straddle images; weight/bias set = image index (APPLY with nsets > 1)
    int pool;             // CONV_3X3 + WCTB200_POOL2: M tile = 2 image rows x 64 columns, 2x2 max-pool in the epilogue
    int pool_tx, pool_ho; // pool: column segments per row pair, row pairs per image
    int nsets;
    int tiles_per_image;
    int flags;
    ActGeom go;           // OUTPUT geometry with its halo mode, made on the host: the epilogue reads it from the parameter bank
    const float* bias;    // [nsets][Cout] or nullptr
    const float* wscale;  // device scalar: 1 / (power-of-two scale the weights were stored with), or nullptr (= 1)
    const int* rexp;      // CONV_APPLY: [nsets][Cout], row i of set n stored times 2^rexp (k_finalize_transform), or nullptr (0)
    __half* out;          // SPF16, Cout channels; UP2: [N, 2H, 2W, Cout]
    unsigned int* err;
    // regions apply (conv_tc2_kernel<.., REG = true>, spatial control): weight/bias set = image * R + region
    const __half* in;     // the input activation (pixels outside every styled region are copied from it)
    const uint8_t* labels;// [N][H][W] region label per pixel
    const int* counts;    // [N*R] pixels per (image, region); a region with fewer than 2 pixels keeps its input
    const uint16_t* amask;// [m_tiles]: bit r set when the tile holds a pixel of region r, bit R when it holds a kept pixel
    int R;
    // weighted apply (conv_tc2_kernel<.., REG, WGT = true>, soft spatial control): R = K transforms per image, pixel weights
    // soft_weight(wts, str, kc, ...); amask bit k: a pixel of the tile has v_k > 0, bit K: one has every v_k = 0
    const float* wts;     // [N][K][H][W] or nullptr (K = 1, weight 1)
    const float* str;     // [N][H][W] strength or nullptr (1)
    const int* kc;        // [N*K] k_c of each transform, -1 = skipped
};

// v_k at row `row` of an APPLY tile (0 on halo and junk rows)
__device__ __forceinline__ float row_weight(const ConvParams& p, long long p0, long long p_end, int row, int k) {
    const unsigned int pos = (unsigned int)p0 + (unsigned int)row;
    if (pos >= (unsigned int)p_end) return 0.f;
    const unsigned int hpwp = (unsigned int)(p.Hp * p.Wp);
    const unsigned int n = pos / hpwp;
    const unsigned int r = pos - n * hpwp;
    const int yy = (int)(r / (unsigned int)p.Wp);
    const int xx = (int)(r - (unsigned int)yy * (unsigned int)p.Wp);
    if (yy < 1 || yy > p.H || xx < 1 || xx > p.W) return 0.f;
    return soft_weight(p.wts, p.str, p.kc, p.R, (int)n, k, (long long)p.H * p.W, (long long)(yy - 1) * p.W + (xx - 1));
}

// region a pixel takes in the regions apply: its label, or R (keep the input) for labels >= R and regions of < 2 pixels
__device__ __forceinline__ int region_of(const uint8_t* labels, const int* counts, int R, int n, int H, int W, int y, int x) {
    const int l = labels[((long long)n * H + y) * W + x];
    return (l < R && counts[n * R + l] >= 2) ? l : R;
}

// ===========================================================================
// Persistent CTAs, warp-specialised (384 threads):
//   warps 0-7: two consumer warpgroups.  Warpgroup w multiplies rows [64w, 64w + 64) of the 128-position tile with
//              wgmma (m64 x N x k16, both operands K-major and 128B-swizzled, fp32 accumulators in registers), writes its
//              rows of the fp32 tile to shared memory and returns to the mainloop;
//   warps 8-11: producer warpgroup; lane 0 of warp 8 issues the TMA loads, warps 9-11 run the epilogue of the tile the
//              consumers handed over while those already multiply the next one.  setmaxnreg moves registers from this
//              warpgroup to the consumers (the register file is allocated in whole warpgroups: 288 threads would cap every
//              thread at 168).
//   * grid = #SMs x oversubscription, every CTA walks a static tile list (cout tile fastest, so CTAs running together
//     share activation tiles in L2 and the whole weight tensor stays L2 resident);
//   * two operand rings, each with its own full / empty mbarriers: the A ring holds activation strips (BN = 128: 2,
//     BN = 64: 3), the B ring one tap's [b_hi | b_lo] per k-iteration (BN = 128: 2, BN = 64: 4).  k-iterations run in
//     the order (filter row, channel slice, column tap), so a strip is released after its last column tap.  With one
//     channel slice (Cin = 64) this is the tap order of a ring without strips, and the sums are the same bit for bit;
//   * accumulation: the tensor core adds into its fp32 accumulator with truncation.  a_hi b_hi accumulates CH k-iterations
//     at a time into a register chunk that starts from zero and is then added into the running sum with round-to-nearest
//     FADDs; the two small cross products (|a_lo| <= 2^-11 |a|, |b_lo| <= 2^-11 |b|) accumulate in ONE accumulator over
//     the whole K, added once at the end, whose truncation error stays below 2^-24 sum |a||b| for K up to 4608
//     (DESIGN.md §3.1).  So a k-iteration is two wgmma groups, a_hi b_hi then the cross products, and at BN = 64 the
//     cross products of one k-iteration still run while the next one is issued;
//   * tile hand-off: one fp32 tile buffer in shared memory and two mbarriers.  Every consumer warp arrives on tile_full
//     after writing its fragment rows; every epilogue warp arrives on tile_empty after its last read.  A consumer waits
//     on tile_empty only before writing the NEXT tile, a whole mainloop later, so the epilogue runs in the shadow of the
//     mainloop as long as it is the shorter of the two;
//   * epilogue: 8 lanes per output position, 8 consecutive channels per lane read straight from the fp32 tile:
//     scale/bias/ReLU/(pool)/split, then 16-byte stores; the 8 lanes of a position write its 128 contiguous bytes per
//     plane, so the stores stay coalesced without a staging buffer.
// ===========================================================================
template <int BN, bool FUSE_>
struct Conv2Cfg {
    static constexpr int BM = 128;
    static constexpr int BK = 64;
    // A ring: one strip per (filter row, 64-channel slice), both planes.  A plane holds the 128 + ncol - 1 rows that the
    // filter row's column taps read (TAPS: ncol = kw <= 16) or, for POOL2, two segments of 64 + 2 rows, each segment
    // starting on a 1024-byte swizzle atom; 144 rows cover every mode.
    static constexpr int STRIP_ROWS = 144;
    static constexpr int POOL_SEG_ROWS = 72;
    static constexpr int PLANE_BYTES = STRIP_ROWS * 128;
    static constexpr int STRIP_BYTES = 2 * PLANE_BYTES;
    // B ring: one tap's [b_hi | b_lo] per k-iteration
    static constexpr int B_BYTES = BN * BK * 2;
    static constexpr int B_SLOT_BYTES = 2 * B_BYTES;
    static constexpr int A_STAGES = BN == 64 ? 3 : 2;
    static constexpr int B_STAGES = BN == 64 ? 4 : 2;
    // FUSE (BN = 64): the products a_hi*b_hi and a_hi*b_lo share the A operand and the two weight planes sit back to back
    // in a stage, so ONE wgmma with N = 2*BN computes both into adjacent accumulator column ranges (summed when the chunk
    // is added up); a_lo*b_hi follows with N = BN into the first range.  2 instead of 3 wgmma per k-step.
    static constexpr bool FUSE = FUSE_ && BN == 64;
    static constexpr int CHUNK_REGS = FUSE ? BN : BN / 2;       // per-thread fp32 registers of one accumulation chunk
    static constexpr int SUM_REGS = BN / 2;                     // per-thread fp32 registers of the m64 x BN running sum
    static constexpr int CH = 2;                                // k-iterations per accumulation chunk
    // wgmma groups a consumer leaves in flight from one k-iteration into the next.  Measured on the H100 (DESIGN.md §6):
    // BN = 64 is 1-7 % faster with its cross products running while it issues the next k-iteration than drained; BN = 128
    // (two B slots) is 20-40 % slower that way, so it drains every k-iteration
    static constexpr int IN_FLIGHT = BN == 64 ? 1 : 0;
    static constexpr int CONSUMERS = 256;
    static constexpr int THREADS = CONSUMERS + 128;
    static constexpr int EPI_WARPS = 3;                         // warps 9-11 of the producer warpgroup
    static constexpr int NB = BN / 64;                          // 64-channel blocks of a tile row
    // fp32 tile row pitch: BN + 8 makes the consumers' float2 fragment writes conflict free (a half-warp's 4 rows land
    // 8 banks apart); the epilogue reads 256 contiguous bytes of one row per 8 lanes, which no pitch affects
    static constexpr int PITCH = BN + 8;
    static constexpr int TILE_BYTES = BM * PITCH * 4;
    static constexpr int AUX_BYTES = 256 + 4 * BN * 4;          // mbarriers + abort flag, then the bias and scale of two passes
    static constexpr int RING_BYTES = A_STAGES * STRIP_BYTES + B_STAGES * B_SLOT_BYTES;
    static constexpr int SMEM_BYTES = RING_BYTES + AUX_BYTES + TILE_BYTES + 1024;
    static_assert(SMEM_BYTES <= 227 * 1024, "conv: shared memory exceeds the 227 KB opt-in limit");
    static_assert(8 * (2 * A_STAGES + 2 * B_STAGES + 2) + 4 <= 256, "conv: mbarriers overflow the aux block");
};

struct TileCoord {
    long long p0, p_end;
    int n0, set;
    int cls;              // UP2: output parity class a*2+b
};

__device__ __forceinline__ TileCoord tile_coord(const ConvParams& p, int tile, int n_tiles, int BN) {
    TileCoord t;
    const int nt = tile % n_tiles;
    int mt = tile / n_tiles;
    const long long HpWp = (long long)p.Hp * p.Wp;
    t.n0 = nt * BN;
    t.cls = 0;
    if (p.pool) {
        // mt = (image * row pairs + pair i) * column segments + t; rows 2i, 2i+1, interior columns [64t, 64t + 64)
        const int t_ = mt % p.pool_tx;
        const int r_ = mt / p.pool_tx;
        const int i_ = r_ % p.pool_ho;
        const int img = r_ / p.pool_ho;
        t.p0 = img * HpWp + (long long)(2 * i_ + 1) * p.Wp + 1 + 64 * t_;     // first position of the UPPER row segment
        t.p_end = p.P;
        t.set = 0;
        t.cls = t_;                          // (reused: column segment; the row pair is recovered from p0)
    } else if (p.mode == CONV_UP2) {
        // cout tile fastest, then the 4 parity classes: CTAs running together share one activation tile in L2
        t.cls = mt & 3;
        mt >>= 2;
        t.p0 = (long long)mt * 128;
        t.p_end = p.P;
        t.set = t.cls;                       // weight set = parity class
    } else if (p.per_image) {
        const int img = mt / p.tiles_per_image;
        const int r = mt - img * p.tiles_per_image;
        t.p0 = img * HpWp + (long long)r * 128;
        t.p_end = (img + 1) * HpWp;
        t.set = p.nsets > 1 ? img : 0;
    } else {
        t.p0 = (long long)mt * 128;
        t.p_end = p.P;
        t.set = 0;
    }
    return t;
}

// One pipeline stage (BK = 64: four 16-wide k-steps) of split-fp16 products, issued as two commit groups.
// conv_stage_ch: `ch`, the chunk accumulator of a_hi b_hi (FUSE: a_hi [b_hi | b_lo]), restarted from zero when `first`.
template <class Cfg>
__device__ __forceinline__ void conv_stage_ch(float (&ch)[Cfg::CHUNK_REGS], uint64_t a_hi, uint64_t b_hi, bool first) {
#pragma unroll
    for (int k = 0; k < Cfg::BK / 16; ++k) {
        const uint64_t ko = (uint64_t)(k * 32 >> 4);
        const uint32_t acc_in = (first && k == 0) ? 0u : 1u;
        // FUSE: [b_hi | b_lo] is one 2*BN-row K-major tile: columns [0,BN) += a_hi b_hi, [BN,2BN) += a_hi b_lo
        if constexpr (Cfg::CHUNK_REGS == 64) wgmma_m64n128k16<0, 0>(ch, a_hi + ko, b_hi + ko, acc_in);
        else wgmma_m64n64k16<0, 0>(ch, a_hi + ko, b_hi + ko, acc_in);
    }
    wgmma_commit();
}

// conv_stage_cx: `cx`, the accumulator of the small cross terms a_hi b_lo + a_lo b_hi (FUSE: a_lo b_hi) over the whole pass,
// zeroed by the caller when the pass starts.  The truncating adds of the cross terms never touch the large a_hi b_hi sum.
// NP = 3: all three products (default), 2: without a_lo b_hi, 1: a_hi b_hi only (experiment knob; the group is empty).
// NP is a template argument so that the wgmma sequence has no branches between its instructions.
template <class Cfg, int NP>
__device__ __forceinline__ void conv_stage_cx(float (&cx)[Cfg::SUM_REGS], uint64_t a_hi, uint64_t a_lo, uint64_t b_hi,
                                              uint64_t b_lo) {
#pragma unroll
    for (int k = 0; k < Cfg::BK / 16; ++k) {
        const uint64_t ko = (uint64_t)(k * 32 >> 4);
        if constexpr (Cfg::FUSE) {
            if (NP >= 3) wgmma_m64n64k16<0, 0>(cx, a_lo + ko, b_hi + ko, 1u);
        } else if constexpr (Cfg::SUM_REGS == 64) {
            if (NP >= 2) wgmma_m64n128k16<0, 0>(cx, a_hi + ko, b_lo + ko, 1u);
            if (NP >= 3) wgmma_m64n128k16<0, 0>(cx, a_lo + ko, b_hi + ko, 1u);
        } else {
            if (NP >= 2) wgmma_m64n64k16<0, 0>(cx, a_hi + ko, b_lo + ko, 1u);
            if (NP >= 3) wgmma_m64n64k16<0, 0>(cx, a_lo + ko, b_hi + ko, 1u);
        }
    }
    wgmma_commit();
}

// sum += acc (FUSE chunk: its two column halves a_hi b_hi + a_hi b_lo added first); WGT: sum = fmaf(v_row s_col, acc, sum)
// with s_col = 2^-rexp of the pass's weight set at that column (cexp: [BN] of the tile, or nullptr), which makes the
// running sum s times the plain one exactly.  Round-to-nearest FADD / FFMA, in the same order in every instantiation, so
// that unit weights give the plain sum's bits.
template <class Cfg, bool WGT, int R>
__device__ __forceinline__ void add_into_sum(float (&sum)[Cfg::SUM_REGS], const float (&acc)[R], const float (&vrow)[2],
                                             const int* cexp = nullptr, int t = 0) {
#pragma unroll
    for (int i = 0; i < Cfg::SUM_REGS; ++i) {
        float a = acc[i];
        if constexpr (R > Cfg::SUM_REGS) a += acc[Cfg::SUM_REGS + i];
        // fragment register i belongs to row r0 + 8 ((i >> 1) & 1) and column 8 (i >> 2) + 2 (t & 3) + (i & 1)
        if constexpr (WGT) {
            const float v = cexp ? vrow[(i >> 1) & 1] * pow2i(-__ldg(cexp + 8 * (i >> 2) + 2 * (t & 3) + (i & 1))) : vrow[(i >> 1) & 1];
            sum[i] = fmaf(v, a, sum[i]);
        } else {
            sum[i] = sum[i] + a;
        }
    }
}

// 8 consecutive fp32 of a tile row.  Lanes 4-7 of each 8-lane group read their two 16-byte halves in the opposite order, so
// each 16-byte load of the 8 lanes (one shared-memory phase) covers all 32 banks once.
__device__ __forceinline__ void tile_load8(const float* src, int c, float (&v)[8]) {
    const float4* s = reinterpret_cast<const float4*>(src);
    const int sw = (c >> 2) & 1;
    const float4 a = s[sw], b = s[sw ^ 1];
    const float4 l = sw ? b : a, h = sw ? a : b;
    v[0] = l.x; v[1] = l.y; v[2] = l.z; v[3] = l.w;
    v[4] = h.x; v[5] = h.y; v[6] = h.z; v[7] = h.w;
}

// *scale + bias, ReLU, split: 8 channels of one output position, biases at s and their scales 2 BN further (the layer's
// one scale, or in CONV_APPLY each row's own).  Every scale is a power of two, so a * scale is exact and the sum rounds
// once, as fmaf(a, scale, bias) would.
template <class Cfg>
__device__ __forceinline__ void finish8(float (&a)[8], const float* s, int c, bool relu, Half8& hi, Half8& lo) {
    float t8[8];
    tile_load8(s + 2 * Cfg::NB * 64, c, t8);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] *= t8[j];
    tile_load8(s, c, t8);
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const float t = a[j] + t8[j];
        v[j] = relu ? fmaxf(t, 0.f) : t;
    }
    split8(v, hi, lo);
}

// Where row `row` of a 128-position tile goes: returns its halo flags and sets its padded output position, or returns -1
// when nothing is stored (halo / junk row of the padded tiling, a pixel of another region, an aborted pipeline).
// REG: the pass stores the pixels of region `want` (R: the pixels that keep their input).
// WGT: the rows whose weight sum V (vsum[row]) is > 0, or (want == R) the rows with V = 0.
// (32-bit position arithmetic: P < 2^31 is checked by the launcher; 64-bit divisions cost ~60 instructions each)
template <bool REG, bool WGT = false>
__device__ __forceinline__ int row_target(const ConvParams& p, const ActGeom& go, const TileCoord& tc, int row, int want,
                                          volatile int* abort_flag, unsigned int& ppos, const float* vsum = nullptr) {
    ppos = 0;
    const unsigned int pos = (unsigned int)tc.p0 + (unsigned int)row;
    if (pos >= (unsigned int)tc.p_end) return -1;
    const unsigned int hpwp = (unsigned int)(p.Hp * p.Wp);
    const unsigned int n = pos / hpwp;
    const unsigned int r = pos - n * hpwp;
    const int yy = (int)(r / (unsigned int)p.Wp);
    const int xx = (int)(r - (unsigned int)yy * (unsigned int)p.Wp);
    if (yy < 1 || yy > p.H || xx < 1 || xx > p.W || *abort_flag) return -1;
    int y = yy - 1, x = xx - 1;
    if (p.mode == CONV_UP2) { y = 2 * y + (tc.cls >> 1); x = 2 * x + (tc.cls & 1); }
    if (WGT) {
        if ((vsum[row] > 0.f) == (want == p.R)) return -1;
    } else if (REG && region_of(p.labels, p.counts, p.R, (int)n, p.H, p.W, y, x) != want) {
        return -1;
    }
    ppos = ((unsigned int)n * (unsigned int)go.Hp + (unsigned int)(y + 1)) * (unsigned int)go.Wp + (unsigned int)(x + 1);
    return halo_flags(go, y, x);
}

// Epilogue of one pass, run by epilogue warp ew (of Cfg::EPI_WARPS).  The work is split into units of 4 positions x 64
// channels (8 lanes per position, 8 channels per lane); unit u = (32-row chunk * 8 + j) * NB + 64-channel block goes to
// warp u % EPI_WARPS.  The lane of a chunk row computes that row's target once; the 8 lanes storing it take it by shuffle.
// KEEP (REG only): copy the input pixels of the rows to keep (hi and lo bytes) instead of finishing the fp32 tile.
// WGT (weighted apply): vst [K + 1][BM] holds v_k and V of every row, `todo` the transforms of the tile; a row finishes as
// sum + v_0 b_0 + v_1 b_1 + ... (+ (1 - V) x where V < 1), in k order, the bias read from global memory.
template <class Cfg, bool REG, bool KEEP, bool WGT = false>
__device__ __forceinline__ void epi_rows(const ConvParams& p, const ActGeom& go, const TileCoord& tc, const float* ctile,
                                         const float* sb, float wsc, bool relu, int want, int ew, int lane,
                                         volatile int* abort_flag, const float* vst = nullptr, unsigned todo = 0u, int img = 0) {
    constexpr int U = 8 * Cfg::NB;                       // units per 32-row chunk
    const int c = lane & 7;
#pragma unroll 1
    for (int chunk = 0; chunk < Cfg::BM / 32; ++chunk) {
        unsigned int pp;
        const int fl = row_target<REG, WGT>(p, go, tc, chunk * 32 + lane, want, abort_flag, pp, WGT ? vst + p.R * Cfg::BM : nullptr);
        for (int v = ((ew - chunk * U) % Cfg::EPI_WARPS + Cfg::EPI_WARPS) % Cfg::EPI_WARPS; v < U; v += Cfg::EPI_WARPS) {
            const int j = v / Cfg::NB, b = v - j * Cfg::NB;
            const int r = j * 4 + (lane >> 3);
            const unsigned int q = __shfl_sync(0xffffffffu, pp, r);
            const int f = __shfl_sync(0xffffffffu, fl, r);
            if (f < 0) continue;
            const int ch = b * 64 + c * 8;               // channel within the tile
            Half8 hi, lo;
            if (KEEP) {
                const __half* src = p.in + (long long)q * p.Cin + tc.n0 + ch;   // APPLY: input and output positions agree
                hi = *reinterpret_cast<const Half8*>(src);
                lo = *reinterpret_cast<const Half8*>(src + (long long)p.P * p.Cin);
            } else if (WGT) {
                const int row = chunk * 32 + r;
                float a[8];
                tile_load8(ctile + row * Cfg::PITCH + ch, c, a);
#pragma unroll
                for (int i = 0; i < 8; ++i) a[i] *= wsc;
                for (unsigned m = todo; m; m &= m - 1u) {    // (v = 1: fmaf is the plain add of the unweighted epilogue)
                    const int k = __ffs(m) - 1;
                    const float vk = vst[k * Cfg::BM + row];
                    if (vk == 0.f) continue;
                    const float4* bk = reinterpret_cast<const float4*>(p.bias + (long long)(img * p.R + k) * p.Cout + tc.n0 + ch);
                    const float4 b0 = __ldg(bk), b1 = __ldg(bk + 1);
                    a[0] = fmaf(vk, b0.x, a[0]); a[1] = fmaf(vk, b0.y, a[1]); a[2] = fmaf(vk, b0.z, a[2]); a[3] = fmaf(vk, b0.w, a[3]);
                    a[4] = fmaf(vk, b1.x, a[4]); a[5] = fmaf(vk, b1.y, a[5]); a[6] = fmaf(vk, b1.z, a[6]); a[7] = fmaf(vk, b1.w, a[7]);
                }
                const float keep = 1.f - vst[p.R * Cfg::BM + row];
                if (keep != 0.f) {          // (skipped at V = 1: -0 + 0 would turn a sign bit)
                    const __half* src = p.in + (long long)q * p.Cin + tc.n0 + ch;
                    float x[8];
                    merge8(*reinterpret_cast<const Half8*>(src), *reinterpret_cast<const Half8*>(src + (long long)p.P * p.Cin), x);
#pragma unroll
                    for (int i = 0; i < 8; ++i) a[i] = fmaf(keep, x[i], a[i]);
                }
                split8(a, hi, lo);
            } else {
                float a[8];
                tile_load8(ctile + (chunk * 32 + r) * Cfg::PITCH + ch, c, a);
                finish8<Cfg>(a, sb + ch, c, relu, hi, lo);
            }
            store8_at(p.out, go, q, f, tc.n0 + ch, hi, lo);
        }
    }
}

// POOL2 epilogue: MaxPooling2D 2x2/2 'same' (vgg_normalised.py:41-42) on the raw accumulators, which commutes with the
// monotone  *scale + bias -> ReLU -> split  that follows.  Tile rows 0..63 = image row 2i, 64..127 = row 2i+1, so pooled
// pixel k of the tile is the max of rows 2k, 2k+1, 64+2k, 65+2k; cells past the right / bottom edge are left out.
// Units of 4 pooled pixels x 64 channels; lane k computes pooled pixel k's target.
template <class Cfg>
__device__ __forceinline__ void epi_pool(const ConvParams& p, const ActGeom& go, const TileCoord& tc, const float* ctile,
                                         const float* sb, float wsc, bool relu, int ew, int lane, volatile int* abort_flag) {
    const unsigned int hpwp = (unsigned int)(p.Hp * p.Wp);
    const unsigned int n = (unsigned int)tc.p0 / hpwp;
    const int yy0 = (int)(((unsigned int)tc.p0 - n * hpwp) / (unsigned int)p.Wp);   // padded row of image row 2i
    const bool lower = yy0 < p.H;                        // image row 2i+1 exists
    unsigned int pp = 0;
    int fl = -1;
    {
        const int x = 64 * tc.cls + 2 * lane;
        if (x < p.W && yy0 - 1 < p.H && !*abort_flag) {
            const int yo = (yy0 - 1) >> 1, xo = x >> 1;
            fl = halo_flags(go, yo, xo);
            pp = (n * (unsigned int)go.Hp + (unsigned int)(yo + 1)) * (unsigned int)go.Wp + (unsigned int)(xo + 1);
        }
    }
    const int c = lane & 7;
    for (int v = ew; v < 8 * Cfg::NB; v += Cfg::EPI_WARPS) {
        const int j = v / Cfg::NB, b = v - j * Cfg::NB;
        const int k = j * 4 + (lane >> 3);
        const unsigned int q = __shfl_sync(0xffffffffu, pp, k);
        const int f = __shfl_sync(0xffffffffu, fl, k);
        if (f < 0) continue;
        const bool right = 64 * tc.cls + 2 * k + 1 < p.W;
        const int ch = b * 64 + c * 8;
        const float* s = ctile + 2 * k * Cfg::PITCH + ch;
        float m[8], a[8];
        tile_load8(s, c, m);
        if (right) {
            tile_load8(s + Cfg::PITCH, c, a);
#pragma unroll
            for (int i = 0; i < 8; ++i) m[i] = fmaxf(m[i], a[i]);
        }
        if (lower) {
            tile_load8(s + 64 * Cfg::PITCH, c, a);
#pragma unroll
            for (int i = 0; i < 8; ++i) m[i] = fmaxf(m[i], a[i]);
            if (right) {
                tile_load8(s + 65 * Cfg::PITCH, c, a);
#pragma unroll
                for (int i = 0; i < 8; ++i) m[i] = fmaxf(m[i], a[i]);
            }
        }
        Half8 hi, lo;
        finish8<Cfg>(m, sb + ch, c, relu, hi, lo);
        store8_at(p.out, go, q, f, tc.n0 + ch, hi, lo);
    }
}

// REG (spatial control, CONV_APPLY only): every tile runs one mainloop + epilogue pass per region present in it (its own
// weight set, stores only the rows of that region), then copies the rows to keep; a tile inside one region costs what the
// plain apply costs.
// WGT (with REG: the weighted apply of soft spatial control, DESIGN.md §3.3.11): one mainloop pass per transform k present
// in the tile, each chunk added as fmaf(v_k(row), ch, sum) and the pass's cross products as fmaf(v_k(row), cx, sum) into
// ONE running sum across the passes; the epilogue finishes the tile once (sum_k v_k b_k and the keep term) and copies the
// rows whose weights are all 0.  v = 1 gives the plain add, so one-hot weights give REG's bits.
template <int BN, bool FUSE_, bool REG = false, bool WGT = false>
__global__ void __launch_bounds__(Conv2Cfg<BN, FUSE_>::THREADS, 1)
conv_tc2_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, const ConvParams p,
                const int total_tiles, const int n_tiles) {
    using Cfg = Conv2Cfg<BN, FUSE_>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* bring = smem + Cfg::A_STAGES * Cfg::STRIP_BYTES;
    uint8_t* aux = smem + Cfg::RING_BYTES;
    uint64_t* fullA = reinterpret_cast<uint64_t*>(aux);
    uint64_t* emptyA = fullA + Cfg::A_STAGES;
    uint64_t* full = emptyA + Cfg::A_STAGES;             // B ring
    uint64_t* empty = full + Cfg::B_STAGES;
    uint64_t* tile_full = empty + Cfg::B_STAGES;         // the fp32 tile is written (one arrival per consumer warp)
    uint64_t* tile_empty = tile_full + 1;                // the fp32 tile is read (one arrival per epilogue warp)
    volatile int* abort_flag = reinterpret_cast<volatile int*>(tile_empty + 1);
    float* sbias = reinterpret_cast<float*>(aux + 256);  // [2][BN] bias, then [2][BN] scale of the pass (by pass parity)
    float* ctile = reinterpret_cast<float*>(aux + Cfg::AUX_BYTES);
    float* vst = ctile + Cfg::BM * Cfg::PITCH;           // WGT: [K + 1][BM] v_k and V of the rows of the epilogue's tile

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    {
        __shared__ unsigned int s_prev_err;
        if (threadIdx.x == 0) s_prev_err = *reinterpret_cast<volatile unsigned int*>(p.err);
        __syncthreads();
        if (s_prev_err != 0u) return;
    }
    if (threadIdx.x == 0) {
        for (int s = 0; s < Cfg::A_STAGES; ++s) {
            mbar_init(&fullA[s], 1);
            mbar_init(&emptyA[s], Cfg::CONSUMERS / 32);     // one arrival per consumer warp
        }
        for (int s = 0; s < Cfg::B_STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], Cfg::CONSUMERS / 32);
        }
        mbar_init(tile_full, Cfg::CONSUMERS / 32);
        mbar_init(tile_empty, Cfg::EPI_WARPS);
        *abort_flag = 0;
        fence_barrier_init();
        tma_prefetch_desc(&mapA);
        tma_prefetch_desc(&mapB);
    }
    __syncthreads();

    // k-iteration order: (filter row, channel slice, column tap), column tap innermost, so that one strip feeds ncol
    // consecutive k-iterations
    const int ksl = p.Cin / Cfg::BK;
    const int kiters = p.taps * ksl;
    const int ncol = REG ? 1 : p.ncol;                   // the regions apply is a 1x1 conv
    const bool pool = !REG && p.pool;

    // register split, checked with ptxas -v to spill nothing (but 8 bytes in the weighted apply at BN = 128, whose consumers
    // also read the row scales of each pass): the consumers of BN = 128 need more than 200 and the epilogue
    // warps more than 56 (REG: 80).  setmaxnreg.inc only receives what the other warpgroups released, so the split must
    // stay within the 3 x 128 x 168 registers the CTA was launched with, or the consumers wait for registers forever.
    constexpr int EPI_REGS = REG ? (BN == 128 ? 88 : 104) : 72;
    constexpr int MMA_REGS = REG ? (BN == 128 ? 208 : 200) : 216;
    static_assert(2 * 128 * MMA_REGS + 128 * EPI_REGS <= 3 * 128 * 168, "setmaxnreg split exceeds the CTA's registers");
    if (warp >= Cfg::CONSUMERS / 32) {
        setmaxnreg_dec<EPI_REGS>();
        if (warp == Cfg::CONSUMERS / 32) {
            if (lane != 0) return;
            // the whole box counts towards the transaction bytes, rows zero-filled outside [0, P) included
            const uint32_t strip_tx = (pool ? 4u : 2u) * (uint32_t)p.strip_rows * 128u;
            uint32_t itg = 0, stg = 0;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const TileCoord tc = tile_coord(p, tile, n_tiles, BN);
                unsigned todo = 1u;                      // passes over the tile (REG: one per region present)
                if constexpr (REG) todo = p.amask[tile / n_tiles] & ((1u << p.R) - 1u);
                for (; todo; todo &= todo - 1u) {
                const int set = REG ? (tile / n_tiles) / p.tiles_per_image * p.R + (__ffs(todo) - 1) : tc.set;
                int fr = 0, ks = 0, kx = 0;                  // filter row, channel slice, column tap of k-iteration it
                for (int it = 0; it < kiters; ++it, ++itg) {
                    if (kx == 0) {
                        // the strip of (fr, ks): the first row its column tap 0 reads
                        const int sa = stg % Cfg::A_STAGES;
                        mbar_wait(&emptyA[sa], ((stg / Cfg::A_STAGES) & 1) ^ 1u, abort_flag, p.err, 0x110u + sa);
                        int off = 0;
                        if (p.mode == CONV_3X3) off = (fr - 1) * p.Wp - 1;
                        else if (p.mode == CONV_TAPS) off = fr * p.Wp;
                        else if (p.mode == CONV_UP2) off = (fr - 1 + (tc.cls >> 1)) * p.Wp + (tc.cls & 1) - 1;
                        const int row = (int)(tc.p0 + off);
                        uint8_t* sp = smem + sa * Cfg::STRIP_BYTES;
                        mbar_arrive_expect_tx(&fullA[sa], strip_tx);
                        if (pool) {
                            // two segments per plane: the one of image row 2i and the one below it
                            constexpr int SEG = Cfg::POOL_SEG_ROWS * 128;
                            tma_load_3d(sp, &mapA, &fullA[sa], ks * Cfg::BK, row, 0);
                            tma_load_3d(sp + SEG, &mapA, &fullA[sa], ks * Cfg::BK, row + p.Wp, 0);
                            tma_load_3d(sp + Cfg::PLANE_BYTES, &mapA, &fullA[sa], ks * Cfg::BK, row, 1);
                            tma_load_3d(sp + Cfg::PLANE_BYTES + SEG, &mapA, &fullA[sa], ks * Cfg::BK, row + p.Wp, 1);
                        } else {
                            tma_load_3d(sp, &mapA, &fullA[sa], ks * Cfg::BK, row, 0);
                            tma_load_3d(sp + Cfg::PLANE_BYTES, &mapA, &fullA[sa], ks * Cfg::BK, row, 1);
                        }
                    }
                    const int s = itg % Cfg::B_STAGES;
                    const uint32_t ph = (itg / Cfg::B_STAGES) & 1;
                    mbar_wait(&empty[s], ph ^ 1u, abort_flag, p.err, 0x100u + s);
                    const int k0 = (fr * ncol + kx) * p.Cin + ks * Cfg::BK;
                    uint8_t* sp = bring + s * Cfg::B_SLOT_BYTES;
                    mbar_arrive_expect_tx(&full[s], Cfg::B_SLOT_BYTES);
                    tma_load_3d(sp, &mapB, &full[s], k0, tc.n0, set * 2);
                    tma_load_3d(sp + Cfg::B_BYTES, &mapB, &full[s], k0, tc.n0, set * 2 + 1);
                    if (++kx == ncol) {
                        kx = 0;
                        ++stg;
                        if (++ks == ksl) { ks = 0; ++fr; }
                    }
                }
                }
            }
            return;
        }

        // ---- epilogue warps 9-11: the same tile list and passes as the consumers, one tile hand-off per pass ----
        const int ew = warp - Cfg::CONSUMERS / 32 - 1;
        const ActGeom& go = p.go;
        const bool relu = (p.flags & WCTB200_RELU) != 0;
        const float wsc = p.wscale ? __ldg(p.wscale) : 1.f;
        uint32_t pass = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            const TileCoord tc = tile_coord(p, tile, n_tiles, BN);
            const int mt = tile / n_tiles;
            unsigned todo = 1u;
            if constexpr (REG) todo = p.amask[mt] & ((1u << p.R) - 1u);
            if constexpr (WGT) {
                const int img = mt / p.tiles_per_image;
                asm volatile("bar.sync 1, %0;" ::"r"(32 * Cfg::EPI_WARPS) : "memory");   // the previous tile's vst is read
                for (int row = threadIdx.x - (Cfg::CONSUMERS + 32); row < Cfg::BM; row += 32 * Cfg::EPI_WARPS) {
                    float V = 0.f;
                    for (int k = 0; k < p.R; ++k) {
                        const float v = ((todo >> k) & 1u) ? row_weight(p, tc.p0, tc.p_end, row, k) : 0.f;
                        vst[k * Cfg::BM + row] = v;
                        V += v;
                    }
                    vst[p.R * Cfg::BM + row] = V;
                }
                if (todo) {
                    mbar_wait(tile_full, pass & 1, abort_flag, p.err, 0x301u);
                    asm volatile("bar.sync 1, %0;" ::"r"(32 * Cfg::EPI_WARPS) : "memory");
                    epi_rows<Cfg, REG, false, true>(p, go, tc, ctile, sbias, wsc, relu, 0, ew, lane, abort_flag, vst, todo, img);
                    __syncwarp();
                    if (lane == 0) mbar_arrive(tile_empty);
                    ++pass;
                } else {
                    asm volatile("bar.sync 1, %0;" ::"r"(32 * Cfg::EPI_WARPS) : "memory");
                }
                if ((p.amask[mt] >> p.R) & 1u)
                    epi_rows<Cfg, REG, true, true>(p, go, tc, ctile, sbias, wsc, relu, p.R, ew, lane, abort_flag, vst, 0u, img);
                continue;
            }
            for (; todo; todo &= todo - 1u, ++pass) {
                const int region = __ffs(todo) - 1;
                const int set = REG ? mt / p.tiles_per_image * p.R + region : tc.set;
                // bias of this pass into the buffer of its parity: that buffer was last read two passes ago, before every
                // epilogue warp passed the previous pass's barrier
                float* sb = sbias + (pass & 1) * BN;
                for (int i = threadIdx.x - (Cfg::CONSUMERS + 32); i < BN; i += 32 * Cfg::EPI_WARPS) {
                    sb[i] = p.bias ? __ldg(p.bias + (long long)(p.mode == CONV_APPLY ? set : 0) * p.Cout + tc.n0 + i) : 0.f;   // UP2: set = weight parity class, ONE bias
                    sb[2 * BN + i] = p.rexp ? pow2i(-__ldg(p.rexp + (long long)set * p.Cout + tc.n0 + i)) : wsc;
                }
                mbar_wait(tile_full, pass & 1, abort_flag, p.err, 0x301u);
                asm volatile("bar.sync 1, %0;" ::"r"(32 * Cfg::EPI_WARPS) : "memory");
                if (p.pool) epi_pool<Cfg>(p, go, tc, ctile, sb, wsc, relu, ew, lane, abort_flag);
                else epi_rows<Cfg, REG, false>(p, go, tc, ctile, sb, wsc, relu, region, ew, lane, abort_flag);
                __syncwarp();
                if (lane == 0) mbar_arrive(tile_empty);  // the consumers may write the next tile
            }
            if constexpr (REG) {
                if ((p.amask[mt] >> p.R) & 1u) epi_rows<Cfg, REG, true>(p, go, tc, ctile, sbias, wsc, relu, p.R, ew, lane, abort_flag);
            }
        }
        return;
    }

    // ---- consumer warpgroups ----
    setmaxnreg_inc<MMA_REGS>();
    const int wg = warp >> 2;                            // rows [64 wg, 64 wg + 64) of the tile
    const int t = threadIdx.x & 127;
    uint32_t itg = 0, stg = 0, pass = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        unsigned todo = 1u;
        if constexpr (REG) todo = p.amask[tile / n_tiles] & ((1u << p.R) - 1u);
        if (WGT && !todo) continue;                       // the epilogue only copies the kept rows
        float sum[Cfg::SUM_REGS];
        if constexpr (WGT) {
#pragma unroll
            for (int i = 0; i < Cfg::SUM_REGS; ++i) sum[i] = 0.f;
        }
        for (; todo; todo &= todo - 1u) {
        float vrow[2] = {1.f, 1.f};                      // WGT: v_k of this thread's two fragment rows
        const int* cexp = nullptr;                       // WGT: the row exponents of transform k at the tile's channels
        if constexpr (WGT) {
            const TileCoord tc = tile_coord(p, tile, n_tiles, BN);
            const int k = __ffs(todo) - 1;
            const int r0 = 64 * wg + 16 * (t >> 5) + ((t & 31) >> 2);
            vrow[0] = row_weight(p, tc.p0, tc.p_end, r0, k);
            vrow[1] = row_weight(p, tc.p0, tc.p_end, r0 + 8, k);
            if (p.rexp) cexp = p.rexp + (long long)((tile / n_tiles) / p.tiles_per_image * p.R + k) * p.Cout + tc.n0;
        } else {
#pragma unroll
            for (int i = 0; i < Cfg::SUM_REGS; ++i) sum[i] = 0.f;
        }
        // ch restarts every CH k-iterations and is added into sum at each chunk end; cx runs over the whole pass and is added
        // once, after the last chunk (DESIGN.md §3.1)
        float ch[Cfg::CHUNK_REGS], cx[Cfg::SUM_REGS];
#pragma unroll
        for (int i = 0; i < Cfg::CHUNK_REGS; ++i) ch[i] = 0.f;
#pragma unroll
        for (int i = 0; i < Cfg::SUM_REGS; ++i) cx[i] = 0.f;
        int kx = 0;
        for (int it = 0; it < kiters; ++it, ++itg) {
            const int sa = stg % Cfg::A_STAGES;
            if (kx == 0) mbar_wait(&fullA[sa], (stg / Cfg::A_STAGES) & 1, abort_flag, p.err, 0x210u + sa);
            const int s = itg % Cfg::B_STAGES;
            const uint32_t ph = (itg / Cfg::B_STAGES) & 1;
            mbar_wait(&full[s], ph, abort_flag, p.err, 0x200u + s);
            // this warpgroup's operand rows: tile rows 64 wg .. (POOL2: the second segment), column tap kx kx rows further
            const uint32_t sta = smem_u32(smem + sa * Cfg::STRIP_BYTES) + (wg * (pool ? Cfg::POOL_SEG_ROWS : 64) + kx) * 128;
            const uint64_t a_hi = gmma_desc_sw128(sta);
            const uint64_t a_lo = gmma_desc_sw128(sta + Cfg::PLANE_BYTES);
            const uint32_t stb = smem_u32(bring + s * Cfg::B_SLOT_BYTES);
            const uint64_t b_hi = gmma_desc_sw128(stb);
            const uint64_t b_lo = gmma_desc_sw128(stb + Cfg::B_BYTES);
            // IN_FLIGHT: in flight at the top of every k-iteration but the pass's first is the cx group of k-iteration it - 1,
            // nothing else.  Each wait below leaves exactly one group running, so the same group is in flight on every path
            // into the loop's back edge: where the paths differ, ptxas serialises every wgmma of the kernel.
            wgmma_fence();
            conv_stage_ch<Cfg>(ch, a_hi, b_hi, it % Cfg::CH == 0);
            wgmma_wait<1>();                             // IN_FLIGHT: cx of k-iteration it - 1 has retired
            // (REG runs APPLY convs, which the products knob leaves at 3: one wgmma sequence keeps the regions apply at
            // BN = 128 within its 208 registers)
            if (REG || p.products >= 3) conv_stage_cx<Cfg, 3>(cx, a_hi, a_lo, b_hi, b_lo);
            else if (p.products == 2) conv_stage_cx<Cfg, 2>(cx, a_hi, a_lo, b_hi, b_lo);
            else conv_stage_cx<Cfg, 1>(cx, a_hi, a_lo, b_hi, b_lo);
            if constexpr (Cfg::IN_FLIGHT) {
                // free the B slot of k-iteration it - 1, and its strip after its last column tap (after the issue above, so
                // that the cross products are queued first)
                if (it > 0) {
                    __syncwarp();
                    if (lane == 0) {
                        mbar_arrive(&empty[(itg - 1) % Cfg::B_STAGES]);
                        if (kx == 0) mbar_arrive(&emptyA[(stg - 1) % Cfg::A_STAGES]);
                    }
                }
            }
            wgmma_wait<Cfg::IN_FLIGHT>();                // ch of this k-iteration has retired (IN_FLIGHT: its cx runs on)
            if constexpr (!Cfg::IN_FLIGHT) {             // free this k-iteration's slot, and its strip after the last tap
                __syncwarp();
                if (lane == 0) {
                    mbar_arrive(&empty[s]);
                    if (kx + 1 == ncol) mbar_arrive(&emptyA[sa]);
                }
            }
            if (++kx == ncol) {
                kx = 0;
                ++stg;
            }
            if ((it + 1) % Cfg::CH == 0) {              // chunk end
                acc_fence(ch);
                add_into_sum<Cfg, WGT>(sum, ch, vrow, cexp, t);
            }
        }
        wgmma_wait<0>();
        acc_fence(ch);
        acc_fence(cx);
        if constexpr (Cfg::IN_FLIGHT) {
            __syncwarp();
            if (lane == 0) {                             // the last k-iteration is the last column tap of its strip
                mbar_arrive(&empty[(itg - 1) % Cfg::B_STAGES]);
                mbar_arrive(&emptyA[(stg - 1) % Cfg::A_STAGES]);
            }
        }
        if (kiters % Cfg::CH != 0) add_into_sum<Cfg, WGT>(sum, ch, vrow, cexp, t);   // the last chunk is a short one
        add_into_sum<Cfg, WGT>(sum, cx, vrow, cexp, t);

        if constexpr (!WGT) {
            // ---- hand the fp32 tile to the epilogue warps (row-major in shared memory: a wgmma fragment spreads one row
            // over 4 lanes); the previous tile must have been read, which it normally was during this mainloop ----
            mbar_wait(tile_empty, (pass & 1) ^ 1u, abort_flag, p.err, 0x300u);
            frag_to_tile(sum, ctile, Cfg::PITCH, 64 * wg, t);
            __syncwarp();
            if (lane == 0) mbar_arrive(tile_full);
            ++pass;
        }
        }
        if constexpr (WGT) {                              // every pass is in the running sum: one hand-off per tile
            mbar_wait(tile_empty, (pass & 1) ^ 1u, abort_flag, p.err, 0x300u);
            frag_to_tile(sum, ctile, Cfg::PITCH, 64 * wg, t);
            __syncwarp();
            if (lane == 0) mbar_arrive(tile_full);
            ++pass;
        }
    }
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_encodeTiled>(ptr);
    }
    return fn;
}

// 3-D fp16 tensor map [d2][d1][d0] (d0 contiguous), box {64, box1, 1}, 128B swizzle, zero OOB fill
int make_tensor_map_3d(CUtensorMap* m, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1_bytes,
                    uint64_t stride2_bytes, uint32_t box1) {
    PFN_encodeTiled enc = get_encode();
    if (!enc) {
        set_error("cuTensorMapEncodeTiled entry point not available");
        return WCTB200_ECUDA;
    }
    cuuint64_t dims[3] = {d0, d1, d2};
    cuuint64_t strides[2] = {stride1_bytes, stride2_bytes};
    cuuint32_t box[3] = {64, box1, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed (%d): dims %llu %llu %llu strides %llu %llu box1 %u", (int)r,
                  (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)d2,
                  (unsigned long long)stride1_bytes, (unsigned long long)stride2_bytes, box1);
        return WCTB200_ECUDA;
    }
    return 0;
}

int g_conv_oversub = 4;

template <int BN, bool FUSE_, bool REG = false, bool WGT = false>
static int launch2_bn(const CUtensorMap& mA, const CUtensorMap& mB, const ConvParams& p, int total_tiles, int n_tiles,
                      cudaStream_t st) {
    using Cfg = Conv2Cfg<BN, FUSE_>;
    // WGT: the rows' v_k and V ([9][BM] fp32) after the fp32 tile
    constexpr int SMEM = Cfg::SMEM_BYTES + (WGT ? 9 * Cfg::BM * 4 : 0);
    static_assert(SMEM <= 227 * 1024, "conv: shared memory exceeds the 227 KB opt-in limit");
    WCTB_ENSURE_SMEM((conv_tc2_kernel<BN, FUSE_, REG, WGT>), SMEM);
    // Over-subscribed persistent grid: with g_conv_oversub x #SMs CTAs (1 resident per SM) the
    // hardware block scheduler hands queued CTAs to whichever SMs are free, so a conv launched
    // while the Jacobi clusters of the other stream hold half the SMs still balances its tiles
    // (a grid of exactly #SMs would run as two unbalanced waves).
    int grid = device_sm_count() * (g_conv_oversub > 0 ? g_conv_oversub : 1);
    if (grid > total_tiles) grid = total_tiles;
    conv_tc2_kernel<BN, FUSE_, REG, WGT><<<grid, Cfg::THREADS, SMEM, st>>>(mA, mB, p, total_tiles, n_tiles);
    WCTB_CHECK_LAUNCH("conv_tc2_kernel");
    return 0;
}

int g_conv_products = 3;     // experiment knob (wctb200_debug_set_conv_products): split-fp16 products per MAC
int g_conv_fuse = -1;        // -1 auto, 0 never, 1 whenever the tile allows (wctb200_debug_set_conv_fuse)
int g_conv_bn_override = 0;  // test/tuning hook: force the N tile (64/128; 256 runs as 128)

// mode CONV_3X3  : in [N,H,W,Cin], w_split [2][Cout][9*Cin],          out [N,H,W,Cout]
// mode CONV_APPLY: in [N,H,W,Cin], w_split [nsets][2][Cout][Cin],     out [N,H,W,Cout]   (per-image weight sets; rexp
//                  [nsets][Cout]: row i stored times 2^rexp, or nullptr)
// mode CONV_UP2  : in [N,H,W,Cin] (edge halo), w_split [4][2][Cout][4*Cin], out [N,2H,2W,Cout]
// mode CONV_TAPS : in [N,H,W,Cin], w_split [2][Cout][kw*kw*Cin],      out [N,H,W,Cout]: top-left anchored kw x kw correlation
// regions (spatial control, CONV_APPLY with C = Cin = Cout): w_split [N*R][2][C][C], bias [N*R][C]; labels / counts / amask
// as in ConvParams
// N tile of a conv with Cout output channels: 128 when it divides Cout (or the test hook's forced tile)
int conv_tc_bn(int Cout) {
    int BN = Cout % 128 == 0 ? 128 : 64;
    if (g_conv_bn_override && Cout % g_conv_bn_override == 0) BN = g_conv_bn_override > 128 ? 128 : g_conv_bn_override;
    return BN;
}

static int conv_tc_impl(int mode, const __half* in, int N, int H, int W, int Cin, const __half* w_split, int nsets,
                        const float* wscale, const float* bias, int Cout, int flags, __half* out, cudaStream_t st, int kw,
                        const uint8_t* labels, const int* counts, const uint16_t* amask, int R, int bn_req = 0,
                        long long wplane = 0, const float* wts = nullptr, const float* str = nullptr, const int* kc = nullptr,
                        const int* rexp = nullptr) {
    const bool wgt = kc != nullptr;
    const bool reg = labels != nullptr || wgt;
    WCTB_REQUIRE(!reg || (mode == CONV_APPLY && Cin == Cout && nsets == N * R && flags == 0), "conv: bad regions apply");
    if (reg) nsets = N;                                   // per-image tiling; the region picks the set inside an image
    WCTB_REQUIRE(N >= 1 && H >= 2 && W >= 2, "conv: bad geometry N=%d H=%d W=%d", N, H, W);
    WCTB_REQUIRE(Cin % 64 == 0 && Cout % 64 == 0 && Cin >= 64 && Cout >= 64, "conv: Cin=%d Cout=%d must be multiples of 64", Cin, Cout);
    WCTB_REQUIRE(mode == CONV_3X3 || mode == CONV_APPLY || mode == CONV_UP2 || mode == CONV_TAPS, "conv: bad mode %d", mode);
    WCTB_REQUIRE(mode != CONV_TAPS || (kw >= 1 && kw <= 16), "conv: bad filter width %d", kw);
    WCTB_REQUIRE(nsets == 1 || (mode == CONV_APPLY && nsets == N), "conv: nsets must be 1 (or N in apply mode)");
    ActGeom gi(N, H, W, Cin);
    WCTB_REQUIRE(gi.P < (1ll << 31) - 4096, "conv: too many padded positions (%lld)", gi.P);
    WCTB_REQUIRE(mode != CONV_UP2 || ActGeom(N, 2 * H, 2 * W, Cout).P < (1ll << 31), "conv: too many output positions");
    const int taps = mode == CONV_3X3 ? 9 : (mode == CONV_UP2 ? 4 : (mode == CONV_TAPS ? kw * kw : 1));
    const int wsets = mode == CONV_UP2 ? 4 : (reg ? N * R : nsets);

    const bool pool = (flags & WCTB200_POOL2) != 0;
    WCTB_REQUIRE(!pool || (mode == CONV_3X3 && (H + 1) / 2 >= 2 && (W + 1) / 2 >= 2), "conv: POOL2 needs the 3x3 mode and a pooled output >= 2x2");
    // N tile: at most 128 (a 64 x 256 fp32 chunk plus the running sum would not fit a warpgroup's registers)
    int BN = bn_req ? bn_req : conv_tc_bn(Cout);
    WCTB_REQUIRE((BN == 64 || BN == 128) && Cout % BN == 0, "conv: N tile %d does not divide Cout=%d", BN, Cout);

    // one strip box per (filter row, channel slice) holds the rows of all its column taps
    const int ncol = mode == CONV_3X3 ? 3 : (mode == CONV_UP2 ? 2 : (mode == CONV_TAPS ? kw : 1));
    const int strip_rows = pool ? 64 + 2 : 127 + ncol;
    CUtensorMap mA, mB;
    int rc = make_tensor_map_3d(&mA, in, (uint64_t)Cin, (uint64_t)gi.P, 2, (uint64_t)Cin * 2, (uint64_t)gi.plane * 2,
                                (uint32_t)strip_rows);
    if (rc) return rc;
    const uint64_t K = (uint64_t)taps * Cin;
    // weight planes [2 * wsets][Cout][K]; a slice of the rows of a larger filter bank keeps that bank's plane stride
    const uint64_t wstride = wplane ? (uint64_t)wplane : K * Cout;
    WCTB_REQUIRE(wstride >= K * Cout, "conv: weight plane stride %llu < %llu", (unsigned long long)wstride, (unsigned long long)(K * Cout));
    rc = make_tensor_map_3d(&mB, w_split, K, (uint64_t)Cout, (uint64_t)2 * wsets, K * 2, wstride * 2, (uint32_t)BN);
    if (rc) return rc;

    ConvParams p;
    p.N = N; p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout; p.Hp = gi.Hp; p.Wp = gi.Wp; p.P = gi.P;
    p.mode = mode;
    p.taps = taps;
    p.kw = kw;
    p.ncol = ncol;
    p.strip_rows = strip_rows;
    p.products = (mode == CONV_3X3 || mode == CONV_UP2) ? g_conv_products : 3;    // the knob only touches the encoder / decoder convs
    p.nsets = nsets;
    p.per_image = nsets > 1 ? 1 : 0;
    p.tiles_per_image = cdiv((long long)gi.Hp * gi.Wp, 128);
    p.pool = pool ? 1 : 0;
    p.pool_tx = cdiv(W, 64);
    p.pool_ho = (H + 1) / 2;
    p.flags = flags;
    p.go = ActGeom(N, mode == CONV_UP2 ? 2 * H : (pool ? (H + 1) / 2 : H), mode == CONV_UP2 ? 2 * W : (pool ? (W + 1) / 2 : W), Cout);
    p.go.set_halo(flags);
    p.bias = bias;
    p.wscale = wscale;
    p.rexp = mode == CONV_APPLY ? rexp : nullptr;
    p.out = out;
    p.err = device_error_word();
    p.in = in;
    p.labels = labels;
    p.counts = counts;
    p.amask = amask;
    p.R = R;
    p.wts = wts;
    p.str = str;
    p.kc = kc;
    if (reg) {
        p.per_image = 1;
        p.nsets = N;
    }
    const int m_tiles = pool ? N * p.pool_ho * p.pool_tx : (p.per_image ? N * p.tiles_per_image : cdiv(gi.P, 128));
    const int n_tiles = Cout / BN;
    const int total = m_tiles * n_tiles * (mode == CONV_UP2 ? 4 : 1);
    if (wgt) {
        switch (BN) {
            case 64: return g_conv_fuse == 0 ? launch2_bn<64, false, true, true>(mA, mB, p, total, n_tiles, st)
                                             : launch2_bn<64, true, true, true>(mA, mB, p, total, n_tiles, st);
            default: return launch2_bn<128, false, true, true>(mA, mB, p, total, n_tiles, st);
        }
    }
    if (reg) {
        switch (BN) {
            case 64: return g_conv_fuse == 0 ? launch2_bn<64, false, true>(mA, mB, p, total, n_tiles, st)
                                             : launch2_bn<64, true, true>(mA, mB, p, total, n_tiles, st);
            default: return launch2_bn<128, false, true>(mA, mB, p, total, n_tiles, st);
        }
    }
    switch (BN) {
        // fused [b_hi|b_lo] wgmma (Conv2Cfg::FUSE) at BN=64 unless switched off; at BN=128 it would need N = 256
        case 64: return g_conv_fuse == 0 ? launch2_bn<64, false>(mA, mB, p, total, n_tiles, st)
                                         : launch2_bn<64, true>(mA, mB, p, total, n_tiles, st);
        default: return launch2_bn<128, false>(mA, mB, p, total, n_tiles, st);
    }
}

int launch_conv_tc(int mode, const __half* in, int N, int H, int W, int Cin, const __half* w_split, int nsets,
                   const float* wscale, const float* bias, int Cout, int flags, __half* out, cudaStream_t st, int kw) {
    return conv_tc_impl(mode, in, N, H, W, Cin, w_split, nsets, wscale, bias, Cout, flags, out, st, kw, nullptr, nullptr, nullptr, 1);
}
// CONV_TAPS over output channels [n0, n0 + Cout) of a bank of `wplane / (kw*kw*Cin)` filters: w_split points at row n0 of the
// hi plane, the lo plane sits `wplane` elements further, and the N tile is `bn` (the bank's own, so that every output element
// runs the same kernel variant and k order as in one launch over the whole bank)
int launch_conv_taps_rows(const __half* in, int N, int H, int W, int Cin, const __half* w_split, long long wplane, int Cout, int bn,
                          __half* out, cudaStream_t st, int kw) {
    return conv_tc_impl(CONV_TAPS, in, N, H, W, Cin, w_split, 1, nullptr, nullptr, Cout, 0, out, st, kw, nullptr, nullptr, nullptr, 1,
                        bn, wplane);
}
// out = M_{n,r} x + bias_{n,r} for the pixels of region r of image n, out = x for the rest (wct.cu: launch_wct_apply_regions)
int launch_conv_apply(const __half* in, int N, int H, int W, int C, const __half* w_split, int nsets, const int* rexp,
                      const float* bias, __half* out, cudaStream_t st) {
    return conv_tc_impl(CONV_APPLY, in, N, H, W, C, w_split, nsets, nullptr, bias, C, 0, out, st, 3, nullptr, nullptr, nullptr, 1, 0, 0,
                        nullptr, nullptr, nullptr, rexp);
}
int launch_conv_apply_regions(const __half* in, int N, int H, int W, int C, const __half* w_split, const int* rexp, const float* bias,
                              const uint8_t* labels, const int* counts, const uint16_t* amask, int R, __half* out, cudaStream_t st) {
    return conv_tc_impl(CONV_APPLY, in, N, H, W, C, w_split, N * R, nullptr, bias, C, 0, out, st, 3, labels, counts, amask, R, 0, 0,
                        nullptr, nullptr, nullptr, rexp);
}
// out = sum_k v_k (M_{n,k} x + bias_{n,k}) + (1 - sum_k v_k) x, v_k = soft_weight(wts, str, kc, ...) (wct.cu:
// launch_wct_transform_apply_weighted); amask as in ConvParams
int launch_conv_apply_weighted(const __half* in, int N, int H, int W, int C, const __half* w_split, const int* rexp, const float* bias,
                               const float* wts, const float* str, const int* kc, const uint16_t* amask, int K, __half* out,
                               cudaStream_t st) {
    return conv_tc_impl(CONV_APPLY, in, N, H, W, C, w_split, N * K, nullptr, bias, C, 0, out, st, 3, nullptr, nullptr, amask, K, 0, 0,
                        wts, str, kc, rexp);
}

}  // namespace wctb
