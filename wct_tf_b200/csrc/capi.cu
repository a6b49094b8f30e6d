// extern "C" surface of libwctb200 (declared in include/wctb200.h).
#include <float.h>
#include <limits.h>
#include <stdarg.h>
#include <string.h>

#include <map>
#include <mutex>
#include <tuple>

#include "common.cuh"
#include "wctb200_debug.h"

namespace wctb {

static thread_local char t_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(t_err, sizeof(t_err), fmt, ap);
    va_end(ap);
}
int cuda_fail(cudaError_t e, const char* what) {
    set_error("CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
    return WCTB200_ECUDA;
}

// Per-stream scratch cache.  Work on one stream is ordered, so a stream can reuse ONE grow-only buffer per slot for every
// call it serves.  (The first version used cudaMallocAsync/cudaFreeAsync: the stream-ordered pool only re-uses a block
// across streams once a dependency exists, so with 8 streams it kept growing at unpredictable moments AFTER the warm-up
// steps -- each growth maps hundreds of MB and showed up as a one-off 75..500 ms step in some bench runs.)
int scratch_alloc(void** ptr, size_t bytes, cudaStream_t st, int slot) {
    struct Entry { void* p; size_t cap; };
    static std::mutex mu;
    static std::map<std::tuple<int, cudaStream_t, int>, Entry> cache;
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> lock(mu);
    Entry& e = cache[std::make_tuple(dev, st, slot)];
    if (e.cap < bytes) {
        if (e.p) {
            WCTB_CUDA(cudaStreamSynchronize(st));
            WCTB_CUDA(cudaFree(e.p));
            e.p = nullptr;
            e.cap = 0;
        }
        const size_t cap = bytes + bytes / 8 + 256;
        WCTB_CUDA(cudaMalloc(&e.p, cap));
        e.cap = cap;
    }
    *ptr = e.p;
    return 0;
}

__device__ unsigned int g_device_error = 0;

unsigned int* device_error_word() {
    static unsigned int* ptr[64] = {nullptr};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    if (!ptr[dev]) {
        void* p = nullptr;
        if (cudaGetSymbolAddress(&p, g_device_error) == cudaSuccess) ptr[dev] = static_cast<unsigned int*>(p);
    }
    return ptr[dev];
}

int device_sm_count() {
    static std::atomic<int> sms[64];
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    int v = sms[dev].load(std::memory_order_relaxed);
    if (v <= 0) {
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 148;
        sms[dev].store(v, std::memory_order_relaxed);
    }
    return v;
}

// launchers (layers.cu / wct.cu)
int launch_u8_to_f32(const uint8_t*, size_t, float*, cudaStream_t);
int launch_f32_to_u8(const float*, size_t, uint8_t*, cudaStream_t);
size_t resize_workspace_bytes(int N, int Hs, int Ws, int C, int Hd, int Wd, int Wout);
int launch_resize_u8(const uint8_t* src, int N, int Hs, int Ws, int C, int Hd, int Wd, int y0, int x0, int Hout, int Wout,
                     uint8_t* dst, void* ws, size_t ws_bytes, cudaStream_t st);
int launch_rgb_moments(const uint8_t* img, long long npix, unsigned long long* sums, cudaStream_t st);
int launch_rgb_moments_batch(const uint8_t* img, int N, long long npf, unsigned long long* sums, cudaStream_t st);
int launch_luma_match(const uint8_t* src, int N, long long npf, const float* kb, uint8_t* dst, cudaStream_t st);
int launch_luma_merge(const uint8_t* content, const uint8_t* styl, int N, long long npf, const float* kb, uint8_t* dst,
                      cudaStream_t st);
int launch_coral_apply(const uint8_t* src, long long npix, const double* A, const double* sm, const double* ss, const double* tm,
                       const double* ts, uint8_t* dst, cudaStream_t st);
int launch_noise_u8(uint8_t* out, int N, long long frame_bytes, unsigned long long seed, long long first_index, cudaStream_t st);
int launch_coarse_join(const uint8_t* content, const uint8_t* coarse, const uint8_t* styl, int N, int H, int W, int h, int w,
                       uint8_t* dst, cudaStream_t st);
int launch_luminance(const uint8_t* rgb, long long npix, float* Y, cudaStream_t st);
size_t flow_pairs_workspace_bytes(int M, int H, int W);
int launch_flow_pairs(const float* Y, int M, int H, int W, float* flows, void* ws, size_t ws_bytes, cudaStream_t st);
int launch_flow_confidence(const float* Y, int M, int H, int W, const float* flows, uint8_t* mask, int* counts, cudaStream_t st);
int launch_temporal_blend(uint8_t* frames, int N, int H, int W, const uint8_t* prev, const float* flows, const uint8_t* masks,
                          float beta, cudaStream_t st);
int launch_act_from_f32(const float*, ActGeom, __half*, cudaStream_t);
int launch_act_to_f32(const __half*, ActGeom, float*, cudaStream_t);
int launch_act_halo(__half*, ActGeom, cudaStream_t);
int launch_prep_weights(const float*, int, int, int, __half*, cudaStream_t);
int launch_prep_weights_up2(const float*, int, int, __half*, cudaStream_t);
size_t style_swap_workspace_bytes(int C, int Hc, int Wc, int Hs, int Ws, int P, int S);
int launch_style_swap_level(const __half* content, int Hc, int Wc, const __half* style, int Hs, int Ws, int C, int patch, int stride,
                            float alpha, float eps_cov, float thresh, __half* out, int32_t* k_out, void* ws, size_t ws_bytes,
                            cudaStream_t st);
size_t style_swap_state_bytes(int C, int Hs, int Ws, int P, int S);
size_t style_swap_prepare_workspace_bytes(int C);
size_t style_swap_apply_workspace_bytes(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int P, int S);
size_t style_swap_apply_min_workspace_bytes(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int P, int S);
int launch_style_swap_prepare(const __half* style, int Hs, int Ws, int C, int patch, int stride, float eps_cov, float thresh,
                              void* state, int32_t* k_out, void* ws, size_t ws_bytes, cudaStream_t st);
int launch_style_swap_apply(const __half* content, int Nc, int Hc, int Wc, int C, const void* state, int Hs, int Ws, int patch,
                            int stride, float alpha, float eps_cov, float thresh, __half* out, int32_t* k_out, void* ws, size_t ws_bytes,
                            cudaStream_t st);
size_t style_swap_labels_workspace_bytes(int Ncl, int Hc, int Wc, int Hs, int Ws, int P, int S);
int launch_style_swap_apply_labels(const __half* content, int Nc, int Hc, int Wc, int C, const void* state, int Hs, int Ws,
                                   int patch, int stride, float alpha, float eps_cov, float thresh, const uint8_t* content_labels,
                                   int Ncl, int Hm, int Wm, const uint8_t* style_labels, int Hms, int Wms, __half* out,
                                   int32_t* k_out, void* ws, size_t ws_bytes, void* label_buf, size_t label_bytes, cudaStream_t st);
void style_swap_debug_layout(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int P, int S, long long* out);
size_t style_swap_softmax_workspace_bytes(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int P, int S);
size_t style_swap_softmax_min_workspace_bytes(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int P, int S);
int style_swap_softmax_launches(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int P, int S, size_t ws_bytes, int labelled);
int launch_style_swap_apply_softmax(const __half* content, int Nc, int Hc, int Wc, int C, const void* state, int Hs, int Ws,
                                    int patch, int stride, float alpha, float eps_cov, float thresh, float temperature,
                                    const uint8_t* content_labels, int Ncl, int Hm, int Wm, const uint8_t* style_labels, int Hms,
                                    int Wms, __half* out, int32_t* k_out, void* ws, size_t ws_bytes, void* label_buf,
                                    size_t label_bytes, cudaStream_t st);
size_t style_swap_balanced_workspace_bytes(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int P, int S);
size_t style_swap_balanced_min_workspace_bytes(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int P, int S);
int style_swap_balanced_launches(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int P, int S, size_t ws_bytes, int labelled,
                                 int iters, int want_cols);
int launch_style_swap_apply_balanced(const __half* content, int Nc, int Hc, int Wc, int C, const void* state, int Hs, int Ws,
                                     int patch, int stride, float alpha, float eps_cov, float thresh, float temperature, int iters,
                                     const uint8_t* content_labels, int Ncl, int Hm, int Wm, const uint8_t* style_labels, int Hms,
                                     int Wms, __half* out, int32_t* k_out, float* col_sums, void* ws, size_t ws_bytes,
                                     void* label_buf, size_t label_bytes, cudaStream_t st);
size_t wct_style_state_layout(int C, int Ns, size_t* off_mean, size_t* off_cs, size_t* off_k);
size_t adain_style_state_layout(int C, int Ns, size_t* off_mean, size_t* off_var);
int launch_adain_style_prepare(const __half* style, int Ns, int Hs, int Ws, int C, void* state, cudaStream_t st);
int launch_adain_apply(const __half* content, int Nc, int Hc, int Wc, int C, const void* state, int Ns, float alpha, float eps,
                       __half* out, void* ws, size_t ws_bytes, cudaStream_t st);
int launch_adain_apply_blend(const __half* content, int Nc, int Hc, int Wc, int C, const void* const* states, int K,
                             const float* weights, int Nw, float alpha, float eps, __half* out, void* ws, size_t ws_bytes,
                             cudaStream_t st);
size_t stats_record_layout(int C, int N, int diag, size_t* off_n, size_t* off_t, size_t* off_s, size_t* off_S);
int launch_wct_stats_rect(const __half* act, int N, int H, int W, int C, int y0, int x0, int h, int w, void* record, cudaStream_t st);
int launch_adain_stats_rect(const __half* act, int N, int H, int W, int C, int y0, int x0, int h, int w, void* record, cudaStream_t st);
int launch_stats_accumulate(void* rec_a, const void* rec_b, int C, int N, int diag, cudaStream_t st);
size_t wct_transform_layout(int C, int N, size_t* off_m, size_t* off_bias, size_t* off_k, size_t* off_exp);
size_t adain_transform_layout(int C, int N, size_t* off_mean, size_t* off_var, size_t* off_inv, size_t* off_ms);
int launch_wct_transform_from_stats(const void* record, int Nc, int C, const void* state, int Ns, float alpha, float eps_cov,
                                    float eps_eig, float thresh, int readd, void* transform, void* ws, size_t ws_bytes, cudaStream_t st);
int launch_wct_transform_apply(const __half* act, int N, int H, int W, int C, const void* transform, __half* out, cudaStream_t st);
size_t ost_workspace_bytes(int C, int Nc);
int launch_ost_apply(const __half* content, int Nc, int Hc, int Wc, int C, const void* state, int Ns, float alpha, float eps_cov,
                     float eps_eig, float thresh, int readd, __half* out, int32_t* k_out, void* ws, size_t ws_bytes, cudaStream_t st);
int launch_ost_transform_from_stats(const void* record, int Nc, int C, const void* state, int Ns, float alpha, float eps_cov,
                                    float eps_eig, float thresh, int readd, void* transform, void* ws, size_t ws_bytes, cudaStream_t st);
int launch_adain_transform_from_stats(const void* record, int Nc, int C, const void* state, int Ns, float eps, void* transform,
                                      cudaStream_t st);
int launch_adain_transform_apply(const __half* act, int N, int H, int W, int C, const void* transform, float alpha, __half* out,
                                 cudaStream_t st);
int launch_mask_feather(const uint8_t* labels, int N, int Hm, int Wm, int R, float sigma, float* out, cudaStream_t st);
int launch_weights_resize_area(const float* src, int N, int K, int Hm, int Wm, int Hf, int Wf, float* dst, cudaStream_t st);
int launch_wct_stats_weighted(const __half* act, int N, int H, int W, int C, const float* wts, int K, void* record, cudaStream_t st);
int launch_wct_transform_apply_weighted(const __half* act, int N, int H, int W, int C, const void* transform, int K, const float* wts,
                                        const float* str, __half* out, cudaStream_t st);
int launch_adain_transform_apply_strength(const __half* act, int N, int H, int W, int C, const void* transform, float alpha,
                                          const float* strength, __half* out, cudaStream_t st);
int launch_conv3x3_ref(const __half*, ActGeom, const float*, const float*, int, int, __half*, cudaStream_t);
int launch_conv_head(const float*, int, int, int, const float*, const float*, int, __half*, cudaStream_t);
int launch_conv_tail(const __half*, ActGeom, const float*, const float*, int, float*, cudaStream_t);
int launch_maxpool2(const __half*, ActGeom, __half*, cudaStream_t);
int launch_upsample2(const __half*, ActGeom, __half*, cudaStream_t);
size_t wct_workspace_bytes(int, int, int);
int launch_wct_level(const __half*, int, int, int, const __half*, int, int, int, int, float, float, float, float, int,
                     __half*, int32_t*, void*, size_t, cudaStream_t);
int launch_adain_level(const __half*, int, int, int, const __half*, int, int, int, int, float, float, __half*, void*,
                       size_t, cudaStream_t);
size_t wct_style_state_bytes(int, int);
int launch_wct_style_prepare(const __half*, int, int, int, int, float, float, float, void*, void*, size_t, cudaStream_t);
int launch_wct_apply(const __half*, int, int, int, int, const void*, int, float, float, float, float, int, __half*, int32_t*,
                     void*, size_t, cudaStream_t);
int launch_covariance(const __half*, int, int, int, int, float, float*, float*, cudaStream_t);
size_t wct_blend_workspace_bytes(int C, int Nc, int K, int Nw);
int launch_wct_apply_blend(const __half*, int, int, int, int, const void* const*, int, const float*, int, float, float, float, float,
                           int, __half*, int32_t*, void*, size_t, cudaStream_t);
size_t adain_blend_workspace_bytes(int C, int Nc, int K);
int launch_adain_blend(const __half*, int, int, int, int, const void* const*, const int*, const int*, int, const float*, int, float,
                       float, __half*, void*, size_t, cudaStream_t);
size_t wct_regions_workspace_bytes(int C, int Nc, int R, int Hc, int Wc);
int launch_wct_apply_regions(const __half*, int, int, int, int, const uint8_t*, int, const void* const*, float, float, float, float,
                             int, __half*, int32_t*, void*, size_t, cudaStream_t);
int launch_labels_resize(const uint8_t* src, int N, int Hm, int Wm, int Hf, int Wf, uint8_t* dst, cudaStream_t st);
size_t mst_clusters_workspace_bytes(int Hs, int Ws, int C, int K);
int launch_mst_style_clusters(const __half* style, int Hs, int Ws, int C, int K, int level, uint8_t* labels, float* centres,
                              int32_t* info, void* ws, size_t ws_bytes, cudaStream_t st);
int launch_mst_data_term(const __half* act, int N, int H, int W, int C, const float* centres, const int32_t* counts, int K, float* D,
                         cudaStream_t st);
int launch_mst_smooth(const float* D, int N, int H, int W, int K, float lambda, int sweeps, uint8_t* labels, cudaStream_t st);
size_t efdm_style_state_bytes(int C, int Ns, int Hs, int Ws);
size_t efdm_style_workspace_bytes(int C, int Ns, int Hs, int Ws, int max_segments);
size_t efdm_workspace_bytes(int C, int N, int H, int W, int max_segments);
int launch_efdm_style_prepare(const __half* style, int Ns, int Hs, int Ws, int C, const float* R, float* state, void* ws,
                              size_t ws_bytes, cudaStream_t st);
size_t efdm_planes_bytes(int C, int N, int H, int W);
int launch_efdm_sliced_step(const __half* content, const float* src, int N, int H, int W, int C, const float* G, const float* state,
                            int Ns, int Hs, int Ws, float alpha, float* out_planes, __half* out, void* ws, size_t ws_bytes,
                            cudaStream_t st);
int launch_efdm_apply(const __half* content, int N, int H, int W, int C, const float* state, int Ns, int Hs, int Ws, float alpha,
                      __half* out, void* ws, size_t ws_bytes, cudaStream_t st);
size_t wct_style_prepare_regions_workspace_bytes(int C, int R, int Hs, int Ws);
int launch_wct_style_prepare_regions(const __half*, int, int, int, const uint8_t*, int, float, float, float, void*, int32_t*, void*,
                                     size_t, cudaStream_t);
int launch_covariance_regions(const __half*, int, int, int, int, const uint8_t*, int, float, float*, float*, int*, cudaStream_t);
int launch_jacobi(float*, int, int, float*, int*, cudaStream_t, const int* skip, float thresh);
int launch_eig_post(const float*, const float*, float*, int, int, float, float, int, float*, float*, int*, cudaStream_t, const int* skip);
extern int g_conv_bn_override;
extern int g_conv_oversub;
extern int g_conv_fuse;
extern int g_conv_products;
extern int g_conv_tail_tc;
extern int g_conv_head_tc;
int launch_matfun_ns(const float* A, int C, int count, int n_first, float thresh, float eps_eig, float* out, int* ok, int* kcount,
                     cudaStream_t st, float* info);
extern int g_matfun;
extern int g_matfun_max_it;
extern int g_cov_max_stages;
int set_jacobi_tolq(float v);
extern int g_jacobi_lg;
extern int g_jacobi_stagger;

// kernels index elements with 32-bit arithmetic: keep every element count (incl. a 2x upsampled output) below 2^32
static bool geom_ok(int N, int H, int W, int C) {
    return N >= 1 && H >= 2 && W >= 2 && C >= 8 && C % 8 == 0 &&
           (long long)N * (2ll * H + 2) * (2ll * W + 2) * (C / 8) < (1ll << 32) && (long long)H * W < (1ll << 31);
}

}  // namespace wctb

using namespace wctb;

#define ST(s) static_cast<cudaStream_t>(s)
#define HP(p) static_cast<__half*>(p)
#define HCP(p) static_cast<const __half*>(p)

extern "C" {

int wctb200_abi_version(void) { return WCTB200_ABI_VERSION; }
const char* wctb200_last_error(void) { return t_err; }

int wctb200_check_device(void* stream) {
    WCTB_CUDA(cudaStreamSynchronize(ST(stream)));
    unsigned int* w = device_error_word();
    if (!w) {
        set_error("device error word unavailable (no CUDA device?)");
        return WCTB200_ECUDA;
    }
    unsigned int v = 0;
    WCTB_CUDA(cudaMemcpy(&v, w, sizeof(v), cudaMemcpyDeviceToHost));
    if (v != 0) {
        unsigned int zero = 0;
        cudaMemcpy(w, &zero, sizeof(zero), cudaMemcpyHostToDevice);
        set_error("device-side pipeline time-out, code 0x%x (0x1xx producer wait, 0x2xx MMA wait, 0x3xx epilogue wait)", v);
        return WCTB200_EDEVICE;
    }
    return 0;
}

size_t wctb200_act_bytes(int N, int H, int W, int C) {
    if (!geom_ok(N, H, W, C)) return 0;
    ActGeom g(N, H, W, C);
    return (size_t)g.plane * 2 * sizeof(__half);
}

int wctb200_act_from_f32(const float* nhwc, int N, int H, int W, int C, void* act, void* stream) {
    WCTB_REQUIRE(geom_ok(N, H, W, C) && nhwc && act, "act_from_f32: bad arguments");
    return launch_act_from_f32(nhwc, ActGeom(N, H, W, C), HP(act), ST(stream));
}
int wctb200_act_to_f32(const void* act, int N, int H, int W, int C, float* nhwc, void* stream) {
    WCTB_REQUIRE(geom_ok(N, H, W, C) && nhwc && act, "act_to_f32: bad arguments");
    return launch_act_to_f32(HCP(act), ActGeom(N, H, W, C), nhwc, ST(stream));
}
int wctb200_act_halo(void* act, int N, int H, int W, int C, int flags, void* stream) {
    WCTB_REQUIRE(geom_ok(N, H, W, C) && act, "act_halo: bad arguments");
    WCTB_REQUIRE((flags & ~(WCTB200_HALO_EDGE | WCTB200_HALO_WRAP_X | WCTB200_HALO_WRAP_Y)) == 0, "act_halo: unknown flag bits 0x%x",
                 flags);
    ActGeom g(N, H, W, C);
    g.set_halo(flags);
    return launch_act_halo(HP(act), g, ST(stream));
}

int wctb200_image_u8_to_f32(const uint8_t* img, size_t count, float* out, void* stream) {
    WCTB_REQUIRE(img && out, "image_u8_to_f32: null pointer");
    if (count == 0) return 0;
    return launch_u8_to_f32(img, count, out, ST(stream));
}
int wctb200_image_f32_to_u8(const float* img, size_t count, uint8_t* out, void* stream) {
    WCTB_REQUIRE(img && out, "image_f32_to_u8: null pointer");
    if (count == 0) return 0;
    return launch_f32_to_u8(img, count, out, ST(stream));
}

static bool resize_args_ok(int N, int Hs, int Ws, int C, int Hd, int Wd) {
    return N >= 1 && Hs >= 1 && Ws >= 1 && C >= 1 && C <= 4 && Hd >= 1 && Wd >= 1 && Hs <= (1 << 15) && Ws <= (1 << 15) &&
           Hd <= (1 << 15) && Wd <= (1 << 15);
}
size_t wctb200_resize_workspace_bytes(int N, int Hs, int Ws, int C, int Hd, int Wd, int Wout) {
    if (!resize_args_ok(N, Hs, Ws, C, Hd, Wd) || Wout < 1 || Wout > Wd) return 0;
    return resize_workspace_bytes(N, Hs, Ws, C, Hd, Wd, Wout);
}
int wctb200_resize_bilinear_u8(const uint8_t* src, int N, int Hs, int Ws, int C, int Hd, int Wd, int y0, int x0, int Hout,
                               int Wout, uint8_t* dst, void* ws, size_t ws_bytes, void* stream) {
    WCTB_REQUIRE(src && dst && ws, "resize_bilinear_u8: null pointer");
    WCTB_REQUIRE(resize_args_ok(N, Hs, Ws, C, Hd, Wd), "resize_bilinear_u8: bad geometry N=%d %dx%dx%d -> %dx%d", N, Hs, Ws, C, Hd, Wd);
    WCTB_REQUIRE(y0 >= 0 && x0 >= 0 && Hout >= 1 && Wout >= 1 && y0 + Hout <= Hd && x0 + Wout <= Wd,
                 "resize_bilinear_u8: window [%d,%d)x[%d,%d) outside %dx%d", y0, y0 + Hout, x0, x0 + Wout, Hd, Wd);
    return launch_resize_u8(src, N, Hs, Ws, C, Hd, Wd, y0, x0, Hout, Wout, dst, ws, ws_bytes, ST(stream));
}
int wctb200_rgb_moments_u8(const uint8_t* img, long long npix, unsigned long long* sums, void* stream) {
    WCTB_REQUIRE(img && sums && npix >= 1 && npix < (1ll << 40), "rgb_moments_u8: bad arguments");
    return launch_rgb_moments(img, npix, sums, ST(stream));
}
// N frames of npf pixels: every byte offset is 64-bit inside the kernels, and N * npf < 2^40 keeps the integer sums exact
static bool frames_ok(int N, long long npf) { return N >= 1 && npf >= 1 && npf < (1ll << 40) && (long long)N * npf < (1ll << 40); }
int wctb200_rgb_moments_batch_u8(const uint8_t* img, int N, long long npix_per_frame, unsigned long long* sums, void* stream) {
    WCTB_REQUIRE(img && sums, "rgb_moments_batch_u8: null pointer");
    WCTB_REQUIRE(frames_ok(N, npix_per_frame), "rgb_moments_batch_u8: bad geometry N=%d npix=%lld", N, npix_per_frame);
    return launch_rgb_moments_batch(img, N, npix_per_frame, sums, ST(stream));
}
int wctb200_luminance_match_u8(const uint8_t* src, int N, long long npix_per_frame, const float* kb, uint8_t* dst, void* stream) {
    WCTB_REQUIRE(src && kb && dst, "luminance_match_u8: null pointer");
    WCTB_REQUIRE(((uintptr_t)kb & 7) == 0, "luminance_match_u8: kb must be 8-byte aligned");
    WCTB_REQUIRE(frames_ok(N, npix_per_frame), "luminance_match_u8: bad geometry N=%d npix=%lld", N, npix_per_frame);
    return launch_luma_match(src, N, npix_per_frame, kb, dst, ST(stream));
}
int wctb200_luminance_merge_u8(const uint8_t* content, const uint8_t* stylised, int N, long long npix_per_frame, const float* kb,
                               uint8_t* dst, void* stream) {
    WCTB_REQUIRE(content && stylised && kb && dst, "luminance_merge_u8: null pointer");
    WCTB_REQUIRE(((uintptr_t)kb & 7) == 0, "luminance_merge_u8: kb must be 8-byte aligned");
    WCTB_REQUIRE(frames_ok(N, npix_per_frame), "luminance_merge_u8: bad geometry N=%d npix=%lld", N, npix_per_frame);
    return launch_luma_merge(content, stylised, N, npix_per_frame, kb, dst, ST(stream));
}
int wctb200_coarse_join_u8(const uint8_t* content, const uint8_t* coarse_content, const uint8_t* coarse_stylised, int N, int H,
                           int W, int h, int w, uint8_t* dst, void* stream) {
    WCTB_REQUIRE(content && coarse_content && coarse_stylised && dst, "coarse_join_u8: null pointer");
    WCTB_REQUIRE(N >= 1 && H >= 1 && W >= 1 && h >= 1 && w >= 1 && H <= (1 << 15) && W <= (1 << 15) && h <= (1 << 15) &&
                 w <= (1 << 15) && (long long)N * H * W < (1ll << 40),
                 "coarse_join_u8: bad geometry N=%d %dx%d from %dx%d", N, H, W, h, w);
    return launch_coarse_join(content, coarse_content, coarse_stylised, N, H, W, h, w, dst, ST(stream));
}
int wctb200_coral_apply_u8(const uint8_t* src, long long npix, const double* A, const double* src_mean, const double* src_std,
                           const double* tgt_mean, const double* tgt_std, uint8_t* dst, void* stream) {
    WCTB_REQUIRE(src && dst && A && src_mean && src_std && tgt_mean && tgt_std && npix >= 1, "coral_apply_u8: bad arguments");
    return launch_coral_apply(src, npix, A, src_mean, src_std, tgt_mean, tgt_std, dst, ST(stream));
}
int wctb200_noise_u8(uint8_t* out, int N, int H, int W, int C, unsigned long long seed, long long first_index, void* stream) {
    WCTB_REQUIRE(out, "noise_u8: null pointer");
    WCTB_REQUIRE(N >= 1 && H >= 1 && W >= 1 && C >= 1 && C <= 4, "noise_u8: bad geometry N=%d %dx%dx%d", N, H, W, C);
    WCTB_REQUIRE((long long)H * W <= (1ll << 62) / C / N, "noise_u8: %d x %dx%dx%d bytes is too large", N, H, W, C);
    WCTB_REQUIRE(first_index >= 0 && first_index <= LLONG_MAX - N, "noise_u8: first_index=%lld with N=%d is out of range",
                 first_index, N);
    return launch_noise_u8(out, N, (long long)H * W * C, seed, first_index, ST(stream));
}

// the flow kernels index a plane with 32-bit pixel coordinates and a stack with 64-bit offsets
static bool flow_geom_ok(int M, int H, int W) {
    return M >= 2 && M <= 65536 && H >= 1 && W >= 1 && H <= (1 << 15) && W <= (1 << 15);
}
int wctb200_luminance_u8(const uint8_t* rgb, long long npix, float* Y, void* stream) {
    WCTB_REQUIRE(rgb && Y && npix >= 1 && npix < (1ll << 40), "luminance_u8: bad arguments");
    return launch_luminance(rgb, npix, Y, ST(stream));
}
size_t wctb200_flow_pairs_workspace_bytes(int M, int H, int W) {
    if (!flow_geom_ok(M, H, W)) return 0;
    return flow_pairs_workspace_bytes(M, H, W);
}
int wctb200_flow_pairs(const float* Y, int M, int H, int W, float* flows, void* ws, size_t ws_bytes, void* stream) {
    WCTB_REQUIRE(Y && flows && ws, "flow_pairs: null pointer");
    WCTB_REQUIRE(flow_geom_ok(M, H, W), "flow_pairs: bad geometry M=%d %dx%d (M >= 2 frames)", M, H, W);
    return launch_flow_pairs(Y, M, H, W, flows, ws, ws_bytes, ST(stream));
}
int wctb200_flow_confidence(const float* Y, int M, int H, int W, const float* flows, uint8_t* mask, int32_t* counts,
                            void* stream) {
    WCTB_REQUIRE(Y && flows && mask && counts, "flow_confidence: null pointer");
    WCTB_REQUIRE(flow_geom_ok(M, H, W), "flow_confidence: bad geometry M=%d %dx%d (M >= 2 frames)", M, H, W);
    return launch_flow_confidence(Y, M, H, W, flows, mask, counts, ST(stream));
}
int wctb200_temporal_blend_u8(uint8_t* frames, int N, int H, int W, const uint8_t* prev, const float* flows, const uint8_t* masks,
                              float beta, void* stream) {
    WCTB_REQUIRE(frames && flows && masks, "temporal_blend_u8: null pointer");
    WCTB_REQUIRE(N >= 1 && H >= 1 && W >= 1 && H <= (1 << 15) && W <= (1 << 15), "temporal_blend_u8: bad geometry N=%d %dx%d", N,
                 H, W);
    WCTB_REQUIRE(prev || N >= 2, "temporal_blend_u8: one frame without a predecessor has nothing to blend");
    WCTB_REQUIRE(beta >= 0.f && beta < 1.f, "temporal_blend_u8: beta=%g outside [0, 1)", (double)beta);
    return launch_temporal_blend(frames, N, H, W, prev, flows, masks, beta, ST(stream));
}

size_t wctb200_conv_weight_bytes(int taps, int Cin, int Cout) {
    if (taps < 1 || Cin < 1 || Cout < 1) return 0;
    return (size_t)2 * taps * Cin * Cout * sizeof(__half) + 256;     // + trailer: the power-of-two scale (layers.cu)
}
int wctb200_prep_conv_weights(const float* w_hwio, int taps, int Cin, int Cout, void* w_split, void* stream) {
    WCTB_REQUIRE(w_hwio && w_split && (taps == 9 || taps == 1) && Cin >= 1 && Cout >= 1, "prep_conv_weights: bad arguments");
    return launch_prep_weights(w_hwio, taps, Cin, Cout, HP(w_split), ST(stream));
}

int wctb200_prep_conv_weights_up2(const float* w_hwio, int Cin, int Cout, void* w_up2, void* stream) {
    WCTB_REQUIRE(w_hwio && w_up2 && Cin >= 1 && Cout >= 1, "prep_conv_weights_up2: bad arguments");
    return launch_prep_weights_up2(w_hwio, Cin, Cout, HP(w_up2), ST(stream));
}

int wctb200_conv3x3(const void* act_in, int N, int H, int W, int Cin, const void* w_split, const float* bias, int Cout,
                    int flags, void* act_out, void* stream) {
    WCTB_REQUIRE(act_in && w_split && act_out, "conv3x3: null pointer");
    WCTB_REQUIRE((flags & ~(WCTB200_RELU | WCTB200_HALO_EDGE | WCTB200_POOL2 | WCTB200_HALO_WRAP_X | WCTB200_HALO_WRAP_Y)) == 0,
                 "conv3x3: unknown flag bits 0x%x", flags);
    return launch_conv_tc(CONV_3X3, HCP(act_in), N, H, W, Cin, HCP(w_split), 1, weight_scale_ptr(HCP(w_split), 9, Cin, Cout),
                          bias, Cout, flags, HP(act_out), ST(stream));
}
int wctb200_conv3x3_up2(const void* act_in, int N, int H, int W, int Cin, const void* w_up2, const float* bias, int Cout,
                        int flags, void* act_out, void* stream) {
    WCTB_REQUIRE(act_in && w_up2 && act_out, "conv3x3_up2: null pointer");
    WCTB_REQUIRE((flags & ~(WCTB200_RELU | WCTB200_HALO_WRAP_X | WCTB200_HALO_WRAP_Y)) == 0, "conv3x3_up2: unknown flag bits 0x%x",
                 flags);
    WCTB_REQUIRE(geom_ok(N, 2 * H, 2 * W, Cout), "conv3x3_up2: output geometry too large");
    return launch_conv_tc(CONV_UP2, HCP(act_in), N, H, W, Cin, HCP(w_up2), 1, weight_scale_ptr(HCP(w_up2), 16, Cin, Cout),
                          bias, Cout, flags, HP(act_out), ST(stream));
}
int wctb200_conv3x3_ref(const void* act_in, int N, int H, int W, int Cin, const float* w_hwio, const float* bias, int Cout,
                        int flags, void* act_out, void* stream) {
    WCTB_REQUIRE(act_in && w_hwio && act_out && geom_ok(N, H, W, Cin) && Cout >= 1, "conv3x3_ref: bad arguments");
    return launch_conv3x3_ref(HCP(act_in), ActGeom(N, H, W, Cin), w_hwio, bias, Cout, flags, HP(act_out), ST(stream));
}
int wctb200_conv_head(const float* img, int N, int H, int W, const float* w, const float* b, void* act_out, void* stream) {
    WCTB_REQUIRE(img && w && b && act_out && geom_ok(N, H, W, 64), "conv_head: bad arguments");
    return launch_conv_head(img, N, H, W, w, b, 0, HP(act_out), ST(stream));
}
int wctb200_conv_head_flags(const float* img, int N, int H, int W, const float* w, const float* b, int flags, void* act_out,
                            void* stream) {
    WCTB_REQUIRE(img && w && b && act_out && geom_ok(N, H, W, 64), "conv_head_flags: bad arguments");
    WCTB_REQUIRE((flags & ~(WCTB200_HALO_WRAP_X | WCTB200_HALO_WRAP_Y)) == 0, "conv_head_flags: unknown flag bits 0x%x", flags);
    return launch_conv_head(img, N, H, W, w, b, flags, HP(act_out), ST(stream));
}
int wctb200_conv_tail(const void* act_in, int N, int H, int W, int Cin, const float* w, const float* b, int flags,
                      float* img_out, void* stream) {
    WCTB_REQUIRE(act_in && w && b && img_out && geom_ok(N, H, W, Cin) && Cin <= 1024, "conv_tail: bad arguments");
    return launch_conv_tail(HCP(act_in), ActGeom(N, H, W, Cin), w, b, flags, img_out, ST(stream));
}
int wctb200_maxpool2(const void* act_in, int N, int H, int W, int C, void* act_out, void* stream) {
    WCTB_REQUIRE(act_in && act_out && geom_ok(N, H, W, C) && (H + 1) / 2 >= 2 && (W + 1) / 2 >= 2, "maxpool2: bad arguments (output must be >= 2x2)");
    return launch_maxpool2(HCP(act_in), ActGeom(N, H, W, C), HP(act_out), ST(stream));
}
int wctb200_upsample2(const void* act_in, int N, int H, int W, int C, void* act_out, void* stream) {
    WCTB_REQUIRE(act_in && act_out && geom_ok(N, H, W, C), "upsample2: bad arguments");
    return launch_upsample2(HCP(act_in), ActGeom(N, H, W, C), HP(act_out), ST(stream));
}

size_t wctb200_wct_workspace_bytes(int C, int Nc, int Ns) {
    if (C < 8 || Nc < 0 || Ns < 0 || Nc + Ns < 1) return 0;     // Nc = 0 / Ns = 0: style-only / content-only calls
    return wct_workspace_bytes(C, Nc, Ns);
}
int wctb200_wct_level(const void* content, int Nc, int Hc, int Wc, const void* style, int Ns, int Hs, int Ws, int C,
                      float alpha, float eps_cov, float eps_eig, float thresh, int readd_content_mean, void* out,
                      int32_t* k_out, void* ws, size_t ws_bytes, void* stream) {
    WCTB_REQUIRE(content && style && out && ws, "wct_level: null pointer");
    WCTB_REQUIRE(geom_ok(Nc, Hc, Wc, C) && geom_ok(Ns, Hs, Ws, C), "wct_level: bad geometry");
    return launch_wct_level(HCP(content), Nc, Hc, Wc, HCP(style), Ns, Hs, Ws, C, alpha, eps_cov, eps_eig, thresh,
                            readd_content_mean, HP(out), k_out, ws, ws_bytes, ST(stream));
}
size_t wctb200_wct_style_state_bytes(int C, int Ns) {
    if (C < 8 || Ns < 1) return 0;
    return wct_style_state_bytes(C, Ns);
}
int wctb200_wct_style_prepare(const void* style, int Ns, int Hs, int Ws, int C, float eps_cov, float eps_eig, float thresh,
                              void* state, void* ws, size_t ws_bytes, void* stream) {
    WCTB_REQUIRE(style && state && ws, "wct_style_prepare: null pointer");
    WCTB_REQUIRE(geom_ok(Ns, Hs, Ws, C), "wct_style_prepare: bad geometry");
    return launch_wct_style_prepare(HCP(style), Ns, Hs, Ws, C, eps_cov, eps_eig, thresh, state, ws, ws_bytes, ST(stream));
}
int wctb200_wct_apply(const void* content, int Nc, int Hc, int Wc, int C, const void* state, int Ns, float alpha,
                      float eps_cov, float eps_eig, float thresh, int readd_content_mean, void* out, int32_t* k_out,
                      void* ws, size_t ws_bytes, void* stream) {
    WCTB_REQUIRE(content && state && out && ws, "wct_apply: null pointer");
    WCTB_REQUIRE(geom_ok(Nc, Hc, Wc, C), "wct_apply: bad geometry");
    return launch_wct_apply(HCP(content), Nc, Hc, Wc, C, state, Ns, alpha, eps_cov, eps_eig, thresh, readd_content_mean,
                            HP(out), k_out, ws, ws_bytes, ST(stream));
}
size_t wctb200_wct_regions_workspace_bytes(int C, int Nc, int R, int Hc, int Wc) {
    if (C < 8 || Nc < 1 || R < 1 || R > 8 || Hc < 2 || Wc < 2) return 0;
    return wct_regions_workspace_bytes(C, Nc, R, Hc, Wc);
}
int wctb200_wct_apply_regions(const void* content, int Nc, int Hc, int Wc, int C, const uint8_t* labels, int R,
                              const void* const* states, float alpha, float eps_cov, float eps_eig, float thresh,
                              int readd_content_mean, void* out, int32_t* k_out, void* ws, size_t ws_bytes, void* stream) {
    WCTB_REQUIRE(content && labels && states && out && ws, "wct_apply_regions: null pointer");
    WCTB_REQUIRE(R >= 1 && R <= 8, "wct_apply_regions: R=%d not in 1..8", R);
    WCTB_REQUIRE(geom_ok(Nc, Hc, Wc, C), "wct_apply_regions: bad geometry");
    return launch_wct_apply_regions(HCP(content), Nc, Hc, Wc, C, labels, R, states, alpha, eps_cov, eps_eig, thresh,
                                    readd_content_mean, HP(out), k_out, ws, ws_bytes, ST(stream));
}
size_t wctb200_wct_style_prepare_regions_workspace_bytes(int C, int R, int Hs, int Ws) {
    if (C < 8 || R < 1 || R > 8 || Hs < 2 || Ws < 2) return 0;
    return wct_style_prepare_regions_workspace_bytes(C, R, Hs, Ws);
}
int wctb200_wct_style_prepare_regions(const void* style, int Hs, int Ws, int C, const uint8_t* labels, int R, float eps_cov,
                                      float eps_eig, float thresh, void* state, int32_t* k_out, void* ws, size_t ws_bytes,
                                      void* stream) {
    WCTB_REQUIRE(style && labels && state && ws, "wct_style_prepare_regions: null pointer");
    WCTB_REQUIRE(R >= 1 && R <= 8, "wct_style_prepare_regions: R=%d not in 1..8", R);
    WCTB_REQUIRE(geom_ok(1, Hs, Ws, C), "wct_style_prepare_regions: bad geometry");
    return launch_wct_style_prepare_regions(HCP(style), Hs, Ws, C, labels, R, eps_cov, eps_eig, thresh, state, k_out, ws, ws_bytes,
                                            ST(stream));
}
size_t wctb200_wct_blend_workspace_bytes(int C, int Nc, int K, int Nw) {
    if (C < 8 || Nc < 1 || K < 1 || K > 8 || (Nw != 1 && Nw != Nc)) return 0;
    return wct_blend_workspace_bytes(C, Nc, K, Nw);
}
int wctb200_wct_apply_blend(const void* content, int Nc, int Hc, int Wc, int C, const void* const* states, int K, const float* weights,
                            int Nw, float alpha, float eps_cov, float eps_eig, float thresh, int readd_content_mean, void* out,
                            int32_t* k_out, void* ws, size_t ws_bytes, void* stream) {
    WCTB_REQUIRE(content && states && weights && out && ws, "wct_apply_blend: null pointer");
    WCTB_REQUIRE(K >= 1 && K <= 8, "wct_apply_blend: K=%d not in 1..8", K);
    WCTB_REQUIRE(geom_ok(Nc, Hc, Wc, C), "wct_apply_blend: bad geometry");
    return launch_wct_apply_blend(HCP(content), Nc, Hc, Wc, C, states, K, weights, Nw, alpha, eps_cov, eps_eig, thresh,
                                  readd_content_mean, HP(out), k_out, ws, ws_bytes, ST(stream));
}
size_t wctb200_adain_blend_workspace_bytes(int C, int Nc, int K) {
    if (C < 8 || Nc < 1 || K < 1 || K > 8) return 0;
    return adain_blend_workspace_bytes(C, Nc, K);
}
int wctb200_adain_blend(const void* content, int Nc, int Hc, int Wc, int C, const void* const* styles, const int* Hs, const int* Ws,
                        int K, const float* weights, int Nw, float alpha, float eps, void* out, void* ws, size_t ws_bytes,
                        void* stream) {
    WCTB_REQUIRE(content && styles && Hs && Ws && weights && out && ws, "adain_blend: null pointer");
    WCTB_REQUIRE(K >= 1 && K <= 8, "adain_blend: K=%d not in 1..8", K);
    WCTB_REQUIRE(geom_ok(Nc, Hc, Wc, C), "adain_blend: bad geometry");
    for (int k = 0; k < K; ++k)
        WCTB_REQUIRE(geom_ok(1, Hs[k], Ws[k], C), "adain_blend: bad geometry of style %d", k);
    return launch_adain_blend(HCP(content), Nc, Hc, Wc, C, styles, Hs, Ws, K, weights, Nw, alpha, eps, HP(out), ws, ws_bytes,
                              ST(stream));
}
// multimodal style transfer (mst.cu): one channel count of the encoder levels, K in 1..8
static bool mst_args_ok(int C, int K) { return (C == 64 || C == 128 || C == 256 || C == 512) && K >= 1 && K <= 8; }
size_t wctb200_mst_style_clusters_workspace_bytes(int Hs, int Ws, int C, int K) {
    if (!mst_args_ok(C, K) || !geom_ok(1, Hs, Ws, C)) return 0;
    return mst_clusters_workspace_bytes(Hs, Ws, C, K);
}
int wctb200_mst_style_clusters(const void* style, int Hs, int Ws, int C, int K, int level, uint8_t* labels_out, float* centres_out,
                               int32_t* info_out, void* ws, size_t ws_bytes, void* stream) {
    WCTB_REQUIRE(style && labels_out && centres_out && info_out && ws, "mst_style_clusters: null pointer");
    WCTB_REQUIRE(mst_args_ok(C, K) && geom_ok(1, Hs, Ws, C) && level >= 0,
                 "mst_style_clusters: bad arguments %dx%d C=%d K=%d level=%d (C in {64,128,256,512}, K in 1..8)", Hs, Ws, C, K, level);
    return launch_mst_style_clusters(HCP(style), Hs, Ws, C, K, level, labels_out, centres_out, info_out, ws, ws_bytes, ST(stream));
}
int wctb200_mst_data_term(const void* content, int N, int H, int W, int C, const float* centres, const int32_t* counts, int K,
                          float* D_out, void* stream) {
    WCTB_REQUIRE(content && centres && counts && D_out, "mst_data_term: null pointer");
    WCTB_REQUIRE(mst_args_ok(C, K) && geom_ok(N, H, W, C), "mst_data_term: bad arguments N=%d %dx%d C=%d K=%d", N, H, W, C, K);
    return launch_mst_data_term(HCP(content), N, H, W, C, centres, counts, K, D_out, ST(stream));
}
int wctb200_mst_smooth(const float* D, int N, int H, int W, int K, float lambda, int sweeps, uint8_t* labels_out, void* stream) {
    WCTB_REQUIRE(D && labels_out, "mst_smooth: null pointer");
    WCTB_REQUIRE(N >= 1 && H >= 1 && W >= 1 && (long long)N * H * W < (1ll << 40) && K >= 1 && K <= 8 && sweeps >= 0 &&
                     sweeps <= 1024 && lambda >= 0.f && lambda <= FLT_MAX,
                 "mst_smooth: bad arguments N=%d %dx%d K=%d lambda=%g sweeps=%d", N, H, W, K, (double)lambda, sweeps);
    return launch_mst_smooth(D, N, H, W, K, lambda, sweeps, labels_out, ST(stream));
}
// exact feature distribution matching (efdm.cu).  A style map may be 1x1 (only its interior is read); the content is an
// activation of at least 2x2, which its reflect halo needs.
static bool efdm_style_ok(int Ns, int Hs, int Ws, int C) {
    return Ns >= 1 && Hs >= 1 && Ws >= 1 && C >= 8 && C % 8 == 0 && (long long)Hs * Ws < (1ll << 31) &&
           (long long)Ns * (Hs + 2) * (Ws + 2) * (C / 8) < (1ll << 32);
}
size_t wctb200_efdm_style_state_bytes(int C, int Ns, int Hs, int Ws) {
    if (!efdm_style_ok(Ns, Hs, Ws, C)) return 0;
    return efdm_style_state_bytes(C, Ns, Hs, Ws);
}
size_t wctb200_efdm_style_workspace_bytes(int C, int Ns, int Hs, int Ws, int max_segments) {
    if (!efdm_style_ok(Ns, Hs, Ws, C) || max_segments < 1) return 0;
    return efdm_style_workspace_bytes(C, Ns, Hs, Ws, max_segments);
}
int wctb200_efdm_style_prepare(const void* style, int Ns, int Hs, int Ws, int C, void* state, void* ws, size_t ws_bytes,
                               void* stream) {
    WCTB_REQUIRE(style && state && ws, "efdm_style_prepare: null pointer");
    WCTB_REQUIRE(efdm_style_ok(Ns, Hs, Ws, C), "efdm_style_prepare: bad geometry Ns=%d %dx%d C=%d", Ns, Hs, Ws, C);
    return launch_efdm_style_prepare(HCP(style), Ns, Hs, Ws, C, nullptr, static_cast<float*>(state), ws, ws_bytes, ST(stream));
}
size_t wctb200_efdm_workspace_bytes(int C, int N, int H, int W, int max_segments) {
    if (!geom_ok(N, H, W, C) || max_segments < 1) return 0;
    return efdm_workspace_bytes(C, N, H, W, max_segments);
}
int wctb200_efdm_apply(const void* content, int N, int H, int W, int C, const void* state, int Ns, int Hs, int Ws, float alpha,
                       void* out, void* ws, size_t ws_bytes, void* stream) {
    WCTB_REQUIRE(content && state && out && (ws || alpha == 0.f), "efdm_apply: null pointer");
    WCTB_REQUIRE(geom_ok(N, H, W, C) && efdm_style_ok(Ns, Hs, Ws, C) && (Ns == 1 || Ns == N),
                 "efdm_apply: bad geometry N=%d %dx%d C=%d, Ns=%d %dx%d (Ns in {1, N})", N, H, W, C, Ns, Hs, Ws);
    WCTB_REQUIRE(alpha >= -FLT_MAX && alpha <= FLT_MAX, "efdm_apply: alpha must be finite");
    return launch_efdm_apply(HCP(content), N, H, W, C, static_cast<const float*>(state), Ns, Hs, Ws, alpha, HP(out), ws, ws_bytes,
                             ST(stream));
}
// sliced distribution matching (efdm.cu, DESIGN.md §3.3.14): the rotation mixes whole 64-channel blocks of a frame
size_t wctb200_efdm_planes_bytes(int C, int N, int H, int W) {
    if (!geom_ok(N, H, W, C) || C % 64) return 0;
    return efdm_planes_bytes(C, N, H, W);
}
int wctb200_efdm_rotated_style_prepare(const void* style, int Ns, int Hs, int Ws, int C, const float* R, void* state, void* ws,
                                       size_t ws_bytes, void* stream) {
    WCTB_REQUIRE(style && R && state && ws, "efdm_rotated_style_prepare: null pointer");
    WCTB_REQUIRE(efdm_style_ok(Ns, Hs, Ws, C) && C % 64 == 0, "efdm_rotated_style_prepare: bad geometry Ns=%d %dx%d C=%d (C %% 64 == 0)",
                 Ns, Hs, Ws, C);
    return launch_efdm_style_prepare(HCP(style), Ns, Hs, Ws, C, R, static_cast<float*>(state), ws, ws_bytes, ST(stream));
}
int wctb200_efdm_sliced_step(const void* content, const float* src, int N, int H, int W, int C, const float* G, const void* state,
                             int Ns, int Hs, int Ws, float alpha, float* out_planes, void* out, void* ws, size_t ws_bytes,
                             void* stream) {
    WCTB_REQUIRE(G && state && ws && (content || src) && (out_planes ? !out : (content && out)),
                 "efdm_sliced_step: null pointer (content or src in; out_planes, or content and out)");
    WCTB_REQUIRE(geom_ok(N, H, W, C) && C % 64 == 0 && efdm_style_ok(Ns, Hs, Ws, C) && (Ns == 1 || Ns == N),
                 "efdm_sliced_step: bad geometry N=%d %dx%d C=%d, Ns=%d %dx%d (C %% 64 == 0, Ns in {1, N})", N, H, W, C, Ns, Hs, Ws);
    WCTB_REQUIRE(alpha >= -FLT_MAX && alpha <= FLT_MAX, "efdm_sliced_step: alpha must be finite");
    return launch_efdm_sliced_step(HCP(content), src, N, H, W, C, G, static_cast<const float*>(state), Ns, Hs, Ws, alpha, out_planes,
                                   HP(out), ws, ws_bytes, ST(stream));
}
int wctb200_labels_resize_nearest(const uint8_t* src, int N, int Hm, int Wm, int Hf, int Wf, uint8_t* dst, void* stream) {
    WCTB_REQUIRE(src && dst, "labels_resize_nearest: null pointer");
    WCTB_REQUIRE(N >= 1 && Hm >= 1 && Wm >= 1 && Hf >= 1 && Wf >= 1 && Hm <= (1 << 15) && Wm <= (1 << 15) && Hf <= (1 << 15) &&
                     Wf <= (1 << 15),
                 "labels_resize_nearest: bad geometry N=%d %dx%d -> %dx%d", N, Hm, Wm, Hf, Wf);
    return launch_labels_resize(src, N, Hm, Wm, Hf, Wf, dst, ST(stream));
}
int wctb200_adain_level(const void* content, int Nc, int Hc, int Wc, const void* style, int Ns, int Hs, int Ws, int C,
                        float alpha, float eps, void* out, void* ws, size_t ws_bytes, void* stream) {
    WCTB_REQUIRE(content && style && out && ws, "adain_level: null pointer");
    WCTB_REQUIRE(geom_ok(Nc, Hc, Wc, C) && geom_ok(Ns, Hs, Ws, C), "adain_level: bad geometry");
    return launch_adain_level(HCP(content), Nc, Hc, Wc, HCP(style), Ns, Hs, Ws, C, alpha, eps, HP(out), ws, ws_bytes,
                              ST(stream));
}

int wctb200_covariance(const void* act, int N, int H, int W, int C, float eps_cov, float* mean, float* cov, void* stream) {
    WCTB_REQUIRE(act && mean && cov && geom_ok(N, H, W, C), "covariance: bad arguments");
    return launch_covariance(HCP(act), N, H, W, C, eps_cov, mean, cov, ST(stream));
}

int wctb200_covariance_regions(const void* act, int N, int H, int W, int C, const uint8_t* labels, int R, float eps_cov,
                               float* mean, float* cov, int32_t* counts, void* stream) {
    WCTB_REQUIRE(act && labels && mean && cov && counts && geom_ok(N, H, W, C), "covariance_regions: bad arguments");
    WCTB_REQUIRE(R >= 1 && R <= 8, "covariance_regions: R=%d not in 1..8", R);
    return launch_covariance_regions(HCP(act), N, H, W, C, labels, R, eps_cov, mean, cov, counts, ST(stream));
}

int wctb200_jacobi_eigh(float* a, int C, int count, float* sigma, int32_t* sweeps, void* stream) {
    WCTB_REQUIRE(a && sigma && count >= 1, "jacobi_eigh: bad arguments");
    WCTB_REQUIRE(C == 64 || C == 128 || C == 256 || C == 512, "jacobi_eigh: C=%d not in {64,128,256,512}", C);
    // scratch: convergence words (16 floats per matrix), a pristine copy of the input (Rayleigh quotients), lambda
    const size_t nmat = (size_t)count * C * C;
    float* scratch = nullptr;
    {
        int rc0 = scratch_alloc(reinterpret_cast<void**>(&scratch), ((size_t)count * 16 + nmat + (size_t)count * C) * sizeof(float), ST(stream), 2);
        if (rc0) return rc0;
    }
    float* conv = scratch;
    float* a0 = scratch + (size_t)count * 16;
    float* lam = a0 + nmat;
    cudaError_t ce = cudaMemcpyAsync(a0, a, nmat * sizeof(float), cudaMemcpyDeviceToDevice, ST(stream));
    int rc = ce == cudaSuccess ? launch_jacobi(a, C, count, conv, sweeps, ST(stream), nullptr, 0.f) : cuda_fail(ce, "cudaMemcpyAsync");
    if (!rc) rc = launch_eig_post(a, a0, lam, C, count, 0.f, 0.f, count, sigma, nullptr, nullptr, ST(stream), nullptr);
    return rc;
}

size_t wctb200_style_swap_workspace_bytes(int C, int Hc, int Wc, int Hs, int Ws, int patch, int stride) {
    if (!geom_ok(1, Hc, Wc, C) || !geom_ok(1, Hs, Ws, C) || patch < 1 || patch > 16 || stride < 1 || stride > 16 || Hc < patch ||
        Wc < patch || Hs < patch || Ws < patch)
        return 0;
    return style_swap_workspace_bytes(C, Hc, Wc, Hs, Ws, patch, stride);
}
int wctb200_style_swap_level(const void* content, int Hc, int Wc, const void* style, int Hs, int Ws, int C, int patch, int stride,
                             float alpha, float eps_cov, float thresh, void* out, int32_t* k_out, void* ws, size_t ws_bytes,
                             void* stream) {
    WCTB_REQUIRE(content && style && out && ws, "style_swap_level: null pointer");
    WCTB_REQUIRE(geom_ok(1, Hc, Wc, C) && geom_ok(1, Hs, Ws, C), "style_swap_level: bad geometry");
    return launch_style_swap_level(HCP(content), Hc, Wc, HCP(style), Hs, Ws, C, patch, stride, alpha, eps_cov, thresh, HP(out), k_out, ws,
                                   ws_bytes, ST(stream));
}
static bool swap_style_ok(int C, int Hs, int Ws, int patch, int stride) {
    return geom_ok(1, Hs, Ws, C) && patch >= 1 && patch <= 16 && stride >= 1 && stride <= 16 && Hs >= patch && Ws >= patch;
}
size_t wctb200_style_swap_state_bytes(int C, int Hs, int Ws, int patch, int stride) {
    if (!swap_style_ok(C, Hs, Ws, patch, stride)) return 0;
    return style_swap_state_bytes(C, Hs, Ws, patch, stride);
}
size_t wctb200_style_swap_prepare_workspace_bytes(int C, int Hs, int Ws, int patch, int stride) {
    if (!swap_style_ok(C, Hs, Ws, patch, stride)) return 0;
    return style_swap_prepare_workspace_bytes(C);
}
int wctb200_style_swap_prepare(const void* style, int Hs, int Ws, int C, int patch, int stride, float eps_cov, float thresh, void* state,
                               int32_t* k_out, void* ws, size_t ws_bytes, void* stream) {
    WCTB_REQUIRE(style && state && ws, "style_swap_prepare: null pointer");
    WCTB_REQUIRE(geom_ok(1, Hs, Ws, C), "style_swap_prepare: bad geometry");
    return launch_style_swap_prepare(HCP(style), Hs, Ws, C, patch, stride, eps_cov, thresh, state, k_out, ws, ws_bytes, ST(stream));
}
size_t wctb200_style_swap_apply_workspace_bytes(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int patch, int stride) {
    if (!swap_style_ok(C, Hs, Ws, patch, stride) || !geom_ok(Nc, Hc, Wc, C) || Hc < patch || Wc < patch) return 0;
    return style_swap_apply_workspace_bytes(C, Nc, Hc, Wc, Hs, Ws, patch, stride);
}
size_t wctb200_style_swap_apply_min_workspace_bytes(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int patch, int stride) {
    if (!swap_style_ok(C, Hs, Ws, patch, stride) || !geom_ok(Nc, Hc, Wc, C) || Hc < patch || Wc < patch) return 0;
    return style_swap_apply_min_workspace_bytes(C, Nc, Hc, Wc, Hs, Ws, patch, stride);
}
int wctb200_style_swap_apply(const void* content, int Nc, int Hc, int Wc, int C, const void* state, int Hs, int Ws, int patch, int stride,
                             float alpha, float eps_cov, float thresh, void* out, int32_t* k_out, void* ws, size_t ws_bytes,
                             void* stream) {
    WCTB_REQUIRE(content && state && out && ws, "style_swap_apply: null pointer");
    WCTB_REQUIRE(Nc >= 1, "style_swap_apply: Nc=%d < 1", Nc);
    WCTB_REQUIRE(geom_ok(Nc, Hc, Wc, C) && geom_ok(1, Hs, Ws, C), "style_swap_apply: bad geometry");
    return launch_style_swap_apply(HCP(content), Nc, Hc, Wc, C, state, Hs, Ws, patch, stride, alpha, eps_cov, thresh, HP(out), k_out,
                                   ws, ws_bytes, ST(stream));
}
static bool swap_label_map_ok(int N, int Hm, int Wm) {
    return N >= 1 && Hm >= 1 && Wm >= 1 && Hm <= (1 << 15) && Wm <= (1 << 15);
}
size_t wctb200_style_swap_labels_workspace_bytes(int Ncl, int Hc, int Wc, int Hs, int Ws, int patch, int stride) {
    if (!swap_style_ok(64, Hs, Ws, patch, stride) || !geom_ok(Ncl, Hc, Wc, 64) || Hc < patch || Wc < patch) return 0;
    return style_swap_labels_workspace_bytes(Ncl, Hc, Wc, Hs, Ws, patch, stride);
}
int wctb200_style_swap_apply_labels(const void* content, int Nc, int Hc, int Wc, int C, const void* state, int Hs, int Ws, int patch,
                                    int stride, float alpha, float eps_cov, float thresh, const uint8_t* content_labels, int Ncl,
                                    int Hm, int Wm, const uint8_t* style_labels, int Hms, int Wms, void* out, int32_t* k_out, void* ws,
                                    size_t ws_bytes, void* label_buf, size_t label_bytes, void* stream) {
    WCTB_REQUIRE(content && state && out && ws && content_labels && style_labels && label_buf,
                 "style_swap_apply_labels: null pointer");
    WCTB_REQUIRE(Nc >= 1, "style_swap_apply_labels: Nc=%d < 1", Nc);
    WCTB_REQUIRE(geom_ok(Nc, Hc, Wc, C) && geom_ok(1, Hs, Ws, C), "style_swap_apply_labels: bad geometry");
    WCTB_REQUIRE(swap_label_map_ok(Ncl, Hm, Wm) && (Ncl == 1 || Ncl == Nc) && swap_label_map_ok(1, Hms, Wms),
                 "style_swap_apply_labels: %d content label maps of %dx%d for %d frames, style labels %dx%d", Ncl, Hm, Wm, Nc,
                 Hms, Wms);
    return launch_style_swap_apply_labels(HCP(content), Nc, Hc, Wc, C, state, Hs, Ws, patch, stride, alpha, eps_cov, thresh,
                                          content_labels, Ncl, Hm, Wm, style_labels, Hms, Wms, HP(out), k_out, ws, ws_bytes,
                                          label_buf, label_bytes, ST(stream));
}
size_t wctb200_style_swap_softmax_workspace_bytes(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int patch, int stride) {
    if (!swap_style_ok(C, Hs, Ws, patch, stride) || !geom_ok(Nc, Hc, Wc, C) || Hc < patch || Wc < patch) return 0;
    return style_swap_softmax_workspace_bytes(C, Nc, Hc, Wc, Hs, Ws, patch, stride);
}
size_t wctb200_style_swap_softmax_min_workspace_bytes(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int patch, int stride) {
    if (!swap_style_ok(C, Hs, Ws, patch, stride) || !geom_ok(Nc, Hc, Wc, C) || Hc < patch || Wc < patch) return 0;
    return style_swap_softmax_min_workspace_bytes(C, Nc, Hc, Wc, Hs, Ws, patch, stride);
}
int wctb200_style_swap_softmax_launches(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int patch, int stride, size_t ws_bytes,
                                         int labelled) {
    if (!swap_style_ok(C, Hs, Ws, patch, stride) || !geom_ok(Nc, Hc, Wc, C) || Hc < patch || Wc < patch) return 0;
    return style_swap_softmax_launches(C, Nc, Hc, Wc, Hs, Ws, patch, stride, ws_bytes, labelled);
}
int wctb200_style_swap_apply_softmax(const void* content, int Nc, int Hc, int Wc, int C, const void* state, int Hs, int Ws, int patch,
                                     int stride, float alpha, float eps_cov, float thresh, float temperature,
                                     const uint8_t* content_labels, int Ncl, int Hm, int Wm, const uint8_t* style_labels, int Hms,
                                     int Wms, void* out, int32_t* k_out, void* ws, size_t ws_bytes, void* label_buf,
                                     size_t label_bytes, void* stream) {
    WCTB_REQUIRE(content && state && out && ws, "style_swap_apply_softmax: null pointer");
    WCTB_REQUIRE(Nc >= 1, "style_swap_apply_softmax: Nc=%d < 1", Nc);
    WCTB_REQUIRE(geom_ok(Nc, Hc, Wc, C) && geom_ok(1, Hs, Ws, C), "style_swap_apply_softmax: bad geometry");
    if (content_labels || style_labels) {
        WCTB_REQUIRE(content_labels && style_labels && label_buf, "style_swap_apply_softmax: null label pointer");
        WCTB_REQUIRE(swap_label_map_ok(Ncl, Hm, Wm) && (Ncl == 1 || Ncl == Nc) && swap_label_map_ok(1, Hms, Wms),
                     "style_swap_apply_softmax: %d content label maps of %dx%d for %d frames, style labels %dx%d", Ncl, Hm, Wm,
                     Nc, Hms, Wms);
    }
    return launch_style_swap_apply_softmax(HCP(content), Nc, Hc, Wc, C, state, Hs, Ws, patch, stride, alpha, eps_cov, thresh,
                                           temperature, content_labels, Ncl, Hm, Wm, style_labels, Hms, Wms, HP(out), k_out, ws,
                                           ws_bytes, label_buf, label_bytes, ST(stream));
}
size_t wctb200_style_swap_balanced_workspace_bytes(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int patch, int stride) {
    if (!swap_style_ok(C, Hs, Ws, patch, stride) || !geom_ok(Nc, Hc, Wc, C) || Hc < patch || Wc < patch) return 0;
    return style_swap_balanced_workspace_bytes(C, Nc, Hc, Wc, Hs, Ws, patch, stride);
}
size_t wctb200_style_swap_balanced_min_workspace_bytes(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int patch, int stride) {
    if (!swap_style_ok(C, Hs, Ws, patch, stride) || !geom_ok(Nc, Hc, Wc, C) || Hc < patch || Wc < patch) return 0;
    return style_swap_balanced_min_workspace_bytes(C, Nc, Hc, Wc, Hs, Ws, patch, stride);
}
int wctb200_style_swap_balanced_launches(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int patch, int stride, size_t ws_bytes,
                                         int labelled, int iters, int want_cols) {
    if (!swap_style_ok(C, Hs, Ws, patch, stride) || !geom_ok(Nc, Hc, Wc, C) || Hc < patch || Wc < patch) return 0;
    return style_swap_balanced_launches(C, Nc, Hc, Wc, Hs, Ws, patch, stride, ws_bytes, labelled, iters, want_cols);
}
int wctb200_style_swap_apply_balanced(const void* content, int Nc, int Hc, int Wc, int C, const void* state, int Hs, int Ws,
                                      int patch, int stride, float alpha, float eps_cov, float thresh, float temperature, int iters,
                                      const uint8_t* content_labels, int Ncl, int Hm, int Wm, const uint8_t* style_labels, int Hms,
                                      int Wms, void* out, int32_t* k_out, float* col_sums, void* ws, size_t ws_bytes,
                                      void* label_buf, size_t label_bytes, void* stream) {
    WCTB_REQUIRE(content && state && out && ws, "style_swap_apply_balanced: null pointer");
    WCTB_REQUIRE(Nc >= 1, "style_swap_apply_balanced: Nc=%d < 1", Nc);
    WCTB_REQUIRE(geom_ok(Nc, Hc, Wc, C) && geom_ok(1, Hs, Ws, C), "style_swap_apply_balanced: bad geometry");
    if (content_labels || style_labels) {
        WCTB_REQUIRE(content_labels && style_labels && label_buf, "style_swap_apply_balanced: null label pointer");
        WCTB_REQUIRE(swap_label_map_ok(Ncl, Hm, Wm) && (Ncl == 1 || Ncl == Nc) && swap_label_map_ok(1, Hms, Wms),
                     "style_swap_apply_balanced: %d content label maps of %dx%d for %d frames, style labels %dx%d", Ncl, Hm, Wm,
                     Nc, Hms, Wms);
    }
    return launch_style_swap_apply_balanced(HCP(content), Nc, Hc, Wc, C, state, Hs, Ws, patch, stride, alpha, eps_cov, thresh,
                                            temperature, iters, content_labels, Ncl, Hm, Wm, style_labels, Hms, Wms, HP(out), k_out,
                                            col_sums, ws, ws_bytes, label_buf, label_bytes, ST(stream));
}
size_t wctb200_wct_style_state_layout(int C, int Ns, size_t* off_mean, size_t* off_cs, size_t* off_k) {
    if (C < 8 || Ns < 1) return 0;
    return wct_style_state_layout(C, Ns, off_mean, off_cs, off_k);
}
size_t wctb200_adain_style_state_bytes(int C, int Ns) {
    if (C < 8 || C % 8 != 0 || Ns < 1) return 0;
    return adain_style_state_layout(C, Ns, nullptr, nullptr);
}
size_t wctb200_adain_style_state_layout(int C, int Ns, size_t* off_mean, size_t* off_var) {
    if (C < 8 || C % 8 != 0 || Ns < 1) return 0;
    return adain_style_state_layout(C, Ns, off_mean, off_var);
}
int wctb200_adain_style_prepare(const void* style, int Ns, int Hs, int Ws, int C, void* state, void* stream) {
    WCTB_REQUIRE(style && state, "adain_style_prepare: null pointer");
    WCTB_REQUIRE(geom_ok(Ns, Hs, Ws, C), "adain_style_prepare: bad geometry");
    return launch_adain_style_prepare(HCP(style), Ns, Hs, Ws, C, state, ST(stream));
}
int wctb200_adain_apply(const void* content, int Nc, int Hc, int Wc, int C, const void* state, int Ns, float alpha, float eps,
                        void* out, void* ws, size_t ws_bytes, void* stream) {
    WCTB_REQUIRE(content && state && out && ws, "adain_apply: null pointer");
    WCTB_REQUIRE(geom_ok(Nc, Hc, Wc, C), "adain_apply: bad geometry");
    return launch_adain_apply(HCP(content), Nc, Hc, Wc, C, state, Ns, alpha, eps, HP(out), ws, ws_bytes, ST(stream));
}
int wctb200_adain_apply_blend(const void* content, int Nc, int Hc, int Wc, int C, const void* const* states, int K,
                              const float* weights, int Nw, float alpha, float eps, void* out, void* ws, size_t ws_bytes,
                              void* stream) {
    WCTB_REQUIRE(content && states && weights && out && ws, "adain_apply_blend: null pointer");
    WCTB_REQUIRE(K >= 1 && K <= 8, "adain_apply_blend: K=%d not in 1..8", K);
    WCTB_REQUIRE(geom_ok(Nc, Hc, Wc, C), "adain_apply_blend: bad geometry");
    return launch_adain_apply_blend(HCP(content), Nc, Hc, Wc, C, states, K, weights, Nw, alpha, eps, HP(out), ws, ws_bytes,
                                    ST(stream));
}
// ---- tiled stylisation: statistics records and transforms (DESIGN.md §3.3.7) ----
static bool wct_channels_ok(int C) { return C == 64 || C == 128 || C == 256 || C == 512; }
static bool rect_ok(int H, int W, int y0, int x0, int h, int w) {
    return y0 >= 0 && x0 >= 0 && h >= 1 && w >= 1 && (long long)y0 + h <= H && (long long)x0 + w <= W;
}
size_t wctb200_stats_record_layout(int C, int N, int diag, size_t* off_n, size_t* off_t, size_t* off_s, size_t* off_S) {
    if (C < 8 || C % 8 != 0 || C > 2048 || N < 1 || (diag != 0 && diag != 1)) return 0;
    return stats_record_layout(C, N, diag, off_n, off_t, off_s, off_S);
}
int wctb200_wct_stats_rect(const void* act, int N, int H, int W, int C, int y0, int x0, int h, int w, void* record, void* stream) {
    WCTB_REQUIRE(act && record, "wct_stats_rect: null pointer");
    WCTB_REQUIRE(geom_ok(N, H, W, C) && wct_channels_ok(C), "wct_stats_rect: bad geometry");
    WCTB_REQUIRE(rect_ok(H, W, y0, x0, h, w), "wct_stats_rect: rectangle (%d,%d)+%dx%d outside %dx%d", y0, x0, h, w, H, W);
    return launch_wct_stats_rect(HCP(act), N, H, W, C, y0, x0, h, w, record, ST(stream));
}
int wctb200_adain_stats_rect(const void* act, int N, int H, int W, int C, int y0, int x0, int h, int w, void* record, void* stream) {
    WCTB_REQUIRE(act && record, "adain_stats_rect: null pointer");
    WCTB_REQUIRE(geom_ok(N, H, W, C) && C <= 2048, "adain_stats_rect: bad geometry");
    WCTB_REQUIRE(rect_ok(H, W, y0, x0, h, w), "adain_stats_rect: rectangle (%d,%d)+%dx%d outside %dx%d", y0, x0, h, w, H, W);
    return launch_adain_stats_rect(HCP(act), N, H, W, C, y0, x0, h, w, record, ST(stream));
}
int wctb200_stats_accumulate(void* record_a, const void* record_b, int C, int N, int diag, void* stream) {
    WCTB_REQUIRE(record_a && record_b, "stats_accumulate: null pointer");
    WCTB_REQUIRE(wctb200_stats_record_layout(C, N, diag, nullptr, nullptr, nullptr, nullptr) > 0, "stats_accumulate: bad arguments");
    return launch_stats_accumulate(record_a, record_b, C, N, diag, ST(stream));
}
size_t wctb200_wct_transform_layout(int C, int N, size_t* off_m, size_t* off_bias, size_t* off_k) {
    if (!wct_channels_ok(C) || N < 1) return 0;
    return wct_transform_layout(C, N, off_m, off_bias, off_k, nullptr);
}
size_t wctb200_wct_transform_row_exp_offset(int C, int N) {
    if (!wct_channels_ok(C) || N < 1) return 0;
    size_t off;
    wct_transform_layout(C, N, nullptr, nullptr, nullptr, &off);
    return off;
}
int wctb200_wct_transform_from_stats(const void* record, int Nc, int C, const void* state, int Ns, float alpha, float eps_cov,
                                     float eps_eig, float thresh, int readd_content_mean, void* transform, void* ws, size_t ws_bytes,
                                     void* stream) {
    WCTB_REQUIRE(record && state && transform && ws, "wct_transform_from_stats: null pointer");
    WCTB_REQUIRE(wct_channels_ok(C) && Nc >= 1, "wct_transform_from_stats: bad arguments");
    return launch_wct_transform_from_stats(record, Nc, C, state, Ns, alpha, eps_cov, eps_eig, thresh, readd_content_mean, transform,
                                           ws, ws_bytes, ST(stream));
}
int wctb200_wct_transform_apply(const void* act, int N, int H, int W, int C, const void* transform, void* out, void* stream) {
    WCTB_REQUIRE(act && transform && out, "wct_transform_apply: null pointer");
    WCTB_REQUIRE(geom_ok(N, H, W, C) && wct_channels_ok(C), "wct_transform_apply: bad geometry");
    return launch_wct_transform_apply(HCP(act), N, H, W, C, transform, HP(out), ST(stream));
}
size_t wctb200_ost_workspace_bytes(int C, int Nc) {
    if (!wct_channels_ok(C) || Nc < 1) return 0;
    return ost_workspace_bytes(C, Nc);
}
int wctb200_ost_apply(const void* content, int Nc, int Hc, int Wc, int C, const void* state, int Ns, float alpha, float eps_cov,
                      float eps_eig, float thresh, int readd_content_mean, void* out, int32_t* k_out, void* ws, size_t ws_bytes,
                      void* stream) {
    WCTB_REQUIRE(content && state && out && ws, "ost_apply: null pointer");
    WCTB_REQUIRE(geom_ok(Nc, Hc, Wc, C), "ost_apply: bad geometry");
    return launch_ost_apply(HCP(content), Nc, Hc, Wc, C, state, Ns, alpha, eps_cov, eps_eig, thresh, readd_content_mean, HP(out),
                            k_out, ws, ws_bytes, ST(stream));
}
int wctb200_ost_transform_from_stats(const void* record, int Nc, int C, const void* state, int Ns, float alpha, float eps_cov,
                                     float eps_eig, float thresh, int readd_content_mean, void* transform, void* ws, size_t ws_bytes,
                                     void* stream) {
    WCTB_REQUIRE(record && state && transform && ws, "ost_transform_from_stats: null pointer");
    WCTB_REQUIRE(wct_channels_ok(C) && Nc >= 1, "ost_transform_from_stats: bad arguments");
    return launch_ost_transform_from_stats(record, Nc, C, state, Ns, alpha, eps_cov, eps_eig, thresh, readd_content_mean, transform,
                                           ws, ws_bytes, ST(stream));
}
size_t wctb200_adain_transform_layout(int C, int N, size_t* off_mean, size_t* off_var, size_t* off_inv, size_t* off_ms) {
    if (C < 8 || C % 8 != 0 || C > 2048 || N < 1) return 0;
    return adain_transform_layout(C, N, off_mean, off_var, off_inv, off_ms);
}
int wctb200_adain_transform_from_stats(const void* record, int Nc, int C, const void* state, int Ns, float eps, void* transform,
                                       void* stream) {
    WCTB_REQUIRE(record && state && transform, "adain_transform_from_stats: null pointer");
    WCTB_REQUIRE(C >= 8 && C % 8 == 0 && C <= 2048 && Nc >= 1, "adain_transform_from_stats: bad arguments");
    return launch_adain_transform_from_stats(record, Nc, C, state, Ns, eps, transform, ST(stream));
}
int wctb200_adain_transform_apply(const void* act, int N, int H, int W, int C, const void* transform, float alpha, void* out,
                                  void* stream) {
    WCTB_REQUIRE(act && transform && out, "adain_transform_apply: null pointer");
    WCTB_REQUIRE(geom_ok(N, H, W, C) && C <= 2048, "adain_transform_apply: bad geometry");
    return launch_adain_transform_apply(HCP(act), N, H, W, C, transform, alpha, HP(out), ST(stream));
}
// ---- soft spatial control (DESIGN.md §3.3.11) ----
int wctb200_mask_feather(const uint8_t* labels, int N, int Hm, int Wm, int R, float sigma, float* out, void* stream) {
    WCTB_REQUIRE(labels && out, "mask_feather: null pointer");
    WCTB_REQUIRE(N >= 1 && Hm >= 1 && Wm >= 1 && (long long)N * R * Hm * Wm < (1ll << 40), "mask_feather: bad geometry");
    return launch_mask_feather(labels, N, Hm, Wm, R, sigma, out, ST(stream));
}
int wctb200_weights_resize_area(const float* src, int N, int K, int Hm, int Wm, int Hf, int Wf, float* dst, void* stream) {
    WCTB_REQUIRE(src && dst, "weights_resize_area: null pointer");
    WCTB_REQUIRE(N >= 1 && K >= 1 && Hm >= 1 && Wm >= 1 && Hf >= 1 && Wf >= 1 && Hm <= 65536 && Wm <= 65536 && Hf <= 65536 && Wf <= 65536,
                 "weights_resize_area: bad geometry N=%d K=%d %dx%d -> %dx%d", N, K, Hm, Wm, Hf, Wf);
    return launch_weights_resize_area(src, N, K, Hm, Wm, Hf, Wf, dst, ST(stream));
}
int wctb200_wct_stats_weighted(const void* act, int N, int H, int W, int C, const float* weights, int K, void* record, void* stream) {
    WCTB_REQUIRE(act && weights && record, "wct_stats_weighted: null pointer");
    WCTB_REQUIRE(geom_ok(N, H, W, C) && wct_channels_ok(C), "wct_stats_weighted: bad geometry");
    WCTB_REQUIRE(K >= 1 && K <= 8, "wct_stats_weighted: K=%d not in 1..8", K);
    return launch_wct_stats_weighted(HCP(act), N, H, W, C, weights, K, record, ST(stream));
}
int wctb200_wct_transform_apply_weighted(const void* act, int N, int H, int W, int C, const void* transform, int K, const float* weights,
                                         const float* strength, void* out, void* stream) {
    WCTB_REQUIRE(act && transform && out, "wct_transform_apply_weighted: null pointer");
    WCTB_REQUIRE(geom_ok(N, H, W, C) && wct_channels_ok(C), "wct_transform_apply_weighted: bad geometry");
    return launch_wct_transform_apply_weighted(HCP(act), N, H, W, C, transform, K, weights, strength, HP(out), ST(stream));
}
int wctb200_adain_transform_apply_strength(const void* act, int N, int H, int W, int C, const void* transform, float alpha,
                                           const float* strength, void* out, void* stream) {
    WCTB_REQUIRE(act && transform && strength && out, "adain_transform_apply_strength: null pointer");
    WCTB_REQUIRE(geom_ok(N, H, W, C) && C <= 2048, "adain_transform_apply_strength: bad geometry");
    return launch_adain_transform_apply_strength(HCP(act), N, H, W, C, transform, alpha, strength, HP(out), ST(stream));
}
// tuning hooks (wctb200_debug.h; not part of the stable ABI)
int wctb200_debug_set_conv_bn(int bn) {
    g_conv_bn_override = bn;
    return 0;
}
int wctb200_debug_set_conv_oversub(int k) {
    g_conv_oversub = k < 1 ? 1 : (k > 16 ? 16 : k);
    return g_conv_oversub;
}
int wctb200_debug_set_conv_fuse(int mode) {
    g_conv_fuse = mode < 0 ? -1 : (mode ? 1 : 0);
    return g_conv_fuse;
}
int wctb200_debug_set_jacobi_tolq(float tolq) { return set_jacobi_tolq(tolq); }
int wctb200_debug_set_cov_stages(int n) {
    if (n >= 1 && n <= 12) g_cov_max_stages = n;
    return g_cov_max_stages;
}
int wctb200_debug_matfun(const float* A, int C, int count, int n_first, float thresh, float eps_eig, float* out, int* ok,
                         float* info, void* stream) {
    WCTB_REQUIRE(A && out && ok && count >= 1 && n_first >= 0 && n_first <= count, "debug_matfun: bad arguments");
    const int rc = launch_matfun_ns(A, C, count, n_first, thresh, eps_eig, out, ok, nullptr, ST(stream), info);
    return rc < 0 ? rc : 0;
}
int wctb200_debug_set_matfun(int mode, int max_it) {
    if (mode == 0 || mode == 1) g_matfun = mode;
    if (max_it >= 1 && max_it <= 64) g_matfun_max_it = max_it;
    return g_matfun;
}
int wctb200_debug_style_swap_layout(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int patch, int stride, long long* out) {
    WCTB_REQUIRE(out, "debug_style_swap_layout: null pointer");
    WCTB_REQUIRE(swap_style_ok(C, Hs, Ws, patch, stride) && geom_ok(Nc, Hc, Wc, C) && Hc >= patch && Wc >= patch,
                 "debug_style_swap_layout: bad geometry");
    style_swap_debug_layout(C, Nc, Hc, Wc, Hs, Ws, patch, stride, out);
    return 0;
}
int wctb200_debug_set_conv_head_tc(int on) {
    if (on == 0 || on == 1) g_conv_head_tc = on;
    return g_conv_head_tc;
}
int wctb200_debug_set_conv_tail_tc(int on) {
    if (on == 0 || on == 1) g_conv_tail_tc = on;
    return g_conv_tail_tc;
}
int wctb200_debug_set_conv_products(int n) {
    if (n >= 1 && n <= 3) g_conv_products = n;
    return g_conv_products;
}

int wctb200_debug_set_jacobi(int lg_groups, int stagger_cycles) {
    if (lg_groups <= 4) g_jacobi_lg = lg_groups < 0 ? -1 : lg_groups;              // negative: back to the per-size default
    g_jacobi_stagger = stagger_cycles < 0 ? -1 : stagger_cycles;
    return g_jacobi_lg;
}

}  // extern "C"
