/*
 * libwctb200 -- C-ABI of the H100-native (sm_90a) WCT inference hot path.
 *
 * The reference (eridgd/WCT-TF) has no native boundary: its operator surface is
 * Python (`WCT.predict` wct.py:70, `WCTModel` model.py:33, `wct_np/wct_tf/adain`
 * ops.py:24,92,282) executed inside one TF `sess.run` (wct.py:97).  This header
 * is the boundary a maintainer binds with ctypes (see INTEGRATION.md); every
 * entry point names the reference code it replaces.
 *
 * Conventions (all functions):
 *   - return 0 on success, <0 on error (WCTB200_E*); `wctb200_last_error()` gives a
 *     thread-local message; nothing throws;
 *   - plain pointers and sizes only; every buffer is a CUDA DEVICE pointer owned by
 *     the caller (e.g. `torch.Tensor.data_ptr()`), kept alive until `stream` is synced;
 *   - asynchronous on `stream` (a `cudaStream_t` passed as void*; 0 = default stream);
 *     the caller selects the device (`cudaSetDevice`) before the call;
 *   - no CPU fallback: without an sm_90 device the kernels fail with WCTB200_ECUDA.
 *
 * Activation format "SPF16" (split-pair fp16, reflect-padded NHWC):
 *   one allocation of `wctb200_act_bytes(N,H,W,C)` bytes holding two fp16 planes
 *   [plane 0 = hi | plane 1 = lo], each [N][H+2][W+2][C]; the fp32 value of an
 *   element is hi+lo: 22-23 significant bits for |x| >= 0.125, an absolute error <= 3e-8 below that (lo is an fp16
 *   subnormal there), |x| saturates at 65000 (fp16 range).  The 1-pixel halo already holds the
 *   REFLECT padding of ops.py:12-15 (mirror without edge repeat), written by the
 *   producer, so a 3x3 'valid' conv over the padded plane equals Conv2DReflect
 *   (ops.py:17-19).  C must be a multiple of 8; H,W >= 2.
 *   Halo modes.  Each axis of the halo has one of three modes, named by the interior row (column) that feeds padded row 0
 *   and the one that feeds row H+1: REFLECT (the default) 1 and H-2; EDGE (WCTB200_HALO_EDGE, the input of
 *   wctb200_conv3x3_up2) 0 and H-1; WRAP (WCTB200_HALO_WRAP_X / _Y, seamless stylisation) H-1 and 0, so that a conv over
 *   the padded plane pads that axis circularly.  Corner cells follow from the two axes.  The producers that take flags
 *   (conv3x3, conv3x3_up2, conv_head_flags) write the mode they are given; every other producer writes REFLECT, and
 *   wctb200_act_halo rewrites the halo of any activation in any mode.
 */
#ifndef WCTB200_H
#define WCTB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define WCTB200_API __attribute__((visibility("default")))
#else
#define WCTB200_API
#endif

#define WCTB200_ABI_VERSION 1

#define WCTB200_OK       0
#define WCTB200_EINVAL  -1   /* bad argument / unsupported shape */
#define WCTB200_ECUDA   -2   /* CUDA runtime / driver error (incl. no sm_90 device) */
#define WCTB200_EWS     -3   /* workspace too small */
#define WCTB200_EDEVICE -4   /* a kernel flagged an internal error (pipeline timeout) */

/* conv / transform flags */
#define WCTB200_RELU     1   /* ReLU epilogue                     (vgg_normalised.py:40, model.py:291) */
#define WCTB200_CLIP01   2   /* clip to [0,1] (tail conv only)    (model.py:17,86) */
#define WCTB200_HALO_EDGE 4  /* conv3x3: write an EDGE-replicated halo instead of the reflect halo -- for an output
                                that is consumed by wctb200_conv3x3_up2 only (UpSampling2D follows, model.py:293) */

#define WCTB200_POOL2    8   /* conv3x3: MaxPooling2D 2x2/2 'same' (vgg_normalised.py:41-42) folded into the epilogue: the
                                output is [N, ceil(H/2), ceil(W/2), Cout] (>= 2x2) and the full-resolution tensor is never
                                written -- for conv1_2 / 2_2 / 3_4 / 4_4, whose only consumer is the pool */
#define WCTB200_HALO_WRAP_X 16  /* conv3x3, conv3x3_up2, conv_head_flags, act_halo: write a WRAPPED halo along x (padded column
                                   0 holds interior column W-1, column W+1 holds column 0), so the next conv pads x circularly
                                   (seamless stylisation).  With WCTB200_HALO_EDGE the other axis keeps the edge halo. */
#define WCTB200_HALO_WRAP_Y 32  /* the same along y (padded row 0 holds interior row H-1, row H+1 holds row 0) */

WCTB200_API int         wctb200_abi_version(void);
WCTB200_API const char* wctb200_last_error(void);
/* Synchronises `stream` and returns WCTB200_EDEVICE if any kernel since the last
 * call recorded an internal error (mbarrier timeout in a TMA / wgmma pipeline). */
WCTB200_API int         wctb200_check_device(void* stream);

/* ---- SPF16 activations ---------------------------------------------------- */
WCTB200_API size_t wctb200_act_bytes(int N, int H, int W, int C);
/* fp32 NHWC -> SPF16 (interior + reflect halo).  Test / interop helper. */
WCTB200_API int wctb200_act_from_f32(const float* nhwc, int N, int H, int W, int C, void* act, void* stream);
/* SPF16 -> fp32 NHWC (interior only). */
WCTB200_API int wctb200_act_to_f32(const void* act, int N, int H, int W, int C, float* nhwc, void* stream);
/* Rewrites, in place, every halo cell of an SPF16 activation [N,H,W,C] from its interior in the mode of `flags`: 0 =
 * REFLECT, WCTB200_HALO_EDGE, and the wrap bits WCTB200_HALO_WRAP_X / _Y (see "Halo modes" above).  The interior is not
 * touched.  Other flag bits are WCTB200_EINVAL.  Seamless stylisation runs it after every transform, whose outputs carry
 * the reflect halo. */
WCTB200_API int wctb200_act_halo(void* act, int N, int H, int W, int C, int flags, void* stream);

/* ---- image pre/post: WCT.preprocess / WCT.postprocess (wct.py:60-68) -------- */
/* out[i] = img[i] / 255 */
WCTB200_API int wctb200_image_u8_to_f32(const uint8_t* img, size_t count, float* out, void* stream);
/* out[i] = (uint8) (clip(img[i],0,1) * 255)   -- truncation, like np.uint8 */
WCTB200_API int wctb200_image_f32_to_u8(const float* img, size_t count, uint8_t* out, void* stream);

/* ---- CLI image steps on the device (scope row 8f-3) ------------------------- */
/* utils.resize_to / center_crop / center_crop_to (utils.py:29-67) -> scipy.misc.imresize(interp='bilinear'), i.e. Pillow's
 * 8-bit ImagingResample: bit-exact restatement (separable triangle filter with support max(1, in/out), 22-bit fixed-point
 * coefficients, horizontal pass first, uint8 rounding between the passes).  src [N][Hs][Ws][C] uint8 is resampled to
 * Hd x Wd and the window rows [y0, y0+Hout) x columns [x0, x0+Wout) of the result is written to dst [N][Hout][Wout][C]
 * (the centre crop of utils.py:29-53 folded in; y0 = x0 = 0, Hout = Hd, Wout = Wd for a plain resize; Hd = Hs, Wd = Ws
 * for a plain crop).  ws: wctb200_resize_workspace_bytes(N, Hs, Ws, C, Hd, Wd, Wout) bytes of device scratch. */
WCTB200_API size_t wctb200_resize_workspace_bytes(int N, int Hs, int Ws, int C, int Hd, int Wd, int Wout);
WCTB200_API int wctb200_resize_bilinear_u8(const uint8_t* src, int N, int Hs, int Ws, int C, int Hd, int Wd, int y0, int x0,
                                           int Hout, int Wout, uint8_t* dst, void* ws, size_t ws_bytes, void* stream);
/* --keep-colors, the pixel-sized parts of coral.coral_numpy (coral.py:13-39; utils.preserve_colors_np utils.py:87-90).
 * rgb_moments: sums[0..2] = sum x_c, sums[3..8] = sum x0x0, x0x1, x0x2, x1x1, x1x2, x2x2 over the npix RGB pixels, exact
 * uint64 on the DEVICE (9 words).  coral_apply: dst = uint8(clip((A ((x/255 - src_mean)/src_std)) * tgt_std + tgt_mean, 0, 1)
 * * 255) in double precision; A (3x3 row-major), the means and the stds are HOST arrays (the 3x3 algebra that produces them
 * from the moments -- numpy's SVD inside the reference's matSqrt, coral.py:8-11 -- is host work). */
WCTB200_API int wctb200_rgb_moments_u8(const uint8_t* img, long long npix, unsigned long long* sums, void* stream);
WCTB200_API int wctb200_coral_apply_u8(const uint8_t* src, long long npix, const double* A, const double* src_mean,
                                       const double* src_std, const double* tgt_mean, const double* tgt_std, uint8_t* dst,
                                       void* stream);
/* rgb_moments of each of N frames img [N][npix_per_frame][3]: sums [N][9] on the DEVICE, frame n's words as rgb_moments_u8
 * gives them for that frame alone (rgb_moments_u8 is the N = 1 case).  N >= 1, npix_per_frame >= 1, N * npix_per_frame
 * < 2^40, else WCTB200_EINVAL. */
WCTB200_API int wctb200_rgb_moments_batch_u8(const uint8_t* img, int N, long long npix_per_frame, unsigned long long* sums,
                                             void* stream);
/* Luminance-only transfer (DESIGN.md §3.3.15).  Y = (299 R + 587 G + 114 B) / 1000 per pixel, in fp32 (one correctly
 * rounded division of the exact integer).  kb: DEVICE float32 [N][2], 8-byte aligned, one (k, b) per frame.
 * match: dst[n] = clip(rint(k_n Y + b_n), 0, 255) replicated to R = G = B; k = 1, b = 0 makes the grey of an image.
 * merge: dst[n]_c = clip(rint(content_c + ((k_n Y(stylised) + b_n) - Y(content))), 0, 255) for c in R, G, B.
 * Every operation is a rounded fp32 fma / add / division in that order (rint: half to even), so frame n's bytes do not
 * depend on N.  Images are uint8 [N][npix_per_frame][3]; geometry as for rgb_moments_batch_u8. */
WCTB200_API int wctb200_luminance_match_u8(const uint8_t* src, int N, long long npix_per_frame, const float* kb, uint8_t* dst,
                                           void* stream);
WCTB200_API int wctb200_luminance_merge_u8(const uint8_t* content, const uint8_t* stylised, int N, long long npix_per_frame,
                                           const float* kb, uint8_t* dst, void* stream);
/* Coarse-to-fine join (DESIGN.md §3.3.16): content [N][H][W][3], coarse_content and coarse_stylised [N][h][w][3], all uint8
 * on the device; dst [N][H][W][3] = clip(rint(content + U(coarse_stylised - coarse_content)), 0, 255), the content with its
 * low band replaced by the stylised one.  U is bilinear upsampling (or downsampling, for h > H) with half-pixel centres: per
 * axis sy = h / H (one fp32 division), ys = (y + 0.5) sy - 0.5 clamped to [0, h - 1], taps y0 = floor(ys), y1 =
 * min(y0 + 1, h - 1), weight wy = ys - y0; the same for x.  The four differences are exact; a = d00 + wx (d01 - d00), b
 * likewise for row y1, v = a + wy (b - a), each a rounded fp32 operation with no contraction, rint half to even.  Frame n's
 * bytes do not depend on N.  1 <= H, W, h, w <= 2^15, N H W < 2^40, else WCTB200_EINVAL. */
WCTB200_API int wctb200_coarse_join_u8(const uint8_t* content, const uint8_t* coarse_content, const uint8_t* coarse_stylised,
                                       int N, int H, int W, int h, int w, uint8_t* dst, void* stream);
/* Texture synthesis input (--noise, webcam.py:191-192 np.random.randint(0, 256, shape, np.uint8)): N frames of uniform random
 * bytes, out device uint8 [N][H][W][C].  Frame n has the absolute index f = first_index + n; byte j of its H*W*C bytes
 * (row-major HWC) is byte j % 16 of Philox4x32-10 (Random123) with counter (b_lo, b_hi, f_lo, f_hi), b = j / 16 (64-bit), and
 * key (seed_lo, seed_hi), where the 16 bytes are x0..x3, each little-endian; a frame's last block is truncated at its end.
 * A frame therefore depends only on (seed, f, H, W, C): not on N or on how a run is cut into calls.
 * N, H, W >= 1, C in 1..4, first_index >= 0 and first_index + N representable, else WCTB200_EINVAL. */
WCTB200_API int wctb200_noise_u8(uint8_t* out, int N, int H, int W, int C, unsigned long long seed, long long first_index,
                                 void* stream);

/* ---- temporal stabilisation of video (DESIGN.md §3.3.6; flow.cu) ------------
 * Luminance Y = (0.299 R + 0.587 G + 0.114 B) / 255 of npix RGB uint8 pixels, float32 out [npix]. */
WCTB200_API int wctb200_luminance_u8(const uint8_t* rgb, long long npix, float* Y, void* stream);
/* Optical flow (coarse-to-fine Horn-Schunck with warping) of the M - 1 consecutive pairs of Y float32 [M][H][W], M >= 2:
 * flows float32 [2 (M - 1)][2][H][W] (u, v planes); problem 2t is the backward flow from frame t+1 to frame t, problem
 * 2t+1 the forward flow from frame t to frame t+1.  Returns 0 from the query on bad geometry. */
WCTB200_API size_t wctb200_flow_pairs_workspace_bytes(int M, int H, int W);
WCTB200_API int wctb200_flow_pairs(const float* Y, int M, int H, int W, float* flows, void* ws, size_t ws_bytes, void* stream);
/* Confidence of frame t+1 against frame t for t < M - 1: mask uint8 [M - 1][H][W] (0/1), counts int32 [M - 1] = the
 * confident pixels before the cut rule (a pair with fewer than half its pixels confident gets mask 0 everywhere). */
WCTB200_API int wctb200_flow_confidence(const float* Y, int M, int H, int W, const float* flows, uint8_t* mask, int32_t* counts,
                                        void* stream);
/* The recurrent blend, in place on frames uint8 [N][H][W][3]: O = round(P + beta c (O_prev(x + w_b) - P)), 0 <= beta < 1.
 * With prev (uint8 [H][W][3], the stabilised frame before frame 0), frame i uses pair i (flows 2i, mask i); with prev NULL
 * frame 0 is left as it is and frame i >= 1 uses pair i - 1.  One launch per frame, in order. */
WCTB200_API int wctb200_temporal_blend_u8(uint8_t* frames, int N, int H, int W, const uint8_t* prev, const float* flows,
                                          const uint8_t* masks, float beta, void* stream);

/* ---- encoder / decoder layers ---------------------------------------------- */
/* Weight preparation (one-time, device side):
 * w_hwio fp32 [3][3][Cin][Cout] (Keras kernel layout, vgg_normalised.py:33 /
 * model.py:291) -> split-fp16 GEMM operand [2 planes][Cout][9*Cin], k = tap*Cin + cin, stored scaled by a per-layer
 * power of two (max|w| -> [512,1024); the factor sits in a trailer of the buffer and is undone in the conv epilogue)
 * so that the lo plane of small weights does not fall into the fp16 subnormals.
 * `taps` is 9 (3x3) or 1 (a [Cin][Cout] matrix). */
WCTB200_API size_t wctb200_conv_weight_bytes(int taps, int Cin, int Cout);
WCTB200_API int wctb200_prep_conv_weights(const float* w_hwio, int taps, int Cin, int Cout, void* w_split, void* stream);
/* Weights of `UpSampling2D() -> Conv2DReflect` (model.py:291-293) as ONE conv over the low-resolution input: four
 * 2x2-tap kernels (one per output parity) whose taps are sums of the 3x3 taps that land on the same low-resolution
 * pixel; [4 parities][2 planes][Cout][4*Cin].  Buffer size: wctb200_conv_weight_bytes(16, Cin, Cout). */
WCTB200_API int wctb200_prep_conv_weights_up2(const float* w_hwio, int Cin, int Cout, void* w_up2, void* stream);

/* Conv2DReflect 3x3 (+bias, optional ReLU) on tensor cores (wgmma, split-fp16 x3):
 * replaces `Lambda(pad_reflect) -> Conv2D(valid)` of vgg_normalised.py:28-40 and
 * model.py:291.  Cin, Cout multiples of 64.  in/out: SPF16 [N,H,W,Cin] -> [N,H,W,Cout]
 * ([N,ceil(H/2),ceil(W/2),Cout] with WCTB200_POOL2).  flags: WCTB200_RELU, WCTB200_HALO_EDGE, WCTB200_POOL2 and the wrap
 * bits WCTB200_HALO_WRAP_X / _Y, which set the halo mode of the output (the conv reads its input's halo as it is). */
WCTB200_API int wctb200_conv3x3(const void* act_in, int N, int H, int W, int Cin,
                    const void* w_split, const float* bias, int Cout, int flags,
                    void* act_out, void* stream);
/* UpSampling2D (nearest x2, model.py:293) followed by Conv2DReflect 3x3 (+bias, optional ReLU), fused: act_in is the
 * LOW-resolution SPF16 [N,H,W,Cin] whose halo is EDGE-replicated (its producer ran with WCTB200_HALO_EDGE), act_out is
 * SPF16 [N,2H,2W,Cout] with the usual reflect halo.  4/9 of the MACs of the unfused pair and no upsampled tensor.
 * flags: WCTB200_RELU and the wrap bits.  Circular padding of the upsampled map lands on the wrapped low-resolution halo
 * (u[-1] = u[2W-1] = L[W-1]), so a wrapped axis needs act_in's halo wrapped on that axis (its producer ran with
 * WCTB200_HALO_EDGE and the wrap bit) and wraps act_out's halo there. */
WCTB200_API int wctb200_conv3x3_up2(const void* act_in, int N, int H, int W, int Cin,
                        const void* w_up2, const float* bias, int Cout, int flags,
                        void* act_out, void* stream);
/* Same contract on CUDA cores in plain fp32 (validation kernel, fp32 weights [3][3][Cin][Cout]). */
WCTB200_API int wctb200_conv3x3_ref(const void* act_in, int N, int H, int W, int Cin,
                        const float* w_hwio, const float* bias, int Cout, int flags,
                        void* act_out, void* stream);
/* Encoder head: the 1x1 'preprocess' conv (vgg_normalised.py:25-26) folded into
 * conv1_1 3->64 + ReLU.  img fp32 NHWC [N,H,W,3] in [0,1]; w fp32 [27][64] (k = tap*3+cin),
 * b fp32 [64]; out SPF16 [N,H,W,64]. */
WCTB200_API int wctb200_conv_head(const float* img, int N, int H, int W, const float* w, const float* b,
                      void* act_out, void* stream);
/* wctb200_conv_head with halo flags: the wrap bits WCTB200_HALO_WRAP_X / _Y pad the image circularly along those axes
 * (the head reads it with wrapped indices) and write a wrapped halo along them; the other axes reflect.  flags = 0 is
 * wctb200_conv_head.  Other bits are WCTB200_EINVAL. */
WCTB200_API int wctb200_conv_head_flags(const float* img, int N, int H, int W, const float* w, const float* b, int flags,
                                        void* act_out, void* stream);
/* Decoder tail: Conv2DReflect Cin->3, no activation (model.py:297-298), optional
 * clip to [0,1] (model.py:86).  w fp32 [9*Cin][3], b fp32 [3]; out fp32 NHWC [N,H,W,3]. */
WCTB200_API int wctb200_conv_tail(const void* act_in, int N, int H, int W, int Cin, const float* w, const float* b,
                      int flags, float* img_out, void* stream);
/* MaxPooling2D(2x2, stride 2, padding='same') (vgg_normalised.py:41-42): out [N,ceil(H/2),ceil(W/2),C]. */
WCTB200_API int wctb200_maxpool2(const void* act_in, int N, int H, int W, int C, void* act_out, void* stream);
/* UpSampling2D nearest x2 (model.py:293): out [N,2H,2W,C]. */
WCTB200_API int wctb200_upsample2(const void* act_in, int N, int H, int W, int C, void* act_out, void* stream);

/* ---- feature transforms ------------------------------------------------------ */
/* Whiten-colour transform of one relu level for a batch: replaces wct_tf (ops.py:24-90,
 * what the graph runs) and wct_np (ops.py:92-140, the named oracle) -- semantics flags:
 *   eps_cov            added to the covariance diagonal           (wct_tf 1e-8 | wct_np 0)
 *   eps_eig            added to the kept eigenvalues              (wct_tf 0    | wct_np 1e-5)
 *   thresh             keep eigenvalues > thresh                  (1e-5, ops.py:68,112)
 *   readd_content_mean blend with fc+mc (ops.py:83) or fc (ops.py:133)
 * content SPF16 [Nc,Hc,Wc,C]; style SPF16 [Ns,Hs,Ws,C] with Ns == Nc (frame i uses
 * style i) or Ns == 1 (shared).  out SPF16 [Nc,Hc,Wc,C].  k_out (device int32
 * [2*(Nc+Ns)], may be NULL): k_c per content then k_s per style, then sweep counts.
 * C in {64,128,256,512}.  ws: device scratch of wctb200_wct_workspace_bytes(). */
WCTB200_API size_t wctb200_wct_workspace_bytes(int C, int Nc, int Ns);
WCTB200_API int wctb200_wct_level(const void* content, int Nc, int Hc, int Wc,
                      const void* style, int Ns, int Hs, int Ws, int C,
                      float alpha, float eps_cov, float eps_eig, float thresh, int readd_content_mean,
                      void* out, int32_t* k_out, void* ws, size_t ws_bytes, void* stream);
/* Split form of wctb200_wct_level (same arithmetic, same semantics flags): the style side --
 * means, covariance, eigendecomposition and colouring matrix C_s = E_s D_s^1/2 E_s^T of
 * ops.py:48-55,76 -- depends only on the style features, so a host can run it on a second
 * stream (it overlaps the content convolutions) or cache it for a batch that shares one style.
 * `state`: device buffer of wctb200_wct_style_state_bytes(C, Ns) bytes.  Workspace sizes:
 * wctb200_wct_workspace_bytes(C, Nc, Ns) is enough for either call. */
WCTB200_API size_t wctb200_wct_style_state_bytes(int C, int Ns);
WCTB200_API int wctb200_wct_style_prepare(const void* style, int Ns, int Hs, int Ws, int C,
                              float eps_cov, float eps_eig, float thresh,
                              void* state, void* ws, size_t ws_bytes, void* stream);
WCTB200_API int wctb200_wct_apply(const void* content, int Nc, int Hc, int Wc, int C, const void* state, int Ns,
                      float alpha, float eps_cov, float eps_eig, float thresh, int readd_content_mean,
                      void* out, int32_t* k_out, void* ws, size_t ws_bytes, void* stream);
/* Layout of a wctb200_wct_style_prepare state, so that a host can pack, unpack, save and load states without repeating
 * the alignment rule: fp32 mean_s [Ns][C] at *off_mean (0), fp32 C_s [Ns][C][C] at *off_cs, int32 [k_s x Ns | sweeps_s x Ns]
 * at *off_k.  Returns the total (= wctb200_wct_style_state_bytes), 0 for C < 8 or Ns < 1.  Any pointer may be NULL. */
WCTB200_API size_t wctb200_wct_style_state_layout(int C, int Ns, size_t* off_mean, size_t* off_cs, size_t* off_k);
/* Spatial control (WCT paper, section 4): a label map splits each content frame into regions and region r takes style r.
 * Per (frame, region r < R) with at least 2 pixels the transform is wctb200_wct_apply's (same semantics flags) restricted
 * to the region's pixels: mean, covariance and whitening over those pixels only, colouring with style r.  Every other
 * pixel -- labels >= R, and regions with fewer than 2 pixels -- keeps its content feature bit for bit (interior and halo).
 * labels: device uint8 [Nc][Hc][Wc], at the level's feature resolution (wctb200_labels_resize_nearest).
 * states: HOST array of R device pointers, each a state of wctb200_wct_style_prepare with Ns = 1 (styles may have any size).
 * R in 1..8, else WCTB200_EINVAL.  ws: device scratch of wctb200_wct_regions_workspace_bytes(C, Nc, R, Hc, Wc).
 * k_out (device int32 [2*(Nc*R + R)], may be NULL): [k_c x Nc*R | k_s x R | sweeps_c x Nc*R | sweeps_s x R], entry
 * n*R + r for frame n / region r; k_c = -1 (and 0 sweeps) for a skipped (frame, region).
 * A state with k_s = -1 (an empty style region of wctb200_wct_style_prepare_regions) makes region r keep its content
 * feature in every frame, as a region of fewer than 2 pixels does; k_out reports k_c = -1 for it.
 * With R = 1 and every label 0 the output is byte-identical to wctb200_wct_apply's. */
WCTB200_API size_t wctb200_wct_regions_workspace_bytes(int C, int Nc, int R, int Hc, int Wc);
WCTB200_API int wctb200_wct_apply_regions(const void* content, int Nc, int Hc, int Wc, int C, const uint8_t* labels, int R,
                              const void* const* states, float alpha, float eps_cov, float eps_eig, float thresh,
                              int readd_content_mean, void* out, int32_t* k_out, void* ws, size_t ws_bytes, void* stream);
/* Style masks for spatial control: the style side of R regions from ONE style and its label map.  Writes one state of
 * wctb200_wct_style_state_bytes(C, R) bytes (layout wctb200_wct_style_state_layout(C, R)) whose entry r is
 * wctb200_wct_style_prepare's (same semantics flags) over the style pixels labelled r only.  When every pixel is labelled r,
 * entry r is byte-identical to wctb200_wct_style_prepare of the style.  An entry whose region has fewer than 2 pixels is
 * the sentinel k_s = -1 with 0 sweeps, mean 0 and C_s 0: wctb200_wct_apply_regions keeps that region's content.
 * style SPF16 [1,Hs,Ws,C]; labels device uint8 [Hs][Ws] at the level's style feature resolution
 * (wctb200_labels_resize_nearest; labels >= R belong to no entry).  C in {64,128,256,512}, R in 1..8, else
 * WCTB200_EINVAL (also for a null pointer).  ws: device scratch of wctb200_wct_style_prepare_regions_workspace_bytes(C, R, Hs,
 * Ws).  k_out (device int32 [2*R], may be NULL): [k_s x R | sweeps x R]. */
WCTB200_API size_t wctb200_wct_style_prepare_regions_workspace_bytes(int C, int R, int Hs, int Ws);
WCTB200_API int wctb200_wct_style_prepare_regions(const void* style, int Hs, int Ws, int C, const uint8_t* labels, int R,
                                      float eps_cov, float eps_eig, float thresh, void* state, int32_t* k_out,
                                      void* ws, size_t ws_bytes, void* stream);
/* Style interpolation (WCT paper, section 4): the transform of wctb200_wct_apply (same semantics flags) against a weighted
 * blend of K styles.  The transform is affine in the style statistics, so the blend runs on the states: frame n is coloured
 * with C_w = sum_k w_k C_sk and shifted by m_w = sum_k w_k m_sk (an fp32 fmaf chain in k order), so that
 *   out = sum_k w_k * wct_apply(states[k])   when a row sums to 1.
 * The weights are used as given (no normalisation).  A one-hot row, or K = 1 with weight 1, is byte-identical to
 * wctb200_wct_apply with that state.
 * states: HOST array of K device pointers, each a state of wctb200_wct_style_prepare with Ns = 1 (styles may have any size).
 * weights: DEVICE fp32 [Nw][K], Nw = 1 (one row for every frame) or Nw = Nc (row n for frame n).
 * K in 1..8, Nw in {1, Nc}, else WCTB200_EINVAL (also for a null state).  ws: device scratch of
 * wctb200_wct_blend_workspace_bytes(C, Nc, K, Nw).  k_out (device int32 [2*(Nc+K)], may be NULL):
 * [k_c x Nc | k_s x K | sweeps_c x Nc | sweeps_s x K]. */
WCTB200_API size_t wctb200_wct_blend_workspace_bytes(int C, int Nc, int K, int Nw);
WCTB200_API int wctb200_wct_apply_blend(const void* content, int Nc, int Hc, int Wc, int C,
                            const void* const* states, int K, const float* weights, int Nw,
                            float alpha, float eps_cov, float eps_eig, float thresh, int readd_content_mean,
                            void* out, int32_t* k_out, void* ws, size_t ws_bytes, void* stream);
/* AdaIN against a weighted blend of K styles: the moments of each style, then per (frame, channel)
 * y = (x-mc)*rsqrt(vc+eps)*sum_k w_k sqrt(v_sk) + sum_k w_k m_sk, out = alpha*y + (1-alpha)*x, so that
 *   out = sum_k w_k * adain_level(styles[k])   when a row sums to 1.
 * styles: HOST array of K device pointers, style k SPF16 [1,Hs[k],Ws[k],C]; Hs, Ws: HOST int arrays of K.  weights as for
 * wctb200_wct_apply_blend (DEVICE fp32 [Nw][K], Nw in {1, Nc}, used as given).  K in 1..8, else WCTB200_EINVAL.
 * ws: device scratch of wctb200_adain_blend_workspace_bytes(C, Nc, K).  K = 1 with weight 1 is byte-identical to
 * wctb200_adain_level with Ns = 1. */
WCTB200_API size_t wctb200_adain_blend_workspace_bytes(int C, int Nc, int K);
WCTB200_API int wctb200_adain_blend(const void* content, int Nc, int Hc, int Wc, int C,
                        const void* const* styles, const int* Hs, const int* Ws, int K,
                        const float* weights, int Nw, float alpha, float eps,
                        void* out, void* ws, size_t ws_bytes, void* stream);
/* Label map resampling for spatial control: src device uint8 [N][Hm][Wm] -> dst [N][Hf][Wf] by proportional nearest
 * sampling in integer arithmetic, dst[y][x] = src[((2y+1)*Hm) / (2*Hf)][((2x+1)*Wm) / (2*Wf)] (no divisibility needed). */
WCTB200_API int wctb200_labels_resize_nearest(const uint8_t* src, int N, int Hm, int Wm, int Hf, int Wf, uint8_t* dst,
                                  void* stream);
/* AdaIN (ops.py:282-294): biased per-channel moments of content and style,
 * y = (x-mc)*rsqrt(vc+eps)*sqrt(vs)+ms, out = alpha*y + (1-alpha)*x.  The moments are summed centred on a sampled
 * per-channel shift, in a split of each frame that depends on C, H and W only: a frame's output is bit-identical
 * whatever batch it runs in. */
WCTB200_API int wctb200_adain_level(const void* content, int Nc, int Hc, int Wc,
                        const void* style, int Ns, int Hs, int Ws, int C,
                        float alpha, float eps, void* out, void* ws, size_t ws_bytes, void* stream);
/* Split form of wctb200_adain_level and wctb200_adain_blend: the style side is the biased per-channel moments of the style,
 * which depend on the style features only, so a host can prepare them once and apply them to any number of calls.
 * wctb200_adain_level is prepare followed by apply, and wctb200_adain_blend is K prepares followed by apply_blend, so
 * the split form gives the same bytes.
 *   state: device buffer of wctb200_adain_style_state_bytes(C, Ns) bytes, fp32 mean [Ns][C] at *off_mean (0) and var [Ns][C]
 *   at *off_var (wctb200_adain_style_state_layout; 0 for C not a multiple of 8 or Ns < 1).
 *   prepare: style SPF16 [Ns,Hs,Ws,C]; needs no workspace (it uses the library's per-stream scratch).
 *   apply: content SPF16 [Nc,Hc,Wc,C] against a state of Ns in {1, Nc} styles (frame i takes style i, or the shared one).
 *   apply_blend: states is a HOST array of K device pointers, each a state with Ns = 1; weights as for
 *   wctb200_adain_blend (DEVICE fp32 [Nw][K], Nw in {1, Nc}, used as given).
 * Both applies take a workspace of wctb200_wct_workspace_bytes(C, Nc, 0) bytes and only read the states.  A null state,
 * Ns not in {1, Nc}, K outside 1..8 or Nw not in {1, Nc} is WCTB200_EINVAL. */
WCTB200_API size_t wctb200_adain_style_state_bytes(int C, int Ns);
WCTB200_API size_t wctb200_adain_style_state_layout(int C, int Ns, size_t* off_mean, size_t* off_var);
WCTB200_API int wctb200_adain_style_prepare(const void* style, int Ns, int Hs, int Ws, int C, void* state, void* stream);
WCTB200_API int wctb200_adain_apply(const void* content, int Nc, int Hc, int Wc, int C, const void* state, int Ns,
                        float alpha, float eps, void* out, void* ws, size_t ws_bytes, void* stream);
WCTB200_API int wctb200_adain_apply_blend(const void* content, int Nc, int Hc, int Wc, int C,
                              const void* const* states, int K, const float* weights, int Nw,
                              float alpha, float eps, void* out, void* ws, size_t ws_bytes, void* stream);

/* ---- tiled stylisation (DESIGN.md §3.3.7) -------------------------------------
 * A level's content statistics are sums, so a frame too large for one pass is encoded tile by tile: the statistics of
 * each tile's interior go into a record, the records are folded into one per frame in a fixed tile order, the record
 * becomes the level's transform once, and a second pass applies that transform to every tile.
 *
 * Statistics record of N frames: fp64 n [N] (pixels), t [N][C] (the centring shift), s [N][C] = sum (x - t) and
 * S = sum (x - t)(x - t)^T: [N][C][C] for WCT (diag = 0), its diagonal [N][C] for AdaIN (diag = 1).  Offsets from
 * wctb200_stats_record_layout (returns the total, 0 for C not a multiple of 8 or > 2048, N < 1 or diag not 0/1).
 *
 * stats_rect: the record of the rectangle [y0, y0+h) x [x0, x0+w) of every frame of an SPF16 map [N,H,W,C] (h, w >= 1,
 * inside the map).  The split into CTA slots and the sampled shift are those of an h x w map, so the whole-map rectangle
 * gives the sums of wctb200_wct_apply / wctb200_adain_apply bit for bit.  WCT: C in {64,128,256,512}.
 * stats_accumulate: folds record B into record A (same C, N, diag): B's sums are re-centred on A's shift in fp64 and
 * added; a frame of A with n = 0 takes B's as they are.  Folding in a fixed order gives a deterministic result.
 *
 * Transforms from a record (frames with n >= 2): the content side of wctb200_wct_apply / wctb200_adain_apply from the
 * record against a style state of Ns in {1, Nc} styles, written to a transform buffer instead of applied:
 *   WCT: split-fp16 M [Nc][2][C][C] at *off_m, bias fp32 [Nc][C] at *off_bias, int32 [k_c x Nc | sweeps_c x Nc] at *off_k
 *        (wctb200_wct_transform_layout; 0 for C not in {64,128,256,512} or N < 1); ws of wctb200_wct_workspace_bytes(C, Nc, 0).
 *        Row exponents int32 e [Nc][C] at wctb200_wct_transform_row_exp_offset(C, Nc) (inside the total): row i of M is
 *        stored times 2^e_i and the apply multiplies it back exactly.  The library picks e_i so that max_j |M_ij| 2^e_i is in
 *        [512, 1024), keeping every lo half that matters a normal fp16 number; e = 0 (a zeroed slot) is a row stored as is.
 *   AdaIN: fp32 mean_c, var_c, inv = rsqrt(var_c + eps) sqrt(var_s), ms, each [Nc][C] (wctb200_adain_transform_layout).
 * transform_apply: out = the transform of frame i applied to frame i of any SPF16 map [N,H,W,C] of those frames (a tile
 * with its halo); AdaIN takes alpha here.  A record of whole frames, then its transform, then the apply, gives the bytes
 * of wctb200_wct_apply / wctb200_adain_apply. */
WCTB200_API size_t wctb200_stats_record_layout(int C, int N, int diag, size_t* off_n, size_t* off_t, size_t* off_s, size_t* off_S);
WCTB200_API int wctb200_wct_stats_rect(const void* act, int N, int H, int W, int C, int y0, int x0, int h, int w, void* record,
                                       void* stream);
WCTB200_API int wctb200_adain_stats_rect(const void* act, int N, int H, int W, int C, int y0, int x0, int h, int w, void* record,
                                         void* stream);
WCTB200_API int wctb200_stats_accumulate(void* record_a, const void* record_b, int C, int N, int diag, void* stream);
WCTB200_API size_t wctb200_wct_transform_layout(int C, int N, size_t* off_m, size_t* off_bias, size_t* off_k);
WCTB200_API size_t wctb200_wct_transform_row_exp_offset(int C, int N);
WCTB200_API int wctb200_wct_transform_from_stats(const void* record, int Nc, int C, const void* state, int Ns, float alpha,
                                                 float eps_cov, float eps_eig, float thresh, int readd_content_mean,
                                                 void* transform, void* ws, size_t ws_bytes, void* stream);
WCTB200_API int wctb200_wct_transform_apply(const void* act, int N, int H, int W, int C, const void* transform, void* out,
                                            void* stream);
WCTB200_API size_t wctb200_adain_transform_layout(int C, int N, size_t* off_mean, size_t* off_var, size_t* off_inv,
                                                  size_t* off_ms);
WCTB200_API int wctb200_adain_transform_from_stats(const void* record, int Nc, int C, const void* state, int Ns, float eps,
                                                   void* transform, void* stream);
WCTB200_API int wctb200_adain_transform_apply(const void* act, int N, int H, int W, int C, const void* transform, float alpha,
                                              void* out, void* stream);

/* ---- optimal-transport transform (OST, DESIGN.md §3.3.8) ----------------------
 * The closed-form Monge map between the content Gaussian N(m_c, A_c) and the style's, in place of WCT's T = C_s W_c:
 *   M = W_c B^1/2 W_c,  B = S_c C_s C_s S_c,  S_c = E_k diag((lambda + eps_eig)^+1/2) E_k^T,
 *   out = alpha (M (x - m_c) + m_s) + (1 - alpha) base   (base and the semantics flags as for wctb200_wct_apply).
 * W_c, the kept set and C_s are wctb200_wct_apply's, so the style state is a wctb200_wct_style_prepare state unchanged.
 * B^1/2 = V diag(sqrt(max(mu, 0))) V^T has no threshold: the matrix-function fast path where it converges, elsewhere the
 * singular values of P = S_c C_s (B = P P^T) by the one-sided Jacobi solver, a column below its null level counting as 0.
 * ost_apply: content SPF16 [Nc,Hc,Wc,C], state of Ns in {1, Nc} styles, out SPF16 [Nc,Hc,Wc,C].  C in {64,128,256,512} and
 * Ns in {1, Nc}, else WCTB200_EINVAL; ws of wctb200_ost_workspace_bytes(C, Nc) bytes, else WCTB200_EWS.
 * k_out (device int32 [5*Nc], may be NULL): [k_c x Nc | sweeps_c x Nc | ns_c x Nc | ns_b x Nc | sweeps_b x Nc]: the kept
 * count and eigensolver sweeps of the content, then 1 where W_c (ns_c) and B^1/2 (ns_b) took the Newton-Schulz fast path
 * (0: the eigensolver), then the eigensolver sweeps of B (0 on the fast path).
 * ost_transform_from_stats: ost_apply's transform from a statistics record, in the layout of wctb200_wct_transform_layout
 * (its int32 slot: [k_c x Nc | sweeps_c x Nc]), applied by wctb200_wct_transform_apply.  A record of whole frames gives
 * the bytes of wctb200_ost_apply. */
WCTB200_API size_t wctb200_ost_workspace_bytes(int C, int Nc);
WCTB200_API int wctb200_ost_apply(const void* content, int Nc, int Hc, int Wc, int C, const void* state, int Ns, float alpha,
                                  float eps_cov, float eps_eig, float thresh, int readd_content_mean, void* out, int32_t* k_out,
                                  void* ws, size_t ws_bytes, void* stream);
WCTB200_API int wctb200_ost_transform_from_stats(const void* record, int Nc, int C, const void* state, int Ns, float alpha,
                                                 float eps_cov, float eps_eig, float thresh, int readd_content_mean,
                                                 void* transform, void* ws, size_t ws_bytes, void* stream);

/*
 * wct_style_swap (ops.py:145-217) + style_swap (ops.py:219-278) for ONE content/style pair: whiten both encodings, take every
 * patch x patch window of the whitened style at `stride` (--ss-patch-size / --ss-stride, stylize.py:33-34), replace every
 * content window (same stride, VALID) by its best-correlated style patch (filters normalised per tap across patches, first
 * arg-max, overlaps averaged), colour with the style, blend with `alpha` (= --ss-alpha).  The swapped encoding must tile the
 * content encoding exactly -- (ho-1)*stride + patch == Hc -- which is what wct.py:84-90 (utils.swap_filter_fit) ensures by
 * cropping the content image; otherwise WCTB200_EINVAL.  k_out (may be NULL): [k_c, k_s].
 * Used at relu5_1 when --swap5 is given (model.py:148-152).
 */
WCTB200_API size_t wctb200_style_swap_workspace_bytes(int C, int Hc, int Wc, int Hs, int Ws, int patch, int stride);
WCTB200_API int wctb200_style_swap_level(const void* content, int Hc, int Wc, const void* style, int Hs, int Ws, int C,
                             int patch, int stride, float alpha, float eps_cov, float thresh, void* out, int32_t* k_out,
                             void* ws, size_t ws_bytes, void* stream);
/*
 * Split form of wctb200_style_swap_level, batched over content frames.  The style side depends only on the style encoding,
 * the patch and the stride, so it is prepared once into a state, and an apply swaps Nc >= 1 frames against it in one call.
 * wctb200_style_swap_level is prepare followed by apply with Nc = 1.  Frame i of an apply is bit-identical to
 * wctb200_style_swap_level on that frame alone.
 *   state: device buffer of wctb200_style_swap_state_bytes(C, Hs, Ws, patch, stride) bytes (0 for a bad geometry) holding the
 *   style mean and k_s, the whitened style encoding the gather reads, the per-tap norms and the split-fp16 patch filters,
 *   and the colouring operand (C_s split) with its bias.  Its layout is private to the library; it is rebuilt from the style
 *   encoding, not stored.
 *   prepare: style SPF16 [1,Hs,Ws,C]; ws of wctb200_style_swap_prepare_workspace_bytes(C, Hs, Ws, patch, stride) bytes;
 *   k_out (may be NULL): [k_s].
 *   apply: content SPF16 [Nc,Hc,Wc,C]; out SPF16 [Nc,Hc,Wc,C]; ws of
 *   wctb200_style_swap_apply_workspace_bytes(C, Nc, Hc, Wc, Hs, Ws, patch, stride) bytes; k_out (may be NULL):
 *   [k_c x Nc | k_s].  The apply only reads the state.
 * A null state, Nc < 1, C not in {64,128,256,512}, a patch or stride outside 1..16, a map smaller than the patch, or a
 * patch / stride that does not tile the content encoding ((ho-1)*stride + patch == Hc, and the same for Wc) is
 * WCTB200_EINVAL.
 */
WCTB200_API size_t wctb200_style_swap_state_bytes(int C, int Hs, int Ws, int patch, int stride);
WCTB200_API size_t wctb200_style_swap_prepare_workspace_bytes(int C, int Hs, int Ws, int patch, int stride);
WCTB200_API int wctb200_style_swap_prepare(const void* style, int Hs, int Ws, int C, int patch, int stride,
                               float eps_cov, float thresh, void* state, int32_t* k_out,
                               void* ws, size_t ws_bytes, void* stream);
WCTB200_API size_t wctb200_style_swap_apply_workspace_bytes(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int patch, int stride);
WCTB200_API int wctb200_style_swap_apply(const void* content, int Nc, int Hc, int Wc, int C, const void* state,
                             int Hs, int Ws, int patch, int stride, float alpha, float eps_cov, float thresh,
                             void* out, int32_t* k_out, void* ws, size_t ws_bytes, void* stream);
/*
 * The apply also runs in less workspace, down to wctb200_style_swap_apply_min_workspace_bytes(C, Nc, Hc, Wc, Hs, Ws, patch,
 * stride) (0 for a bad geometry): it then correlates the patches in chunks, each the largest multiple of the correlation's N
 * tile that fits, and keeps a running first arg-max across them.  The output and k_out are byte-identical for every workspace
 * size from that minimum up; from wctb200_style_swap_apply_workspace_bytes up the apply runs in one chunk.  Less than the
 * minimum is WCTB200_EWS.  This is what makes the swap affordable at the finer levels (relu3_1 of a 512^2 image has 15 876
 * patches: about 1.1 GB of scores per frame in one chunk).
 */
WCTB200_API size_t wctb200_style_swap_apply_min_workspace_bytes(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int patch, int stride);
/*
 * Labelled style swap (DESIGN.md §3.3.13; neural doodle): wctb200_style_swap_apply in which each content anchor draws only
 * on the style patches that carry its own label.  content_labels: device uint8 [Ncl][Hm][Wm], Ncl in {1, Nc} (1: every
 * frame shares the map); style_labels: device uint8 [Hms][Wms], the labels of the state's style.  Maps of any resolution
 * (1..32768 per side) are sampled onto the content / style feature grids by the rule of wctb200_labels_resize_nearest.  With
 * o = (patch-1)/2, patch n = py*pcol + px carries the style label at (py*stride + o, px*stride + o), and the anchor (y, x)
 * of frame i the content label at (y*stride + o, x*stride + o).  The anchor takes the first maximum of its scores over the
 * patches of its label, or over every patch when no patch carries that label.  Labels are compared for equality only.
 *   label_buf: device scratch of wctb200_style_swap_labels_workspace_bytes(Ncl, Hc, Wc, Hs, Ws, patch, stride) bytes (0 for
 *   a bad geometry) for the sampled maps and the patch labels, separate from ws, which is sized and chunked exactly as for
 *   wctb200_style_swap_apply.  A smaller label_buf is WCTB200_EWS; the other errors are wctb200_style_swap_apply's.
 * Identities: with one label everywhere (or any labelling in which every anchor may take every patch) the output and k_out
 * are byte-identical to wctb200_style_swap_apply's; every workspace size from the minimum up gives the same bytes; frame i
 * of an apply is bit-identical to the apply of that frame alone with its own map.
 */
WCTB200_API size_t wctb200_style_swap_labels_workspace_bytes(int Ncl, int Hc, int Wc, int Hs, int Ws, int patch, int stride);
WCTB200_API int wctb200_style_swap_apply_labels(const void* content, int Nc, int Hc, int Wc, int C, const void* state,
                                    int Hs, int Ws, int patch, int stride, float alpha, float eps_cov, float thresh,
                                    const uint8_t* content_labels, int Ncl, int Hm, int Wm,
                                    const uint8_t* style_labels, int Hms, int Wms,
                                    void* out, int32_t* k_out, void* ws, size_t ws_bytes, void* label_buf, size_t label_bytes,
                                    void* stream);

/*
 * Softmax style swap (DESIGN.md §3.3.17): wctb200_style_swap_apply (or _apply_labels when both label maps are given) with
 * each anchor's arg-max replaced by a softmax over the patches at temperature tau = `temperature`.  With s(a,n) the hard
 * swap's scores, ||c_a|| the l2 norm of the whitened content over the anchor's window, K = patch*patch*C and n_p the number
 * of real patches, z(a,n) = s(a,n) / (||c_a|| sqrt(K / n_p)) (0 where ||c_a|| = 0) and
 * w(a,n) = exp((z(a,n) - M_a) / tau) / sum_{m in A(a)} exp((z(a,m) - M_a) / tau) on the allowed set A(a) (every patch, or
 * wctb200_style_swap_apply_labels's set), M_a the maximum of z over A(a).  Every anchor pastes sum_n w(a,n) times the raw
 * whitened patch n; overlaps are averaged, coloured and blended with `alpha` as in the hard swap.  tau -> 0 gives the hard
 * swap wherever an anchor's maximum is unique; a large tau the mean of A(a).  The state is the hard swap's, unchanged.
 *   ws: wctb200_style_swap_softmax_workspace_bytes(C, Nc, Hc, Wc, Hs, Ws, patch, stride) bytes run the apply in one chunk;
 *   down to wctb200_style_swap_softmax_min_workspace_bytes (one block of patches) it runs in chunks of whole blocks, and
 *   every size gives the same bytes.  The workspace begins with wctb200_style_swap_apply's layout (the offsets of
 *   wctb200_debug_style_swap_layout hold).  Less than the minimum is WCTB200_EWS.
 *   content_labels / style_labels: both NULL (every patch allowed) or both given, with label_buf, as for
 *   wctb200_style_swap_apply_labels.
 * A temperature that is not a finite, normal float > 0 (a subnormal has no finite 1/tau) is WCTB200_EINVAL; the other errors
 * are wctb200_style_swap_apply_labels's.  Frame i of an apply is bit-identical to the apply of that frame alone.
 * wctb200_style_swap_softmax_launches: the number of kernels an apply with ws_bytes of workspace launches (it grows with
 * the chunks and the patch blocks), counted as the library's other calls count theirs; 0 for a bad geometry or too
 * small a workspace.
 */
WCTB200_API size_t wctb200_style_swap_softmax_workspace_bytes(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int patch, int stride);
WCTB200_API size_t wctb200_style_swap_softmax_min_workspace_bytes(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int patch,
                                                                  int stride);
WCTB200_API int wctb200_style_swap_softmax_launches(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int patch, int stride,
                                                    size_t ws_bytes, int labelled);
WCTB200_API int wctb200_style_swap_apply_softmax(const void* content, int Nc, int Hc, int Wc, int C, const void* state,
                                     int Hs, int Ws, int patch, int stride, float alpha, float eps_cov, float thresh,
                                     float temperature, const uint8_t* content_labels, int Ncl, int Hm, int Wm,
                                     const uint8_t* style_labels, int Hms, int Wms,
                                     void* out, int32_t* k_out, void* ws, size_t ws_bytes, void* label_buf, size_t label_bytes,
                                     void* stream);

/*
 * Balanced style swap (DESIGN.md §3.3.18): wctb200_style_swap_apply_softmax with `iters` Sinkhorn iterations that balance
 * how much each style patch is used.  With z(a,n), tau and the allowed sets A(a) of the softmax swap, the column targets are
 * c_n = sum_{a : n in A(a)} 1 / |A(a)| (Na / n_p without labels; with labels cnt(l(n)) / np(l(n)) + F / n_p, from exact
 * counts: cnt the anchors of a label the style carries, np the patches of that label, F the anchors of absent labels).
 * Potentials h_n (fp32, one per frame and patch, in units of z) start at 0; x(a,n) = z(a,n) + h_n, rounded once.
 *   row step:    M_a = max_{n in A(a)} x(a,n),  Z_a = sum_{n in A(a)} exp((x(a,n) - M_a) / tau);
 *   column step: S_n = sum_{a : n in A(a)} exp((x(a,n) - M_a) / tau) / Z_a (a log-sum-exp over anchor blocks of 256 per
 *                frame, combined in block order),  h_n += tau (log c_n - log S_n) for every n with c_n > 0.
 * The apply runs the row step of h = 0, `iters` times a column step then a row step, and folds
 * w(a,n) = exp((x(a,n) - M_a) / tau) / Z_a as the softmax swap folds its weights: rows sum to 1, columns tend to c_n.
 * iters = 0 is the softmax swap, launch for launch and byte for byte.  Each iteration costs one pass over the scores: the
 * correlation again when the apply runs in chunks.
 *   col_sums: NULL, or float [Nc][n_p] that receives S_n of the final plan (one more column pass, no extra correlation).
 *   ws: wctb200_style_swap_balanced_workspace_bytes run in one chunk, down to _balanced_min_workspace_bytes (one block of
 *   patches) in chunks of whole blocks, and every size gives the same bytes.  The workspace begins with
 *   wctb200_style_swap_apply's layout.
 * iters < 0 or > 256 is WCTB200_EINVAL; the other errors are wctb200_style_swap_apply_softmax's.  Frame i of an apply is
 * bit-identical to the apply of that frame alone.
 * wctb200_style_swap_balanced_launches: the kernels an apply with ws_bytes of workspace launches (labelled: label maps
 * given; want_cols: col_sums given); 0 for a bad geometry, a bad iters or too small a workspace.
 */
WCTB200_API size_t wctb200_style_swap_balanced_workspace_bytes(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int patch, int stride);
WCTB200_API size_t wctb200_style_swap_balanced_min_workspace_bytes(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int patch,
                                                                   int stride);
WCTB200_API int wctb200_style_swap_balanced_launches(int C, int Nc, int Hc, int Wc, int Hs, int Ws, int patch, int stride,
                                                     size_t ws_bytes, int labelled, int iters, int want_cols);
WCTB200_API int wctb200_style_swap_apply_balanced(const void* content, int Nc, int Hc, int Wc, int C, const void* state,
                                      int Hs, int Ws, int patch, int stride, float alpha, float eps_cov, float thresh,
                                      float temperature, int iters, const uint8_t* content_labels, int Ncl, int Hm, int Wm,
                                      const uint8_t* style_labels, int Hms, int Wms,
                                      void* out, int32_t* k_out, float* col_sums, void* ws, size_t ws_bytes, void* label_buf,
                                      size_t label_bytes, void* stream);

/* ---- multimodal style transfer (DESIGN.md §3.3.10; mst.cu) ----------------
 * Spherical k-means of one style feature (SPF16 [1,Hs,Ws,C], C in {64,128,256,512}) into K in 1..8 clusters of the unit
 * directions u_p = f_p / max(|f_p|, 1e-12): k-means++ seeding with Philox4x32-10 draws (counter (j, level, 0, 0)), then at
 * most 16 Lloyd iterations (argmax_k u.c_k, ties to the lowest k; c_k = normalised sum of its u_p, fp64 in a fixed order;
 * an empty cluster keeps its centre), stopping after the first iteration that changes no label -- decided on the device.
 * labels_out uint8 [Hs*Ws], centres_out fp32 [K][C], info_out int32 [K init pixel indices | iterations | K pixel counts].
 * The result depends only on the feature, K and level.  ws: wctb200_mst_style_clusters_workspace_bytes bytes (0: bad
 * arguments).  2K + 31 launches. */
WCTB200_API size_t wctb200_mst_style_clusters_workspace_bytes(int Hs, int Ws, int C, int K);
WCTB200_API int wctb200_mst_style_clusters(const void* style, int Hs, int Ws, int C, int K, int level, uint8_t* labels_out,
                                           float* centres_out, int32_t* info_out, void* ws, size_t ws_bytes, void* stream);
/* Data term of the content side: D_out fp32 [N][H][W][K] = 1 - u_p . c_k for the centres fp32 [K][C]; +inf where counts[k]
 * (device int32 [K], the style pixels of cluster k) is below 2.  Reads the content once; one launch. */
WCTB200_API int wctb200_mst_data_term(const void* content, int N, int H, int W, int C, const float* centres, const int32_t* counts,
                                      int K, float* D_out, void* stream);
/* Red-black ICM on D fp32 [N][H][W][K] with a Potts term of weight lambda >= 0 per disagreeing 4-neighbour inside the image:
 * labels_out uint8 [N][H][W] starts at argmin_k D (ties: lowest k); each of `sweeps` sweeps updates the pixels with (y + x)
 * even, then those with (y + x) odd, to argmin_k D[p,k] + lambda n_k(p), keeping the current label when it is among the
 * minima and taking the lowest k otherwise; cost = __fadd_rn(D, __fmul_rn(lambda, n_k)).  1 + 2 sweeps launches. */
WCTB200_API int wctb200_mst_smooth(const float* D, int N, int H, int W, int K, float lambda, int sweeps, uint8_t* labels_out,
                                   void* stream);

/* ---- exact feature distribution matching (EFDM, DESIGN.md §3.3.12; efdm.cu) ------
 * A segment is one (frame, channel) of a feature map.  Each content segment of Nc = H*W values x_p takes the distribution of
 * the same channel of its style (Q_0 <= ... <= Q_{Ms-1}, Ms = Hs*Ws) by rank: with the content sorted,
 *   q(r) = Q linearly interpolated at u(r) = clamp((2r+1) Ms / (2 Nc) - 1/2, 0, Ms-1)   (q(r) = Q_r when Ms = Nc),
 * every run [r0, r1) of equal content values takes t = mean of q over the run (fp64 prefix sums in a fixed order), and
 *   out_p = alpha t + (1 - alpha) x_p,   x_p = hi + lo of the SPF16 input, -0 counted as +0.
 * out is SPF16 [N,H,W,C] with the reflect halo; alpha = 0 copies the content's bytes.  C a multiple of 8; the content is at
 * least 2x2; a style may be 1x1.
 * style_prepare: style SPF16 [Ns,Hs,Ws,C] -> state, the sorted values fp32 [Ns][C][Ms], of
 * wctb200_efdm_style_state_bytes(C, Ns, Hs, Ws) bytes (0: bad geometry).  Workspace: wctb200_efdm_style_workspace_bytes(C, Ns,
 * Hs, Ws, S) bytes sort S segments at a time (14 launches per chunk of S).
 * apply: content SPF16 [N,H,W,C] against a state of Ns in {1, N} styles (frame n takes style n, or style 0), WCTB200_EINVAL
 * otherwise.  ws: wctb200_efdm_workspace_bytes(C, N, H, W, S) bytes process S whole segments at a time (18 launches per chunk;
 * 1 launch for alpha = 0, which reads no workspace); less than one segment's is WCTB200_EWS.  The output is byte-identical
 * for every workspace size, and a frame's bytes do not depend on the other frames of the call. */
WCTB200_API size_t wctb200_efdm_style_state_bytes(int C, int Ns, int Hs, int Ws);
WCTB200_API size_t wctb200_efdm_style_workspace_bytes(int C, int Ns, int Hs, int Ws, int max_segments);
WCTB200_API int wctb200_efdm_style_prepare(const void* style, int Ns, int Hs, int Ws, int C, void* state, void* ws, size_t ws_bytes,
                                           void* stream);
WCTB200_API size_t wctb200_efdm_workspace_bytes(int C, int N, int H, int W, int max_segments);
WCTB200_API int wctb200_efdm_apply(const void* content, int N, int H, int W, int C, const void* state, int Ns, int Hs, int Ws,
                                   float alpha, void* out, void* ws, size_t ws_bytes, void* stream);

/* ---- sliced distribution matching (DESIGN.md §3.3.14; efdm.cu) ----------------------------------------------------
 * EFDM in K random orthonormal bases of each level's channels, chained: y_1 = G_1 x_0, m_k = EFDM(y_k, S_k) at alpha = 1,
 * y_{k+1} = G_{k+1} m_k for k = 1..K+1, out = alpha m_{K+1} + (1 - alpha) x_0 (G_k = R_k R_{k-1}^T folds the back- and
 * forward-rotations; G_{K+1} = R_K^T; S_{K+1} the plain EFDM state).  C a multiple of 64.
 * rotated_style_prepare: the state of one step, the sorted values of R y for the style SPF16 [Ns,Hs,Ws,C] and R fp32 C x C
 * (row-major, y_c = sum_j R[c][j] v_j), in wctb200_efdm_style_state_bytes / _style_workspace_bytes as the plain prepare.
 * sliced_step: m = EFDM(G v, state) at alpha = 1, with v the fp32 planes src [N][C][H*W] or, when src is NULL, the SPF16
 * content [N,H,W,C]; written to the fp32 planes out_planes [N][C][H*W] (wctb200_efdm_planes_bytes, 0: bad geometry) or,
 * when out_planes is NULL, as alpha m + (1 - alpha) content to SPF16 out with the reflect halo (alpha = 0 copies the
 * content's bytes).  out_planes must not alias src.  ws: wctb200_efdm_workspace_bytes(C, N, H, W, S), as for the apply.
 * G v is one fmaf chain per value over the input channels in index order, so a frame's bytes depend on nothing but its own
 * values, its style's and G: the same for every workspace size, batch and chunking. */
WCTB200_API size_t wctb200_efdm_planes_bytes(int C, int N, int H, int W);
WCTB200_API int wctb200_efdm_rotated_style_prepare(const void* style, int Ns, int Hs, int Ws, int C, const float* R, void* state,
                                                   void* ws, size_t ws_bytes, void* stream);
WCTB200_API int wctb200_efdm_sliced_step(const void* content, const float* src, int N, int H, int W, int C, const float* G,
                                         const void* state, int Ns, int Hs, int Ws, float alpha, float* out_planes, void* out,
                                         void* ws, size_t ws_bytes, void* stream);

/* ---- soft spatial control (DESIGN.md §3.3.11) -----------------------------------
 * mask_feather: labels device uint8 [N][Hm][Wm], R in 1..8, sigma in (0, 1024] mask pixels -> out fp32 [N][R][Hm][Wm]: the
 * one-hot plane of label r blurred by a separable Gaussian (taps exp(-d^2 / 2 sigma^2), |d| <= ceil(3 sigma), normalised in
 * fp64, clamp-to-edge).  Labels >= R are the keep plane, which is what the R planes leave.
 * weights_resize_area: fp32 [N][K][Hm][Wm] -> [N][K][Hf][Wf] by the exact area average (fractional box coverage, fp64 sum,
 * rounded once): the identity at equal size, for up- and downsampling alike.
 * wct_stats_weighted: the statistics records of N*K problems (problem n*K + k: frame n under weight plane k of weights
 * fp32 [N][K][H][W], weights >= 0) in the layout of wctb200_stats_record_layout(C, N*K, 0): with W = sum w, Q = sum w^2,
 * n = W^2 / Q (0 without weight) and s, S of the weighted sums scaled by n / W, so that wctb200_wct_transform_from_stats
 * (or ost_transform_from_stats) over the N*K problems gives mean t + s / W and cov (S - s s^T / W) / (W - Q / W).  A
 * record of n < 2, or a style entry with k_s = -1, gets k_c = -1 in the transform.  C in {64,128,256,512}, K in 1..8.
 * wct_transform_apply_weighted: out(p) = sum_k v_k (M_{n,k} x + b_{n,k}) + (1 - sum_k v_k) x with v_k = s(p) w_k(p) over
 * the transforms of N*K problems (a k_c = -1 transform has v = 0); weights [N][K][H][W] or NULL (K = 1, weight 1), strength
 * fp32 [N][H][W] in [0,1] or NULL (1); sum_k w_k <= 1.  A pixel with every v_k = 0 keeps its input bytes.  One-hot
 * weights give the bytes of wctb200_wct_apply_regions, and weights = strength = NULL those of wctb200_wct_transform_apply.
 * adain_transform_apply_strength: wctb200_adain_transform_apply with alpha s(p) at pixel p, strength fp32 [N][H][W]. */
WCTB200_API int wctb200_mask_feather(const uint8_t* labels, int N, int Hm, int Wm, int R, float sigma, float* out, void* stream);
WCTB200_API int wctb200_weights_resize_area(const float* src, int N, int K, int Hm, int Wm, int Hf, int Wf, float* dst, void* stream);
WCTB200_API int wctb200_wct_stats_weighted(const void* act, int N, int H, int W, int C, const float* weights, int K, void* record,
                                           void* stream);
WCTB200_API int wctb200_wct_transform_apply_weighted(const void* act, int N, int H, int W, int C, const void* transform, int K,
                                                     const float* weights, const float* strength, void* out, void* stream);
WCTB200_API int wctb200_adain_transform_apply_strength(const void* act, int N, int H, int W, int C, const void* transform, float alpha,
                                                       const float* strength, void* out, void* stream);

/* Stand-alone pieces of the transform, exposed for parity tests and profiling:
 * per-channel mean [N][C] and covariance [N][C][C] = fc fc^T/(HW-1) + eps_cov*I of a feature batch
 * (ops.py:43-45,105-108), fp32 outputs. */
WCTB200_API int wctb200_covariance(const void* act, int N, int H, int W, int C, float eps_cov, float* mean, float* cov,
                       void* stream);
/* The same per (image, region): labels device uint8 [N][H][W], R in 1..8; mean [N*R][C], cov [N*R][C][C] over the pixels
 * labelled r (entry n*R + r), counts device int32 [N*R] = those pixels; cov = I where a region has fewer than 2 pixels. */
WCTB200_API int wctb200_covariance_regions(const void* act, int N, int H, int W, int C, const uint8_t* labels, int R,
                               float eps_cov, float* mean, float* cov, int32_t* counts, void* stream);
/*
 * symmetric eigen-decomposition of `count` CxC fp32 matrices by one-sided Jacobi.
 * a: [count][C][C] symmetric (overwritten: column i becomes s_i * u_i, u_i the unit eigenvector, s_i within 2e-4 relative of
 * sigma_i -- only the direction of a column is significant),
 * sigma: [count][C] = |lambda_i| (Rayleigh quotients against the input), sweeps: [count] (may be NULL). */
WCTB200_API int wctb200_jacobi_eigh(float* a, int C, int count, float* sigma, int32_t* sweeps, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* WCTB200_H */
