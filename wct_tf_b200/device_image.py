"""The CLI's image steps on the device (scope row 8f-3): same names, arguments and results as the reference's helpers
(``utils.resize_to`` / ``center_crop`` / ``center_crop_to`` utils.py:29-67, ``utils.preserve_colors_np`` utils.py:87-90,
the ``--concat`` thumbnail stylize.py:107-111), operating on ``torch.uint8`` CUDA tensors HxWx3 (or NxHxWx3) through the C ABI
(``wctb200_resize_bilinear_u8``, ``wctb200_rgb_moments_u8``, ``wctb200_coral_apply_u8``).  A decoded image goes to the GPU once
and stays there through resize, crop, CORAL, every ``--passes`` round and the concat; only the finished frame comes back.
``noise_u8`` makes the noise frames of texture synthesis (``--noise``) on the device (``wctb200_noise_u8``).  The
``luminance_*`` functions are the pixel steps of luminance-only transfer (``--luminance-only``, DESIGN.md §3.3.15): exact
per-frame luminance moments, the matched grey and the merge of a stylised luminance into the content's colours.

There is no CPU fallback: the functions raise ``WctB200Error`` when the library or a CUDA device is missing.  The only host
arithmetic is the 3x3 algebra of CORAL (the reference's ``matSqrt`` goes through ``np.linalg.svd`` and, as written, depends on
its sign conventions -- coral.py:8-11 -- so the same call is made here on the 3x3 matrices built from the device's exact
integer moments).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _capi


def _stream():
    return torch.cuda.current_stream().cuda_stream


def to_device(img, device="cuda:0"):
    """numpy / torch uint8 HxWxC -> contiguous CUDA tensor (one H2D copy)."""
    if not torch.cuda.is_available():
        raise _capi.WctB200Error("no CUDA device: the image steps have no CPU fallback")
    t = img if isinstance(img, torch.Tensor) else torch.from_numpy(np.array(img, dtype=np.uint8, order="C"))   # own, writable copy (PIL arrays are read-only)
    if t.dtype != torch.uint8:
        raise TypeError("expected a uint8 image, got %s" % t.dtype)
    return t.to(device, non_blocking=True).contiguous()


def to_host(img):
    """uint8 CUDA tensor -> numpy (synchronous D2H)."""
    return img.cpu().numpy()


def _as_batch(img):
    if img.dim() == 3:
        return img.unsqueeze(0), True
    if img.dim() == 4:
        return img, False
    raise ValueError("expected HxWxC or NxHxWxC, got shape %s" % (tuple(img.shape),))


def imresize(img, hw, window=None):
    """``scipy.misc.imresize(img, (H, W), interp='bilinear')`` (utils.py:48,67; bit-exact with Pillow's resample); ``window`` =
    (y0, x0, Hout, Wout) returns that crop of the result without computing the rest."""
    lib = _capi.load()
    x, single = _as_batch(img)
    if not x.is_cuda:
        raise _capi.WctB200Error("device_image works on CUDA tensors (use to_device)")
    x = x.contiguous()
    N, Hs, Ws, Cc = x.shape
    Hd, Wd = int(hw[0]), int(hw[1])
    y0, x0, Ho, Wo = (0, 0, Hd, Wd) if window is None else [int(v) for v in window]
    with torch.cuda.device(x.device):
        nbytes = lib.wctb200_resize_workspace_bytes(N, Hs, Ws, Cc, Hd, Wd, Wo)
        if nbytes == 0:
            raise _capi.WctB200Error("resize: bad geometry %s -> %s" % ((N, Hs, Ws, Cc), (Hd, Wd)))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
        out = torch.empty((N, Ho, Wo, Cc), dtype=torch.uint8, device=x.device)
        _capi.check(lib.wctb200_resize_bilinear_u8(x.data_ptr(), N, Hs, Ws, Cc, Hd, Wd, y0, x0, Ho, Wo, out.data_ptr(),
                                                   ws.data_ptr(), nbytes, _stream()))
    return out[0] if single else out


def _short_side_shape(height, width, resize):
    # utils.py:57-65 (Python 3 round: banker's rounding, as in the reference)
    if height < width:
        return resize, int(round(width / (height / resize)))
    return int(round(height / (width / resize))), resize


def resize_to(img, resize=512):
    """utils.py:55-67: SHORT side to ``resize``, aspect ratio kept."""
    h, w = (img.shape[0], img.shape[1]) if img.dim() == 3 else (img.shape[1], img.shape[2])
    return imresize(img, _short_side_shape(h, w, resize))


def center_crop(img, size=256):
    """utils.py:29-38; the resize (when a side is too small) and the crop are one launch sequence: only the window is computed."""
    h, w = (img.shape[0], img.shape[1]) if img.dim() == 3 else (img.shape[1], img.shape[2])
    hd, wd = (h, w) if (h >= size and w >= size) else _short_side_shape(h, w, size)
    return imresize(img, (hd, wd), window=((hd - size) // 2, (wd - size) // 2, size, size))


def center_crop_to(img, H_target, W_target):
    """utils.py:40-53"""
    h, w = (img.shape[0], img.shape[1]) if img.dim() == 3 else (img.shape[1], img.shape[2])
    hd, wd = h, w
    if h < H_target or w < W_target:
        rat = max(H_target / h, W_target / w)
        hd, wd = int(h * rat), int(w * rat)          # imresize(img, <float>): both sides scaled by the fraction, truncated
    return imresize(img, (hd, wd), window=((hd - H_target) // 2, (wd - W_target) // 2, H_target, W_target))


def rgb_moments(img):
    """(npix, sum x_c [3], sum x_c x_d [3][3]) of an RGB uint8 image -- exact integers from the device."""
    lib = _capi.load()
    x = img.contiguous()
    if x.shape[-1] != 3:
        raise ValueError("expected an RGB image")
    npix = x.numel() // 3
    with torch.cuda.device(x.device):
        sums = torch.empty(9, dtype=torch.int64, device=x.device)
        _capi.check(lib.wctb200_rgb_moments_u8(x.data_ptr(), npix, sums.data_ptr(), _stream()))
        s = [int(v) for v in sums.cpu().tolist()]
    s1 = np.array(s[:3], dtype=object)
    s2 = np.empty((3, 3), dtype=object)
    s2[0, 0], s2[0, 1], s2[0, 2], s2[1, 1], s2[1, 2], s2[2, 2] = s[3:]
    s2[1, 0], s2[2, 0], s2[2, 1] = s2[0, 1], s2[0, 2], s2[1, 2]
    return npix, s1, s2


def _mat_sqrt(x):
    # coral.py:8-11 as written: U diag(sqrt D) (V^T)^T with numpy's (u, s, vh) -- for the symmetric input U sqrt(D) U
    u, d, vh = np.linalg.svd(x)
    return (u * np.sqrt(d)) @ vh.T


def _standardised_stats(img):
    """mean, std (population, np.std) and norm . norm^T + I of the [0,1]-scaled channels (coral.py:23-32), from the moments."""
    npix, s1, s2 = rgb_moments(img)
    mean = np.array([float(v) / npix for v in s1]) / 255.0
    # population covariance of x/255 from exact integers: (n*S2 - s s^T) / n^2 / 255^2 (the integer numerator is exact)
    cov = np.array([[float(npix * s2[i, j] - s1[i] * s1[j]) for j in range(3)] for i in range(3)]) / (float(npix) ** 2) / 255.0 ** 2
    std = np.sqrt(np.diag(cov))
    gram = npix * cov / np.outer(std, std) + np.eye(3)
    return mean, std, gram


def preserve_colors_np(style_rgb, content_rgb):
    """utils.py:87-90 (--keep-colors): CORAL of the style to the content's colour statistics; uint8 CUDA tensors in and out."""
    lib = _capi.load()
    src = style_rgb.contiguous()
    sm, ss, cs = _standardised_stats(src)
    tm, ts, ct = _standardised_stats(content_rgb)
    A = np.ascontiguousarray(_mat_sqrt(ct) @ np.linalg.inv(_mat_sqrt(cs)), dtype=np.float64)
    out = torch.empty_like(src)

    def dp(a):
        a = np.ascontiguousarray(a, dtype=np.float64)
        return a, a.ctypes.data_as(C.c_void_p)
    keep = [dp(A), dp(sm), dp(ss), dp(tm), dp(ts)]
    with torch.cuda.device(src.device):
        _capi.check(lib.wctb200_coral_apply_u8(src.data_ptr(), src.numel() // 3, keep[0][1], keep[1][1], keep[2][1], keep[3][1],
                                               keep[4][1], out.data_ptr(), _stream()))
    return out


# BT.601 luma weights in thousandths: L = 299 R + 587 G + 114 B is an exact integer, Y = L / 1000 (flow.cu's k_luminance)
LUMA_WEIGHTS = (299, 587, 114)


def _frames(img):
    x, _ = _as_batch(img)
    if not x.is_cuda:
        raise _capi.WctB200Error("device_image works on CUDA tensors (use to_device)")
    if x.shape[-1] != 3:
        raise ValueError("expected RGB frames, got shape %s" % (tuple(x.shape),))
    return x.contiguous()


def luminance_moments(img):
    """(npix per frame, [sum L], [sum L^2]) of uint8 RGB frames [H,W,3] or [N,H,W,3], L = 299 R + 587 G + 114 B: exact Python
    integers per frame, from the device's nine integer sums per frame (``wctb200_rgb_moments_batch_u8``) as w.s1 and
    w^T S2 w."""
    lib = _capi.load()
    x = _frames(img)
    N, npf = x.shape[0], x.shape[1] * x.shape[2]
    with torch.cuda.device(x.device):
        sums = torch.empty((N, 9), dtype=torch.int64, device=x.device)
        _capi.check(lib.wctb200_rgb_moments_batch_u8(x.data_ptr(), N, npf, sums.data_ptr(), _stream()))
        rows = sums.cpu().tolist()
    w0, w1, w2 = LUMA_WEIGHTS
    s1 = [w0 * r[0] + w1 * r[1] + w2 * r[2] for r in rows]
    s2 = [w0 * w0 * r[3] + 2 * w0 * w1 * r[4] + 2 * w0 * w2 * r[5] + w1 * w1 * r[6] + 2 * w1 * w2 * r[7] + w2 * w2 * r[8]
          for r in rows]
    return npf, s1, s2


def luminance_stats_from_moments(npix, s1, s2):
    """(mean, population std) of Y = L / 1000 in float64 from exact moments of L (scalars or per-frame lists): the
    variance's numerator n S2 - S1^2 is an exact integer."""
    one = not isinstance(s1, (list, tuple))
    s1, s2 = ([s1], [s2]) if one else (s1, s2)
    mean = np.array([a / (1000.0 * npix) for a in s1])
    sd = np.sqrt(np.array([float(npix * b - a * a) for a, b in zip(s1, s2)]) / (float(npix) ** 2 * 1e6))
    return (mean[0], sd[0]) if one else (mean, sd)


def luminance_stats(img):
    """Per-frame (mean, population std) of the luminance Y = (299 R + 587 G + 114 B) / 1000 of uint8 RGB frames on the
    device: two float64 arrays [N] from exact integer moments."""
    return luminance_stats_from_moments(*luminance_moments(img))


def _kb(k, b, n, device):
    """Per-frame (k, b) as a device float32 [n, 2] (k and b: scalars or length-n sequences, float64 on the host)."""
    kb = np.empty((n, 2), np.float32)
    kb[:, 0], kb[:, 1] = np.broadcast_to(np.asarray(k, np.float64), n), np.broadcast_to(np.asarray(b, np.float64), n)
    return torch.from_numpy(kb).to(device, non_blocking=True)


def luminance_match(img, k, b):
    """Replicated grey clip(rint(k Y + b)) of uint8 RGB frames on the device (``wctb200_luminance_match_u8``); ``k`` and
    ``b`` per frame (or one for all)."""
    lib = _capi.load()
    x = _frames(img)
    N, npf = x.shape[0], x.shape[1] * x.shape[2]
    with torch.cuda.device(x.device):
        kb = _kb(k, b, N, x.device)
        out = torch.empty_like(x)
        _capi.check(lib.wctb200_luminance_match_u8(x.data_ptr(), N, npf, kb.data_ptr(), out.data_ptr(), _stream()))
    return out if img.dim() == 4 else out[0]


def luminance_grey(img):
    """The grey of uint8 RGB frames: clip(rint(Y)) in R = G = B."""
    return luminance_match(img, 1.0, 0.0)


def luminance_merge(content, stylised, k_inv, b):
    """Content frames with their luminance replaced by k_inv Y(stylised) + b (per frame), the same difference added to R, G
    and B so that the content's chrominance stays (``wctb200_luminance_merge_u8``).  Both uint8 RGB, of one shape."""
    lib = _capi.load()
    c, s = _frames(content), _frames(stylised)
    if c.shape != s.shape:
        raise ValueError("luminance_merge: content %s and stylised %s frames differ in shape" % (tuple(c.shape), tuple(s.shape)))
    N, npf = c.shape[0], c.shape[1] * c.shape[2]
    with torch.cuda.device(c.device):
        kb = _kb(k_inv, b, N, c.device)
        out = torch.empty_like(c)
        _capi.check(lib.wctb200_luminance_merge_u8(c.data_ptr(), s.data_ptr(), N, npf, kb.data_ptr(), out.data_ptr(), _stream()))
    return out if content.dim() == 4 else out[0]


def luminance_params(mean_c, sd_c, mean_s, sd_s):
    """Per-frame parameters of luminance-only transfer from the content's and the style's luminance statistics (float64):
    k = sd_s / sd_c (1 when either is 0), the match (k, mean_s - k mean_c) and the merge (1/k, mean_c - mean_s / k)."""
    mean_c, sd_c, mean_s, sd_s = np.broadcast_arrays(*(np.asarray(v, np.float64) for v in (mean_c, sd_c, mean_s, sd_s)))
    k = np.where((sd_c > 0) & (sd_s > 0), sd_s / np.where(sd_c > 0, sd_c, 1.0), 1.0)
    return (k, mean_s - k * mean_c), (1.0 / k, mean_c - mean_s / k)


def coarse_join(content, coarse_content, coarse_stylised):
    """The join of coarse-to-fine stylisation (DESIGN.md §3.3.16): clip(rint(C + U(S - D))) on the device
    (``wctb200_coarse_join_u8``), the content frames C [H,W,3] or [N,H,W,3] with their low band, the coarse content D
    [h,w,3] or [N,h,w,3], replaced by the stylised low band S of D's shape; U is bilinear resampling from h x w to H x W.
    All uint8 on one CUDA device; returns uint8 of C's shape."""
    lib = _capi.load()
    c, d, s = _frames(content), _frames(coarse_content), _frames(coarse_stylised)
    if d.shape != s.shape or d.shape[0] != c.shape[0] or not (c.device == d.device == s.device):
        raise ValueError("coarse_join: content %s, coarse content %s and coarse stylised %s frames must be [N,H,W,3], [N,h,w,3] "
                         "and [N,h,w,3] on one device" % (tuple(c.shape), tuple(d.shape), tuple(s.shape)))
    N, H, W = c.shape[:3]
    h, w = d.shape[1:3]
    with torch.cuda.device(c.device):
        out = torch.empty_like(c)
        _capi.check(lib.wctb200_coarse_join_u8(c.data_ptr(), d.data_ptr(), s.data_ptr(), N, H, W, h, w, out.data_ptr(),
                                               _stream()))
    return out if content.dim() == 4 else out[0]


def noise_u8(count, height, width, seed=0, first_index=0, device="cuda:0"):
    """--noise (webcam.py:191-192, ``np.random.randint(0, 256, shape, np.uint8)``): ``count`` frames of uniform random bytes,
    a uint8 CUDA tensor [count, height, width, 3] made on the device (``wctb200_noise_u8``) on the current stream.  Frame i
    is a pure function of (seed, first_index + i, height, width): counter-based Philox4x32-10, so it does not depend on
    ``count`` or on how a run is cut into calls.  ``seed``: 0 .. 2^64 - 1; ``first_index`` >= 0."""
    if not torch.cuda.is_available():
        raise _capi.WctB200Error("no CUDA device: the image steps have no CPU fallback")
    count, height, width, seed, first_index = int(count), int(height), int(width), int(seed), int(first_index)
    if count < 1 or height < 1 or width < 1:
        raise ValueError("noise_u8: count, height and width must be >= 1, got %d, %d, %d" % (count, height, width))
    if not 0 <= seed < 2 ** 64 or not 0 <= first_index < 2 ** 63:
        raise ValueError("noise_u8: seed must be in [0, 2^64) and first_index in [0, 2^63)")
    lib = _capi.load()
    with torch.cuda.device(device):
        out = torch.empty((count, height, width, 3), dtype=torch.uint8, device=device)
        _capi.check(lib.wctb200_noise_u8(out.data_ptr(), count, height, width, 3, seed, first_index, _stream()))
    return out


def concat_with_style(style_img, result):
    """--concat (stylize.py:107-111): [style resized to the result's height, square | result]"""
    edge = result.shape[0]
    return torch.cat([imresize(style_img, (edge, edge)), result], dim=1)
