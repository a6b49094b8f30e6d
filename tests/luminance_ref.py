"""Float64 / exact-integer oracle of luminance-only transfer (DESIGN.md §3.3.15), written from the definition and
independent of the package.

Per pixel L = 299 R + 587 G + 114 B (an exact integer) and Y = L / 1000.  grey(s) = clip(rint(Y_s)); the content is matched
to the grey style's luminance mean / spread, g = clip(rint(mu_s + k (Y - mu_c))), k = sd_s / sd_c (1 when either is 0);
after stylising g the result's luminance is mapped back, Y' = mu_c + (Y_S - mu_s) / k, and out_c = clip(rint(content_c + Y'
- Y_content)) for every channel.  The functions that return values before rounding let tests compare within 1 LSB and
exactly away from half-integers."""
import numpy as np

WEIGHTS = np.array([299, 587, 114], np.int64)


def luma_int(img):
    """uint8 [..., 3] -> int64 L [...]."""
    return np.asarray(img, np.int64) @ WEIGHTS


def moments(frames):
    """(npix per frame, [sum L], [sum L^2]) of uint8 [N,H,W,3] as Python integers."""
    L = luma_int(frames).reshape(frames.shape[0], -1)
    return L.shape[1], [int(r.sum()) for r in L], [int((r * r).sum()) for r in L]


def stats_from_moments(npix, s1, s2):
    """(mean, population std) of Y = L / 1000 from exact moments (one frame)."""
    return s1 / (1000.0 * npix), np.sqrt(float(npix * s2 - s1 * s1) / (float(npix) ** 2 * 1e6))


def stats(frames):
    """Per-frame (mean, std) float64 arrays [N] of the luminance of uint8 [N,H,W,3]."""
    n, s1, s2 = moments(frames)
    st = np.array([stats_from_moments(n, a, b) for a, b in zip(s1, s2)])
    return st[:, 0], st[:, 1]


def weighted_mixture(means, sds, w):
    """Mean / std of the mixture of K distributions under weights w [.., K] that sum to 1."""
    means, sds, w = np.asarray(means, np.float64), np.asarray(sds, np.float64), np.asarray(w, np.float64)
    mu = w @ means
    return mu, np.sqrt(np.maximum(w @ (sds ** 2 + means ** 2) - mu ** 2, 0.0))


def pooled(images):
    """Mean / std of the luminance over the pixels of all ``images`` (uint8 [H_i,W_i,3]) taken together."""
    L = np.concatenate([luma_int(x).ravel() for x in images])
    return stats_from_moments(L.size, int(L.sum()), int((L * L).sum()))


def round_clip(v):
    return np.clip(np.rint(v), 0, 255).astype(np.uint8)


def grey(img):
    """clip(rint(Y)) replicated to R = G = B."""
    Y = luma_int(img) / 1000.0
    return np.repeat(round_clip(Y)[..., None], 3, axis=-1)


def params(mean_c, sd_c, mean_s, sd_s):
    """k per frame (1 when either std is 0)."""
    mean_c, sd_c, mean_s, sd_s = np.broadcast_arrays(*(np.asarray(v, np.float64) for v in (mean_c, sd_c, mean_s, sd_s)))
    ok = (sd_c > 0) & (sd_s > 0)
    return np.where(ok, sd_s / np.where(ok, sd_c, 1.0), 1.0)


def match_pre(frames, mean_c, mean_s, k):
    """mu_s + k (Y - mu_c) per pixel [N,H,W] before rounding (per-frame mean_c, mean_s, k)."""
    Y = luma_int(frames) / 1000.0
    sh = (-1,) + (1,) * (Y.ndim - 1)
    return np.reshape(mean_s, sh) + np.reshape(k, sh) * (Y - np.reshape(mean_c, sh))


def match(frames, mean_c, mean_s, k):
    return np.repeat(round_clip(match_pre(frames, mean_c, mean_s, k))[..., None], 3, axis=-1)


def merge_pre(content, Y_S, mean_c, mean_s, k):
    """content_c + Y' - Y_content per pixel and channel [N,H,W,3] before rounding; Y_S [N,H,W] float (the stylised
    frames' luminance, or any other luminance to merge)."""
    sh = (-1,) + (1,) * (Y_S.ndim - 1)
    Yp = np.reshape(mean_c, sh) + (Y_S - np.reshape(mean_s, sh)) / np.reshape(k, sh)
    d = Yp - luma_int(content) / 1000.0
    return np.asarray(content, np.float64) + d[..., None]


def merge(content, stylised, mean_c, mean_s, k):
    return round_clip(merge_pre(content, luma_int(stylised) / 1000.0, mean_c, mean_s, k))


def iq(img):
    """YIQ I and Q of RGB values [..., 3] (any dtype) in float64."""
    x = np.asarray(img, np.float64)
    return x @ np.array([0.596, -0.274, -0.322]), x @ np.array([0.211, -0.523, 0.312])


# |I(out) - I(content)| <= 0.5 * sum |row| where no channel clips: out_c - content_c = d + e_c with |e_c| <= 0.5, and each
# row sums to 0, so d cancels
IQ_BOUND = (0.5 * (0.596 + 0.274 + 0.322), 0.5 * (0.211 + 0.523 + 0.312))
