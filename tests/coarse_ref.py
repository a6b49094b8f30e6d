"""NumPy oracle of coarse-to-fine stylisation (DESIGN.md §3.3.16): the coarse size rule and the join
J = clip(rint(C + U(S - D))), in float32 with the operation order of ``k_coarse_join_u8``, so that it gives the kernel's
bytes."""
import numpy as np


def coarse_size(H, W, f, g):
    """Each side divided by f, rounded to the nearest multiple of g (halves up), at least g."""
    def side(n):
        q = max(1, int(np.floor(n / (f * g) + 0.5)))
        return g * q
    return side(H), side(W)


def taps(n_out, n_in):
    """(i0, i1, weight) per output coordinate of one axis: s = (i + 0.5) (n_in / n_out) - 0.5 in float32, clamped to
    [0, n_in - 1]; i0 = floor(s), i1 = min(i0 + 1, n_in - 1), weight s - i0."""
    f32 = np.float32
    sc = f32(n_in) / f32(n_out)
    s = (np.arange(n_out, dtype=f32) + f32(0.5)) * sc - f32(0.5)
    s = np.clip(s, f32(0), f32(n_in - 1)).astype(f32)
    i0 = np.floor(s).astype(np.int64)
    i1 = np.minimum(i0 + 1, n_in - 1)
    return i0, i1, (s - i0.astype(f32)).astype(f32)


def upsampled_delta(coarse, stylised, H, W):
    """U(S - D) [N,H,W,3] in float32 before the content is added: the exact differences, interpolated along x in each of
    the two rows, then along y."""
    d = stylised.astype(np.float32) - coarse.astype(np.float32)
    y0, y1, wy = taps(H, d.shape[1])
    x0, x1, wx = taps(W, d.shape[2])
    wx = wx[None, None, :, None]
    wy = wy[None, :, None, None]

    def row(r):
        a, b = d[:, r][:, :, x0], d[:, r][:, :, x1]
        return a + wx * (b - a)
    a, b = row(y0), row(y1)
    return a + wy * (b - a)


def join(content, coarse, stylised):
    """clip(rint(C + U(S - D)), 0, 255) as uint8, rint half to even."""
    v = content.astype(np.float32) + upsampled_delta(coarse, stylised, content.shape[1], content.shape[2])
    return np.clip(np.rint(v), 0, 255).astype(np.uint8)
