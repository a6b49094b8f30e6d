"""Float32 NumPy restatement of the temporal stabilisation of DESIGN.md §3.3.6 (wct_tf_b200/csrc/flow.cu).

Every array is float32 and every operation is one rounded float32 operation, in the order the kernels issue them, so the
device reproduces these results bit for bit.  Flows are [2, H, W] (u = x displacement, v = y displacement); the flows of a
stack of M frames are [2 (M - 1), 2, H, W], problem 2t the backward flow from frame t+1 to frame t and problem 2t+1 the
forward flow from frame t to frame t+1.
"""
import numpy as np

f32 = np.float32

# the constants of wct_tf_b200/csrc/flow.cu (DESIGN.md §3.3.6)
HS_ALPHA2 = f32(0.0025)      # alpha = 0.05, smoothness weight of Horn-Schunck on luminance in [0, 1]
MAX_LEVELS = 6
MIN_SIDE = 32
WARPS = 3
ITERS = 30
FB_A = f32(0.01)
FB_B = f32(0.25)
PHOTO_TAU = f32(0.05)
CUT_PERCENT = 50


def luminance(frames):
    """uint8 [..., H, W, 3] -> float32 [..., H, W]: (0.299 R + 0.587 G + 0.114 B) / 255."""
    x = np.asarray(frames).astype(f32)
    t = f32(0.299) * x[..., 0]
    t = t + f32(0.587) * x[..., 1]
    t = t + f32(0.114) * x[..., 2]
    return t / f32(255)


def level_sizes(H, W):
    sizes = [(H, W)]
    while len(sizes) < MAX_LEVELS:
        h, w = (sizes[-1][0] + 1) // 2, (sizes[-1][1] + 1) // 2
        if min(h, w) < MIN_SIDE:
            break
        sizes.append((h, w))
    return sizes


def sample(img, x, y):
    """Bilinear sample of img [h, w] at (x, y), coordinates clamped to the border."""
    h, w = img.shape
    x = np.minimum(np.maximum(x, f32(0)), f32(w - 1))
    y = np.minimum(np.maximum(y, f32(0)), f32(h - 1))
    x0, y0 = np.floor(x), np.floor(y)
    fx, fy = x - x0, y - y0
    ix0, iy0 = x0.astype(np.int64), y0.astype(np.int64)
    ix1, iy1 = np.minimum(ix0 + 1, w - 1), np.minimum(iy0 + 1, h - 1)
    a, b, c, d = img[iy0, ix0], img[iy0, ix1], img[iy1, ix0], img[iy1, ix1]
    top = a + fx * (b - a)
    bot = c + fx * (d - c)
    return top + fy * (bot - top)


def grid(h, w):
    ys, xs = np.meshgrid(np.arange(h, dtype=f32), np.arange(w, dtype=f32), indexing="ij")
    return xs, ys


def downsample(img):
    """2x2 box average, ceil sizes, edge replication."""
    h, w = img.shape
    ys, xs = 2 * np.arange((h + 1) // 2), 2 * np.arange((w + 1) // 2)
    ys1, xs1 = np.minimum(ys + 1, h - 1), np.minimum(xs + 1, w - 1)
    a, b = img[ys][:, xs], img[ys][:, xs1]
    c, d = img[ys1][:, xs], img[ys1][:, xs1]
    return ((a + b) + (c + d)) * f32(0.25)


def upsample_flow(flow, h, w):
    """[2, hc, wc] -> [2, h, w]: bilinear at the pixel centres, values x2."""
    xs, ys = grid(h, w)
    sx = (xs + f32(0.5)) * f32(0.5) - f32(0.5)
    sy = (ys + f32(0.5)) * f32(0.5) - f32(0.5)
    return np.stack([sample(flow[0], sx, sy) * f32(2), sample(flow[1], sx, sy) * f32(2)])


def warp_coefs(I0, I1, u, v):
    """Linearise I1(x + w) - I0(x) around the current flow: (Ix, Iy, It', den) with It' = It - Ix u - Iy v, so that a
    Jacobi step acts on the whole flow."""
    xs, ys = grid(*I0.shape)
    X, Y = xs + u, ys + v
    Iw = sample(I1, X, Y)
    Ix = (sample(I1, X + f32(1), Y) - sample(I1, X - f32(1), Y)) * f32(0.5)
    Iy = (sample(I1, X, Y + f32(1)) - sample(I1, X, Y - f32(1))) * f32(0.5)
    It = ((Iw - I0) - Ix * u) - Iy * v
    den = (HS_ALPHA2 + Ix * Ix) + Iy * Iy
    return Ix, Iy, It, den


def neighbour_mean(u):
    p = np.pad(u, 1, mode="edge")
    return ((p[:-2, 1:-1] + p[2:, 1:-1]) + (p[1:-1, :-2] + p[1:-1, 2:])) * f32(0.25)


def jacobi(u, v, Ix, Iy, It, den, iters):
    for _ in range(iters):
        ub, vb = neighbour_mean(u), neighbour_mean(v)
        t = ((Ix * ub + Iy * vb) + It) / den
        u, v = ub - Ix * t, vb - Iy * t
    return u, v


def flow(I0, I1):
    """Coarse-to-fine Horn-Schunck with warping: the flow w with I1(x + w(x)) ~ I0(x), float32 [2, H, W]."""
    p0, p1 = [np.asarray(I0, f32)], [np.asarray(I1, f32)]
    sizes = level_sizes(*p0[0].shape)
    for _ in sizes[1:]:
        p0.append(downsample(p0[-1]))
        p1.append(downsample(p1[-1]))
    w = None
    for l in range(len(sizes) - 1, -1, -1):
        h, wd = sizes[l]
        w = np.zeros((2, h, wd), f32) if w is None else upsample_flow(w, h, wd)
        u, v = w[0], w[1]
        for _ in range(WARPS):
            u, v = jacobi(u, v, *warp_coefs(p0[l], p1[l], u, v), ITERS)
        w = np.stack([u, v])
    return w


def flow_pairs(Y):
    """Y float32 [M, H, W] -> flows [2 (M - 1), 2, H, W]: backward (t+1 -> t) and forward (t -> t+1) for every pair."""
    out = []
    for t in range(Y.shape[0] - 1):
        out.append(flow(Y[t + 1], Y[t]))
        out.append(flow(Y[t], Y[t + 1]))
    return np.stack(out) if out else np.zeros((0, 2) + Y.shape[1:], f32)


def confidence(Y, flows):
    """uint8 masks [M - 1, H, W] (mask t for frame t+1 against frame t) and their counts before the cut rule."""
    M, H, W = Y.shape
    xs, ys = grid(H, W)
    masks, counts = [], []
    for t in range(M - 1):
        ub, vb = flows[2 * t]
        uf0, vf0 = flows[2 * t + 1]
        px, py = xs + ub, ys + vb
        inside = (px >= 0) & (px <= f32(W - 1)) & (py >= 0) & (py <= f32(H - 1))
        uf, vf = sample(uf0, px, py), sample(vf0, px, py)
        dx, dy = uf + ub, vf + vb
        lhs = dx * dx + dy * dy
        rhs = FB_A * ((uf * uf + vf * vf) + (ub * ub + vb * vb)) + FB_B
        photo = np.abs(Y[t + 1] - sample(Y[t], px, py)) <= PHOTO_TAU
        c = inside & (lhs <= rhs) & photo
        n = int(c.sum())
        if n * 100 < CUT_PERCENT * H * W:
            c[:] = False
        masks.append(c.astype(np.uint8))
        counts.append(n)
    return (np.stack(masks) if masks else np.zeros((0, H, W), np.uint8)), counts


def blend_one(frame, prev_out, flow_b, mask, beta):
    """O = round(P + beta c (O_prev(x + w_b) - P)) per channel, round = floor(v + 0.5), clamped to 0..255."""
    H, W = frame.shape[:2]
    xs, ys = grid(H, W)
    px, py = xs + flow_b[0], ys + flow_b[1]
    beta = f32(beta)
    out = np.empty_like(frame)
    for ch in range(3):
        P = frame[..., ch].astype(f32)
        s = sample(prev_out[..., ch].astype(f32), px, py)
        v = np.where(mask != 0, P + beta * (s - P), P)
        out[..., ch] = np.clip(np.floor(v + f32(0.5)), 0, 255).astype(np.uint8)
    return out


def blend(frames, prev_out, flows, masks, beta):
    """frames uint8 [N, H, W, 3] stylised; prev_out uint8 [H, W, 3] (the stabilised predecessor of frame 0) or None (frame 0
    starts the clip).  Returns the stabilised frames."""
    out = np.array(frames, copy=True)
    first = 0 if prev_out is not None else 1
    for j in range(out.shape[0] - first):
        i = j + first
        prev = prev_out if i == 0 else out[i - 1]
        out[i] = blend_one(out[i], prev, flows[2 * j], masks[j], beta)
    return out


def stabilize(contents, stylised, beta, prev=None):
    """One call of the recurrence on frames of one size: contents uint8 [N, H, W, 3] at the stylised size, stylised uint8
    [N, H, W, 3], prev = (luminance [H, W], stabilised output [H, W, 3]) of the frame before, or None.  Returns (stabilised
    frames, the new prev)."""
    Y = luminance(contents)
    Ys = Y if prev is None else np.concatenate([prev[0][None], Y])
    out = np.array(stylised, copy=True)
    if Ys.shape[0] >= 2:
        flows = flow_pairs(Ys)
        masks, _ = confidence(Ys, flows)
        out = blend(out, None if prev is None else prev[1], flows, masks, beta)
    return out, (Y[-1], out[-1])


# ---- synthetic clips (seeded) -------------------------------------------------------------------------------------------
def texture(H, W, seed, shift=(0.0, 0.0), n_waves=24):
    """A smooth random RGB texture, a sum of low-frequency waves, sampled at (x - dx, y - dy): an exact sub-pixel shift."""
    rng = np.random.default_rng(seed)
    ys, xs = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    xs, ys = xs - shift[0], ys - shift[1]
    img = np.full((H, W, 3), 128.0)
    for _ in range(n_waves):
        f = rng.uniform(0.01, 0.08, 2) * rng.choice([-1, 1], 2)
        ph = rng.uniform(0, 2 * np.pi)
        amp = rng.uniform(6, 16, 3)
        img += amp * np.cos(2 * np.pi * (f[0] * xs + f[1] * ys) + ph)[..., None]
    return np.clip(np.round(img), 0, 255).astype(np.uint8)


def translating_clip(T, H, W, d=(0.75, 0.5), seed=0, square=None, cut=None):
    """T frames of texture(seed) moved by d px per frame.  square = (size, x0, y0, vx, vy): a square of another texture moving
    by (vx, vy) whole pixels per frame on top (occlusion).  cut = frame index from which the clip shows an unrelated texture."""
    frames = []
    for t in range(T):
        if cut is not None and t >= cut:
            fr = texture(H, W, seed + 1000, (d[0] * (t - cut), d[1] * (t - cut)))
        else:
            fr = texture(H, W, seed, (d[0] * t, d[1] * t))
        if square is not None:
            s, x0, y0, vx, vy = square
            x, y = x0 + vx * t, y0 + vy * t
            patch = 255 - texture(s, s, seed + 2000)
            fr[y:y + s, x:x + s] = patch[:H - y, :W - x]
        frames.append(fr)
    return np.stack(frames)
