"""NumPy oracle of multimodal style transfer (DESIGN.md §3.3.10): the k-means++ draws, spherical Lloyd, the data term in
float64, red-black ICM in explicitly rounded float32, and ``pipeline_mst`` on ``oracle.nets``.  Test infrastructure only.

Features are float arrays [..., C]; the device's are the SPF16 values hi + lo (``tests.gpu_util.split_repr``).  A pixel's
unit direction is u = f / max(|f|, 1e-12)."""
import numpy as np

from oracle import nets
from tests.regions_ref import resize_labels
from tests.style_masks_ref import wct_style_masks
from tests.texture_ref import philox4x32_10

KEY = (0x3154534D, 0x50504D4B)     # Philox key of the k-means++ draws
PIX = 256                          # k-means++ block size
LLOYD_MAX = 16
SWEEPS = 8


def unit(f):
    """float64 unit directions of f [..., C]; a zero vector stays 0."""
    f = np.asarray(f, np.float64)
    n = np.sqrt((f * f).sum(-1, keepdims=True))
    return f / np.maximum(n, 1e-12)


def draw(j, level):
    """x0 of Philox4x32-10 at counter (j, level, 0, 0) under KEY."""
    return int(philox4x32_10(np.array([[j, level, 0, 0]]), KEY)[0, 0])


def kmeanspp_distances(u, centres):
    """d_p = max(0, 1 - max_i u_p . c_i) (float64) for the centres chosen so far [j, C]."""
    return np.maximum(0.0, 1.0 - (u @ np.asarray(centres, np.float64).T).max(axis=1))


def kmeanspp_select(d, j, level):
    """The pixel of draw j >= 1 given d [P]: the first pixel whose running sum (block sums of PIX pixels, each in pixel order,
    added in block order) exceeds v sum(d), v = x0 / 2^32; None when sum(d) = 0 (the centre copies centre 0)."""
    P = d.shape[0]
    bs = [float(np.sum(d[b:b + PIX])) for b in range(0, P, PIX)]
    total = float(np.sum(bs))
    if total <= 0:
        return None
    T = draw(j, level) / 2.0 ** 32 * total
    run = np.cumsum(d)
    return int(min(np.searchsorted(run, T, side="right"), P - 1))


def kmeanspp(u, K, level):
    """Init pixel indices of the k-means++ seeding of u [P, C] (float64 distances)."""
    P = u.shape[0]
    idx = [(draw(0, level) * P) >> 32]
    for j in range(1, K):
        p = kmeanspp_select(kmeanspp_distances(u, u[idx]), j, level)
        idx.append(idx[0] if p is None else p)
    return idx


def check_draws(u, idx, level, tol=1e-9):
    """Asserts that the init indices ``idx`` are k-means++ draws of u [P, C]: index 0 is floor(v P), and index j >= 1 sits on
    the interval of the running sum of d that holds v sum(d), up to ``tol`` (relative to sum(d)) at the interval's edges."""
    P = u.shape[0]
    assert idx[0] == (draw(0, level) * P) >> 32, (idx[0], (draw(0, level) * P) >> 32)
    for j in range(1, len(idx)):
        d = kmeanspp_distances(u, u[list(idx[:j])])
        total = d.sum()
        if total <= tol:
            assert idx[j] == idx[0] or d[idx[j]] <= tol, (j, idx[j])
            continue
        T = draw(j, level) / 2.0 ** 32 * total
        run = np.cumsum(d)
        lo = run[idx[j]] - d[idx[j]]
        assert lo <= T + tol * total and run[idx[j]] >= T - tol * total, (j, idx[j], lo, run[idx[j]], T)


def assign(u, centres):
    """(labels, margins): argmax_k u . c_k (ties to the lowest k) and the gap to the runner-up (inf for K = 1)."""
    s = u @ np.asarray(centres, np.float64).T
    lab = np.argmax(s, axis=1)
    if s.shape[1] == 1:
        return lab, np.full(lab.shape, np.inf)
    top = np.sort(s, axis=1)
    return lab, top[:, -1] - top[:, -2]


def update(u, labels, centres):
    """c_k = normalised sum of the u_p labelled k; an empty cluster keeps its centre."""
    out = np.array(centres, np.float64, copy=True)
    for k in range(out.shape[0]):
        m = labels == k
        if m.any():
            s = u[m].sum(0)
            out[k] = s / max(np.sqrt((s * s).sum()), 1e-12)
    return out


def lloyd(u, init_idx, iters=LLOYD_MAX):
    """Spherical Lloyd from the centres u[init_idx]: (labels, centres, iterations, counts), stopping after the first
    iteration that changes no label."""
    c = u[list(init_idx)].copy()
    prev = None
    for t in range(1, iters + 1):
        lab, _ = assign(u, c)
        if prev is not None and np.array_equal(lab, prev):
            return lab, c, t, np.bincount(lab, minlength=c.shape[0])
        c = update(u, lab, c)
        prev = lab
    return lab, c, iters, np.bincount(lab, minlength=c.shape[0])


def style_clusters(feat, K, level):
    """feat [Hs, Ws, C] -> (labels [Hs, Ws], centres [K, C], init indices, iterations, counts) in float64."""
    Hs, Ws, C = feat.shape
    u = unit(np.asarray(feat).reshape(-1, C))
    idx = kmeanspp(u, K, level)
    lab, c, it, cnt = lloyd(u, idx)
    return lab.reshape(Hs, Ws).astype(np.uint8), c, idx, it, cnt


def data_term(feat, centres, counts):
    """D [..., K] = 1 - u . c_k in float64; +inf for a cluster of fewer than 2 style pixels."""
    D = 1.0 - unit(feat) @ np.asarray(centres, np.float64).T
    D[..., np.asarray(counts) < 2] = np.inf
    return D


def _neighbour_labels(lab):
    """Labels of the 4 neighbours of every pixel of lab [N, H, W], 255 outside the image."""
    pad = np.pad(lab.astype(np.int64), ((0, 0), (1, 1), (1, 1)), constant_values=255)
    return [pad[:, :-2, 1:-1], pad[:, 2:, 1:-1], pad[:, 1:-1, :-2], pad[:, 1:-1, 2:]]


def icm(D, lam, sweeps=SWEEPS, history=None):
    """Red-black ICM on D float32 [N, H, W, K] in explicitly rounded float32 (one product, one sum per cost): labels uint8
    [N, H, W].  ``history`` (a list) receives the labels after the start and after every half-sweep."""
    D = np.asarray(D, np.float32)
    N, H, W, K = D.shape
    lam = np.float32(lam)
    lab = np.argmin(D, axis=-1).astype(np.uint8)
    if history is not None:
        history.append(lab.copy())
    yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    inside = (yy > 0).astype(np.int64) + (yy < H - 1) + (xx > 0) + (xx < W - 1)
    for _ in range(sweeps):
        for parity in (0, 1):
            nbs = _neighbour_labels(lab)
            cost = np.empty(D.shape, np.float32)
            for k in range(K):
                same = sum((nb == k).astype(np.int64) for nb in nbs)
                n = (inside[None] - same).astype(np.float32)
                cost[..., k] = D[..., k] + lam * n          # float32 product, float32 sum: no contraction
            m = cost.min(axis=-1)
            cur = np.take_along_axis(cost, lab[..., None].astype(np.int64), -1)[..., 0]
            first = np.argmax(cost == m[..., None], axis=-1).astype(np.uint8)
            new = np.where(cur == m, lab, first)
            upd = ((yy + xx) % 2 == parity)[None]
            lab = np.where(upd, new, lab).astype(np.uint8)
            if history is not None:
                history.append(lab.copy())
    return lab


def energy(D, lab, lam):
    """Potts energy in float64: sum of D at the labels + lam x the disagreeing 4-neighbour pairs."""
    D = np.asarray(D, np.float64)
    e = np.take_along_axis(D, lab[..., None].astype(np.int64), -1).sum()
    pairs = (lab[:, 1:, :] != lab[:, :-1, :]).sum() + (lab[:, :, 1:] != lab[:, :, :-1]).sum()
    return e + float(np.float32(lam)) * pairs


def content_labels(feat, centres, counts, lam, sweeps=SWEEPS):
    """feat [N, H, W, C] -> labels [N, H, W]: the float64 data term rounded to float32, then ``icm``."""
    return icm(data_term(feat, centres, counts).astype(np.float32), lam, sweeps)


def pipeline_mst(content_u8, style_u8, weights, relu_targets, K, lam=0.05, alpha=1.0, semantics="tf", dtype=np.float32,
                 teacher=None):
    """The MST pipeline on oracle.nets: per level, cluster the style feature (``style_clusters``, seeded by level index
    RELU_LEVEL - 1), label the content (``content_labels``) and apply ``wct_style_masks`` with the K clusters as the regions
    of one style.  ``teacher`` (optional): per level a (style labels [Hs, Ws], content labels [H, W]) pair used instead."""
    relu_targets = list(relu_targets)
    x = nets.preprocess(content_u8).astype(dtype)
    sfeats = nets.encode(nets.preprocess(style_u8).astype(dtype), weights, relu_targets, dtype)
    for i, relu in enumerate(relu_targets):
        if i > 0:
            x = np.clip(x, 0, 1)
        cf = nets.encode(x, weights, [relu], dtype)[relu]
        sf = sfeats[relu]
        if teacher is not None:
            slab, clab = teacher[i]
        else:
            slab, c, _, _, cnt = style_clusters(sf[0], K, int(relu[4]) - 1)
            clab = content_labels(cf, c, cnt, lam)[0]
        f = wct_style_masks(cf, [sf] * K, clab, [slab] * K, alpha, semantics)
        x = nets.decode(np.asarray(f, dtype=dtype), weights, relu, dtype)
    return x


__all__ = ["unit", "draw", "kmeanspp", "check_draws", "assign", "update", "lloyd", "style_clusters", "data_term", "icm",
           "energy", "content_labels", "pipeline_mst", "resize_labels"]
