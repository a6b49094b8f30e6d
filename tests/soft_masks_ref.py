"""Float64 oracle of soft spatial control (DESIGN.md §3.3.11): Gaussian feathering of a label map, the exact area
resample, the reliability-weighted statistics and their Kish-normalised record, and the per-pixel blend of transforms."""
import math

import numpy as np


def feather(labels, R, sigma):
    """uint8 [N,Hm,Wm] -> float64 [N,R,Hm,Wm]: one-hot plane r blurred by a separable Gaussian, truncated at ceil(3 sigma),
    taps normalised, clamp-to-edge borders."""
    rad = int(math.ceil(3.0 * sigma))
    d = np.arange(-rad, rad + 1)
    taps = np.exp(-(d.astype(np.float64) ** 2) / (2.0 * sigma * sigma))
    taps /= taps[rad] + 2.0 * taps[rad + 1:].sum()
    N, H, W = labels.shape
    out = np.zeros((N, R, H, W))
    xi = np.clip(np.arange(W)[:, None] + d[None, :], 0, W - 1)
    yi = np.clip(np.arange(H)[:, None] + d[None, :], 0, H - 1)
    for n in range(N):
        for r in range(R):
            p = (labels[n] == r).astype(np.float64)
            rows = (p[:, xi] * taps).sum(-1)                     # [H, W]
            out[n, r] = (rows[yi, :] * taps[None, :, None]).sum(1)
    return out


def _coverage(m, f):
    """[f, m] overlap weights of the exact area average of m cells onto f cells (in units of 1 / (f m))."""
    A = np.zeros((f, m))
    for y in range(f):
        a, b = y * m, (y + 1) * m
        for i in range(a // f, -(-b // f)):
            A[y, i] = min(b, (i + 1) * f) - max(a, i * f)
    return A


def resize_area(maps, hf, wf):
    """[..., Hm, Wm] -> [..., hf, wf] by the exact area average."""
    hm, wm = maps.shape[-2:]
    Ay, Ax = _coverage(hm, hf), _coverage(wm, wf)
    return np.einsum("yi,...ij,xj->...yx", Ay, maps.astype(np.float64), Ax) / (hm * wm)


def weighted_stats(x, w):
    """x [H,W,C], w [H,W] -> (mean, cov, n_eff) with reliability weights: mean = sum w x / W,
    cov = sum w (x - m)(x - m)^T / (W - Q / W)."""
    f = x.reshape(-1, x.shape[-1]).astype(np.float64)
    v = w.reshape(-1).astype(np.float64)
    W, Q = v.sum(), (v * v).sum()
    if W <= 0:
        return None, None, 0.0
    m = (v[:, None] * f).sum(0) / W
    d = f - m
    cov = (v[:, None] * d).T @ d / (W - Q / W) if W * W > Q else None     # n_eff = 1: no covariance
    return m, cov, W * W / Q


def kish_record(x, w, t):
    """The record (n_eff, t, s', S') of DESIGN.md §3.3.11 for shift t."""
    f = x.reshape(-1, x.shape[-1]).astype(np.float64) - t
    v = w.reshape(-1).astype(np.float64)
    W, Q = v.sum(), (v * v).sum()
    n = W * W / Q
    s = (v[:, None] * f).sum(0) * n / W
    S = (v[:, None] * f).T @ f * n / W
    return n, s, S


def record_stats(n, t, s, S):
    """mean and cov of an ordinary statistics record."""
    return t + s / n, (S - np.outer(s, s) / n) / (n - 1.0)


def apply_soft(x, Ms, bs, v):
    """out(p) = sum_k v_k (M_k x_p + b_k) + (1 - sum_k v_k) x_p; x [H,W,C], Ms [K,C,C], bs [K,C], v [K,H,W]."""
    x = x.astype(np.float64)
    out = (1.0 - v.sum(0))[..., None] * x
    for k in range(len(Ms)):
        out += v[k][..., None] * (x @ Ms[k].T + bs[k])
    return out


SEMS = dict(tf=dict(eps_cov=1e-8, eps_eig=0.0, readd=True), np=dict(eps_cov=0.0, eps_eig=1e-5, readd=False))
THRESH = 1e-5


def frame_stats(x):
    """Mean and unbiased covariance of a feature map [1,H,W,C] (or [H,W,C])."""
    f = np.asarray(x, np.float64).reshape(-1, np.shape(x)[-1])
    m = f.mean(0)
    d = f - m
    return m, d.T @ d / (f.shape[0] - 1)


def transform_from_stats(mc, cov_c, ms, cov_s, alpha, semantics="tf"):
    """The affine map out = M x + b of ``oracle.ref_ops.wct_generic`` from the content and style (mean, cov), with the
    reference's own threshold (keep singular values > 1e-5 of cov + eps_cov I), eps_eig and re-add rule.  Returns
    (M, b, k_c, k_s)."""
    p = SEMS[semantics]
    C = len(mc)
    Ec, wc, _ = np.linalg.svd(cov_c + np.eye(C) * p["eps_cov"])
    k_c = int((wc > THRESH).sum())
    Wc = (Ec[:, :k_c] * (wc[:k_c] + p["eps_eig"]) ** -0.5) @ Ec[:, :k_c].T
    Es, ws, _ = np.linalg.svd(cov_s + np.eye(C) * p["eps_cov"])
    k_s = int((ws > THRESH).sum())
    Cs = (Es[:, :k_s] * np.sqrt(ws[:k_s] + p["eps_eig"])) @ Es[:, :k_s].T
    M = alpha * (Cs @ Wc) + (1.0 - alpha) * np.eye(C)
    b = alpha * ms - M @ mc + ((1.0 - alpha) * mc if p["readd"] else 0.0)
    return M, b, k_c, k_s


def wct_soft(content, styles, weights, strength, alpha, semantics="tf", return_info=False):
    """One level of soft spatial control: content [1,H,W,C], styles K arrays [1,Hs,Ws,C], weights [K,H,W] (None: K = 1,
    weight 1), strength [H,W] (None: 1).  Region k's statistics are the reliability-weighted ones of plane k; a plane of
    n_eff < 2 is skipped (weight 0); then ``apply_soft``.  info per k: k_c (-1 when skipped), k_s."""
    x = np.asarray(content, np.float64)[0]
    H, W, C = x.shape
    K = len(styles)
    w = np.ones((1, H, W)) if weights is None else np.asarray(weights, np.float64)
    s = np.ones((H, W)) if strength is None else np.asarray(strength, np.float64)
    Ms, bs, v, info = [], [], np.zeros((K, H, W)), []
    for k in range(K):
        ms, cs = frame_stats(styles[k])
        m, cov, ne = weighted_stats(x, w[k])
        if ne < 2:
            Ms.append(np.eye(C))
            bs.append(np.zeros(C))
            info.append(dict(k_c=-1))
            continue
        M, b, k_c, k_s = transform_from_stats(m, cov, ms, cs, alpha, semantics)
        Ms.append(M)
        bs.append(b)
        v[k] = s * w[k]
        wc = np.linalg.svd(cov + np.eye(C) * SEMS[semantics]["eps_cov"], compute_uv=False)
        info.append(dict(k_c=k_c, k_s=k_s, wc=wc))
    out = apply_soft(x, np.array(Ms), np.array(bs), v)[None]
    return (out, info) if return_info else out


def pipeline_soft(content_u8, styles_u8, weights_map, strength_map, nets_weights, relu_targets, alpha=1.0, semantics="tf",
                  dtype=np.float64):
    """``oracle.nets.pipeline`` with soft spatial control: at every level the weight planes [K,Hm,Wm] and the strength
    map [Hm,Wm] (either may be None) are area-averaged to the feature grid and ``wct_soft`` replaces the transform."""
    from oracle import nets
    relu_targets = list(relu_targets)
    x = nets.preprocess(content_u8).astype(dtype)
    sfe = [nets.encode(nets.preprocess(s).astype(dtype), nets_weights, relu_targets, dtype) for s in styles_u8]
    for i, relu in enumerate(relu_targets):
        if i > 0:
            x = np.clip(x, 0, 1)
        cf = nets.encode(x, nets_weights, [relu], dtype)[relu]
        h, w = cf.shape[1:3]
        wl = None if weights_map is None else resize_area(weights_map, h, w)
        sl = None if strength_map is None else resize_area(strength_map, h, w)
        f = wct_soft(cf, [sf[relu] for sf in sfe], wl, sl, alpha, semantics)
        x = nets.decode(np.asarray(f, dtype=dtype), nets_weights, relu, dtype)
    return x
