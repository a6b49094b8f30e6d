"""CPU oracle of exact feature distribution matching (EFDM, DESIGN.md §3.3.12).

Per frame n and channel c, with content values x_p (p < Nc = H*W) and the sorted style values Q_0 <= ... <= Q_{Ms-1}:

    u(r) = clamp((2r+1) Ms / (2 Nc) - 1/2, 0, Ms-1),   q(r) = Q linearly interpolated at u(r)   (q(r) = Q_r when Ms = Nc)
    every run [r0, r1) of equal content values in sorted order takes t = mean_{r in [r0, r1)} q(r)
    out_p = alpha t + (1 - alpha) x_p

The run mean is the tie-respecting assignment closest in L2 to the exact one: the output does not depend on spatial order,
and the style's mean is kept exactly when Ms = Nc.  Everything here is float64.
"""
import numpy as np

from oracle import nets


def rank_quantiles(Q, Nc):
    """q(r), r < Nc, of the sorted style values Q (float64)."""
    Q = np.asarray(Q, dtype=np.float64)
    Ms = Q.shape[0]
    r = np.arange(Nc, dtype=np.float64)
    u = np.clip(((2.0 * r + 1.0) * Ms) / (2.0 * Nc) - 0.5, 0.0, Ms - 1)
    i0 = u.astype(np.int64)
    i1 = np.minimum(i0 + 1, Ms - 1)
    f = u - i0
    return Q[i0] + f * (Q[i1] - Q[i0])


def efdm_channel(x, style_values, alpha=1.0):
    """EFDM of one channel: x [Nc] content values, style_values [Ms] (any order)."""
    x = np.asarray(x, dtype=np.float64)
    q = rank_quantiles(np.sort(np.asarray(style_values, dtype=np.float64)), x.shape[0])
    _, inv, counts = np.unique(x, return_inverse=True, return_counts=True)
    r1 = np.cumsum(counts)
    P = np.concatenate([[0.0], np.cumsum(q)])
    t = (P[r1] - P[r1 - counts]) / counts
    return alpha * t[inv.reshape(-1)] + (1.0 - alpha) * x


def efdm(content, style, alpha=1.0):
    """content [N,H,W,C], style [Ns,Hs,Ws,C] with Ns in {1, N}: frame n takes style n (or style 0)."""
    content = np.asarray(content, dtype=np.float64)
    style = np.asarray(style, dtype=np.float64)
    N, H, W, C = content.shape
    Ns = style.shape[0]
    assert Ns in (1, N) and style.shape[3] == C
    out = np.empty_like(content)
    for n in range(N):
        s = style[0 if Ns == 1 else n].reshape(-1, C)
        x = content[n].reshape(-1, C)
        o = out[n].reshape(-1, C)
        for c in range(C):
            o[:, c] = efdm_channel(x[:, c], s[:, c], alpha)
    return out


def floor_w1(content, style):
    """Per-channel 1-D Wasserstein-1 distance between the oracle's EFDM output (alpha = 1) and the style, [N, C]: what is
    left by ties and by interpolating Ms style quantiles at Nc ranks."""
    return w1(efdm(content, style, 1.0), style)


def w1(a, style):
    """Per-channel 1-D Wasserstein-1 distance between the values of a [N,H,W,C] and of style [1|N,Hs,Ws,C], [N, C]: the mean
    absolute difference of the two quantile functions, taken exactly over the union of their breakpoints."""
    a = np.asarray(a, dtype=np.float64)
    style = np.asarray(style, dtype=np.float64)
    N, C = a.shape[0], a.shape[3]
    out = np.empty((N, C))
    for n in range(N):
        A = np.sort(a[n].reshape(-1, C), axis=0)
        B = np.sort(style[0 if style.shape[0] == 1 else n].reshape(-1, C), axis=0)
        na, nb = A.shape[0], B.shape[0]
        cuts = np.union1d(np.arange(na + 1) / na, np.arange(nb + 1) / nb)
        mid = 0.5 * (cuts[1:] + cuts[:-1])
        ia = np.minimum((mid * na).astype(np.int64), na - 1)
        ib = np.minimum((mid * nb).astype(np.int64), nb - 1)
        out[n] = (np.abs(A[ia] - B[ib]) * np.diff(cuts)[:, None]).sum(axis=0)
    return out


def pipeline_efdm(content_u8, style_u8, weights, relu_targets, alpha=1.0, dtype=np.float32):
    """``oracle.nets.pipeline`` with EFDM in place of WCT at every level; the encoder and decoders run in ``dtype``."""
    relu_targets = list(relu_targets)
    x = nets.preprocess(content_u8).astype(dtype)
    style_feats = nets.encode(nets.preprocess(style_u8).astype(dtype), weights, relu_targets, dtype)
    for i, relu in enumerate(relu_targets):
        if i > 0:
            x = np.clip(x, 0, 1)
        cf = nets.encode(x, weights, [relu], dtype)[relu]
        f = efdm(cf, style_feats[relu], alpha)
        x = nets.decode(np.asarray(f, dtype=dtype), weights, relu, dtype)
    return x
