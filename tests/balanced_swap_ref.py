"""float64 oracle of the balanced style swap (DESIGN.md §3.3.18): Sinkhorn iterations on the softmax swap's plan.

With z(a,n), tau and the allowed sets A(a) of ``softmax_swap_ref`` (every patch, or ``swap_labels_ref.allowed``'s set):

    c_n = sum_{a : n in A(a)} 1 / |A(a)|                               column targets (the tau -> inf plan's column sums)
    x(a,n) = z(a,n) + h_n,  h = 0 at the start
    row step:    M_a = max_{A(a)} x,  Z_a = sum_{A(a)} exp((x - M_a) / tau),  w(a,n) = exp((x - M_a) / tau) / Z_a
    column step: S_n = sum_{a : n in A(a)} w(a,n),  h_n += tau (log c_n - log S_n)  (c_n > 0)

T iterations are T (column step, row step) pairs after the first row step; T = 0 is the softmax swap.  Every anchor pastes
sum_n w(a,n) times the raw patch n and the overlaps are averaged, as in the softmax swap.
"""
import numpy as np
from scipy.special import logsumexp

from tests import softmax_swap_ref as SR


def targets(allowed):
    """c_n [n] from the allowed sets [ho, wo, n] (bool)."""
    a = np.asarray(allowed, bool).reshape(-1, np.shape(allowed)[-1])
    return (a / a.sum(axis=1, keepdims=True)).sum(axis=0)


def balanced_weights(scores, norms, K, temperature, iters, allowed=None):
    """(w [ho, wo, n], column sums S [n], targets c [n], potentials h [n], z) after ``iters`` Sinkhorn iterations, from
    the hard swap's scores [ho, wo, n], the anchor norms [ho, wo] and K = P*P*C; ``allowed`` as ``SR.softmax_weights``."""
    tau = float(temperature)
    _, z = SR.softmax_weights(scores, norms, K, tau, allowed)
    mask = np.ones(z.shape, bool) if allowed is None else np.asarray(allowed, bool)
    c = targets(mask)
    h = np.zeros(z.shape[2])

    def row(h):
        xm = np.where(mask, z + h, -np.inf)
        d = (xm - xm.max(axis=2, keepdims=True)) / tau
        e = np.where(mask, np.exp(d), 0.0)
        zsum = e.sum(axis=2, keepdims=True)
        return e / zsum, np.where(mask, d - np.log(zsum), -np.inf)

    w, logw = row(h)
    live = c > 0
    for _ in range(int(iters)):
        log_s = logsumexp(logw.reshape(-1, z.shape[2]), axis=0)
        h = np.where(live, h + tau * (np.log(np.where(live, c, 1.0)) - log_s), h)
        w, logw = row(h)
    return w, w.reshape(-1, z.shape[2]).sum(axis=0), c, h, z


def paste(w, ws_feat, hc, wc, p, s):
    """Every anchor pastes sum_n w(a,n) times the raw patch n of ws_feat [Hs,Ws,C]; the overlaps are averaged."""
    st = np.asarray(ws_feat, np.float64)
    st = st[0] if st.ndim == 4 else st
    P = SR._patches(st, p, s)
    ho, wo = w.shape[:2]
    out = np.zeros((hc, wc, st.shape[2]), np.float64)
    cnt = np.zeros((hc, wc), np.float64)
    blend = np.tensordot(w, P, axes=([2], [0]))                  # [ho, wo, p, p, C]
    for y in range(ho):
        for x in range(wo):
            out[y * s:y * s + p, x * s:x * s + p] += blend[y, x]
            cnt[y * s:y * s + p, x * s:x * s + p] += 1
    return out / cnt[..., None]


def style_swap_balanced(wc_feat, ws_feat, p, s, temperature, iters, allowed=None):
    """The balanced swap of whitened features: content wc_feat [Hc,Wc,C] (or 1xHcxWcxC), style ws_feat [Hs,Ws,C].
    Returns (swapped feature [Hc,Wc,C], info: w, col_sums, c, h, z)."""
    from oracle import ref_ops
    c = np.asarray(wc_feat, np.float64)
    st = np.asarray(ws_feat, np.float64)
    c = c[0] if c.ndim == 4 else c
    st = st[0] if st.ndim == 4 else st
    _, inf = ref_ops.style_swap(c[None], st[None], p, s, return_info=True)
    norms = SR.anchor_norms(c, p, s)
    w, col, tgt, h, z = balanced_weights(inf["scores"], norms, p * p * c.shape[2], temperature, iters, allowed)
    out = paste(w, st, c.shape[0], c.shape[1], p, s)
    return out, dict(w=w, col_sums=col, c=tgt, h=h, z=z, scores=inf["scores"], norms=norms)


def wct_style_swap_balanced(content, style, alpha, temperature, iters, patch_size=3, stride=1, allowed=None):
    """``softmax_swap_ref.wct_style_swap_softmax`` with the balanced swap: whiten, swap, colour with the style, blend."""
    from oracle import ref_ops
    _, winf = ref_ops.wct_style_swap(content, style, alpha, patch_size, stride, return_info=True)
    swapped, _ = style_swap_balanced(winf["wc_feat"], winf["ws_feat"], patch_size, stride, temperature, iters, allowed)
    fcx, shape = ref_ops._flat(np.asarray(content, np.float64))
    fsx, _ = ref_ops._flat(np.asarray(style, np.float64))
    ms = fsx.mean(axis=1, keepdims=True)
    fs = fsx - ms
    fsfs = fs @ fs.T / (fsx.shape[1] - 1) + np.eye(fsx.shape[0]) * 1e-8
    Es, ws, _ = np.linalg.svd(fsfs)
    k_s = int((ws > ref_ops.THRESH).sum())
    ss, _ = ref_ops._flat(swapped[None])
    fcs_hat = (Es[:, :k_s] * np.sqrt(ws[:k_s])) @ Es[:, :k_s].T @ ss + ms
    return ref_ops._unflat(alpha * fcs_hat + (1 - alpha) * fcx, shape)
