"""float64 oracle of the softmax style swap (DESIGN.md §3.3.17): ``ref_ops.style_swap`` with each anchor's arg-max replaced
by a softmax over the patches.

With s(a,n) the scores of ``ref_ops.style_swap`` (filters normalised per tap across patches), ||c_a|| the l2 norm of the
whitened content over the anchor's window, K = P*P*C and n_p the number of patches:

    z(a,n) = s(a,n) / (||c_a|| sqrt(K / n_p))           (0 where ||c_a|| = 0)
    w(a,n) = exp((z(a,n) - M_a) / tau) / sum_{m in A(a)} exp((z(a,m) - M_a) / tau)   on A(a), 0 elsewhere

with M_a the maximum of z over A(a): every patch, or ``swap_labels_ref.allowed``'s set.  Every anchor pastes
sum_n w(a,n) times the raw patch n and the overlaps are averaged; ``wct_style_swap_softmax`` whitens, swaps, colours and
blends as ``ref_ops.wct_style_swap`` does.
"""
import numpy as np

from oracle import ref_ops


def _patches(f, p, s):
    """[n_patches, p, p, C] VALID patches of f [H,W,C] every s pixels, rows then columns."""
    h, w = f.shape[:2]
    rows, cols = (h - p) // s + 1, (w - p) // s + 1
    return np.stack([f[r * s:r * s + p, q * s:q * s + p, :] for r in range(rows) for q in range(cols)])


def anchor_norms(wc_feat, p, s):
    """||c_a|| [ho, wo]: the l2 norm of the whitened content f [H,W,C] over each anchor's p x p window."""
    f = np.asarray(wc_feat, np.float64)
    ho, wo = (f.shape[0] - p) // s + 1, (f.shape[1] - p) // s + 1
    return np.sqrt((_patches(f, p, s) ** 2).sum(axis=(1, 2, 3))).reshape(ho, wo)


def softmax_weights(scores, norms, K, temperature, allowed=None):
    """w [ho, wo, n] from the hard swap's scores [ho, wo, n], the anchor norms [ho, wo] and K = P*P*C; ``allowed``
    [ho, wo, n] bool or None (every patch)."""
    scores = np.asarray(scores, np.float64)
    n = scores.shape[2]
    den = np.asarray(norms, np.float64)[..., None] * np.sqrt(K / n)
    z = np.where(den > 0, scores / np.where(den > 0, den, 1.0), 0.0)
    mask = np.ones(scores.shape, bool) if allowed is None else np.asarray(allowed, bool)
    zm = np.where(mask, z, -np.inf)
    e = np.where(mask, np.exp((zm - zm.max(axis=2, keepdims=True)) / float(temperature)), 0.0)
    return e / e.sum(axis=2, keepdims=True), z


def style_swap_softmax(wc_feat, ws_feat, p, s, temperature, allowed=None, return_info=False):
    """The softmax swap of whitened features: content wc_feat [Hc,Wc,C] (or 1xHcxWcxC), style ws_feat [Hs,Ws,C].  Returns
    the swapped feature [Hc,Wc,C] (and info: weights, z, scores, anchor norms)."""
    c = np.asarray(wc_feat, np.float64)
    st = np.asarray(ws_feat, np.float64)
    c = c[0] if c.ndim == 4 else c
    st = st[0] if st.ndim == 4 else st
    _, inf = ref_ops.style_swap(c[None], st[None], p, s, return_info=True)
    scores = inf["scores"]
    norms = anchor_norms(c, p, s)
    w, z = softmax_weights(scores, norms, p * p * c.shape[2], temperature, allowed)
    P = _patches(st, p, s)
    ho, wo = scores.shape[:2]
    out = np.zeros(c.shape, np.float64)
    cnt = np.zeros(c.shape[:2], np.float64)
    blend = np.tensordot(w, P, axes=([2], [0]))                  # [ho, wo, p, p, C]
    for y in range(ho):
        for x in range(wo):
            out[y * s:y * s + p, x * s:x * s + p] += blend[y, x]
            cnt[y * s:y * s + p, x * s:x * s + p] += 1
    out /= cnt[..., None]
    if return_info:
        return out, dict(w=w, z=z, scores=scores, norms=norms, hard_idx=inf["idx"])
    return out


def uniform_swap(ws_feat, hc, wc, p, s, allowed=None):
    """The tau -> infinity limit: every anchor pastes the mean of its allowed patches, overlaps averaged."""
    st = np.asarray(ws_feat, np.float64)
    st = st[0] if st.ndim == 4 else st
    P = _patches(st, p, s)
    ho, wo = (hc - p) // s + 1, (wc - p) // s + 1
    out = np.zeros((hc, wc, st.shape[2]), np.float64)
    cnt = np.zeros((hc, wc), np.float64)
    for y in range(ho):
        for x in range(wo):
            m = P.mean(axis=0) if allowed is None else P[np.asarray(allowed)[y, x]].mean(axis=0)
            out[y * s:y * s + p, x * s:x * s + p] += m
            cnt[y * s:y * s + p, x * s:x * s + p] += 1
    return out / cnt[..., None]


def wct_style_swap_softmax(content, style, alpha, temperature, patch_size=3, stride=1, allowed=None, eps=1e-8,
                           thresh=ref_ops.THRESH, return_info=False):
    """``ref_ops.wct_style_swap`` (content 1xHcxWcxC, style 1xHsxWsxC) with the softmax swap at ``temperature``.  info:
    ``style_swap_softmax``'s plus the whitened features and eigenvalues of ``ref_ops.wct_style_swap``."""
    _, winf = ref_ops.wct_style_swap(content, style, alpha, patch_size, stride, eps=eps, thresh=thresh, return_info=True)
    swapped, inf = style_swap_softmax(winf["wc_feat"], winf["ws_feat"], patch_size, stride, temperature, allowed,
                                      return_info=True)
    fcx, shape = ref_ops._flat(np.asarray(content, np.float64))
    fsx, _ = ref_ops._flat(np.asarray(style, np.float64))
    mc = fcx.mean(axis=1, keepdims=True)
    ms = fsx.mean(axis=1, keepdims=True)
    fs = fsx - ms
    fsfs = fs @ fs.T / (fsx.shape[1] - 1) + np.eye(fsx.shape[0]) * eps
    Es, ws, _ = np.linalg.svd(fsfs)
    k_s = int((ws > thresh).sum())
    ss, _ = ref_ops._flat(swapped[None])
    fcs_hat = (Es[:, :k_s] * np.sqrt(ws[:k_s])) @ Es[:, :k_s].T @ ss + ms
    out = ref_ops._unflat(alpha * fcs_hat + (1 - alpha) * fcx, shape)
    if return_info:
        inf.update(swapped=swapped, wc_feat=winf["wc_feat"], ws_feat=winf["ws_feat"], wc=winf["wc"], ws=winf["ws"],
                   k_c=winf["k_c"], k_s=winf["k_s"])
        return out, inf
    return out
