"""NumPy restatement of the reference feature transforms (TEST INFRASTRUCTURE).

Follows /root/reference/ops.py:
  wct_np   ops.py:92-140   (the named oracle; pinned by tests/golden/wct_np_*.npz)
  wct_tf   ops.py:24-90    (what the reference graph really executes; pinned by tests/golden/pipeline_*.npz:
                            the reference's own wct_tf source evaluated over the NumPy TF stand-in np_tf1.py)
  adain    ops.py:282-294  (pinned the same way, pipeline_adain4_a07.npz)
  wct_style_swap / style_swap  ops.py:145-278  (pinned the same way, pipeline_swap5_*.npz)

All functions take features shaped 1xHxWxC (or HxWxC) like the reference and
are dtype-polymorphic: float64 inputs give an fp64 "truth" run of the same
arithmetic, float32 inputs mimic the reference numerics.
"""
from __future__ import annotations

import numpy as np

THRESH = 1e-5  # ops.py:68-69 / ops.py:112,125  -- hard-coded singular value cut


def _flat(x):
    """1xHxWxC (or HxWxC) -> C x HW, as ops.py:98-103 / ops.py:32-40."""
    x = np.asarray(x)
    if x.ndim == 4:
        assert x.shape[0] == 1, "WCT assumes batch 1 (ops.py:32 tf.squeeze)"
        x = x[0]
    h, w, c = x.shape
    return np.ascontiguousarray(x.reshape(h * w, c).T), (h, w, c)


def _unflat(flat, shape):
    h, w, c = shape
    return flat.T.reshape(1, h, w, c)


def wct_generic(content, style, alpha, *, eps_cov, eps_eig, thresh=THRESH,
                readd_content_mean, out_dtype=None, return_info=False):
    """Single parametrised statement of both reference variants.

    eps_cov            added to the covariance diagonal before the SVD (ops.py:45,50; wct_tf: 1e-8, wct_np: none)
    eps_eig            added to the kept singular values (ops.py:114,127; wct_np: 1e-5, wct_tf: none)
    thresh             keep singular values > thresh (ops.py:68-69,112,125)
    readd_content_mean blend with fc+mc (ops.py:83, wct_tf) or with fc only (ops.py:133, wct_np)
    """
    fcx, shape = _flat(content)
    fsx, _ = _flat(style)
    dt = fcx.dtype
    n_c = fcx.shape[1]
    n_s = fsx.shape[1]

    mc = fcx.mean(axis=1, keepdims=True)
    fc = fcx - mc
    fcfc = fc @ fc.T / dt.type(n_c - 1)
    if eps_cov:
        fcfc = fcfc + np.eye(fcfc.shape[0], dtype=dt) * dt.type(eps_cov)
    Ec, wc, _ = np.linalg.svd(fcfc)
    k_c = int((wc > thresh).sum())
    dc = (wc[:k_c] + dt.type(eps_eig)) ** dt.type(-0.5)
    fc_hat = (Ec[:, :k_c] * dc) @ Ec[:, :k_c].T @ fc

    ms = fsx.mean(axis=1, keepdims=True)
    fs = fsx - ms
    fsfs = fs @ fs.T / dt.type(n_s - 1)
    if eps_cov:
        fsfs = fsfs + np.eye(fsfs.shape[0], dtype=dt) * dt.type(eps_cov)
    Es, ws, _ = np.linalg.svd(fsfs)
    k_s = int((ws > thresh).sum())
    ds = np.sqrt(ws[:k_s] + dt.type(eps_eig))
    fcs_hat = (Es[:, :k_s] * ds) @ Es[:, :k_s].T @ fc_hat
    fcs_hat = fcs_hat + ms

    base = fc + mc if readd_content_mean else fc
    blended = dt.type(alpha) * fcs_hat + dt.type(1 - alpha) * base
    out = _unflat(blended, shape)
    if out_dtype is not None:
        out = out.astype(out_dtype)
    if return_info:
        return out, dict(k_c=k_c, k_s=k_s, wc=wc, ws=ws)
    return out


def wct_np(content, style, alpha=0.6, eps=1e-5, return_info=False):
    """ops.py:92-140.  No covariance regulariser, +eps on kept eigenvalues,
    blend with the CENTRED content (ops.py:133), result cast to float32 (ops.py:140)."""
    return wct_generic(content, style, alpha, eps_cov=0.0, eps_eig=eps,
                       readd_content_mean=False, out_dtype=np.float32,
                       return_info=return_info)


def wct_tf(content, style, alpha, eps=1e-8, return_info=False):
    """ops.py:24-90.  +eps*I on the covariance (ops.py:45,50), S^-1/2 / S^1/2
    without eigenvalue eps (ops.py:72,76), blend with fc+mc (ops.py:83)."""
    return wct_generic(content, style, alpha, eps_cov=eps, eps_eig=0.0,
                       readd_content_mean=True, return_info=return_info)


def adain(content_features, style_features, alpha, epsilon=1e-5):
    """ops.py:282-294.  tf.nn.moments over axes [1,2] (biased variance) and
    tf.nn.batch_normalization(x, mean, var, offset=style_mean,
    scale=sqrt(style_var), eps):  y = (x-mean)*rsqrt(var+eps)*scale + offset."""
    c = np.asarray(content_features)
    s = np.asarray(style_features)
    if c.ndim == 3:
        c = c[None]
    if s.ndim == 3:
        s = s[None]
    dt = c.dtype
    sm = s.mean(axis=(1, 2), keepdims=True)
    sv = s.var(axis=(1, 2), keepdims=True)
    cm = c.mean(axis=(1, 2), keepdims=True)
    cv = c.var(axis=(1, 2), keepdims=True)
    inv = (cv + dt.type(epsilon)) ** dt.type(-0.5) * np.sqrt(sv)
    norm = (c - cm) * inv + sm
    return dt.type(alpha) * norm + dt.type(1 - alpha) * c


def style_swap(content, style, patch_size=3, stride=1, return_info=False, idx=None):
    """ops.py:219-278 on 1xHxWxC arrays.  Every patch_size x patch_size patch of ``style`` (VALID, ``stride``) becomes
    a conv filter; the filters are l2-normalised along the PATCH axis (``tf.nn.l2_normalize(style_patches, dim=3)`` on a
    [p,p,C,n_patches] tensor, ops.py:233 -- i.e. per filter tap, across patches, not per patch); the content is
    cross-correlated with them (VALID), each position takes the arg-max patch (first maximum, like tf.argmax), the
    UN-normalised patch is pasted back by the transposed conv and overlaps are averaged (ops.py:255-276).

    ``idx`` (int [ho, wo]): paste these patches instead of the arg-max (the rest of the op evaluated at another
    implementation's choice); the correlation is then not computed and ``return_info`` holds only ``idx``."""
    c = np.asarray(content)
    st = np.asarray(style)
    c = c[0] if c.ndim == 4 else c
    st = st[0] if st.ndim == 4 else st
    dt = c.dtype
    hc, wc, nc = c.shape
    hs, ws, _ = st.shape
    p = int(patch_size)
    rows, cols = (hs - p) // stride + 1, (ws - p) // stride + 1
    # [n_patches, p, p, C]   (tf.extract_image_patches order: rows then cols)
    patches = np.stack([st[r * stride:r * stride + p, q * stride:q * stride + p, :] for r in range(rows) for q in range(cols)])
    norm = np.sqrt(np.maximum((patches ** 2).sum(axis=0, keepdims=True), dt.type(1e-12)))      # l2_normalize epsilon 1e-12
    pn = patches / norm
    ho, wo = (hc - p) // stride + 1, (wc - p) // stride + 1
    given = idx is not None
    if given:
        idx = np.asarray(idx)
        assert idx.shape == (ho, wo) and idx.min() >= 0 and idx.max() < len(patches), "idx must name a patch per position"
    else:
        flat = pn.reshape(len(patches), -1)
        scores = np.empty((ho, wo, len(patches)), dtype=dt)
        for y in range(ho):
            for x in range(wo):
                scores[y, x] = flat @ c[y * stride:y * stride + p, x * stride:x * stride + p, :].reshape(-1)
        idx = scores.argmax(axis=2)
    out = np.zeros((1, (ho - 1) * stride + p, (wo - 1) * stride + p, nc), dtype=dt)
    cnt = np.zeros(out.shape[1:3], dtype=dt)
    for y in range(ho):
        for x in range(wo):
            out[0, y * stride:y * stride + p, x * stride:x * stride + p, :] += patches[idx[y, x]]
            cnt[y * stride:y * stride + p, x * stride:x * stride + p] += 1
    out = out / cnt[None, :, :, None]
    if return_info and given:
        return out, dict(idx=idx)
    if return_info:
        srt = np.sort(scores, axis=2)
        return out, dict(idx=idx, margin=srt[:, :, -1] - srt[:, :, -2], scores=scores)
    return out


def wct_style_swap(content, style, alpha, patch_size=3, stride=1, eps=1e-8, thresh=THRESH, return_info=False, idx=None):
    """ops.py:145-217: whiten content AND style (S^-1/2 on the kept eigenvalues of cov + eps*I), style-swap the
    whitened encodings, colour the result with the style (S^+1/2), add the style mean, blend with fc + mc.
    ``idx``: the patch per position to paste instead of the arg-max (``style_swap``).  ``return_info`` adds the whitened
    content and style as 1xHxWxC arrays (``wc_feat``, ``ws_feat``)."""
    fcx, shape = _flat(content)
    fsx, sshape = _flat(style)
    dt = fcx.dtype
    mc = fcx.mean(axis=1, keepdims=True)
    fc = fcx - mc
    fcfc = fc @ fc.T / dt.type(fcx.shape[1] - 1) + np.eye(fcx.shape[0], dtype=dt) * dt.type(eps)
    ms = fsx.mean(axis=1, keepdims=True)
    fs = fsx - ms
    fsfs = fs @ fs.T / dt.type(fsx.shape[1] - 1) + np.eye(fsx.shape[0], dtype=dt) * dt.type(eps)
    Ec, wc, _ = np.linalg.svd(fcfc)
    Es, ws, _ = np.linalg.svd(fsfs)
    k_c, k_s = int((wc > thresh).sum()), int((ws > thresh).sum())
    fc_hat = (Ec[:, :k_c] * wc[:k_c] ** dt.type(-0.5)) @ Ec[:, :k_c].T @ fc
    fs_hat = (Es[:, :k_s] * ws[:k_s] ** dt.type(-0.5)) @ Es[:, :k_s].T @ fs
    wc_feat, ws_feat = _unflat(fc_hat, shape), _unflat(fs_hat, sshape)
    swapped, inf = style_swap(wc_feat, ws_feat, patch_size, stride, return_info=True, idx=idx)
    assert swapped.shape[1:3] == shape[:2], "style swap changed the encoding size (wct.py:84-90 refits the content for stride > 1)"
    ss, _ = _flat(swapped)
    fcs_hat = (Es[:, :k_s] * np.sqrt(ws[:k_s])) @ Es[:, :k_s].T @ ss + ms
    out = _unflat(dt.type(alpha) * fcs_hat + dt.type(1 - alpha) * (fc + mc), shape)
    if return_info:
        inf.update(k_c=k_c, k_s=k_s, wc=wc, ws=ws, wc_feat=wc_feat, ws_feat=ws_feat)
        return out, inf
    return out


def spectral_gap_ok(w, lo=1e-6, hi=1e-4):
    """SURVEY 8c: a parity vector is only well posed when no covariance
    eigenvalue sits near the hard 1e-5 cut (ops.py:112): assert none in [lo, hi]."""
    w = np.asarray(w)
    return not bool(((w >= lo) & (w <= hi)).any())


def load_reference_ops(path="/root/reference"):
    """Import the reference's own ops.py (pure-NumPy wct_np body) with
    TensorFlow / Keras stubbed out.  Only possible in the build container
    (/root/reference does not exist on the GPU box); returns None otherwise."""
    import os
    import sys
    import types
    if not os.path.isfile(os.path.join(path, "ops.py")):
        return None
    names = ["tensorflow", "keras", "keras.layers", "tensorflow.python",
             "tensorflow.python.layers", "tensorflow.python.layers.utils"]
    saved = {n: sys.modules.get(n) for n in names}
    try:
        for n in names:
            sys.modules[n] = types.ModuleType(n)
        sys.modules["keras.layers"].Conv2D = object
        sys.modules["keras.layers"].Lambda = object
        sys.modules["tensorflow.python.layers"].utils = sys.modules["tensorflow.python.layers.utils"]
        import importlib.util
        spec = importlib.util.spec_from_file_location("_wct_reference_ops", os.path.join(path, "ops.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        return mod
    finally:
        for n, m in saved.items():
            if m is None:
                sys.modules.pop(n, None)
            else:
                sys.modules[n] = m
