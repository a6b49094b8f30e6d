"""CPU oracle of style interpolation (WCT paper, section 4): the weighted sum of the single-style outputs.

The oracle follows the paper's definition at the OUTPUT level -- sum_k w_k transform(content, style_k) with the reference's
own transforms (``oracle.ref_ops.wct_tf`` / ``wct_np`` / ``adain``) -- not the engine's blend of the style statistics.  That
the two agree (both transforms are affine in the style statistics) is what tests/test_interp_cpu.py checks.
"""
import numpy as np

from oracle import nets, ref_ops


def wct_interp(content, styles, weights, alpha, semantics="tf", return_info=False):
    """content 1xHxWxC, styles: K arrays 1xHsxWsxC, weights [K].  sum_k w_k wct_tf|wct_np(content, style_k, alpha).
    info per style: k_c, k_s, wc, ws."""
    fn = ref_ops.wct_tf if semantics == "tf" else ref_ops.wct_np
    out, infos = None, []
    for s, w in zip(styles, weights):
        f, inf = fn(content, s, alpha, return_info=True)
        f = np.asarray(f, dtype=np.asarray(content).dtype)
        out = f * w if out is None else out + f * w
        infos.append(inf)
    if return_info:
        return out, infos
    return out


def adain_interp(content, styles, weights, alpha):
    """sum_k w_k adain(content, style_k, alpha)."""
    out = None
    for s, w in zip(styles, weights):
        f = ref_ops.adain(content, s, alpha)
        out = f * w if out is None else out + f * w
    return out


def level_interp(content, styles, weights, alpha, semantics="tf", adain=False, return_info=False):
    if adain:
        out = adain_interp(content, styles, weights, alpha)
        return (out, None) if return_info else out
    return wct_interp(content, styles, weights, alpha, semantics, return_info=return_info)


def pipeline_interp(content_u8, styles_u8, weights, params, relu_targets, alpha=1.0, semantics="tf", adain=False,
                    dtype=np.float32, return_info=False):
    """``oracle.nets.pipeline`` with a style blend: at every level the interpolated transform replaces the single-style
    one (mirrors tests/regions_ref.pipeline_regions)."""
    relu_targets = list(relu_targets)
    w = np.asarray(weights, dtype=dtype)
    x = nets.preprocess(content_u8).astype(dtype)
    style_feats = [nets.encode(nets.preprocess(s).astype(dtype), params, relu_targets, dtype) for s in styles_u8]
    info = []
    for i, relu in enumerate(relu_targets):
        if i > 0:
            x = np.clip(x, 0, 1)
        cf = nets.encode(x, params, [relu], dtype)[relu]
        f, inf = level_interp(cf, [sf[relu] for sf in style_feats], w, alpha, semantics, adain, return_info=True)
        info.append(inf)
        x = nets.decode(np.asarray(f, dtype=dtype), params, relu, dtype)
    if return_info:
        return x, info
    return x
