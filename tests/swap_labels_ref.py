"""CPU oracle of the labelled style swap (DESIGN.md §3.3.13): ``ref_ops.wct_style_swap`` with the arg-max restricted, per
content anchor, to the style patches that carry the anchor's label.

Both label maps are sampled onto their feature grids by the rule of spatial control (``regions_ref.resize_labels``).  With
o = (P-1)//2, patch n = py*pcol + px carries the sampled style label at (py*S + o, px*S + o) and the anchor (y, x) the
sampled content label at (y*S + o, x*S + o).  An anchor takes the first maximum of its float64 scores over the patches of
its label, or over every patch when no patch carries it; the rest of the op is ``ref_ops.wct_style_swap(..., idx=)``.
"""
import numpy as np

from oracle import nets, ref_ops
from tests.regions_ref import resize_labels


def patch_labels(style_labels, hs, ws, p, s):
    """l(n) of every VALID p x p patch every s pixels of an hs x ws style feature, from a label map of any size."""
    lab = resize_labels(style_labels, hs, ws)
    o = (p - 1) // 2
    rows, cols = (hs - p) // s + 1, (ws - p) // s + 1
    return lab[o:o + (rows - 1) * s + 1:s, o:o + (cols - 1) * s + 1:s].reshape(-1)


def anchor_labels(content_labels, hc, wc, p, s):
    """The label of every VALID anchor [ho, wo] of an hc x wc content feature, from a label map of any size."""
    lab = resize_labels(content_labels, hc, wc)
    o = (p - 1) // 2
    ho, wo = (hc - p) // s + 1, (wc - p) // s + 1
    return lab[o:o + (ho - 1) * s + 1:s, o:o + (wo - 1) * s + 1:s]


def allowed(alab, plab):
    """[ho, wo, n_patches]: whether anchor (y, x) may take patch n (its own label, or any patch for an absent label)."""
    alab, plab = np.asarray(alab), np.asarray(plab)
    mask = alab[..., None] == plab[None, None, :]
    absent = ~np.isin(alab, plab)
    return mask | absent[..., None]


def masked_argmax(scores, alab, plab):
    """First maximum of ``scores`` [ho, wo, n] over each anchor's allowed patches (ties to the lower index)."""
    return np.where(allowed(alab, plab), scores, -np.inf).argmax(axis=2)


def wct_style_swap_labels(content, style, alpha, content_labels, style_labels, patch_size=3, stride=1, return_info=False):
    """content 1xHcxWcxC, style 1xHsxWsxC, label maps [Hm,Wm] / [Hm',Wm'] of any size.  info: that of
    ``ref_ops.wct_style_swap`` at the labelled indices, plus the unlabelled ``scores`` and the labels."""
    hc, wc = np.shape(content)[1:3]
    hs, ws = np.shape(style)[1:3]
    _, inf = ref_ops.wct_style_swap(content, style, alpha, patch_size, stride, return_info=True)
    alab = anchor_labels(content_labels, hc, wc, patch_size, stride)
    plab = patch_labels(style_labels, hs, ws, patch_size, stride)
    idx = masked_argmax(inf["scores"], alab, plab)
    out, info = ref_ops.wct_style_swap(content, style, alpha, patch_size, stride, return_info=True, idx=idx)
    info.update(scores=inf["scores"], free_idx=inf["idx"], anchor_labels=alab, patch_labels=plab)
    if return_info:
        return out, info
    return out


def pipeline_labels(content_u8, style_u8, weights, relu_targets, swap_targets, content_labels, style_labels, alpha=1.0,
                    ss_alpha=0.6, ss_patch_size=3, ss_stride=1, dtype=np.float32, return_info=False):
    """``tests.swap_levels_ref.pipeline_levels`` (WCT in the TF semantics at the other levels) with the labelled swap at
    every level of ``swap_targets``."""
    relu_targets = list(relu_targets)
    x = nets.preprocess(content_u8).astype(dtype)
    style_feats = nets.encode(nets.preprocess(style_u8).astype(dtype), weights, relu_targets, dtype)
    info = []
    for i, relu in enumerate(relu_targets):
        if i > 0:
            x = np.clip(x, 0, 1)
        cf = nets.encode(x, weights, [relu], dtype)[relu]
        sf = style_feats[relu]
        if relu in swap_targets:
            f, inf = wct_style_swap_labels(cf, sf, ss_alpha, content_labels, style_labels, ss_patch_size, ss_stride,
                                           return_info=True)
        else:
            f, inf = ref_ops.wct_tf(cf, sf, alpha, return_info=True)
        inf["relu"] = relu
        info.append(inf)
        x = nets.decode(np.asarray(f, dtype=dtype), weights, relu, dtype)
    if return_info:
        return x, info
    return x
