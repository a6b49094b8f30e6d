"""CPU oracle of style masks (spatial control with a label map on the style side too).

Region r of a frame is transformed as in ``tests.regions_ref.wct_regions``, but against the pixels of style r labelled r
only, taken as a 1 x 1 x m x C feature map (mean and covariance do not depend on where the pixels sit).  A style entry
without a mask (None) is the whole style.  A style region with fewer than 2 pixels at a level leaves region r of the
content as it is, as a content region of fewer than 2 pixels does.  The style mask is sampled to each level's style
feature grid by the rule of ``resize_labels``.
"""
import numpy as np

from oracle import nets
from tests.regions_ref import resize_labels, wct_regions


def restrict_style(style, style_labels, r):
    """style 1xHsxWsxC, labels HsxWs (or None) -> the pixels labelled r as a 1x1xmxC map, the style itself for None, and
    None when fewer than 2 pixels are labelled r."""
    if style_labels is None:
        return style
    idx = np.asarray(style_labels) == r
    if int(idx.sum()) < 2:
        return None
    return np.asarray(style)[0][idx][None, None]


def wct_style_masks(content, styles, labels, style_labels, alpha, semantics="tf", return_info=False):
    """content 1xHxWxC, styles: R arrays 1xHsxWsxC, labels HxW, style_labels: R entries, None or the HsxWs labels of style
    r.  ``wct_regions`` with style r restricted to its pixels labelled r; an empty style region keeps region r of the
    content (info k_c = k_s = -1)."""
    labels = np.asarray(labels)
    subs = [restrict_style(s, sl, r) for r, (s, sl) in enumerate(zip(styles, style_labels))]
    empty = [r for r, s in enumerate(subs) if s is None]
    keep = labels.copy()
    for r in empty:
        keep[labels == r] = 255                                     # no region: the content stays
    out, infos = wct_regions(content, [styles[r] if s is None else s for r, s in enumerate(subs)], keep, alpha, semantics,
                             return_info=True)
    for r in empty:
        infos[r] = dict(k_c=-1, k_s=-1, wc=None, ws=None)
    if return_info:
        return out, infos
    return out


def pipeline_style_masks(content_u8, styles_u8, mask, style_masks, weights, relu_targets, alpha=1.0, semantics="tf",
                         dtype=np.float32, return_info=False):
    """``tests.regions_ref.pipeline_regions`` with style masks: at every level the content mask is sampled to the content
    feature grid, each style mask to its style's feature grid, and ``wct_style_masks`` replaces ``wct_regions``."""
    relu_targets = list(relu_targets)
    x = nets.preprocess(content_u8).astype(dtype)
    style_feats = [nets.encode(nets.preprocess(s).astype(dtype), weights, relu_targets, dtype) for s in styles_u8]
    info = []
    for i, relu in enumerate(relu_targets):
        if i > 0:
            x = np.clip(x, 0, 1)
        cf = nets.encode(x, weights, [relu], dtype)[relu]
        lab = resize_labels(mask, cf.shape[1], cf.shape[2])
        sfs = [sf[relu] for sf in style_feats]
        slabs = [None if m is None else resize_labels(m, sf.shape[1], sf.shape[2]) for m, sf in zip(style_masks, sfs)]
        f, inf = wct_style_masks(cf, sfs, lab, slabs, alpha, semantics, return_info=True)
        info.append(inf)
        x = nets.decode(np.asarray(f, dtype=dtype), weights, relu, dtype)
    if return_info:
        return x, info
    return x
