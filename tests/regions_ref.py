"""CPU oracle of spatial control (WCT paper, section 4): the reference transform restricted to pixel sets.

Spatial control adds no new mathematics: region r of a frame is transformed by ``oracle.ref_ops.wct_generic`` (through
wct_tf / wct_np) as if its pixels were a 1 x 1 x n_r x C feature map, against the features of style r, and scattered
back; every other pixel keeps its content feature.  The label map is sampled to each level's feature grid by the
integer proportional-nearest rule of ``resize_labels``.
"""
import numpy as np

from oracle import nets, ref_ops


def resize_labels(mask, Hf, Wf):
    """[..., Hm, Wm] -> [..., Hf, Wf]:  L[((2y+1) Hm) // (2 Hf)][((2x+1) Wm) // (2 Wf)]."""
    mask = np.asarray(mask)
    Hm, Wm = mask.shape[-2:]
    ys = ((2 * np.arange(Hf) + 1) * Hm) // (2 * Hf)
    xs = ((2 * np.arange(Wf) + 1) * Wm) // (2 * Wf)
    return mask[..., ys[:, None], xs[None, :]]


def mask_regions(gray, R):
    """8-bit grayscale mask file -> region labels: gray value v maps to region v*R // 256."""
    return ((np.asarray(gray, dtype=np.int64) * R) // 256).astype(np.uint8)


def wct_regions(content, styles, labels, alpha, semantics="tf", return_info=False):
    """content 1xHxWxC, styles: R arrays 1xHsxWsxC, labels HxW (integers).  For every region r < R with at least 2 pixels,
    wct_tf (or wct_np) of its pixels against style r; the rest of the map is returned unchanged.
    info per region: k_c (-1 when skipped), k_s, wc, ws."""
    fn = ref_ops.wct_tf if semantics == "tf" else ref_ops.wct_np
    c = np.asarray(content)
    out = c.copy()
    labels = np.asarray(labels)
    assert labels.shape == c.shape[1:3]
    infos = []
    for r, style in enumerate(styles):
        idx = labels == r
        n = int(idx.sum())
        if n < 2:
            _, inf = fn(c[:, :2, :2], style, alpha, return_info=True)    # k_s of the style all the same
            infos.append(dict(k_c=-1, k_s=inf["k_s"], wc=None, ws=inf["ws"]))
            continue
        sub = c[0][idx][None, None]                                    # 1 x 1 x n_r x C
        f, inf = fn(sub, style, alpha, return_info=True)
        out[0][idx] = f[0, 0]
        infos.append(inf)
    if return_info:
        return out, infos
    return out


def pipeline_regions(content_u8, styles_u8, mask, weights, relu_targets, alpha=1.0, semantics="tf", dtype=np.float32,
                     return_info=False):
    """``oracle.nets.pipeline`` with a label map: at every level the map is sampled to the feature grid and
    ``wct_regions`` replaces the whole-frame transform."""
    relu_targets = list(relu_targets)
    x = nets.preprocess(content_u8).astype(dtype)
    style_feats = [nets.encode(nets.preprocess(s).astype(dtype), weights, relu_targets, dtype) for s in styles_u8]
    info = []
    for i, relu in enumerate(relu_targets):
        if i > 0:
            x = np.clip(x, 0, 1)
        cf = nets.encode(x, weights, [relu], dtype)[relu]
        lab = resize_labels(mask, cf.shape[1], cf.shape[2])
        f, inf = wct_regions(cf, [sf[relu] for sf in style_feats], lab, alpha, semantics, return_info=True)
        info.append(inf)
        x = nets.decode(np.asarray(f, dtype=dtype), weights, relu, dtype)
    if return_info:
        return x, info
    return x
