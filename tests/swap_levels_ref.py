"""Oracle of the style swap at any level: ``oracle.nets.pipeline`` with the swap at every level of ``swap_targets``.

``nets.pipeline`` swaps at relu5_1 only (``swap5``).  This is the same level loop (model.py:60-94: encode the clipped
level input, transform, decode) with ``ref_ops.wct_style_swap`` at each level of ``swap_targets`` instead of WCT / AdaIN.
Without ``swap_targets`` it is ``nets.pipeline`` itself.
"""
import numpy as np

from oracle import nets, ref_ops


def pipeline_levels(content_u8, style_u8, weights, relu_targets, alpha=1.0, adain=False, semantics="tf", dtype=np.float32,
                    return_info=False, swap5=False, ss_alpha=0.6, ss_patch_size=3, ss_stride=1, swap_targets=None):
    if swap_targets is None:
        return nets.pipeline(content_u8, style_u8, weights, relu_targets, alpha=alpha, adain=adain, semantics=semantics,
                             dtype=dtype, return_info=return_info, swap5=swap5, ss_alpha=ss_alpha, ss_patch_size=ss_patch_size,
                             ss_stride=ss_stride)
    if swap5:
        raise ValueError("give swap5 or swap_targets, not both")
    relu_targets = list(relu_targets)
    for relu in swap_targets:
        if relu not in relu_targets:
            raise ValueError("swap_targets: %s is not a relu target" % relu)
    content = nets.preprocess(content_u8).astype(dtype)
    style = nets.preprocess(style_u8).astype(dtype)
    style_feats = nets.encode(style, weights, relu_targets, dtype)
    info = []
    x = content
    for i, relu in enumerate(relu_targets):
        if i > 0:
            x = np.clip(x, 0, 1)
        cf = nets.encode(x, weights, [relu], dtype)[relu]
        sf = style_feats[relu]
        if relu in swap_targets:
            f, inf = ref_ops.wct_style_swap(cf, sf, ss_alpha, ss_patch_size, ss_stride, return_info=True)
        elif adain:
            f, inf = ref_ops.adain(cf, sf, alpha), {}
        else:
            fn = ref_ops.wct_tf if semantics == "tf" else ref_ops.wct_np
            f, inf = fn(cf, sf, alpha, return_info=True)
        inf["relu"] = relu
        info.append(inf)
        x = nets.decode(np.asarray(f, dtype=dtype), weights, relu, dtype)
    if return_info:
        return x, info
    return x
