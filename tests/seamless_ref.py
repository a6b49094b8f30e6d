"""CPU oracle of seamless stylisation (DESIGN.md §3.3.9): the encoder, decoders and pipeline of oracle/nets.py with every
3x3 conv of the content path padded circularly along the wrapped axes and by reflection along the others.

``wrap`` is "" (today's reflect padding everywhere: the same values as oracle/nets.py), "x", "y" or "xy".  The style is
encoded as in oracle/nets.py, unwrapped.  The transforms are the reference's (oracle/ref_ops.py, tests/ost_ref.py): they
read interior pixels only, so padding does not touch them.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle import nets, ref_ops


def pad(x, wrap):
    """1-pixel padding of an NCHW tensor: circular along the wrapped axes, reflect along the others (x first, then y, so
    that the corners follow from the two axes)."""
    x = F.pad(x, (1, 1, 0, 0), mode="circular" if "x" in wrap else "reflect")
    return F.pad(x, (0, 0, 1, 1), mode="circular" if "y" in wrap else "reflect")


def _conv(x, w_hwio, b, padded, wrap):
    w = torch.from_numpy(np.ascontiguousarray(np.transpose(w_hwio, (3, 2, 0, 1)))).to(x.dtype)
    bb = torch.from_numpy(np.asarray(b)).to(x.dtype)
    return F.conv2d(pad(x, wrap) if padded else x, w, bb)


def encode(img_nhwc, weights, targets, dtype=np.float32, wrap=""):
    """oracle.nets.encode with the wrapped axes padded circularly."""
    targets = list(targets)
    deepest = sorted(targets)[-1]
    vgg = {l["name"]: l for l in weights["vgg"]}
    x = nets._t(img_nhwc, dtype)
    feats = {}
    pad_next = False
    for typ, name in nets.VGG_MODULES:
        if typ == "pad":
            pad_next = True
        elif typ == "conv":
            l = vgg[name]
            x = _conv(x, np.transpose(np.asarray(l["weight"]), (2, 3, 1, 0)), l["bias"], pad_next, wrap)
            pad_next = False
        elif typ == "relu":
            x = torch.relu(x)
        elif typ == "pool":
            x = F.max_pool2d(x, 2, 2, ceil_mode=True)
        if name in targets:
            feats[name] = nets._n(x)
        if name == deepest:
            break
    return feats


def decode(feat_nhwc, weights, relu_target, dtype=np.float32, wrap=""):
    """oracle.nets.decode with the wrapped axes padded circularly."""
    layers = {l["name"]: l for l in weights["decoders"][relu_target]}
    x = nets._t(feat_nhwc, dtype)
    for typ, name, _filters, relu in nets.decoder_layers(relu_target):
        if typ == "conv":
            l = layers[name]
            x = _conv(x, np.asarray(l["kernel"]), l["bias"], True, wrap)
            if relu:
                x = torch.relu(x)
        else:
            x = x.repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)
    return nets._n(x)


def transform(cf, sf, alpha, adain=False, ost=False, semantics="tf"):
    """The level transform of the pipeline: AdaIN, OST (tests/ost_ref.py) or WCT."""
    if adain:
        return ref_ops.adain(cf, sf, alpha)
    if ost:
        from tests import ost_ref
        return ost_ref.ost(cf, sf, alpha, semantics=semantics)
    fn = ref_ops.wct_tf if semantics == "tf" else ref_ops.wct_np
    return fn(cf, sf, alpha)


def pipeline(content_u8, style_u8, weights, relu_targets, alpha=1.0, adain=False, ost=False, semantics="tf",
             dtype=np.float32, wrap=""):
    """oracle.nets.pipeline (model.py:60-94) with the content path padded circularly along the wrapped axes."""
    relu_targets = list(relu_targets)
    content = nets.preprocess(content_u8).astype(dtype)
    style_feats = nets.encode(nets.preprocess(style_u8).astype(dtype), weights, relu_targets, dtype)
    x = content
    for i, relu in enumerate(relu_targets):
        if i > 0:
            x = np.clip(x, 0, 1)
        cf = encode(x, weights, [relu], dtype, wrap)[relu]
        f = transform(cf, style_feats[relu], alpha, adain, ost, semantics)
        x = decode(np.asarray(f, dtype=dtype), weights, relu, dtype, wrap)
    return x
