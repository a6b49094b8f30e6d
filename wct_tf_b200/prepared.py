"""Prepared styles: the style side of the pipeline, computed once and reused across calls, passes, clips and runs.

The style side -- the VGG encode of the style image and, per relu level, the WCT state (mean ``m_s``, colouring matrix
``C_s`` and ``k_s``) and the AdaIN moments -- depends only on the style image, the encoder weights and the semantics.
A ``PreparedStyle`` holds it on the device for ``n`` styles (one shared style, or one per frame), together with the
style feature of relu5_1 when it is a target and of every level it was prepared to swap at (the style swap is prepared
from them on first use, per level, patch and stride) and the uint8 style image on the host.

``PreparedStyle.save`` / ``load_file`` write and read a ``.wctstyle`` file: an ``np.savez`` container, read with
``allow_pickle=False``.  Per level it stores a fingerprint of the encoder weights up to that relu, so a file serves any
model that shares the encoder (any decoders, any subset of the targets) and is refused by any other.
"""
from __future__ import annotations

import ctypes
import hashlib
import os

import numpy as np
import torch

from .model import RELU_CHANNELS, VGG_CONVS

FORMAT = "wctstyle"
VERSION = 1
EXT = ".wctstyle"
SEMANTIC_KEYS = ("eps_cov", "eps_eig", "thresh")


def encoder_fingerprints(vgg_layers, targets):
    """SHA-256 over the encoder weights up to each relu of ``targets``: ``preprocess``, ``conv1_1`` ... in VGG order, each
    layer as its name, its weight shape and the fp32 bytes of its weight and bias, as given in the weights dict.
    Returns {relu: hex digest}."""
    vgg = {l["name"]: l for l in vgg_layers}
    want = set(targets)
    h = hashlib.sha256()
    out = {}
    for name in ["preprocess"] + [c[0] for c in VGG_CONVS]:
        l = vgg[name]
        w = np.ascontiguousarray(np.asarray(l["weight"], dtype=np.float32))
        b = np.ascontiguousarray(np.asarray(l["bias"], dtype=np.float32))
        h.update(name.encode())
        h.update(np.asarray(w.shape, dtype=np.int64).tobytes())
        h.update(w.tobytes())
        h.update(b.tobytes())
        relu = name.replace("conv", "relu")
        if relu in want:
            out[relu] = h.hexdigest()
        if len(out) == len(want):
            break
    return out


class PreparedStyle(object):
    """The style side of ``n`` styles for one encoder and one set of semantics (see the module docstring).

    Made by ``WCT.prepare_style`` or ``WCT.load_style``; accepted wherever a style image is.  Applies only read it, so one
    prepared style may serve any number of calls, on any stream: every use waits for the events of the prepare and marks
    the buffers as in use on its stream."""

    def __init__(self, n, semantics, targets):
        self.n = int(n)
        self.semantics = dict(semantics)          # eps_cov, eps_eig, thresh
        self.targets = list(targets)              # relu targets the states cover
        self.wct = {}                             # relu -> device uint8 WCT state (wctb200_wct_style_prepare, Ns = n)
        self.adain = {}                           # relu -> device uint8 AdaIN state (wctb200_adain_style_prepare, Ns = n)
        self.feats = {}                           # relu -> engine.Act: SPF16 style feature [n,Hs,Ws,C] of a swap level
        self.events = {}                          # relu -> torch.cuda.Event recorded when that level's side is complete
        self.side = None                          # stream the side was enqueued on
        self.image = None                         # host uint8 [n,H,W,3] (prepare_style / load_style)
        self.fingerprints = {}                    # relu -> encoder fingerprint (prepare_style / load_style)
        self.swap = {}                            # (relu, patch, stride) -> (device swap state, event)
        self.entries = None                       # style-masked side (Engine._style_side): its n styles, one by one
        self.mst = {}                             # relu -> dict(labels, centres, info): MST clusters (Engine._style_side)
        self.mst_k = 0                            # K of an MST side (its n = K styles are the clusters), 0 otherwise
        self.efdm = {}                            # relu -> dict(state, H, W, slices, rot): sorted style values, and those of
                                                  # the K rotated bases of a shared sliced side (Engine._style_side)

    @property
    def feat5(self):
        """The relu5_1 style feature (``feats["relu5_1"]``), or None."""
        return self.feats.get("relu5_1")

    @feat5.setter
    def feat5(self, act):
        if act is None:
            self.feats.pop("relu5_1", None)
        else:
            self.feats["relu5_1"] = act

    def __repr__(self):
        return "PreparedStyle(n=%d, targets=%s)" % (self.n, self.targets)

    def wait(self, stream, relu=None):
        """Make ``stream`` wait for the prepare (of level ``relu``, or of every level)."""
        evs = [self.events.get(relu)] if relu is not None else list(self.events.values())
        for ev in evs:
            if ev is not None:
                stream.wait_event(ev)

    def tensors(self):
        ts = list(self.wct.values()) + list(self.adain.values()) + [st for st, _ in self.swap.values()]
        ts += [f.buf for f in self.feats.values()]
        ts += [t for m in self.mst.values() for t in m.values()]
        ts += [e["state"] for e in self.efdm.values()]
        ts += [t for e in self.efdm.values() for t in e.get("rot") or ()]
        return ts

    def record_stream(self, stream):
        """The caching allocator may recycle these buffers only once ``stream``'s work queued so far is done."""
        for t in self.tensors():
            t.record_stream(stream)

    # ------------------------------------------------------------------ file
    def save(self, path):
        """Write the prepared style to ``path`` (a ``.wctstyle`` file, see the module docstring).  Synchronous."""
        from . import _capi
        lib = _capi.load()
        if self.image is None or not self.fingerprints:
            raise ValueError("only a style made by WCT.prepare_style or WCT.load_style can be saved")
        torch.cuda.synchronize(self.wct_device())
        arrays = dict(format=np.array(FORMAT), version=np.array(VERSION, dtype=np.int64), image=np.ascontiguousarray(self.image),
                      targets=np.array(self.targets))
        for k in SEMANTIC_KEYS:
            arrays[k] = np.array(self.semantics[k], dtype=np.float64)
        for relu in self.targets:
            C = RELU_CHANNELS[relu]
            mean, cs, k = unpack_wct_state(lib, self.wct[relu], C, self.n)
            am, av = unpack_adain_state(lib, self.adain[relu], C, self.n)
            arrays.update({"%s/fingerprint" % relu: np.array(self.fingerprints[relu]), "%s/wct_mean" % relu: mean,
                           "%s/wct_cs" % relu: cs, "%s/wct_k" % relu: k, "%s/adain_mean" % relu: am, "%s/adain_var" % relu: av})
        for relu, f in self.feats.items():
            raw = f.buf[: 2 * f.N * (f.H + 2) * (f.W + 2) * f.C * 2].cpu().numpy()
            arrays["%s/feat" % relu] = raw.view(np.float16).reshape(2, f.N, f.H + 2, f.W + 2, f.C)
        if not str(path).endswith(EXT):
            raise ValueError("a prepared style file must end in %s: %r" % (EXT, path))
        tmp = str(path) + ".tmp.npz"
        np.savez(tmp, **arrays)
        os.replace(tmp, path)

    def wct_device(self):
        for t in self.tensors():
            return t.device
        return torch.device("cuda")


def read_file(path):
    """The arrays of a ``.wctstyle`` file as a dict, after the format and version checks."""
    with np.load(path, allow_pickle=False) as z:
        data = {k: z[k] for k in z.files}
    if "format" not in data or str(data["format"]) != FORMAT:
        raise ValueError("%s: format: not a %s file" % (path, FORMAT))
    if "version" not in data or int(data["version"]) != VERSION:
        raise ValueError("%s: version: unknown version %s (this build reads %d)" % (path, data.get("version"), VERSION))
    return data


def check_file(data, path, semantics, targets, fingerprints):
    """ValueError naming the field when the file does not serve a model with these semantics, targets and fingerprints."""
    for k in SEMANTIC_KEYS:
        if k not in data or float(data[k]) != float(semantics[k]):
            raise ValueError("%s: %s: the file was prepared with %s = %s, this model uses %s"
                             % (path, k, k, data.get(k), semantics[k]))
    have = [str(t) for t in data["targets"]]
    for relu in targets:
        if relu not in have:
            raise ValueError("%s: targets: %s is not prepared in the file (it has %s)" % (path, relu, ", ".join(have)))
        key = "%s/fingerprint" % relu
        if str(data[key]) != fingerprints[relu]:
            raise ValueError("%s: %s: the encoder weights up to %s differ from this model's" % (path, key, relu))


# ---------------------------------------------------------------------------------------------------------- state packing
def _layout_wct(lib, C, n):
    a, b, c = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_size_t()
    total = lib.wctb200_wct_style_state_layout(C, n, ctypes.byref(a), ctypes.byref(b), ctypes.byref(c))
    return total, a.value, b.value, c.value


def _layout_adain(lib, C, n):
    a, b = ctypes.c_size_t(), ctypes.c_size_t()
    total = lib.wctb200_adain_style_state_layout(C, n, ctypes.byref(a), ctypes.byref(b))
    return total, a.value, b.value


def unpack_wct_state(lib, state, C, n):
    """Device WCT state -> host (mean_s fp32 [n,C], C_s fp32 [n,C,C], int32 [n,2] = (k_s, sweeps))."""
    _, om, oc, ok = _layout_wct(lib, C, n)
    h = state.cpu().numpy()
    mean = h[om:om + n * C * 4].view(np.float32).reshape(n, C).copy()
    cs = h[oc:oc + n * C * C * 4].view(np.float32).reshape(n, C, C).copy()
    k = h[ok:ok + 2 * n * 4].view(np.int32).reshape(2, n).T.copy()
    return mean, cs, k


def pack_wct_state(lib, mean, cs, k, device):
    n, C = mean.shape
    total, om, oc, ok = _layout_wct(lib, C, n)
    h = np.zeros(total, dtype=np.uint8)
    h[om:om + n * C * 4] = np.ascontiguousarray(mean, np.float32).view(np.uint8).ravel()
    h[oc:oc + n * C * C * 4] = np.ascontiguousarray(cs, np.float32).view(np.uint8).ravel()
    h[ok:ok + 2 * n * 4] = np.ascontiguousarray(np.asarray(k, np.int32).T).view(np.uint8).ravel()
    return torch.from_numpy(h).to(device)


def unpack_adain_state(lib, state, C, n):
    _, om, ov = _layout_adain(lib, C, n)
    h = state.cpu().numpy()
    return h[om:om + n * C * 4].view(np.float32).reshape(n, C).copy(), h[ov:ov + n * C * 4].view(np.float32).reshape(n, C).copy()


def pack_adain_state(lib, mean, var, device):
    n, C = mean.shape
    total, om, ov = _layout_adain(lib, C, n)
    h = np.zeros(total, dtype=np.uint8)
    h[om:om + n * C * 4] = np.ascontiguousarray(mean, np.float32).view(np.uint8).ravel()
    h[ov:ov + n * C * 4] = np.ascontiguousarray(var, np.float32).view(np.uint8).ravel()
    return torch.from_numpy(h).to(device)


def slice_wct_state(lib, state, C, n, lo, hi):
    """Styles lo..hi-1 of a WCT state of n styles as a state of hi - lo styles (device copies, exact)."""
    m = hi - lo
    _, om, oc, ok = _layout_wct(lib, C, n)
    total2, om2, oc2, ok2 = _layout_wct(lib, C, m)
    out = torch.zeros(total2, dtype=torch.uint8, device=state.device)
    out[om2:om2 + m * C * 4] = state[om + lo * C * 4:om + hi * C * 4]
    out[oc2:oc2 + m * C * C * 4] = state[oc + lo * C * C * 4:oc + hi * C * C * 4]
    out[ok2:ok2 + m * 4] = state[ok + lo * 4:ok + hi * 4]
    out[ok2 + m * 4:ok2 + 2 * m * 4] = state[ok + (n + lo) * 4:ok + (n + hi) * 4]
    return out


def slice_adain_state(lib, state, C, n, lo, hi):
    m = hi - lo
    _, om, ov = _layout_adain(lib, C, n)
    total2, om2, ov2 = _layout_adain(lib, C, m)
    out = torch.zeros(total2, dtype=torch.uint8, device=state.device)
    out[om2:om2 + m * C * 4] = state[om + lo * C * 4:om + hi * C * 4]
    out[ov2:ov2 + m * C * 4] = state[ov + lo * C * 4:ov + hi * C * 4]
    return out


def slice_act_planes(buf, n, H, W, C, lo, hi, out):
    """Frames lo..hi-1 of an SPF16 buffer of n frames (both planes, halo included) into ``out`` (uint8, of hi - lo frames)."""
    fb = (H + 2) * (W + 2) * C * 2
    m = hi - lo
    out[:m * fb] = buf[lo * fb:hi * fb]
    out[m * fb:2 * m * fb] = buf[(n + lo) * fb:(n + hi) * fb]
    return out
