"""Executes the multi-level WCT plan (model.py) on one GPU through libwctb200.

Host side of the hot path ``WCT.predict`` (wct.py:70-106): PyTorch is used only
for device memory, streams and H2D/D2H copies; every arithmetic step is a
hand-written sm_90a kernel behind the C-ABI (include/wctb200.h).
"""
from __future__ import annotations

import collections
import ctypes
import dataclasses

import numpy as np
import torch

from . import _capi, options, sliced
from .model import WCTModel, RELU_CHANNELS, RELU_LEVEL, check_seamless, seamless_axes
from .prepared import (PreparedStyle, SEMANTIC_KEYS, encoder_fingerprints, slice_act_planes, slice_adain_state,
                       slice_wct_state)

# wct_tf (ops.py:24-90, what the graph executes) vs wct_np (ops.py:92-140, the named oracle)
SEMANTICS = {
    "tf": dict(eps_cov=1e-8, eps_eig=0.0, thresh=1e-5, readd=1),
    "np": dict(eps_cov=0.0, eps_eig=1e-5, thresh=1e-5, readd=0),
}

# Workspace of one style-swap apply: all of its scores when they fit this size, else at least one N tile of them.  The
# apply then correlates the patches in chunks; the output is the same byte for byte (wctb200_style_swap_apply_min_workspace_
# bytes).  At 512^2 a relu5_1 swap (4.4 MB of scores per frame) runs in one chunk, a relu3_1 swap (1.08 GB) in two.
SWAP_WORKSPACE_BYTES = 1 << 30

# Multimodal style transfer (DESIGN.md §3.3.10): red-black ICM sweeps of the content labelling per level
MST_SWEEPS = 8

# Exact feature distribution matching (DESIGN.md §3.3.12): device scratch of one level's sort, in bytes.  The apply sorts
# as many whole (frame, channel) segments at a time as this holds (24 bytes a value, so 2 GB is 85 M values: the relu1_1
# level of 5 frames at 512^2, or a quarter of one 4096^2 frame); the bytes do not depend on it.
EFDM_WORKSPACE_BYTES = 2 << 30


class Act(object):
    """SPF16 activation: device buffer + logical NHWC shape."""
    __slots__ = ("buf", "N", "H", "W", "C")

    def __init__(self, buf, N, H, W, C):
        self.buf, self.N, self.H, self.W, self.C = buf, N, H, W, C

    @property
    def ptr(self):
        return self.buf.data_ptr()


def style_states(adain=False, efdm=False, efdm_slices=0):
    """The per-level style states a call applies, as keywords of ``Engine._style_side``: the WCT states (also read by OST),
    the AdaIN moments, or the EFDM states of ``efdm_slices`` slices."""
    return dict(wct=not adain and not efdm, adain=adain, efdm=efdm, efdm_slices=efdm_slices)


# the style swap of a call (DESIGN.md §3.3.5, §3.3.13, §3.3.17, §3.3.18): patch and stride, the relu levels it replaces the
# transform at, ss_alpha, the (content, style) label maps or None, the softmax temperature or None, the Sinkhorn iterations
Swap = collections.namedtuple("Swap", "patch stride levels alpha labels temperature balance")


@dataclasses.dataclass(frozen=True)
class Plan(object):
    """What one ``Engine.stylize`` call runs, decided once from its checked arguments."""
    run: list                       # the levels to run (``run_levels``)
    alpha: float
    transform: str = "wct"          # of the levels that do not swap: "wct", "ost", "adain" or "efdm"
    slices: int = 0                 # with "efdm": the K rotated bases of sliced EFDM
    swap: Swap = None
    mode: str = None                # several styles: "regions", "interp" or "mst"; None for one style side
    labels: torch.Tensor = None     # "regions": the label maps [N,Hm,Wm]
    masks: list = None              # "regions": the style masks (``check_region_masks``) or None
    weights: torch.Tensor = None    # "interp": the weight rows [1|N,K]
    mst: tuple = None               # "mst": (K, lambda)
    soft: tuple = None              # soft spatial control: (strength [N,Hm,Wm] | None, weights [N,K,Hm,Wm] | None)
    seamless: str = None

    @property
    def states(self):
        return style_states(self.transform == "adain", self.transform == "efdm", self.slices)

    def frames(self, lo, hi):
        """The plan of frames [lo, hi): the per-frame maps and rows are sliced, a shared one ([1,...]) is kept."""
        def cut(t):
            return t if t is None or t.shape[0] == 1 else t[lo:hi]
        swap = self.swap
        if swap is not None and swap.labels is not None:
            swap = swap._replace(labels=tuple(cut(t) for t in swap.labels))
        return dataclasses.replace(self, swap=swap, labels=cut(self.labels), weights=cut(self.weights),
                                   soft=None if self.soft is None else tuple(cut(m) for m in self.soft))


class Engine(object):
    def __init__(self, weights, relu_targets, device="cuda:0", semantics="tf", fuse_upsample=True, fuse_pool=True):
        if not torch.cuda.is_available():
            raise _capi.WctB200Error("no CUDA device: the WCT engine has no CPU fallback")
        self.lib = _capi.load()
        self.device = torch.device(device)
        self.model = WCTModel(mode="test", relu_targets=relu_targets)
        if semantics not in SEMANTICS:
            raise ValueError("semantics must be 'tf' or 'np'")
        self.semantics = semantics
        self.last_info = None
        self._ws = {}
        self.overlap_style = True  # run the style side (encode + per-level eigendecompositions) on a second stream
        self.groups = 1            # >1: split a batch into sub-batches that run as independent stream-pairs
        self.group_priorities = False
        self._group = 0
        self._style_streams = {}
        self._group_streams = {}
        self.fuse_pool = bool(fuse_pool)          # MaxPooling2D folded into the epilogue of the conv before it (WCTB200_POOL2)
        self.fuse_upsample = bool(fuse_upsample)  # UpSampling2D folded into the next conv (4 parity kernels, 4/9 of the MACs); fixed at construction
        self.launches = 0          # kernels launched through the C-ABI (bench.py "gpu_launches")
        self.profile = None        # optional dict: key -> [torch.cuda.Event pairs, flops, bytes]
        self._tag = None           # profiling only: "style" / relu target of the level being enqueued
        self._vgg_layers = weights["vgg"]          # encoder fingerprints of prepared styles (computed on first use)
        self._fingerprints = None
        self._sliced = {}                 # (C, K) -> device bases and step matrices of sliced EFDM
        with torch.cuda.device(self.device):
            self._upload(weights)

    # ------------------------------------------------------------------ weights
    def _dev(self, a, dtype=torch.float32):
        return torch.from_numpy(np.ascontiguousarray(a)).to(device=self.device, dtype=dtype)

    def _prep_split(self, w_hwio, up2=False):
        """fp32 (kH,kW,Cin,Cout) -> device split-fp16 GEMM operand (``up2``: the four 2x2-tap parity kernels of
        UpSampling2D -> Conv2DReflect, see csrc/conv_tc.cu)."""
        kh, kw, cin, cout = w_hwio.shape
        src = self._dev(w_hwio.astype(np.float32))
        if up2:
            dst = torch.empty(self.lib.wctb200_conv_weight_bytes(16, cin, cout), dtype=torch.uint8, device=self.device)
            _capi.check(self.lib.wctb200_prep_conv_weights_up2(src.data_ptr(), cin, cout, dst.data_ptr(), self._stream()))
            return dst
        dst = torch.empty(self.lib.wctb200_conv_weight_bytes(kh * kw, cin, cout), dtype=torch.uint8, device=self.device)
        _capi.check(self.lib.wctb200_prep_conv_weights(src.data_ptr(), kh * kw, cin, cout, dst.data_ptr(), self._stream()))
        return dst

    @staticmethod
    def _fused_up(ops, i):
        """True when ops[i] is an 'up' that the engine folds into the conv that follows it (model.py:291-293)."""
        return ops[i].kind == "up" and i + 1 < len(ops) and ops[i + 1].kind == "conv" and ops[i + 1].act

    def _upload(self, weights):
        vgg = {l["name"]: l for l in weights["vgg"]}
        # fold the 1x1 'preprocess' conv (vgg_normalised.py:25-26) into conv1_1 (exact: a per-pixel affine
        # map commutes with reflect padding); done in float64 on the host, once.
        w0 = np.asarray(vgg["preprocess"]["weight"], dtype=np.float64)[:, :, 0, 0]  # (O=j, I=i)
        b0 = np.asarray(vgg["preprocess"]["bias"], dtype=np.float64)
        w1 = np.asarray(vgg["conv1_1"]["weight"], dtype=np.float64)                 # (O, j, kH, kW)
        b1 = np.asarray(vgg["conv1_1"]["bias"], dtype=np.float64)
        wf = np.einsum("ojyx,ji->yxio", w1, w0)                                      # (kH,kW,i,O)
        bf = b1 + np.einsum("ojyx,j->o", w1, b0)
        self.head_w = self._dev(wf.reshape(27, 64).astype(np.float32))
        self.head_b = self._dev(bf.astype(np.float32))
        self.enc_w, self.enc_b = {}, {}
        deepest_ops = [op for op in self.model.style_plan if op.kind == "conv" and op.name != "conv1_1"]
        for op in deepest_ops:
            l = vgg[op.name]
            hwio = np.transpose(np.asarray(l["weight"], dtype=np.float32), (2, 3, 1, 0))  # vgg_normalised.py:33
            self.enc_w[op.name] = self._prep_split(hwio)
            self.enc_b[op.name] = self._dev(np.asarray(l["bias"], dtype=np.float32))
        self.dec_w, self.dec_b, self.tail_w, self.tail_b = {}, {}, {}, {}
        for lvl in self.model.levels:
            relu = lvl.relu_target
            if relu in self.tail_w:
                continue
            if relu not in weights["decoders"]:
                raise Exception("No checkpoint found for target {}".format(relu))  # wct.py:57-58
            layers = {l["name"]: l for l in weights["decoders"][relu]}
            ops = self.model.decoder_plan(lvl.index)
            for i, op in enumerate(ops):
                if op.kind != "conv":
                    continue
                l = layers[op.name]
                k = np.asarray(l["kernel"], dtype=np.float32)
                assert k.shape == (3, 3, op.cin, op.cout), (op.name, k.shape)
                if op.act:
                    self.dec_w[op.name] = self._prep_split(k, up2=(self.fuse_upsample and i > 0 and self._fused_up(ops, i - 1)))
                    self.dec_b[op.name] = self._dev(np.asarray(l["bias"], dtype=np.float32))
                else:
                    self.tail_w[relu] = self._dev(k.reshape(9 * op.cin, 3))
                    self.tail_b[relu] = self._dev(np.asarray(l["bias"], dtype=np.float32))
        torch.cuda.synchronize(self.device)

    # ------------------------------------------------------------------ helpers
    def _call(self, key, nkernels, fn, *args, flops=0.0, bytes_=0.0):
        """Run one C-ABI call; count its kernels; optionally bracket it with CUDA events on
        the launching stream (bench.py roofline section)."""
        self.launches += nkernels
        if self.profile is None:
            _capi.check(fn(*args))
            return
        if self._tag:
            key = "%s:%s" % (self._tag, key)      # level the call belongs to (bench.py: per-level conv rates)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _capi.check(fn(*args))
        e1.record()
        rec = self.profile.setdefault(key, dict(events=[], flops=0.0, bytes=0.0, launches=0))
        rec["events"].append((e0, e1))
        rec["flops"] += flops
        rec["bytes"] += bytes_
        rec["launches"] += nkernels

    @staticmethod
    def _matfun_launches(C):
        """kernels the matrix-function fast path adds to a WCT call (matfun_tc.cu: norm + init + 3 products x 16 iterations + guard;
        launches of converged matrices return at once but are launches all the same)"""
        return 3 + 3 * 16 if C >= 128 else 0

    def _stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def _act(self, N, H, W, C):
        nbytes = self.lib.wctb200_act_bytes(N, H, W, C)
        return Act(torch.empty(nbytes, dtype=torch.uint8, device=self.device), N, H, W, C)

    def _workspace(self, C, Nc, Ns):
        key = (self._group, C, Nc, Ns)    # concurrent groups (streams) must not share scratch
        ws = self._ws.get(key)
        if ws is None:
            ws = torch.empty(self.lib.wctb200_wct_workspace_bytes(C, Nc, Ns), dtype=torch.uint8, device=self.device)
            self._ws[key] = ws
        return ws

    # ------------------------------------------------------------------ layers
    @staticmethod
    def wrap_flags(seamless):
        """The halo flag bits of a seamless mode (None, "x", "y", "xy"; DESIGN.md §3.3.9)."""
        wx, wy = seamless_axes(seamless)
        return (_capi.HALO_WRAP_X if wx else 0) | (_capi.HALO_WRAP_Y if wy else 0)

    def halo(self, act, flags):
        """Rewrite the halo of ``act`` in place in the mode of ``flags`` (the wrap bits; wctb200_act_halo)."""
        self._call("act_halo[C%d]" % act.C, 1, self.lib.wctb200_act_halo, act.ptr, act.N, act.H, act.W, act.C, flags,
                   self._stream(), bytes_=8.0 * act.C * act.N * (2 * (act.W + 2) + 2 * act.H))

    def encode(self, img, target, taps=(), seamless=None):
        """img: float32 cuda tensor [N,H,W,3] in [0,1].  Runs the shared encoder up to
        ``target`` (vgg_normalised.py:22-50); returns (act_at_target, {tap: act}).  ``seamless`` ("x", "y", "xy"):
        every conv pads the wrapped axes circularly (DESIGN.md §3.3.9)."""
        N, H, W, _ = img.shape
        st = self._stream()
        lib = self.lib
        wrap = self.wrap_flags(seamless)
        x = self._act(N, H, W, 64)
        head = (lib.wctb200_conv_head_flags, img.data_ptr(), N, H, W, self.head_w.data_ptr(), self.head_b.data_ptr(), wrap) if wrap \
            else (lib.wctb200_conv_head, img.data_ptr(), N, H, W, self.head_w.data_ptr(), self.head_b.data_ptr())
        self._call("conv_head", 1, *head, x.ptr, st, flops=2.0 * 27 * 64 * N * H * W, bytes_=N * H * W * (12.0 + 64 * 4))
        kept = {}
        if "relu1_1" in taps:
            kept["relu1_1"] = x
        from .model import encoder_plan
        plan = encoder_plan(target)[1:]
        skip_pool = False
        for i, op in enumerate(plan):
            if op.kind == "conv":
                relu_name = op.name.replace("conv", "relu")
                # MaxPooling2D folded into the conv that feeds it (conv1_2 / 2_2 / 3_4 / 4_4: the pool is their only consumer)
                pooled = (self.fuse_pool and i + 1 < len(plan) and plan[i + 1].kind != "conv" and relu_name not in taps
                          and (x.H + 1) // 2 >= 2 and (x.W + 1) // 2 >= 2)
                y = self._act(N, (x.H + 1) // 2, (x.W + 1) // 2, op.cout) if pooled else self._act(N, x.H, x.W, op.cout)
                self._call("conv3x3_%s[%dx%d@%d]" % ("pool" if pooled else "tc", op.cin, op.cout, x.H), 1, lib.wctb200_conv3x3, x.ptr,
                           N, x.H, x.W, op.cin, self.enc_w[op.name].data_ptr(), self.enc_b[op.name].data_ptr(), op.cout,
                           _capi.RELU | (_capi.POOL2 if pooled else 0) | wrap, y.ptr, st, flops=2.0 * 9 * op.cin * op.cout * N * x.H * x.W,
                           bytes_=4.0 * N * (x.H * x.W * op.cin + y.H * y.W * op.cout))
                x = y
                skip_pool = pooled
                if relu_name in taps:
                    kept[relu_name] = x
            elif skip_pool:
                skip_pool = False
            else:
                y = self._act(N, (x.H + 1) // 2, (x.W + 1) // 2, x.C)
                self._call("maxpool2", 1, lib.wctb200_maxpool2, x.ptr, N, x.H, x.W, x.C, y.ptr, st,
                           bytes_=4.0 * N * x.C * (x.H * x.W + y.H * y.W))
                if wrap:
                    self.halo(y, wrap)
                x = y
        return x, kept

    def decode(self, feat, level_index, clip, seamless=None):
        """Run decoder ``level_index`` (model.py:279-300) -> float32 image [N,H',W',3];
        ``clip`` applies model.py:86's clip_by_value(0,1).  ``seamless``: the wrapped axes of ``encode``; ``feat``'s halo
        must already be wrapped on them."""
        st = self._stream()
        lib = self.lib
        wrap = self.wrap_flags(seamless)
        relu = self.model.levels[level_index].relu_target
        x = feat
        N = x.N
        ops = self.model.decoder_plan(level_index)
        pending_up = False                     # an UpSampling2D waiting to be folded into the next conv
        for i, op in enumerate(ops):
            if op.kind == "up":
                if self.fuse_upsample and self._fused_up(ops, i):
                    pending_up = True          # x stays low-resolution (its producer wrote an edge halo)
                    continue
                y = self._act(N, x.H * 2, x.W * 2, x.C)
                self._call("upsample2", 1, lib.wctb200_upsample2, x.ptr, N, x.H, x.W, x.C, y.ptr, st,
                           bytes_=4.0 * N * x.C * x.H * x.W * 5)
                if wrap:
                    self.halo(y, wrap)
                x = y
            elif op.act:
                # a conv whose output feeds a folded upsample writes an EDGE-replicated halo (conv_tc.cu, mode UP2)
                edge = self.fuse_upsample and i + 1 < len(ops) and self._fused_up(ops, i + 1)
                flags = _capi.RELU | (_capi.HALO_EDGE if edge else 0) | wrap
                if pending_up:
                    y = self._act(N, 2 * x.H, 2 * x.W, op.cout)
                    self._call("conv3x3_up2[%dx%d@%d]" % (op.cin, op.cout, y.H), 1, lib.wctb200_conv3x3_up2, x.ptr, N, x.H, x.W,
                               op.cin, self.dec_w[op.name].data_ptr(), self.dec_b[op.name].data_ptr(), op.cout,
                               flags, y.ptr, st, flops=2.0 * 4 * op.cin * op.cout * N * y.H * y.W,
                               bytes_=4.0 * N * (x.H * x.W * op.cin + y.H * y.W * op.cout))
                    pending_up = False
                else:
                    y = self._act(N, x.H, x.W, op.cout)
                    self._call("conv3x3_tc[%dx%d@%d]" % (op.cin, op.cout, x.H), 1, lib.wctb200_conv3x3, x.ptr, N, x.H, x.W,
                               op.cin, self.dec_w[op.name].data_ptr(), self.dec_b[op.name].data_ptr(), op.cout,
                               flags, y.ptr, st, flops=2.0 * 9 * op.cin * op.cout * N * x.H * x.W,
                               bytes_=4.0 * N * x.H * x.W * (op.cin + op.cout))
                x = y
            else:
                assert not pending_up
                img = torch.empty((N, x.H, x.W, 3), dtype=torch.float32, device=self.device)
                self._call("conv_tail", 1, lib.wctb200_conv_tail, x.ptr, N, x.H, x.W, op.cin, self.tail_w[relu].data_ptr(),
                           self.tail_b[relu].data_ptr(), _capi.CLIP01 if clip else 0, img.data_ptr(), st,
                           flops=2.0 * 9 * op.cin * 3 * N * x.H * x.W, bytes_=N * x.H * x.W * (4.0 * op.cin + 12))
                return img
        raise AssertionError("decoder plan without a tail conv")

    def transform(self, content, style, alpha, adain, want_info=False):
        """wct_tf / wct_np / adain on one level (model.py:144-158)."""
        st = self._stream()
        out = self._act(content.N, content.H, content.W, content.C)
        ws = self._workspace(content.C, content.N, style.N)
        if adain:
            self._call("adain_level[C%d]" % content.C, 8, self.lib.wctb200_adain_level, content.ptr, content.N, content.H,
                       content.W, style.ptr, style.N, style.H, style.W, content.C, float(alpha), 1e-5, out.ptr,
                       ws.data_ptr(), ws.numel(), st,
                       bytes_=4.0 * content.C * (2 * content.N * content.H * content.W + style.N * style.H * style.W))
            return out, None
        sem = SEMANTICS[self.semantics]
        kbuf = torch.empty(2 * (content.N + style.N), dtype=torch.int32, device=self.device) if want_info else None
        C = content.C
        hwc, hws = content.H * content.W, style.H * style.W
        self._call("wct_level[C%d]" % C, 14 + self._matfun_launches(C), self.lib.wctb200_wct_level, content.ptr, content.N, content.H, content.W,
                   style.ptr, style.N, style.H, style.W, C, float(alpha), sem["eps_cov"], sem["eps_eig"],
                   sem["thresh"], sem["readd"], out.ptr, kbuf.data_ptr() if want_info else None, ws.data_ptr(),
                   ws.numel(), st, flops=2.0 * C * C * (2 * content.N * hwc + style.N * hws),
                   bytes_=4.0 * C * (2 * content.N * hwc + style.N * hws))
        return out, kbuf

    def adain_prepare(self, style):
        """Style side of AdaIN on one level: the per-channel moments of the style, a state read by ``adain_apply``."""
        state = torch.empty(self.lib.wctb200_adain_style_state_bytes(style.C, style.N), dtype=torch.uint8, device=self.device)
        self._call("adain_style[C%d]" % style.C, 3, self.lib.wctb200_adain_style_prepare, style.ptr, style.N, style.H, style.W, style.C,
                   state.data_ptr(), self._stream(), bytes_=4.0 * style.C * style.N * style.H * style.W)
        return state

    def adain_apply(self, content, state, n_style, alpha):
        st = self._stream()
        out = self._act(content.N, content.H, content.W, content.C)
        ws = self._workspace(content.C, content.N, 0)
        self._call("adain_level[C%d]" % content.C, 5, self.lib.wctb200_adain_apply, content.ptr, content.N, content.H, content.W,
                   content.C, state.data_ptr(), n_style, float(alpha), 1e-5, out.ptr, ws.data_ptr(), ws.numel(), st,
                   bytes_=4.0 * content.C * 2 * content.N * content.H * content.W)
        return out, None

    def adain_apply_blend(self, content, states, weights, alpha):
        """AdaIN against the blend of K prepared styles (``adain_prepare`` states, one style each) with the weights of
        ``weights`` (cuda fp32 [1|N, K])."""
        st = self._stream()
        C, N, K, Nw = content.C, content.N, len(states), weights.shape[0]
        out = self._act(N, content.H, content.W, C)
        ws = self._workspace(C, N, 0)
        self._call("adain_blend[C%d]" % C, 5, self.lib.wctb200_adain_apply_blend, content.ptr, N, content.H, content.W, C,
                   _capi.pointer_array([s.data_ptr() for s in states]), K, weights.data_ptr(), Nw, float(alpha), 1e-5, out.ptr,
                   ws.data_ptr(), ws.numel(), st, bytes_=4.0 * C * 2 * N * content.H * content.W)
        return out, None

    def swap_prepare(self, style, patch, stride):
        """Style side of the style swap (whitened style, patch filters, colouring operand) for one style feature."""
        st = self._stream()
        C = style.C
        nbytes = self.lib.wctb200_style_swap_state_bytes(C, style.H, style.W, int(patch), int(stride))
        if nbytes == 0:
            raise ValueError("style swap needs a style encoding of at least %dx%d (style %dx%d)" % (patch, patch, style.H, style.W))
        state = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        ws = torch.empty(self.lib.wctb200_style_swap_prepare_workspace_bytes(C, style.H, style.W, int(patch), int(stride)),
                         dtype=torch.uint8, device=self.device)
        sem = SEMANTICS["tf"]                  # the reference only has the TF graph version of this op
        self._call("swap_style[C%d]" % C, 12, self.lib.wctb200_style_swap_prepare, style.ptr, style.H, style.W, C, int(patch),
                   int(stride), sem["eps_cov"], sem["thresh"], state.data_ptr(), None, ws.data_ptr(), ws.numel(), st)
        return state

    def swap_apply(self, content, state, style_hw, ss_alpha, want_info=False, patch=3, stride=1, labels=None, temperature=None,
                   balance=0):
        """wct_style_swap (ops.py:145-217) of the N content frames against one prepared style (``swap_prepare``).
        ``labels``: (content labels cuda uint8 [1|N,Hm,Wm], style labels cuda uint8 [1,Hm',Wm']) of a labelled swap
        (DESIGN.md §3.3.13), each anchor matched only to the style patches of its own label.  ``temperature``: the softmax
        swap at that temperature (DESIGN.md §3.3.17) instead of the arg-max; None is the hard swap.  ``balance`` = T > 0
        (with ``temperature``): the balanced swap (DESIGN.md §3.3.18), T Sinkhorn iterations that even out how much each
        style patch is used; 0 is the softmax swap."""
        st = self._stream()
        C, N = content.C, content.N
        Hs, Ws = style_hw
        out = self._act(N, content.H, content.W, C)
        geom = (C, N, content.H, content.W, Hs, Ws, int(patch), int(stride))
        soft = temperature is not None
        balance = int(balance)
        if balance and not soft:
            raise ValueError("the balanced swap needs a temperature")
        lib = self.lib
        kind = "balanced" if balance else "softmax" if soft else None
        nbytes = (getattr(lib, "wctb200_style_swap_%s_workspace_bytes" % kind) if kind
                  else lib.wctb200_style_swap_apply_workspace_bytes)(*geom)
        if nbytes == 0:
            raise ValueError("style swap needs encodings of at least %dx%d (content %dx%d, style %dx%d)"
                             % (patch, patch, content.H, content.W, Hs, Ws))
        # the scores of the patch correlation are produced in chunks when they would not fit SWAP_WORKSPACE_BYTES; every
        # chunking gives the same bytes (include/wctb200.h: wctb200_style_swap_apply_min_workspace_bytes,
        # wctb200_style_swap_softmax_min_workspace_bytes, wctb200_style_swap_balanced_min_workspace_bytes)
        least = (getattr(lib, "wctb200_style_swap_%s_min_workspace_bytes" % kind) if kind
                 else lib.wctb200_style_swap_apply_min_workspace_bytes)(*geom)
        nbytes = min(nbytes, max(least, SWAP_WORKSPACE_BYTES))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        kbuf = torch.empty(N + 1, dtype=torch.int32, device=self.device) if want_info else None
        sem = SEMANTICS["tf"]
        cur = torch.cuda.current_stream(self.device)
        lbuf = None
        if labels is not None:
            cl, sl = (t.contiguous() for t in labels)
            lbuf = torch.empty(lib.wctb200_style_swap_labels_workspace_bytes(cl.shape[0], content.H, content.W, Hs, Ws,
                                                                             int(patch), int(stride)),
                               dtype=torch.uint8, device=self.device)
            lab = (cl.data_ptr(), cl.shape[0], cl.shape[1], cl.shape[2], sl.data_ptr(), sl.shape[-2], sl.shape[-1])
        head = (content.ptr, N, content.H, content.W, C, state.data_ptr(), Hs, Ws, int(patch), int(stride), float(ss_alpha),
                sem["eps_cov"], sem["thresh"])
        tail = (out.ptr, kbuf.data_ptr() if want_info else None, ws.data_ptr(), ws.numel())
        if balance:
            self._call("style_swap_balanced[C%d]" % C,
                       lib.wctb200_style_swap_balanced_launches(*geom, nbytes, int(lbuf is not None), balance, 0),
                       lib.wctb200_style_swap_apply_balanced, *head, float(temperature), balance,
                       *(lab if lbuf is not None else (None, 0, 0, 0, None, 0, 0)), *tail[:2], None, *tail[2:],
                       None if lbuf is None else lbuf.data_ptr(), 0 if lbuf is None else lbuf.numel(), st)
        elif soft:
            self._call("style_swap_softmax[C%d]" % C, lib.wctb200_style_swap_softmax_launches(*geom, nbytes, int(lbuf is not None)),
                       lib.wctb200_style_swap_apply_softmax, *head, float(temperature),
                       *(lab if lbuf is not None else (None, 0, 0, 0, None, 0, 0)), *tail,
                       None if lbuf is None else lbuf.data_ptr(), 0 if lbuf is None else lbuf.numel(), st)
        elif lbuf is None:
            self._call("style_swap[C%d]" % C, 11, lib.wctb200_style_swap_apply, *head, *tail, st)
        else:
            self._call("style_swap_labels[C%d]" % C, 14, lib.wctb200_style_swap_apply_labels, *head, *lab, *tail, lbuf.data_ptr(),
                       lbuf.numel(), st)
        if lbuf is not None:
            lbuf.record_stream(cur)
        ws.record_stream(cur)   # freed by the caching allocator only after this stream is done
        return out, kbuf

    def style_prepare(self, style):
        """Style side of one level (ops.py:48-55,76): means, covariance, eigendecomposition, C_s.
        Returns the device state buffer consumed by ``wct_apply``."""
        st = self._stream()
        sem = SEMANTICS[self.semantics]
        C = style.C
        state = torch.empty(self.lib.wctb200_wct_style_state_bytes(C, style.N), dtype=torch.uint8, device=self.device)
        ws = self._workspace(C, 0, style.N)
        hws = style.H * style.W
        self._call("wct_style[C%d]" % C, 7 + self._matfun_launches(C), self.lib.wctb200_wct_style_prepare, style.ptr, style.N, style.H, style.W, C,
                   sem["eps_cov"], sem["eps_eig"], sem["thresh"], state.data_ptr(), ws.data_ptr(), ws.numel(), st,
                   flops=2.0 * C * C * style.N * hws, bytes_=4.0 * C * style.N * hws)
        return state

    def style_prepare_regions(self, style, labels, R):
        """Style side of one level under a style mask: entry r of the returned state of R styles is ``style_prepare`` over
        the pixels of ``style`` (one style) labelled r in ``labels`` (device uint8 [1,Hs,Ws] at the feature resolution).  An
        entry of fewer than 2 pixels has k_s = -1, and ``wct_apply_regions`` keeps the content of that region."""
        st = self._stream()
        sem = SEMANTICS[self.semantics]
        C = style.C
        state = torch.empty(self.lib.wctb200_wct_style_state_bytes(C, R), dtype=torch.uint8, device=self.device)
        ws = self._grow_workspace(("style_regions", C, R),
                                  self.lib.wctb200_wct_style_prepare_regions_workspace_bytes(C, R, style.H, style.W))
        hws = style.H * style.W
        self._call("wct_style_regions[C%d]" % C, 10 + self._matfun_launches(C), self.lib.wctb200_wct_style_prepare_regions, style.ptr,
                   style.H, style.W, C, labels.data_ptr(), R, sem["eps_cov"], sem["eps_eig"], sem["thresh"], state.data_ptr(), None,
                   ws.data_ptr(), ws.numel(), st, flops=2.0 * C * C * hws, bytes_=4.0 * C * hws)
        return state

    def wct_apply(self, content, state, n_style, alpha, want_info=False):
        st = self._stream()
        sem = SEMANTICS[self.semantics]
        C = content.C
        out = self._act(content.N, content.H, content.W, C)
        ws = self._workspace(C, content.N, 0)
        kbuf = torch.empty(2 * (content.N + n_style), dtype=torch.int32, device=self.device) if want_info else None
        hwc = content.H * content.W
        self._call("wct_level[C%d]" % C, 9 + self._matfun_launches(C), self.lib.wctb200_wct_apply, content.ptr, content.N, content.H, content.W, C,
                   state.data_ptr(), n_style, float(alpha), sem["eps_cov"], sem["eps_eig"], sem["thresh"], sem["readd"],
                   out.ptr, kbuf.data_ptr() if want_info else None, ws.data_ptr(), ws.numel(), st,
                   flops=2.0 * C * C * 2 * content.N * hwc, bytes_=4.0 * C * 2 * content.N * hwc)
        return out, kbuf

    def _ost_launches(self, C):
        """kernels OST adds to the WCT content side: the products of S_c, B and M, B^1/2 by the matrix-function fast path
        and the eigensolver (Jacobi on P = S_c C_s, k_root_post, outer product), and the eps_eig term"""
        return 8 + int(SEMANTICS[self.semantics]["eps_eig"] != 0.0) + self._matfun_launches(C)

    def _ost_workspace(self, C, Nc):
        key = ("ost", self._group, C, Nc)
        ws = self._ws.get(key)
        if ws is None:
            ws = torch.empty(self.lib.wctb200_ost_workspace_bytes(C, Nc), dtype=torch.uint8, device=self.device)
            self._ws[key] = ws
        return ws

    def ost_apply(self, content, state, n_style, alpha, want_info=False):
        """The optimal-transport transform (DESIGN.md §3.3.8) of one level against a WCT style state of ``n_style`` styles.
        ``want_info``: the int32 k_out [k_c | sweeps_c | ns_c | ns_b | sweeps_b] x N of ``wctb200_ost_apply``."""
        st = self._stream()
        sem = SEMANTICS[self.semantics]
        C = content.C
        out = self._act(content.N, content.H, content.W, C)
        ws = self._ost_workspace(C, content.N)
        kbuf = torch.empty(5 * content.N, dtype=torch.int32, device=self.device) if want_info else None
        hwc = content.H * content.W
        self._call("ost_level[C%d]" % C, 9 + self._matfun_launches(C) + self._ost_launches(C), self.lib.wctb200_ost_apply,
                   content.ptr, content.N, content.H, content.W, C, state.data_ptr(), n_style, float(alpha), sem["eps_cov"],
                   sem["eps_eig"], sem["thresh"], sem["readd"], out.ptr, kbuf.data_ptr() if want_info else None, ws.data_ptr(),
                   ws.numel(), st, flops=2.0 * C * C * 2 * content.N * hwc, bytes_=4.0 * C * 2 * content.N * hwc)
        return out, kbuf

    def labels_resize(self, labels, H, W):
        """Device uint8 label maps [N,Hm,Wm] -> [N,H,W] by proportional nearest sampling (spatial control)."""
        out = torch.empty((labels.shape[0], H, W), dtype=torch.uint8, device=self.device)
        self._call("labels_resize", 1, self.lib.wctb200_labels_resize_nearest, labels.data_ptr(), labels.shape[0], labels.shape[1],
                   labels.shape[2], H, W, out.data_ptr(), self._stream())
        return out

    def wct_apply_regions(self, content, labels, states, alpha, want_info=False):
        """Spatial control on one level: region r of each frame (``labels`` [N,H,W] at the feature resolution) takes the
        style whose state is ``states[r]``; labels >= R and regions of < 2 pixels keep the content feature."""
        st = self._stream()
        sem = SEMANTICS[self.semantics]
        C, N, R = content.C, content.N, len(states)
        out = self._act(N, content.H, content.W, C)
        ws = self._grow_workspace(("regions", C, N, R), self.lib.wctb200_wct_regions_workspace_bytes(C, N, R, content.H, content.W))
        kbuf = torch.empty(2 * (N * R + R), dtype=torch.int32, device=self.device) if want_info else None
        hwc = content.H * content.W
        self._call("wct_regions[C%d]" % C, 13 + self._matfun_launches(C), self.lib.wctb200_wct_apply_regions, content.ptr, N,
                   content.H, content.W, C, labels.data_ptr(), R, _capi.pointer_array([s.data_ptr() for s in states]),
                   float(alpha), sem["eps_cov"], sem["eps_eig"], sem["thresh"], sem["readd"], out.ptr,
                   kbuf.data_ptr() if want_info else None, ws.data_ptr(), ws.numel(), st,
                   flops=2.0 * C * C * 2 * N * hwc, bytes_=4.0 * C * 2 * N * hwc)
        return out, kbuf

    # ------------------------------------------------------------------ soft spatial control (DESIGN.md §3.3.11)
    def mask_feather(self, labels, R, sigma):
        """Device uint8 label maps [N,Hm,Wm] -> fp32 weight planes [N,R,Hm,Wm]: the one-hot plane of each label r < R blurred
        by a Gaussian of ``sigma`` mask pixels (labels >= R are the keep plane, which the R planes leave)."""
        N, Hm, Wm = labels.shape
        out = torch.empty((N, R, Hm, Wm), dtype=torch.float32, device=self.device)
        self._call("mask_feather", 2, self.lib.wctb200_mask_feather, labels.data_ptr(), N, Hm, Wm, R, float(sigma), out.data_ptr(),
                   self._stream())
        return out

    def weights_resize(self, maps, H, W):
        """Device fp32 maps [N,K,Hm,Wm] -> [N,K,H,W] by the exact area average."""
        N, K, Hm, Wm = maps.shape
        out = torch.empty((N, K, H, W), dtype=torch.float32, device=self.device)
        self._call("weights_resize", 1, self.lib.wctb200_weights_resize_area, maps.data_ptr(), N, K, Hm, Wm, H, W, out.data_ptr(),
                   self._stream())
        return out

    def _gather_states(self, states, N, C):
        """One WCT style state of N*K entries from K states of one style each: entry n*K + k is states[k]."""
        K = len(states)
        om, oc, ok, om2, oc2, ok2 = (ctypes.c_size_t() for _ in range(6))
        self.lib.wctb200_wct_style_state_layout(C, 1, ctypes.byref(om), ctypes.byref(oc), ctypes.byref(ok))
        total = self.lib.wctb200_wct_style_state_layout(C, N * K, ctypes.byref(om2), ctypes.byref(oc2), ctypes.byref(ok2))
        out = torch.zeros(total, dtype=torch.uint8, device=self.device)
        P = N * K
        for name, o1, o2, nb in (("mean", om, om2, 4 * C), ("cs", oc, oc2, 4 * C * C)):
            src = torch.stack([s[o1.value:o1.value + nb] for s in states])            # [K, nb]
            out[o2.value:o2.value + P * nb].view(N, K, nb).copy_(src.unsqueeze(0).expand(N, K, nb))
        ks = torch.stack([s[ok.value:ok.value + 8].view(torch.int32) for s in states])  # [K, 2]: k_s, sweeps
        kv = out[ok2.value:ok2.value + 8 * P].view(torch.int32).view(2, N, K)
        kv.copy_(ks.t().unsqueeze(1).expand(2, N, K))
        return out

    def soft_level(self, cf, soft, states, n_style, alpha, adain=False, ost=False, labels=None):
        """One level of a call with soft spatial control (DESIGN.md §3.3.11).  ``soft`` = (strength [N,Hm,Wm] | None,
        weights [N,K,Hm,Wm] | None) at map resolution; ``states``: the level's style state (one WCT or AdaIN state of
        ``n_style`` styles), or with weights or ``labels`` a list of K states of one style each; ``labels``: the hard label
        map [N,Hm,Wm] of a masked call, whose one-hot planes (nearest sampling) are the weights."""
        st = self._stream()
        sem = SEMANTICS[self.semantics]
        strength, weights = soft
        C, N = cf.C, cf.N
        s_l = self.weights_resize(strength.unsqueeze(1), cf.H, cf.W) if strength is not None else None
        out = self._act(N, cf.H, cf.W, C)
        if weights is None and labels is None:
            record = torch.empty(self.lib.wctb200_stats_record_layout(C, N, int(adain), None, None, None, None), dtype=torch.uint8,
                                 device=self.device)
            self._call("%s_stats_rect[C%d]" % ("adain" if adain else "wct", C), 3,
                       self.lib.wctb200_adain_stats_rect if adain else self.lib.wctb200_wct_stats_rect, cf.ptr, N, cf.H, cf.W, C,
                       0, 0, cf.H, cf.W, record.data_ptr(), st)
            if adain:
                tr = torch.empty(self.lib.wctb200_adain_transform_layout(C, N, None, None, None, None), dtype=torch.uint8,
                                 device=self.device)
                self._call("adain_transform[C%d]" % C, 2, self.lib.wctb200_adain_transform_from_stats, record.data_ptr(), N, C,
                           states.data_ptr(), n_style, 1e-5, tr.data_ptr(), st)
                self._call("adain_apply_strength[C%d]" % C, 1, self.lib.wctb200_adain_transform_apply_strength, cf.ptr, N, cf.H,
                           cf.W, C, tr.data_ptr(), float(alpha), s_l.data_ptr(), out.ptr, st)
                return out, None
            P, K, w_l, state = N, 1, None, states
        else:
            K = len(states)
            if weights is not None:
                w_l = self.weights_resize(weights, cf.H, cf.W)
            else:
                lab = self.labels_resize(labels, cf.H, cf.W)
                w_l = (lab.unsqueeze(1) == torch.arange(K, dtype=torch.uint8, device=self.device).view(1, K, 1, 1)).float()
            P = N * K
            state = self._gather_states(states, N, C)
            n_style = P
            record = torch.empty(self.lib.wctb200_stats_record_layout(C, P, 0, None, None, None, None), dtype=torch.uint8,
                                 device=self.device)
            self._call("wct_stats_weighted[C%d]" % C, 5, self.lib.wctb200_wct_stats_weighted, cf.ptr, N, cf.H, cf.W, C,
                       w_l.data_ptr(), K, record.data_ptr(), st)
        tr = torch.empty(self.lib.wctb200_wct_transform_layout(C, P, None, None, None), dtype=torch.uint8, device=self.device)
        if ost:
            ws = self._ost_workspace(C, P)
            self._call("ost_transform[C%d]" % C, 8 + self._matfun_launches(C) + self._ost_launches(C),
                       self.lib.wctb200_ost_transform_from_stats, record.data_ptr(), P, C, state.data_ptr(), n_style, float(alpha),
                       sem["eps_cov"], sem["eps_eig"], sem["thresh"], sem["readd"], tr.data_ptr(), ws.data_ptr(), ws.numel(), st)
        else:
            ws = self._workspace(C, P, 0)
            self._call("wct_transform[C%d]" % C, 8 + self._matfun_launches(C), self.lib.wctb200_wct_transform_from_stats,
                       record.data_ptr(), P, C, state.data_ptr(), n_style, float(alpha), sem["eps_cov"], sem["eps_eig"],
                       sem["thresh"], sem["readd"], tr.data_ptr(), ws.data_ptr(), ws.numel(), st)
        hwc = cf.H * cf.W
        self._call("wct_apply_weighted[C%d]" % C, 2, self.lib.wctb200_wct_transform_apply_weighted, cf.ptr, N, cf.H, cf.W, C,
                   tr.data_ptr(), K, w_l.data_ptr() if w_l is not None else None, s_l.data_ptr() if s_l is not None else None,
                   out.ptr, st, flops=2.0 * C * C * 2 * N * hwc * K, bytes_=4.0 * C * 2 * N * hwc)
        if w_l is not None:
            w_l.record_stream(torch.cuda.current_stream(self.device))
        return out, None

    # ------------------------------------------------------------------ multimodal style transfer (DESIGN.md §3.3.10)
    check_mst = staticmethod(options.check_mst)                 # (K, lambda) of an MST call: options.check_mst

    def mst_clusters(self, style, K, level):
        """Spherical k-means of the style feature ``style`` (one style) into K clusters, seeded by the draws of ``level`` (0 for
        relu1_1 .. 4 for relu5_1).  Returns device (labels uint8 [1,Hs,Ws], centres fp32 [K,C], info int32 [K init indices |
        iterations | K counts])."""
        C = style.C
        labels = torch.empty((1, style.H, style.W), dtype=torch.uint8, device=self.device)
        centres = torch.empty((K, C), dtype=torch.float32, device=self.device)
        info = torch.empty(2 * K + 1, dtype=torch.int32, device=self.device)
        ws = self._grow_workspace(("mst_clusters",), self.lib.wctb200_mst_style_clusters_workspace_bytes(style.H, style.W, C, K))
        self._call("mst_clusters[C%d@%dx%d]" % (C, style.H, style.W), 2 * K + 31, self.lib.wctb200_mst_style_clusters, style.ptr,
                   style.H, style.W, C, K, int(level), labels.data_ptr(), centres.data_ptr(), info.data_ptr(), ws.data_ptr(),
                   ws.numel(), self._stream(), bytes_=4.0 * C * style.H * style.W * (K + 16))
        return labels, centres, info

    def mst_data_term(self, content, centres, info):
        """D fp32 [N,H,W,K] = 1 - u_p . c_k of the content feature against the K cluster centres (``mst_clusters``); +inf for a
        cluster of fewer than 2 style pixels."""
        K, C = centres.shape[0], content.C
        D = torch.empty((content.N, content.H, content.W, K), dtype=torch.float32, device=self.device)
        hw = content.N * content.H * content.W
        self._call("mst_data_term[C%d]" % C, 1, self.lib.wctb200_mst_data_term, content.ptr, content.N, content.H, content.W, C,
                   centres.data_ptr(), info[K + 1:].data_ptr(), K, D.data_ptr(), self._stream(),
                   flops=2.0 * (K + 1) * C * hw, bytes_=4.0 * hw * (C + K))
        return D

    def mst_smooth(self, D, lam, sweeps=MST_SWEEPS):
        """Content labels uint8 [N,H,W]: red-black ICM on the data term ``D`` with Potts weight ``lam``."""
        N, H, W, K = D.shape
        labels = torch.empty((N, H, W), dtype=torch.uint8, device=self.device)
        self._call("mst_smooth", 1 + 2 * sweeps, self.lib.wctb200_mst_smooth, D.data_ptr(), N, H, W, K, float(lam), int(sweeps),
                   labels.data_ptr(), self._stream(), bytes_=(1 + 2 * sweeps) * N * H * W * (4.0 * K + 1))
        return labels

    def prepare_mst_call(self, style_u8, K):
        """The MST style side of one style image (cuda uint8 [1,Hs,Ws,3]), made once for a call that applies it several times
        (passes)."""
        main = torch.cuda.current_stream(self.device)
        ps = self._style_side(style_u8, main, mst=K)
        style_u8.record_stream(ps.side)
        return ps

    # ------------------------------------------------------------------ exact feature distribution matching (§3.3.12)
    def _efdm_chunk(self, total, per_seg_fn):
        """(segments per chunk, chunks) of an EFDM sort of ``total`` segments within EFDM_WORKSPACE_BYTES."""
        per_seg = per_seg_fn(2) - per_seg_fn(1)
        S = max(1, min(total, (EFDM_WORKSPACE_BYTES - per_seg_fn(1) + per_seg) // max(per_seg, 1)))
        return S, -(-total // S)

    def efdm_prepare(self, style, R=None):
        """Style side of EFDM on one level: every channel's values, sorted (fp32 [n][C][Hs*Ws]).  Returns dict(state, H, W).
        With ``R`` (cuda fp32 C x C) the values are those of R y, the state of one sliced step (§3.3.14)."""
        lib, C, n = self.lib, style.C, style.N
        state = torch.empty(lib.wctb200_efdm_style_state_bytes(C, n, style.H, style.W), dtype=torch.uint8, device=self.device)
        S, chunks = self._efdm_chunk(n * C, lambda k: lib.wctb200_efdm_style_workspace_bytes(C, n, style.H, style.W, k))
        nbytes = lib.wctb200_efdm_style_workspace_bytes(C, n, style.H, style.W, S)
        # the rotated states of a per-frame style are made on the content stream, while the style stream may still be
        # preparing later levels: each has its own scratch
        ws = self._grow_workspace(("efdm_style",) if R is None else ("efdm_style_rot",), nbytes)
        m = n * C * style.H * style.W
        # the exact size of S segments (a grown buffer may be larger): the chunking, and so the launch count, is the one above
        if R is None:
            self._call("efdm_style[C%d]" % C, 14 * chunks, lib.wctb200_efdm_style_prepare, style.ptr, n, style.H, style.W, C,
                       state.data_ptr(), ws.data_ptr(), nbytes, self._stream(), bytes_=84.0 * m)
        else:
            self._call("efdm_style_rot[C%d]" % C, 14 * chunks, lib.wctb200_efdm_rotated_style_prepare, style.ptr, n, style.H,
                       style.W, C, R.data_ptr(), state.data_ptr(), ws.data_ptr(), nbytes, self._stream(),
                       flops=2.0 * C * m, bytes_=84.0 * m)
        return dict(state=state, H=style.H, W=style.W)

    def sliced_matrices(self, C, K):
        """(R_1..R_K, G_1..G_{K+1}) of ``sliced`` as cuda fp32 C x C tensors, made once per (C, K)."""
        key = (int(C), int(K))
        if key not in self._sliced:
            to = lambda a: torch.from_numpy(np.array(a, dtype=np.float32)).to(self.device)
            self._sliced[key] = ([to(R) for R in sliced.rotations(C, K)], [to(G) for G in sliced.step_matrices(C, K)])
        return self._sliced[key]

    def efdm_sliced_apply(self, content, st, n_style, alpha, feat=None):
        """Sliced distribution matching of one level (§3.3.14): the chain of ``st["slices"]`` = K rotated EFDM steps and
        the plain one.  The state of step k is ``st["rot"][k]`` when the side made them (a shared style), otherwise it is
        made from the style feature ``feat`` just before the step and dropped after it."""
        lib, C, N, K = self.lib, content.C, content.N, st["slices"]
        if float(alpha) == 0.0:
            return self.efdm_apply(content, st, n_style, alpha)
        Rs, Gs = self.sliced_matrices(C, K)
        H, W = content.H, content.W
        m = N * C * H * W
        S, chunks = self._efdm_chunk(N * C, lambda k: lib.wctb200_efdm_workspace_bytes(C, N, H, W, k))
        ws_n = lib.wctb200_efdm_workspace_bytes(C, N, H, W, S)
        ws_ptr = self._grow_workspace(("efdm",), ws_n).data_ptr()
        pn = lib.wctb200_efdm_planes_bytes(C, N, H, W)
        # m_k stays in fp32 planes; step k + 1 reads all channels of m_k while writing m_{k+1}, so two buffers take turns
        planes = [self._grow_workspace(("efdm_planes", i), pn).data_ptr() for i in range(min(K, 2))]
        out = self._act(N, H, W, C)
        src = None
        for k in range(K + 1):
            last = k == K
            state = st["state"] if last else (st["rot"][k] if st.get("rot") else self.efdm_prepare(feat, Rs[k])["state"])
            dst = None if last else planes[k % 2]
            self._call("efdm_sliced[C%d]" % C, (18 if last else 17) * chunks, lib.wctb200_efdm_sliced_step, content.ptr, src,
                       N, H, W, C, Gs[k].data_ptr(), state.data_ptr(), n_style, st["H"], st["W"], float(alpha), dst,
                       out.ptr if last else None, ws_ptr, ws_n, self._stream(), flops=2.0 * C * m, bytes_=130.0 * m)
            src = dst
        return out, None

    def efdm_apply(self, content, st, n_style, alpha):
        """EFDM of one level against an ``efdm_prepare`` state of ``n_style`` in {1, N} styles."""
        lib, C, N = self.lib, content.C, content.N
        out = self._act(N, content.H, content.W, C)
        m = N * C * content.H * content.W
        if float(alpha) == 0.0:
            chunks, ws_ptr, ws_n = 0, None, 0
        else:
            S, chunks = self._efdm_chunk(N * C, lambda k: lib.wctb200_efdm_workspace_bytes(C, N, content.H, content.W, k))
            ws_n = lib.wctb200_efdm_workspace_bytes(C, N, content.H, content.W, S)
            ws_ptr = self._grow_workspace(("efdm",), ws_n).data_ptr()
        self._call("efdm_level[C%d]" % C, 18 * chunks if chunks else 1, lib.wctb200_efdm_apply, content.ptr, N, content.H,
                   content.W, C, st["state"].data_ptr(), n_style, st["H"], st["W"], float(alpha), out.ptr, ws_ptr, ws_n,
                   self._stream(), bytes_=(130.0 if chunks else 8.0) * m)
        return out, None

    def _grow_workspace(self, key, nbytes):
        """Grow-only scratch per (group, key): the levels of a call differ in size."""
        key = (self._group,) + key
        ws = self._ws.get(key)
        if ws is None or ws.numel() < nbytes:
            ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
            self._ws[key] = ws
        return ws

    def wct_apply_blend(self, content, states, weights, alpha, want_info=False):
        """Style interpolation on one level: frame n takes the blend of the K style ``states`` with the weights of row n of
        ``weights`` (cuda fp32 [1|N, K]; one row: every frame)."""
        st = self._stream()
        sem = SEMANTICS[self.semantics]
        C, N, K, Nw = content.C, content.N, len(states), weights.shape[0]
        out = self._act(N, content.H, content.W, C)
        ws = self._grow_workspace(("blend", C, N, K, Nw), self.lib.wctb200_wct_blend_workspace_bytes(C, N, K, Nw))
        kbuf = torch.empty(2 * (N + K), dtype=torch.int32, device=self.device) if want_info else None
        hwc = content.H * content.W
        self._call("wct_blend[C%d]" % C, 10 + self._matfun_launches(C), self.lib.wctb200_wct_apply_blend, content.ptr, N, content.H,
                   content.W, C, _capi.pointer_array([s.data_ptr() for s in states]), K, weights.data_ptr(), Nw, float(alpha),
                   sem["eps_cov"], sem["eps_eig"], sem["thresh"], sem["readd"], out.ptr, kbuf.data_ptr() if want_info else None,
                   ws.data_ptr(), ws.numel(), st, flops=2.0 * C * C * 2 * N * hwc, bytes_=4.0 * C * 2 * N * hwc)
        return out, kbuf

    # ------------------------------------------------------------------ pipeline
    def run_levels(self, levels=None):
        """The levels (``model.levels`` entries) a call runs: all for None, else those of ``levels`` in the model's order
        (``options.check_levels``: ValueError for an empty, repeated or foreign target)."""
        if levels is None:
            return self.model.levels
        keep = options.check_levels(levels, self.model.relu_targets)
        return [lvl for lvl in self.model.levels if lvl.relu_target in keep]

    def swap_levels(self, swap5=False, swap_targets=None):
        """The relu levels a call swaps at: ``swap_targets`` (checked against this model's targets), or relu5_1 for
        ``swap5`` when it is a target (model.py:148).  ValueError for both at once or a level that is not a target."""
        have = [l.relu_target for l in self.model.levels]
        if swap_targets is None:
            return ("relu5_1",) if swap5 and "relu5_1" in have else ()
        if swap5:
            raise ValueError("give swap5 or swap_targets, not both (swap5 is swap_targets=['relu5_1'])")
        levels = tuple(dict.fromkeys(str(r) for r in swap_targets))
        for relu in levels:
            if relu not in have:
                raise ValueError("swap_targets: %s is not a relu target of this model (%s)" % (relu, ", ".join(have)))
        return levels

    def stylize(self, content_u8, style_u8, alpha=1.0, adain=False, want_info=False, capture=None, swap5=False, ss_alpha=0.6,
                ss_patch_size=3, ss_stride=1, labels=None, region_styles=None, interp_styles=None, interp_weights=None,
                region_masks=None, swap_targets=None, ost=False, seamless=None, mst=None, mst_smooth=0.05, strength_map=None,
                content_weights=None, mask_feather=None, efdm=False, swap_labels=None, efdm_slices=0, levels=None,
                ss_temperature=None, ss_balance=0):
        """content_u8: cuda uint8 [N,H,W,3]; style_u8: cuda uint8 [Ns,Hs,Ws,3] or a ``PreparedStyle`` of Ns styles, Ns in
        {1, N}.  Returns the float32 ``decoded_output`` [N,H',W',3] (unclipped, model.py:94).
        ``capture`` (dict) receives every level's input image / features for parity tests.

        Every call runs the style side once -- the encode of the style and its per-level states (``_style_side``) -- and
        then applies it; a ``PreparedStyle`` skips the first step.  A shared style swap (``swap5``) swaps the N frames in
        one batched call per sub-batch; with one style per frame the frames run one by one.

        With ``self.groups`` = G > 1 the batch is cut into G sub-batches whose level chains are
        enqueued on G independent stream pairs: frames are independent (wct.py:97-103), and the
        eigendecompositions are latency bound on a few SMs, so one group's Jacobi clusters overlap the
        other groups' convolutions (same arithmetic per frame; only the schedule changes).

        Which of the options below combine is decided by one table, ``wct_tf_b200/options.py``.

        Spatial control: ``labels`` is a cuda uint8 label map [N|1,Hm,Wm] of any resolution and ``region_styles`` a list of
        R (1..8) cuda uint8 images [1,Hs,Ws,3] of any sizes, or prepared styles of one style each; ``style_u8`` is ignored.
        At every level the map is resampled to the feature grid and region r of a frame is transformed against style r;
        labels >= R keep the content feature.  The R styles are encoded and prepared once per call.

        Style masks: ``region_masks`` (with ``labels``) is a list of R entries, each None (the whole style r) or a cuda
        uint8 label map [Hm',Wm'] of style r, of any resolution.  Region r then takes the statistics of the pixels of style
        r labelled r, the map sampled to each level's style feature grid by the rule of ``labels``; where that region has
        fewer than 2 pixels at a level, region r of every frame keeps its content feature.  Entries that are the same
        (style, mask) pair of objects share one encode and one masked prepare (``_region_sides``).

        Style interpolation: ``interp_styles`` is a list of K (1..8) cuda uint8 images [1,Hs,Ws,3] of any sizes, or prepared
        styles of one style each, and ``interp_weights`` a cuda float32 [1|N, K] tensor; ``style_u8`` is ignored.  Frame n is
        stylised with the blend of the K styles under weight row n (one row: every frame), which for a row that sums to 1 is
        the same blend of the K single-style outputs at every level (WCT and AdaIN are affine in the style statistics).  The
        weights are used as given.  The K styles are encoded and prepared once per call.

        Style swap at any level: ``swap_targets`` is a list of relu targets at which the style swap replaces WCT / AdaIN,
        with ``ss_alpha``, ``ss_patch_size`` and ``ss_stride``; ``swap5`` is ``swap_targets=["relu5_1"]``.
        ``swap_labels`` = (content labels, style labels), cuda uint8 [1|N,Hm,Wm] and [1|Ns,Hm',Wm'] of any resolution,
        makes every swap level a labelled swap (DESIGN.md §3.3.13): each content patch draws only on the style patches of
        its own label, or on all of them when the style has none of that label.  The other levels are unchanged.
        ``ss_temperature`` = tau > 0 makes every swap level a softmax swap (DESIGN.md §3.3.17): each content patch is
        rebuilt from the blend of the style patches weighted by a softmax of their scores at temperature tau, instead of
        its single best patch.  None is the hard swap.  ``ss_balance`` = T in 1..256 (with ``ss_temperature``) makes it the
        balanced swap (DESIGN.md §3.3.18): T Sinkhorn iterations spread the blend's use of the style patches evenly; 0 is
        the softmax swap.

        Optimal-transport transform: ``ost=True`` matches each level's content Gaussian to the style's by the Monge map
        (DESIGN.md §3.3.8) instead of WCT, against the same WCT style states; swap levels still swap.

        Seamless stylisation: ``seamless`` = "x", "y" or "xy" pads every conv of the content path circularly along those
        axes (DESIGN.md §3.3.9), so the output equals that of the infinitely tiled content and tiles without a seam.  Each
        wrapped axis must be a multiple of 2^P (P pools up to the deepest target).  The style side is unchanged.

        Multimodal style transfer: ``mst`` = K (1..8) clusters each level's style feature into K modes and labels every
        content pixel with the mode it resembles, smoothed by a Potts term of weight ``mst_smooth`` (DESIGN.md §3.3.10);
        region k of each frame then takes the statistics of style mode k.  ``style_u8`` is one style image.  K = 1 is the
        plain WCT call, byte for byte.

        Soft spatial control (DESIGN.md §3.3.11): ``strength_map`` (cuda fp32 [1|N,Hm,Wm] in [0,1]) scales the stylisation
        per pixel, out = s T(x) + (1 - s) x; ``content_weights`` (cuda fp32
        [1|N,K,Hm,Wm], weights >= 0 summing to <= 1 per pixel, with ``region_styles`` of K styles and no ``labels``) blends
        the K region transforms per pixel, each region's statistics weighted by its plane; ``mask_feather`` = sigma (with
        ``labels``) turns the label map into Gaussian-feathered weights.  Maps of any resolution are area-averaged to each
        level.

        Exact feature distribution matching (DESIGN.md §3.3.12): ``efdm=True`` gives every channel of each level the value
        distribution of the same channel of the style, by rank (ties take the mean of their ranks' style values), instead
        of WCT; swap levels still swap.  ``style_u8`` is one style or one per frame; a ``PreparedStyle`` only as made by
        ``prepare_call(efdm=True)``.

        Sliced distribution matching (DESIGN.md §3.3.14): ``efdm_slices`` = K in 0..32 (with ``efdm``) first runs EFDM in
        K random orthonormal bases of each level's channels, each step rotating the previous one's output, so that the
        joint distribution of the channels approaches the style's; the last step is plain EFDM, and the blend at ``alpha``
        is with the content feature.  K = 0 is plain EFDM.  A ``PreparedStyle`` must come from
        ``prepare_call(efdm=True, efdm_slices=K)`` with the same K.

        Level subset (coarse-to-fine stylisation, DESIGN.md §3.3.16): ``levels`` names some of the model's relu targets
        (``options.check_levels``); only those levels run, in the model's order, each but the last clipped (model.py:86),
        as in an engine built with only those targets and the same weights.  A style side made for every level serves
        any subset.  None runs every level.  Not with ``mst``, whose clustering side runs its own level chain."""
        N = content_u8.shape[0]
        chain = self.run_levels(levels)
        if levels is not None and mst is not None:
            raise ValueError("levels does not combine with mst: its clustering side runs its own level chain")
        options.check({name for name, on in (
            ("adain", adain), ("ost", ost), ("efdm", efdm), ("mst", mst is not None), ("swap", swap5 or swap_targets is not None),
            ("content_mask", labels is not None), ("style_masks", region_masks is not None),
            ("style_weights", interp_styles is not None), ("content_weights", content_weights is not None),
            ("mask_feather", mask_feather is not None), ("strength_map", strength_map is not None),
            ("seamless", seamless is not None)) if on}, options.ENGINE)
        efdm_slices = options.check_efdm_slices(efdm_slices, efdm, options.ENGINE)
        ss_temperature = options.check_ss_temperature(ss_temperature, swap5 or swap_targets is not None, options.ENGINE)
        ss_balance = options.check_ss_balance(ss_balance, ss_temperature, options.ENGINE)
        transform = "adain" if adain else "efdm" if efdm else "ost" if ost else "wct"
        if efdm and isinstance(style_u8, PreparedStyle):
            skip = self.swap_levels(swap5, swap_targets)
            if any(relu not in style_u8.efdm and relu not in skip for relu in self.model.style_taps):
                raise ValueError("efdm sorts the style's features at every level, which a prepared style does not keep: "
                                 "give the style image")
            if any(st["slices"] != efdm_slices for st in style_u8.efdm.values()):
                raise ValueError("the prepared style was made for efdm_slices = %d, the call asks for %d"
                                 % (next(iter(style_u8.efdm.values()))["slices"], efdm_slices))
        soft = None
        if strength_map is not None or content_weights is not None or mask_feather is not None:
            sm = None
            if strength_map is not None:
                sm = strength_map if strength_map.dim() == 3 else strength_map.unsqueeze(0)
                if sm.dtype != torch.float32 or sm.dim() != 3 or sm.shape[0] not in (1, N) or sm.device != self.device:
                    raise ValueError("strength_map must be a float32 tensor [1|N,Hm,Wm] on %s" % self.device)
                sm = sm.expand(N, -1, -1).contiguous()
            cw = None
            if content_weights is not None:
                R = len(region_styles) if region_styles is not None else 0
                cw = content_weights if content_weights.dim() == 4 else content_weights.unsqueeze(0)
                if (cw.dtype != torch.float32 or cw.dim() != 4 or cw.shape[0] not in (1, N) or cw.shape[1] != R or not 1 <= R <= 8
                        or cw.device != self.device):
                    raise ValueError("content_weights must be a float32 tensor [1|N,K,Hm,Wm] on %s with K = 1..8 region styles"
                                     % self.device)
                cw = cw.expand(N, -1, -1, -1).contiguous()
            elif mask_feather is not None:
                sigma = options.check_mask_feather(mask_feather)
                R = len(region_styles) if region_styles is not None else 0
                if not 1 <= R <= 8:
                    raise ValueError("spatial control needs 1..8 region styles, got %d" % R)
                lab = labels if labels.dim() == 3 else labels.unsqueeze(0)
                if lab.dtype != torch.uint8 or lab.dim() != 3 or lab.shape[0] not in (1, N):
                    raise ValueError("labels must be uint8 [Hm,Wm] or [N,Hm,Wm]")
                cw = self.mask_feather(lab.contiguous(), R, sigma).expand(N, -1, -1, -1).contiguous()
            soft = (sm, cw)
            if cw is not None and labels is None:
                # soft weights take the place of the label map: a region call whose labels are never read
                labels = torch.zeros((N, 1, 1), dtype=torch.uint8, device=self.device)
        if mst is not None:
            K, lam = options.check_mst(mst, mst_smooth)
            if isinstance(style_u8, PreparedStyle):
                if style_u8.mst_k != K or any(relu not in style_u8.mst for relu in self.model.style_taps):
                    raise ValueError("mst clusters the style's features at every level, which a prepared style does not keep: "
                                     "give the style image")
            elif style_u8.shape[0] != 1:
                raise ValueError("mst takes one style for the whole batch, got %d" % style_u8.shape[0])
            return self._stylize_call(content_u8, style_u8, Plan(chain, alpha, mode="mst", mst=(K, lam)), want_info, capture)
        if seamless is not None:
            check_seamless(seamless, content_u8.shape[1], content_u8.shape[2], self.model.relu_targets)
        swap_lv = self.swap_levels(swap5, swap_targets)
        if swap_labels is not None:
            n_sty = style_u8.n if isinstance(style_u8, PreparedStyle) else style_u8.shape[0]
            cl, sl = options.check_swap_labels(swap_labels, bool(swap_lv), N, n_sty)
            for t in (cl, sl):
                if not isinstance(t, torch.Tensor) or t.device != self.device:
                    raise ValueError("swap_labels must be uint8 tensors on %s" % self.device)
            swap_labels = (cl.contiguous(), sl.contiguous())
        if interp_styles is not None:
            K = len(interp_styles)
            if not 1 <= K <= 8:
                raise ValueError("style interpolation needs 1..8 styles, got %d" % K)
            w = interp_weights
            if (not isinstance(w, torch.Tensor) or w.dtype != torch.float32 or w.dim() != 2 or w.shape[0] not in (1, N)
                    or w.shape[1] != K or w.device != self.device):
                raise ValueError("interp_weights must be a float32 tensor [1|N, K] on %s" % self.device)
            w = w.contiguous()
            return self._stylize_call(content_u8, list(interp_styles), Plan(chain, alpha, transform, mode="interp", weights=w,
                                                                            seamless=seamless), want_info, capture)
        if labels is not None:
            R = len(region_styles) if region_styles is not None else 0
            if not 1 <= R <= 8:
                raise ValueError("spatial control needs 1..8 region styles, got %d" % R)
            if labels.dim() == 2:
                labels = labels.unsqueeze(0)
            if labels.dtype != torch.uint8 or labels.dim() != 3 or labels.shape[0] not in (1, N):
                raise ValueError("labels must be uint8 [Hm,Wm] or [N,Hm,Wm]")
            labels = labels.expand(N, -1, -1).contiguous()
            if region_masks is not None:
                region_masks = self.check_region_masks(region_masks, region_styles)
            return self._stylize_call(content_u8, list(region_styles), Plan(chain, alpha, mode="regions", labels=labels,
                                                                            masks=region_masks, soft=soft, seamless=seamless),
                                      want_info, capture)
        prepared = isinstance(style_u8, PreparedStyle)
        n_style = style_u8.n if prepared else style_u8.shape[0]
        if n_style not in (1, N):
            raise ValueError("%d styles for %d frames: give one style, or one per frame" % (n_style, N))
        if prepared and not efdm:
            self.check_prepared(style_u8, adain, swap_lv)
        swap = (Swap(int(ss_patch_size), int(ss_stride), swap_lv, ss_alpha, swap_labels, ss_temperature, ss_balance)
                if swap_lv else None)
        return self._stylize_call(content_u8, style_u8, Plan(chain, alpha, transform, efdm_slices, swap=swap, soft=soft,
                                                             seamless=seamless), want_info, capture)

    def _stylize_call(self, content_u8, style, plan, want_info, capture):
        """Run ``plan`` on the frames ``content_u8`` against ``style``: an image batch or ``PreparedStyle`` of 1 or N styles
        (one style side, or the MST side), or the list of styles of a "regions" / "interp" call.

        The style sides that serve the whole batch -- those of a multi-style call, and one shared style image that the
        groups or the swap reuse -- are made here once, on group 1's style stream when the batch is cut into G sub-batch
        groups.  Otherwise each group prepares, or slices, the styles of its own frames.  With one style per frame and a
        swap the frames run one by one, each with its own style side."""
        N = content_u8.shape[0]
        prepared = isinstance(style, PreparedStyle)
        if plan.swap is not None and (style.n if prepared else style.shape[0]) > 1:
            return torch.cat([self._stylize_call(content_u8[i:i + 1], self.slice_prepared(style, i, i + 1) if prepared
                                                 else style[i:i + 1], plan.frames(i, i + 1), want_info, None)
                              for i in range(N)], dim=0)
        main = torch.cuda.current_stream(self.device)
        G = min(self.groups, N) if (capture is None and not want_info) else 1
        sides, owned = None, []
        self._group = 1 if G > 1 else 0
        try:
            if plan.mode == "mst":
                ps = style if prepared else self._style_side(style, main, mst=plan.mst[0])
                sides, owned = ps.entries, [] if prepared else [ps]
            elif plan.mode is not None:
                sides, owned = self._region_sides(style, plan.masks, main, plan.transform == "adain")
            elif prepared and style.n == 1:
                sides = [style]
            elif not prepared and style.shape[0] == 1 and (G > 1 or plan.swap is not None):
                # ONE style for the whole batch (video, configs[2]): its encoder pass and per-level states are made once,
                # every sub-batch group waits for the per-level events
                keep = plan.swap.levels if plan.swap is not None else ()
                sides = owned = [self._style_side(style, main, keep=keep, skip=keep, **plan.states)]
        finally:
            self._group = 0
        if plan.swap is not None:
            for relu in plan.swap.levels:
                self.swap_state(sides[0], relu, plan.swap.patch, plan.swap.stride)

        def group(lo, hi, want_info, capture):
            cur = torch.cuda.current_stream(self.device)
            held, mine = sides, None
            if held is None and prepared:
                held = [style if G == 1 else self.slice_prepared(style, lo, hi)]
            elif held is None:
                assert style.dtype == torch.uint8 and style.shape[0] in (1, N)
                mine = self._style_side(style[lo:hi], cur, **plan.states)
                held = [mine]
            out = self._stylize_one(content_u8[lo:hi], held, plan.frames(lo, hi), want_info, capture)
            for sd in held:
                if sd is not mine:
                    sd.record_stream(cur)      # a prepared style held by the caller may be dropped while this work is queued
            if mine is not None and mine.side is not cur:
                mine.side.wait_stream(cur)     # buffers handed across streams may be recycled only after both are done
                cur.wait_stream(mine.side)
            return out

        out = group(0, N, want_info, capture) if G == 1 else self._in_groups(N, G, main, lambda lo, hi: group(lo, hi, False, None))
        for side in {id(sd.side): sd.side for sd in owned}.values():
            if side is not main:
                side.wait_stream(main)         # the style states are recycled only after every group used them
                if G == 1 or plan.mode is not None:
                    main.wait_stream(side)
        if plan.mode == "mst" and prepared:
            style.record_stream(main)          # the caller's clustered side, whose entries the groups applied
        return out

    def _in_groups(self, N, G, main, run):
        """Cut a batch of N frames into G sub-batches and enqueue ``run(lo, hi)`` for each on its own stream (group g + 1
        owns its scratch); returns the concatenated outputs, ordered on ``main`` after every group."""
        bounds = [(g * N) // G for g in range(G + 1)]
        outs = []
        for g in range(G):
            lo, hi = bounds[g], bounds[g + 1]
            if g not in self._group_streams:
                # descending priority: group 0 runs "in the foreground", later groups fill the SMs it
                # leaves idle while its eigendecompositions are latency bound (self.group_priorities)
                prio = -1 if (self.group_priorities and g == 0) else 0
                self._group_streams[g] = torch.cuda.Stream(device=self.device, priority=prio)
            gs = self._group_streams[g]
            gs.wait_stream(main)
            self._group = g + 1
            try:
                with torch.cuda.stream(gs):
                    outs.append(run(lo, hi))
            finally:
                self._group = 0
        for g in range(G):
            main.wait_stream(self._group_streams[g])
        out = torch.cat(outs, dim=0)
        for g in range(G):                      # sub-batch buffers die here: their streams wait for the cat
            self._group_streams[g].wait_stream(main)
        return out

    def check_region_masks(self, masks, styles):
        """ValueError unless ``masks`` holds one entry per region style, each None or a uint8 label map [Hm',Wm'] (or
        [1,Hm',Wm']) on this device, and no prepared style has a mask.  Returns the list with every map as [1,Hm',Wm'];
        entries that were the same object stay the same object."""
        masks = list(masks)
        if len(masks) != len(styles):
            raise ValueError("%d style masks for %d region styles: give one entry (None or a mask) per style" % (len(masks), len(styles)))
        out, seen = [], {}
        for s, m in zip(styles, masks):
            if m is None:
                out.append(None)
                continue
            if isinstance(s, PreparedStyle):
                raise ValueError("a prepared style has no feature maps to mask: give the style image with its mask")
            if id(m) not in seen:
                if (not isinstance(m, torch.Tensor) or m.dtype != torch.uint8 or m.device != self.device or m.dim() not in (2, 3)
                        or (m.dim() == 3 and m.shape[0] != 1) or m.shape[-2] < 1 or m.shape[-1] < 1):
                    raise ValueError("each style mask must be a uint8 label map [Hm,Wm] on %s" % self.device)
                seen[id(m)] = (m, m.reshape(1, m.shape[-2], m.shape[-1]).contiguous())
            out.append(seen[id(m)][1])
        return out

    def _region_sides(self, styles, masks, main, adain=False):
        """The style sides of a multi-style call: (one side per style, the sides made here).  Without ``masks`` every image
        is prepared on its own.  With ``masks`` (``check_region_masks``) the entries that are the same (style, mask) pair of
        objects share one side: an unmasked entry takes it whole, and a masked entry r takes its entry r, the style prepared
        over its pixels labelled r (``_style_side`` with a mask)."""
        sides, owned, shared = [], [], {}
        R = len(styles)
        for r, s in enumerate(styles):
            m = masks[r] if masks is not None else None
            if isinstance(s, PreparedStyle):
                if s.n != 1:
                    raise ValueError("each region / interpolated style must be one style, got a prepared style of %d" % s.n)
                self.check_prepared(s, adain)
                sides.append(s)
            elif masks is None:
                owned.append(self._style_side(s, main, **style_states(adain)))
                sides.append(owned[-1])
            else:
                key = (id(s), id(m))
                if key not in shared:
                    shared[key] = self._style_side(s, main, labels=m, R=R) if m is not None else self._style_side(s, main)
                    owned.append(shared[key])
                sides.append(shared[key].entries[r] if m is not None else shared[key])
        return sides, owned

    def prepare_regions_call(self, styles, masks):
        """The style sides of a spatial-control call with style masks (``check_region_masks``), made once for a call that
        applies them several times (passes): one prepared style of one style per region."""
        main = torch.cuda.current_stream(self.device)
        sides, owned = self._region_sides(styles, masks, main)
        for s, m in zip(styles, masks):
            if not isinstance(s, PreparedStyle):
                side = self._style_stream() or main
                s.record_stream(side)
                if m is not None:
                    m.record_stream(side)
        return sides

    def _style_stream(self):
        """This group's style stream (the style side overlaps the content work), or None without overlap."""
        if not self.overlap_style:
            return None
        if self._group not in self._style_streams:
            prio = -1 if (self.group_priorities and self._group <= 1) else 0
            self._style_streams[self._group] = torch.cuda.Stream(device=self.device, priority=prio)
        return self._style_streams[self._group]

    def _style_side(self, style_u8, main, wct=True, adain=False, keep=(), skip=(), labels=None, R=0, mst=0, efdm=False,
                    efdm_slices=0):
        """The prepare step: style side of one call (model.py:70-72: ONE encoder pass emitting every target; per level the
        WCT state of ops.py:48-55,76 when ``wct``, the AdaIN moments when ``adain``; levels in ``skip`` get neither), enqueued
        on this group's style stream when overlap is on.  ``keep`` lists the levels whose feature it keeps (the style
        swap is prepared from them).  Returns a
        ``PreparedStyle`` with one event per level.

        With ``labels`` (a style mask, cuda uint8 [1,Hm,Wm] of one style) the WCT state of each level is the masked prepare
        of R regions, so the result is a prepared style of n = R; ``entries[r]`` is its slice r (``slice_prepared``) as a
        prepared style of one style, cut per level as soon as that level is prepared and sharing its events.

        With ``mst`` = K (one style image) each level's style feature is clustered (``mst_clusters``) and its WCT state is
        the masked prepare of the K clusters under the style's own labels: a prepared style of n = K with ``entries`` as
        above, and the labels, centres and info of every level in ``mst``, which the entries share.

        With ``efdm`` every level also gets its EFDM state (``efdm_prepare``: the style's values sorted per channel) in
        ``efdm``.  With ``efdm_slices`` = K > 0 as well (sliced EFDM, §3.3.14), a side of one style also makes the K
        rotated states of each level (``rot``); a side of one style per frame keeps each level's feature instead, from which
        ``efdm_sliced_apply`` makes each state just before its step."""
        lib = self.lib
        side = self._style_stream() or main
        if side is not main:
            side.wait_stream(main)             # style_u8 (and last step's buffers) are ready
        sem = SEMANTICS[self.semantics]
        taps = list(dict.fromkeys(self.model.style_taps))
        if mst:
            R = int(mst)
        ps = PreparedStyle(style_u8.shape[0] if labels is None and not mst else R, {k: sem[k] for k in SEMANTIC_KEYS}, taps)
        ps.side = side
        ps.mst_k = int(mst)
        if labels is not None or mst:
            ps.entries = [PreparedStyle(1, ps.semantics, taps) for _ in range(R)]
            for e in ps.entries:
                e.side, e.events, e.mst = side, ps.events, ps.mst
        with torch.cuda.stream(side):
            tag, self._tag = self._tag, "style"
            style = torch.empty(style_u8.shape, dtype=torch.float32, device=self.device)
            self._call("u8_to_f32", 1, lib.wctb200_image_u8_to_f32, style_u8.data_ptr(), style_u8.numel(), style.data_ptr(),
                       self._stream())
            _, feats = self.encode(style, self.model.deepest_target, taps=self.model.style_taps)
            for relu in taps:
                if relu not in skip:
                    if mst:
                        f = feats[relu]
                        lab, cen, info = self.mst_clusters(f, R, RELU_LEVEL[relu] - 1)
                        ps.mst[relu] = dict(labels=lab, centres=cen, info=info)
                        ps.wct[relu] = self.style_prepare_regions(f, lab, R)
                        for r, e in enumerate(ps.entries):
                            e.wct[relu] = slice_wct_state(lib, ps.wct[relu], f.C, R, r, r + 1)
                    elif labels is not None:
                        f = feats[relu]
                        ps.wct[relu] = self.style_prepare_regions(f, self.labels_resize(labels, f.H, f.W), R)
                        for r, e in enumerate(ps.entries):
                            e.wct[relu] = slice_wct_state(lib, ps.wct[relu], f.C, R, r, r + 1)
                    elif wct:
                        ps.wct[relu] = self.style_prepare(feats[relu])
                    if adain:
                        ps.adain[relu] = self.adain_prepare(feats[relu])
                    if efdm:
                        ps.efdm[relu] = dict(self.efdm_prepare(feats[relu]), slices=int(efdm_slices), rot=None)
                        if efdm_slices and ps.n == 1:
                            ps.efdm[relu]["rot"] = [self.efdm_prepare(feats[relu], R)["state"]
                                                    for R in self.sliced_matrices(feats[relu].C, efdm_slices)[0]]
                        elif efdm_slices:
                            ps.feats[relu] = feats[relu]
                ev = torch.cuda.Event()
                ev.record(side)
                ps.events[relu] = ev
            for relu in keep:
                if relu in feats:
                    ps.feats[relu] = feats[relu]
            self._tag = tag
        return ps

    def prepare(self, style_u8, swap_targets=()):
        """Every part of the style side of ``style_u8`` (cuda uint8 [n,Hs,Ws,3]): WCT states and AdaIN moments of every
        target, and the feature of relu5_1 (when it is a target) and of every level of ``swap_targets``."""
        main = torch.cuda.current_stream(self.device)
        keep = ("relu5_1",) + tuple(r for r in self.swap_levels(False, list(swap_targets)) if r != "relu5_1")
        ps = self._style_side(style_u8, main, wct=True, adain=True, keep=keep)
        style_u8.record_stream(ps.side)        # read on the style stream after the caller may have dropped it
        ps.record_stream(main)
        return ps

    def prepare_call(self, style_u8, adain=False, swap5=False, swap_targets=None, efdm=False, efdm_slices=0):
        """The style side one call needs (WCT states, the AdaIN moments, or the EFDM states, with ``efdm_slices`` those of
        every slice; the features of the swap levels of ``swap5`` / ``swap_targets``), made once for a call that applies it
        several times (passes)."""
        main = torch.cuda.current_stream(self.device)
        ps = self._style_side(style_u8, main, keep=self.swap_levels(swap5, swap_targets), **style_states(adain, efdm, efdm_slices))
        style_u8.record_stream(ps.side)
        return ps

    def check_prepared(self, ps, adain, swap=()):
        """ValueError unless ``ps`` was prepared for this engine's encoder and semantics and covers its targets, with the
        feature of every level in ``swap`` (the swap levels of the call)."""
        sem = SEMANTICS[self.semantics]
        for k in SEMANTIC_KEYS:
            if float(ps.semantics[k]) != float(sem[k]):
                raise ValueError("the prepared style was made with %s = %s, this model uses %s" % (k, ps.semantics[k], sem[k]))
        need = dict.fromkeys(self.model.style_taps)
        have = ps.adain if adain else ps.wct
        for relu in need:
            if relu not in have and relu not in swap:
                raise ValueError("the prepared style has no %s state for %s" % ("AdaIN" if adain else "WCT", relu))
        for relu in swap:
            if relu not in ps.feats:
                raise ValueError("the prepared style has no %s feature for the style swap" % relu)
        if ps.fingerprints:
            mine = self.fingerprints()
            for relu in need:
                if ps.fingerprints.get(relu) != mine[relu]:
                    raise ValueError("the prepared style was made with other encoder weights up to %s" % relu)

    def fingerprints(self):
        """Encoder fingerprint per target (prepared.encoder_fingerprints), computed once."""
        if self._fingerprints is None:
            self._fingerprints = encoder_fingerprints(self._vgg_layers, self.model.style_taps)
        return self._fingerprints

    def slice_prepared(self, ps, lo, hi):
        """Styles lo..hi-1 of a prepared style as a prepared style of their own (exact device copies on the current
        stream, which first waits for the prepare)."""
        cur = torch.cuda.current_stream(self.device)
        if ps.side is not cur:
            ps.wait(cur)
        out = PreparedStyle(hi - lo, ps.semantics, ps.targets)
        out.side = cur
        out.fingerprints = ps.fingerprints
        for relu, st in ps.wct.items():
            out.wct[relu] = slice_wct_state(self.lib, st, RELU_CHANNELS[relu], ps.n, lo, hi)
        for relu, st in ps.adain.items():
            out.adain[relu] = slice_adain_state(self.lib, st, RELU_CHANNELS[relu], ps.n, lo, hi)
        for relu, st in ps.efdm.items():
            per = RELU_CHANNELS[relu] * st["H"] * st["W"] * 4          # the sorted values of one style
            out.efdm[relu] = dict(st, state=st["state"][lo * per:hi * per].clone(),
                                  rot=[r[lo * per:hi * per].clone() for r in st["rot"]] if st.get("rot") else None)
        for relu, f in ps.feats.items():
            out.feats[relu] = self._act(hi - lo, f.H, f.W, f.C)
            slice_act_planes(f.buf, f.N, f.H, f.W, f.C, lo, hi, out.feats[relu].buf)
        ps.record_stream(cur)
        return out

    def swap_state(self, ps, relu, patch, stride):
        """The style-swap state of a prepared style of one style at level ``relu`` for (patch, stride): made on first use
        from its feature at that level (on its style stream when it has one) and cached in it.  Returns (state, event)."""
        key = (relu, int(patch), int(stride))
        if key not in ps.swap:
            main = torch.cuda.current_stream(self.device)
            st = ps.side if ps.side is not None else main
            if st is not main:
                st.wait_stream(main)
            with torch.cuda.stream(st):
                ps.wait(st, relu)
                tag, self._tag = self._tag, "style"
                state = self.swap_prepare(ps.feats[relu], *key[1:])
                self._tag = tag
                ps.feats[relu].buf.record_stream(st)
                ev = torch.cuda.Event()
                ev.record(st)
            ps.swap[key] = (state, ev)
        return ps.swap[key]

    def _stylize_one(self, content_u8, sides, plan, want_info, capture):
        """The level chain of ``plan`` on one (sub-)batch against the style ``sides`` (``_stylize_call``).  With
        ``plan.seamless`` the transforms write a reflect halo, which is rewritten before the decoder reads it."""
        assert content_u8.dtype == torch.uint8
        wrap = self.wrap_flags(plan.seamless)
        content = torch.empty(content_u8.shape, dtype=torch.float32, device=self.device)
        self._call("u8_to_f32", 1, self.lib.wctb200_image_u8_to_f32, content_u8.data_ptr(), content_u8.numel(), content.data_ptr(),
                   self._stream())
        infos = []
        x = content
        for lvl in plan.run:
            relu = lvl.relu_target
            self._tag = relu
            cf, _ = self.encode(x, relu, seamless=plan.seamless)
            f, kbuf = self._level(cf, relu, sides, plan, want_info, capture)
            if wrap:
                self.halo(f, wrap)
            infos.append(kbuf)
            if capture is not None:
                capture.setdefault("level_input", []).append(x)
                capture.setdefault("content_feat", []).append(cf)
                capture.setdefault("transformed", []).append(f)
            # model.py:86: clip between levels; model.py:94: last output unclipped
            x = self.decode(f, lvl.index, clip=lvl is not plan.run[-1], seamless=plan.seamless)
            if capture is not None:
                capture.setdefault("level_output", []).append(x)
        self._tag = None
        if want_info:
            self.last_info = infos
        return x

    def _level(self, cf, relu, sides, plan, want_info, capture):
        """The transform of level ``relu`` of ``plan`` on the content feature ``cf``: the one place that picks it.
        Returns (the transformed feature, the level's info or None)."""
        main = torch.cuda.current_stream(self.device)
        sw, alpha = plan.swap, plan.alpha
        if sw is not None and relu in sw.levels:      # model.py:148-152: style swap wins over AdaIN / WCT at its levels
            state, ev = sides[0].swap[(relu, sw.patch, sw.stride)]
            main.wait_event(ev)
            sf = sides[0].feats[relu]
            return self.swap_apply(cf, state, (sf.H, sf.W), sw.alpha, want_info, sw.patch, sw.stride, labels=sw.labels,
                                   temperature=sw.temperature, balance=sw.balance)
        for sd in sides:
            if sd.side is not main:
                sd.wait(main, relu)
        adain = plan.transform == "adain"
        if plan.mode is None:
            style = sides[0]
            if plan.soft is not None:
                return self.soft_level(cf, plan.soft, style.adain[relu] if adain else style.wct[relu], style.n, alpha, adain,
                                       plan.transform == "ost")
            if adain:
                return self.adain_apply(cf, style.adain[relu], style.n, alpha)
            if plan.transform == "efdm" and plan.slices:
                return self.efdm_sliced_apply(cf, style.efdm[relu], style.n, alpha, style.feats.get(relu))
            if plan.transform == "efdm":
                return self.efdm_apply(cf, style.efdm[relu], style.n, alpha)
            if plan.transform == "ost":
                return self.ost_apply(cf, style.wct[relu], style.n, alpha, want_info)
            return self.wct_apply(cf, style.wct[relu], style.n, alpha, want_info)
        if plan.soft is not None:              # regions: soft weights, or the hard labels' one-hot planes
            return self.soft_level(cf, plan.soft, [sd.wct[relu] for sd in sides], None, alpha,
                                   labels=plan.labels if plan.soft[1] is None else None)
        if plan.mode == "interp" and adain:
            return self.adain_apply_blend(cf, [sd.adain[relu] for sd in sides], plan.weights, alpha)
        if plan.mode == "interp":
            return self.wct_apply_blend(cf, [sd.wct[relu] for sd in sides], plan.weights, alpha, want_info)
        if plan.mode == "regions":
            lab = self.labels_resize(plan.labels, cf.H, cf.W)
            return self.wct_apply_regions(cf, lab, [sd.wct[relu] for sd in sides], alpha, want_info)
        m = sides[0].mst[relu]                 # "mst": label each pixel with its cluster, then regions
        lab = self.mst_smooth(self.mst_data_term(cf, m["centres"], m["info"]), plan.mst[1])
        out = self.wct_apply_regions(cf, lab, [sd.wct[relu] for sd in sides], alpha, want_info)
        if capture is not None:
            for key, val in (("mst_style_labels", m["labels"]), ("mst_centres", m["centres"]), ("mst_info", m["info"]),
                             ("mst_content_labels", lab)):
                capture.setdefault(key, []).append(val)
        return out

    # ------------------------------------------------------------------ tiled stylisation (DESIGN.md §3.3.7)
    check_tile_size = staticmethod(options.check_tile_size)     # the tile edge of a tiled call: options.check_tile_size

    def stats_record(self, C, adain):
        """A zeroed statistics record of one frame (n = 0: the empty record that the first accumulate fills)."""
        nbytes = self.lib.wctb200_stats_record_layout(C, 1, int(adain), None, None, None, None)
        return torch.zeros(nbytes, dtype=torch.uint8, device=self.device)

    def stats_rect(self, feat, y0, x0, h, w, record, adain):
        """Statistics of the rectangle [y0, y0+h) x [x0, x0+w) of ``feat`` into ``record`` (the covariance sums for WCT, the
        per-channel moments for AdaIN)."""
        fn = self.lib.wctb200_adain_stats_rect if adain else self.lib.wctb200_wct_stats_rect
        self._call("%s_stats_rect[C%d]" % ("adain" if adain else "wct", feat.C), 3, fn, feat.ptr, feat.N, feat.H, feat.W, feat.C,
                   int(y0), int(x0), int(h), int(w), record.data_ptr(), self._stream(), bytes_=4.0 * feat.C * feat.N * h * w)

    def stats_accumulate(self, rec_a, rec_b, C, adain):
        self._call("stats_accumulate[C%d]" % C, 2, self.lib.wctb200_stats_accumulate, rec_a.data_ptr(), rec_b.data_ptr(), C, 1,
                   int(adain), self._stream())

    def transform_from_stats(self, record, C, state, alpha, adain, ost=False):
        """The level transform of one frame from its statistics record against the style ``state`` of one style (a WCT
        state, or AdaIN moments); ``ost``: the optimal-transport transform of a WCT state, in the WCT transform layout."""
        st = self._stream()
        if adain:
            tr = torch.empty(self.lib.wctb200_adain_transform_layout(C, 1, None, None, None, None), dtype=torch.uint8, device=self.device)
            self._call("adain_transform[C%d]" % C, 2, self.lib.wctb200_adain_transform_from_stats, record.data_ptr(), 1, C,
                       state.data_ptr(), 1, 1e-5, tr.data_ptr(), st)
            return tr
        sem = SEMANTICS[self.semantics]
        tr = torch.empty(self.lib.wctb200_wct_transform_layout(C, 1, None, None, None), dtype=torch.uint8, device=self.device)
        if ost:
            ws = self._ost_workspace(C, 1)
            self._call("ost_transform[C%d]" % C, 8 + self._matfun_launches(C) + self._ost_launches(C),
                       self.lib.wctb200_ost_transform_from_stats, record.data_ptr(), 1, C, state.data_ptr(), 1, float(alpha),
                       sem["eps_cov"], sem["eps_eig"], sem["thresh"], sem["readd"], tr.data_ptr(), ws.data_ptr(), ws.numel(), st)
            return tr
        ws = self._workspace(C, 1, 0)           # keyed by C alone: the tile shapes of a call never add an entry
        self._call("wct_transform[C%d]" % C, 8 + self._matfun_launches(C), self.lib.wctb200_wct_transform_from_stats,
                   record.data_ptr(), 1, C, state.data_ptr(), 1, float(alpha), sem["eps_cov"], sem["eps_eig"], sem["thresh"],
                   sem["readd"], tr.data_ptr(), ws.data_ptr(), ws.numel(), st)
        return tr

    def transform_apply(self, feat, transform, alpha, adain):
        out = self._act(feat.N, feat.H, feat.W, feat.C)
        hw = feat.N * feat.H * feat.W
        if adain:
            self._call("adain_transform_apply[C%d]" % feat.C, 1, self.lib.wctb200_adain_transform_apply, feat.ptr, feat.N, feat.H,
                       feat.W, feat.C, transform.data_ptr(), float(alpha), out.ptr, self._stream(), bytes_=8.0 * feat.C * hw)
        else:
            self._call("wct_transform_apply[C%d]" % feat.C, 1, self.lib.wctb200_wct_transform_apply, feat.ptr, feat.N, feat.H,
                       feat.W, feat.C, transform.data_ptr(), out.ptr, self._stream(), flops=2.0 * feat.C * feat.C * hw,
                       bytes_=8.0 * feat.C * hw)
        return out

    def tiled_level(self, x, level_index, state, alpha, adain, tile_size, clip, ost=False, seamless=None):
        """One level of tiled stylisation on the float32 image ``x`` [1,H,W,3] against the style ``state`` of one style
        (DESIGN.md §3.3.7).  Pass A encodes every tile's crop (its interior widened by h_A, clipped to the image) and folds
        the statistics of the tile's interior feature into one record in tile order; the record becomes the level's
        transform once.  Pass B encodes every crop widened by h_B, applies the transform to the whole tile feature,
        decodes, and writes the decoded interior into the output image [1, g ceil(H/g), g ceil(W/g), 3].

        ``seamless`` (DESIGN.md §3.3.9), per wrapped axis: when one tile spans the axis the crop is the whole axis and is
        encoded with the wrap flag; otherwise the crop is widened by the same halos modulo the image size (a window of the
        periodic image) and encoded with the reflect halo, which the halos keep out of the interior."""
        from .model import RELU_LEVEL, tile_grid, tile_halos
        lvl = self.model.levels[level_index]
        relu, C = lvl.relu_target, lvl.channels
        g = 2 ** (RELU_LEVEL[relu] - 1)
        h_a, h_b = tile_halos(relu)
        H, W = x.shape[1], x.shape[2]
        tiles = tile_grid(H, W, tile_size)
        wx, wy = seamless_axes(seamless)
        mod_y, mod_x = wy and tile_size < H, wx and tile_size < W        # wrapped axes cut into tiles
        crop_mode = ("x" if wx and not mod_x else "") + ("y" if wy and not mod_y else "") or None
        crop_wrap = self.wrap_flags(crop_mode)

        def span(lo, hi, h, n, modular):
            """The crop [lo - h, hi + h) of an axis of n pixels: clipped to [0, n), or taken modulo n."""
            if modular:
                return lo - h, torch.arange(lo - h, hi + h, device=self.device) % n
            return max(0, lo - h), slice(max(0, lo - h), min(n, hi + h))

        def crop(y0, y1, x0, x1, h):
            cy0, ys = span(y0, y1, h, H, mod_y)
            cx0, xs = span(x0, x1, h, W, mod_x)
            img = x[:, ys] if isinstance(ys, slice) else x.index_select(1, ys)
            img = img[:, :, xs] if isinstance(xs, slice) else img.index_select(2, xs)
            return cy0, cx0, img.contiguous()

        record, part = self.stats_record(C, adain), self.stats_record(C, adain)
        for y0, y1, x0, x1 in tiles:
            cy0, cx0, img = crop(y0, y1, x0, x1, h_a)
            f, _ = self.encode(img, relu, seamless=crop_mode)
            # the interior feature rectangle: [y0/g, ceil(y1/g)) of the whole map, in the crop's coordinates
            fy0, fx0 = (y0 - cy0) // g, (x0 - cx0) // g
            self.stats_rect(f, fy0, fx0, -(-y1 // g) - cy0 // g - fy0, -(-x1 // g) - cx0 // g - fx0, part, adain)
            self.stats_accumulate(record, part, C, adain)
        transform = self.transform_from_stats(record, C, state, alpha, adain, ost)
        out = torch.empty((1, g * -(-H // g), g * -(-W // g), 3), dtype=torch.float32, device=self.device)
        for y0, y1, x0, x1 in tiles:
            cy0, cx0, img = crop(y0, y1, x0, x1, h_b)
            f, _ = self.encode(img, relu, seamless=crop_mode)
            t = self.transform_apply(f, transform, alpha, adain)
            if crop_wrap:
                self.halo(t, crop_wrap)
            dec = self.decode(t, level_index, clip, seamless=crop_mode)
            oy1, ox1 = g * -(-y1 // g), g * -(-x1 // g)
            out[:, y0:oy1, x0:ox1] = dec[:, y0 - cy0:oy1 - cy0, x0 - cx0:ox1 - cx0]
        return out

    def stylize_tiled(self, content_u8, style_u8, alpha=1.0, adain=False, tile_size=1024, ost=False, seamless=None, levels=None):
        """``stylize`` in tiles of ``tile_size`` (a positive multiple of 16) at every level, in bounded device memory: the
        working set follows the largest crop, (tile_size + 2 h_B)^2, not the image.  Each level's statistics are those of
        the whole image, so the result is the untiled one up to the order in which the statistics are summed, and byte
        for byte the same when one tile covers the image.  ``style_u8``: a cuda uint8 image batch or a ``PreparedStyle``
        of 1 or N styles.  The frames run one after another, each with its own statistics; the style side is untiled.
        ``ost``: the optimal-transport transform (DESIGN.md §3.3.8) instead of WCT.  ``seamless``: as for
        ``stylize`` (``tiled_level``).  ``levels``: the subset of levels to run, as for ``stylize``."""
        T = options.check_tile_size(tile_size)
        run = self.run_levels(levels)
        options.check({name for name, on in (("tile_size", True), ("adain", adain), ("ost", ost),
                                             ("seamless", seamless is not None)) if on}, options.ENGINE)
        N = content_u8.shape[0]
        check_seamless(seamless, content_u8.shape[1], content_u8.shape[2], self.model.relu_targets)
        prepared = isinstance(style_u8, PreparedStyle)
        n_style = style_u8.n if prepared else style_u8.shape[0]
        if n_style not in (1, N):
            raise ValueError("%d styles for %d frames: give one style, or one per frame" % (n_style, N))
        if prepared:
            self.check_prepared(style_u8, adain)
        main = torch.cuda.current_stream(self.device)
        side = style_u8 if prepared else self._style_side(style_u8, main, **style_states(adain))
        outs = []
        for i in range(N):
            sd = side if n_style == 1 else self.slice_prepared(side, i, i + 1)
            x = torch.empty((1,) + tuple(content_u8.shape[1:]), dtype=torch.float32, device=self.device)
            self._call("u8_to_f32", 1, self.lib.wctb200_image_u8_to_f32, content_u8[i].data_ptr(), x.numel(), x.data_ptr(),
                       self._stream())
            for lvl in run:
                self._tag = lvl.relu_target
                if sd.side is not main:
                    sd.wait(main, lvl.relu_target)
                state = sd.adain[lvl.relu_target] if adain else sd.wct[lvl.relu_target]
                # model.py:86: clip between levels; model.py:94: last output unclipped
                x = self.tiled_level(x, lvl.index, state, alpha, adain, T, clip=lvl is not run[-1], ost=ost, seamless=seamless)
            self._tag = None
            outs.append(x)
        if prepared:
            style_u8.record_stream(main)       # a prepared style held by the caller may be dropped while this work is queued
        elif side.side is not main:
            side.side.wait_stream(main)        # buffers handed across streams may be recycled only after both are done
            main.wait_stream(side.side)
        return outs[0] if N == 1 else torch.cat(outs, dim=0)

    def to_u8(self, img_f32):
        """WCT.postprocess (wct.py:66-68)."""
        out = torch.empty(img_f32.shape, dtype=torch.uint8, device=self.device)
        self._call("f32_to_u8", 1, self.lib.wctb200_image_f32_to_u8, img_f32.data_ptr(), img_f32.numel(), out.data_ptr(),
                   self._stream())
        return out

    def act_to_f32(self, act):
        out = torch.empty((act.N, act.H, act.W, act.C), dtype=torch.float32, device=self.device)
        _capi.check(self.lib.wctb200_act_to_f32(act.ptr, act.N, act.H, act.W, act.C, out.data_ptr(), self._stream()))
        return out

    def act_from_f32(self, t):
        N, H, W, C = t.shape
        a = self._act(N, H, W, C)
        t = t.contiguous()
        _capi.check(self.lib.wctb200_act_from_f32(t.data_ptr(), N, H, W, C, a.ptr, self._stream()))
        return a

    def check_device(self):
        _capi.check(self.lib.wctb200_check_device(self._stream()))
