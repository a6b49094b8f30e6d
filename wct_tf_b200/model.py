"""Level wiring of the multi-level WCT pipeline (host-side bookkeeping only).

Mirror of the reference's ``WCTModel`` (model.py:30-94, test mode) as an
explicit *plan*: which encoder layers run, which decoder layers run, in which
order, with the reference's layer names.  No tensors live here -- the engine
(`engine.py` -> libwctb200.so) executes the plan on the GPU.

Reference facts restated here (file:line in /root/reference):
  * shared VGG is built up to ``sorted(relu_targets)[-1]``            model.py:60
  * the style image is encoded once per call, all targets in one pass model.py:70-72
  * level i>0 consumes ``clip(prev.decoded, 0, 1)``                    model.py:86
  * the final output is the last decoder's output, UNCLIPPED          model.py:94
  * per-level transform choice                                        model.py:144-158
  * decoder architecture table and ``{relu}_{count}`` layer names     model.py:252-298
  * encoder module walk of vgg_normalised.t7                          vgg_normalised.py:22-50
"""
from __future__ import annotations

from collections import namedtuple

RELU_TARGETS_ALL = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]  # model.py:33 default
RELU_LEVEL = {"relu1_1": 1, "relu2_1": 2, "relu3_1": 3, "relu4_1": 4, "relu5_1": 5}  # model.py:252
RELU_CHANNELS = {"relu1_1": 64, "relu2_1": 128, "relu3_1": 256, "relu4_1": 512, "relu5_1": 512}

# 3x3 convs of the normalised VGG19 up to relu5_1: (name, Cin, Cout)
VGG_CONVS = [
    ("conv1_1", 3, 64), ("conv1_2", 64, 64),
    ("conv2_1", 64, 128), ("conv2_2", 128, 128),
    ("conv3_1", 128, 256), ("conv3_2", 256, 256), ("conv3_3", 256, 256), ("conv3_4", 256, 256),
    ("conv4_1", 256, 512), ("conv4_2", 512, 512), ("conv4_3", 512, 512), ("conv4_4", 512, 512),
    ("conv5_1", 512, 512),
]
_POOL_AFTER = {"conv1_2": "pool1", "conv2_2": "pool2", "conv3_4": "pool3", "conv4_4": "pool4"}

EncOp = namedtuple("EncOp", "kind name cin cout")          # kind: 'conv' (3x3 reflect + ReLU) | 'pool'
DecOp = namedtuple("DecOp", "kind name cin cout act")      # kind: 'conv' | 'up'


def encoder_plan(target):
    """Ops of the shared encoder from the [0,1] RGB image up to ``target``
    (vgg_normalised.py:22-50).  The 1x1 'preprocess' conv (vgg_normalised.py:25-26)
    is not listed: the engine folds it into conv1_1 (exact -- a per-pixel affine
    map commutes with reflect padding)."""
    if target not in RELU_LEVEL and not target.startswith("relu"):
        raise ValueError("unknown target layer %r" % (target,))
    ops = []
    for name, cin, cout in VGG_CONVS:
        ops.append(EncOp("conv", name, cin, cout))
        if name.replace("conv", "relu") == target:
            return ops
        if name in _POOL_AFTER:
            ops.append(EncOp("pool", _POOL_AFTER[name], cout, cout))
    raise ValueError("unknown target layer %r" % (target,))


_DECODER_ARCHS = {  # model.py:255-277
    5: [("conv", 512), ("up",), ("conv", 512), ("conv", 512), ("conv", 512)],
    4: [("conv", 256), ("up",), ("conv", 256), ("conv", 256), ("conv", 256)],
    3: [("conv", 128), ("up",), ("conv", 128)],
    2: [("conv", 64), ("up",)],
    1: [("conv", 64)],
}


def decoder_plan(relu_target):
    """Ops of one decoder, named as the reference names them (model.py:283-298):
    ``count`` runs over convs and upsamples; the last conv has 3 filters and no
    activation."""
    num = RELU_LEVEL[relu_target]
    c = RELU_CHANNELS[relu_target]
    ops, count = [], 0
    for d in reversed(range(1, num + 1)):
        for tup in _DECODER_ARCHS[d]:
            name = "%s_%d" % (relu_target, count)
            if tup[0] == "conv":
                ops.append(DecOp("conv", name, c, tup[1], True))
                c = tup[1]
            else:
                ops.append(DecOp("up", name, c, c, False))
            count += 1
    ops.append(DecOp("conv", "%s_%d" % (relu_target, count), c, 3, False))
    return ops


def _spread(ops, d):
    """Depth (in the pixels after ``ops``) to which a wrong border of depth ``d`` spreads through ``ops``: a 3x3 conv adds 1,
    an aligned 2x2 pool halves it (rounding up), an upsample doubles it."""
    for op in ops:
        if op.kind == "conv":
            d += 1
        elif op.kind == "pool":
            d = -(-d // 2)
        else:
            d *= 2
    return d


def tile_halos(relu_target):
    """Halos of tiled stylisation at level ``relu_target`` (DESIGN.md §3.3.7), in pixels of the level's input image, each a
    multiple of g = 2^(pools to the relu): (h_A, h_B).  A tile's crop widened by h_A encodes to the same relu feature on the
    tile's interior as the whole image does; widened by h_B it also decodes to the same image on the interior.  The cut
    edge of a crop is the wrong border: its depth is walked through ``encoder_plan`` (h_A) and on through
    ``decoder_plan`` (h_B)."""
    g = 2 ** (RELU_LEVEL[relu_target] - 1)
    d_feat = _spread(encoder_plan(relu_target), 0)
    d_img = _spread(decoder_plan(relu_target), d_feat)
    return d_feat * g, -(-d_img // g) * g


def tile_grid(H, W, T):
    """Interiors (y0, y1, x0, x1) of the T x T tiles of an H x W image in row-major order; the last row and column end at
    the image border, so the interiors partition the image."""
    return [(y0, min(y0 + T, H), x0, min(x0 + T, W)) for y0 in range(0, H, T) for x0 in range(0, W, T)]


def coarse_size(H, W, f, g):
    """Size (h, w) of the coarse stage of coarse-to-fine stylisation (DESIGN.md §3.3.16) of an H x W content at factor ``f``:
    each side divided by f and rounded to the nearest multiple of g = 2^(pools to the deepest target), halves up, at least g,
    so that every level of the coarse stage decodes exactly h x w."""
    return tuple(g * max(1, (2 * n + f * g) // (2 * f * g)) for n in (H, W))


SEAMLESS_MODES = (None, "x", "y", "xy")


def seamless_axes(seamless):
    """(wrap x, wrap y) of a seamless mode (DESIGN.md §3.3.9): None, "x" (panoramas), "y" or "xy" (tileable textures);
    ValueError for any other value."""
    if seamless not in SEAMLESS_MODES:
        raise ValueError("seamless must be None, 'x', 'y' or 'xy', got %r" % (seamless,))
    return seamless is not None and "x" in seamless, seamless is not None and "y" in seamless


def check_seamless(seamless, H, W, relu_targets):
    """ValueError unless ``seamless`` is a mode and every wrapped axis of an H x W content is a multiple of 2^P, P the
    pools up to the deepest of ``relu_targets`` (16 for relu5_1): otherwise a 'same' pool would pair pixels across the
    seam and the output would not be periodic.  Returns (wrap x, wrap y)."""
    wx, wy = seamless_axes(seamless)
    m = 2 ** (max(RELU_LEVEL[r] for r in relu_targets) - 1)
    for axis, wrapped, size in (("width", wx, W), ("height", wy, H)):
        if wrapped and size % m:
            raise ValueError("seamless=%r: the content %s %d is not a multiple of %d (2^pools up to the deepest target): "
                             "a pool would pair pixels across the seam" % (seamless, axis, size, m))
    return wx, wy


Level = namedtuple("Level", "index relu_target channels clip_input transform_rule")


class WCTModel(object):
    """Plan-only mirror of the reference ``WCTModel`` (model.py:30-94).

    Same constructor surface: ``WCTModel(mode='test', relu_targets=[...], vgg_path=None, **build_kwargs)``.
    Only ``mode='test'`` (inference) is in scope; ``mode='train'`` raises."""

    def __init__(self, mode="train", relu_targets=RELU_TARGETS_ALL, vgg_path=None, *args, **kwargs):
        if mode != "test":
            raise NotImplementedError("only the inference graph (mode='test') is in scope; "
                                      "decoder training (model.py:178-220) is out of scope")
        relu_targets = list(relu_targets)
        if len(relu_targets) == 0:
            raise ValueError("relu_targets must name at least one layer")
        for r in relu_targets:
            if r not in RELU_LEVEL:
                raise ValueError("unknown relu target %r" % (r,))
        self.mode = mode
        self.relu_targets = relu_targets
        self.vgg_path = vgg_path
        self.ss_patch_size = kwargs.get("ss_patch_size", 3)
        self.ss_stride = kwargs.get("ss_stride", 1)
        # model.py:60 -- plain string sort, exactly like the reference
        self.deepest_target = sorted(relu_targets)[-1]
        # model.py:70-72: the style encoder emits every target in one pass
        self.style_plan = encoder_plan(self.deepest_target)
        self.style_taps = list(relu_targets)
        # model.py:78-90
        self.levels = []
        for i, relu in enumerate(relu_targets):
            rule = "swap5>adain>wct" if relu == "relu5_1" else "adain>wct"  # model.py:144-158
            self.levels.append(Level(i, relu, RELU_CHANNELS[relu], i > 0, rule))
        self.encoder_decoders = self.levels  # reference attribute name (model.py:54)

    def content_plan(self, level_index):
        return encoder_plan(self.levels[level_index].relu_target)  # model.py:135-139

    def decoder_plan(self, level_index):
        return decoder_plan(self.levels[level_index].relu_target)  # model.py:167

    @staticmethod
    def transform_for(relu_target, swap5, use_adain):
        """model.py:144-158: relu5_1 -> tf.case([(swap5, style-swap), (use_adain, adain)], default=wct);
        other levels -> tf.cond(use_adain, adain, wct)."""
        if relu_target == "relu5_1" and swap5:
            return "style_swap"
        return "adain" if use_adain else "wct"
