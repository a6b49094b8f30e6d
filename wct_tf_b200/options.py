"""Which options of a stylising call combine, and the checks of their values.

This is the one statement of that policy.  ``WCT.predict_batch``, ``Engine.stylize`` / ``stylize_tiled`` and the flags of
``stylize.py`` / ``stylize_video.py`` each map their arguments to a set of the canonical option names below and call
``check`` with their vocabulary, so that every caller accepts the same combinations and names them in its own words.

``swap_labels`` (the labelled style swap, ``check_swap_labels``) has no entry in ``SPELLINGS``: it is a parameter of
``swap``, as ``mst_smooth`` is of ``mst``.  It needs the swap, and through it takes the swap's exclusions; it adds none of
its own.  ``ss_temperature`` (the softmax swap, ``check_ss_temperature``) is a parameter of ``swap`` in the same way, and
``ss_balance`` (the balanced swap, ``check_ss_balance``) a parameter of ``ss_temperature``.
``efdm_slices`` (sliced distribution matching, ``check_efdm_slices``) is in the same way a parameter of ``efdm``.

``coarse_to_fine`` (scale control, ``check_coarse_to_fine``) is in ``AROUND`` too: it runs the call on a downscaled
content at every level, joins the result into the content's low band and runs the fine levels on that at full size.
``fine_targets`` is its parameter.  The engine's part is ``levels=``, the subset of relu targets a call runs.

``luminance_only`` (colour preservation) is in ``AROUND``: it runs the whole call on grey frames and merges the colours
into its uint8 result, so it combines with every option of ``SPELLINGS`` but ``return_float``.
"""
import numpy as np

# canonical option -> its spelling as a predict_batch keyword, an Engine.stylize keyword and a CLI flag (None: that caller
# has no such option)
SPELLINGS = {
    "adain": ("adain", "adain", "--adain"),
    "ost": ("ost", "ost", "--ost"),
    "efdm": ("efdm", "efdm", "--efdm"),
    "mst": ("mst", "mst", "--mst"),
    "swap": ("swap5 / swap_targets", "swap5 / swap_targets", "--swap5 / --swap-targets"),
    "content_mask": ("content_mask", "labels", "--content-mask"),
    "style_masks": ("style_masks", "region_masks", "--style-masks"),
    "style_weights": ("style_weights", "interp_styles", "--interp-styles"),
    "content_weights": ("content_weights", "content_weights", "--mask-weights"),
    "mask_feather": ("mask_feather", "mask_feather", "--mask-feather"),
    "strength_map": ("strength_map", "strength_map", "--strength-map"),
    "tile_size": ("tile_size", "tile_size", "--tile-size"),
    "seamless": ("seamless", "seamless", "--seamless"),
    "temporal": ("temporal", None, "--temporal"),
    "return_float": ("return_float", None, None),
    "prepared": ("a prepared style", None, "prepared styles (.wctstyle)"),
    "per_frame_styles": ("one style per frame", None, None),
}
# options that act around the stylising call, on its uint8 frames before and after it (coarse-to-fine: before, between and
# after its two stages); the engine has no such option.  Spelled as SPELLINGS
AROUND = {
    "luminance_only": ("luminance_only", None, "--luminance-only"),
    "coarse_to_fine": ("coarse_to_fine", None, "--coarse-to-fine"),
}
API, ENGINE, CLI = ({name: s[i] for name, s in list(SPELLINGS.items()) + list(AROUND.items())} for i in range(3))

_MASKS = ("content_mask", "style_masks", "content_weights", "mask_feather")

# (option, the options it does not combine with, why); checked in this order
EXCLUDES = [
    ("efdm", ("adain", "ost", "mst"), "each level takes one transform"),
    ("efdm", _MASKS + ("strength_map", "style_weights"), "the sorted-value map has no region, weighted or blended form"),
    ("efdm", ("tile_size",), "the ranks are taken over the whole image"),
    ("efdm", ("prepared",), "it sorts the style's features at every level, which a prepared style does not keep"),
    ("content_weights", ("content_mask",), "the soft weights replace the label map; give one of them"),
    ("strength_map", ("style_weights", "swap", "mst", "tile_size"),
     "the per-pixel blend runs on untiled WCT, OST and AdaIN levels"),
    ("content_weights", ("style_weights", "swap", "mst", "tile_size", "adain", "ost"),
     "the weighted statistics and their blend are WCT's"),
    ("mask_feather", ("style_weights", "swap", "mst", "tile_size", "adain", "ost"),
     "feathering makes soft weights, whose statistics and blend are WCT's"),
    ("mst", ("adain", "ost"), "AdaIN / OST per cluster is not defined"),
    ("mst", ("content_mask", "style_masks", "style_weights"), "MST makes the regions itself"),
    ("mst", ("swap",), "every level runs WCT per cluster"),
    ("mst", ("tile_size",), "the clustering and the labelling need the whole level"),
    ("mst", ("seamless",), "red-black smoothing on a wrapped ring of odd length is not an independent set"),
    ("mst", ("prepared",), "it clusters the style's features at every level, which a prepared style does not keep"),
    ("mst", ("per_frame_styles",), "the style is clustered once for every frame"),
    ("seamless", ("swap",), "the swap's VALID patches are not periodic"),
    ("seamless", ("temporal",), "the optical flow does not see across the seam"),
    ("ost", ("adain",), "OST is a transform of the WCT style states"),
    ("ost", ("content_mask", "style_masks", "style_weights"), "M is not affine in the style statistics"),
    ("tile_size", ("content_mask", "style_masks", "style_weights"), "the tiled levels take the statistics of one whole style"),
    ("tile_size", ("swap",), "the swap's gather needs a patch-sized extra halo"),
    ("tile_size", ("temporal",), "the tiled path has no stabilisation pass"),
    ("temporal", ("return_float",), "temporal stabilisation works on the uint8 frames"),
    ("style_weights", ("content_mask", "swap"), "interpolation blends the transforms of whole styles"),
    ("content_mask", ("adain", "swap"), "spatial control is WCT only"),
    ("luminance_only", ("return_float",), "the colours are merged into the uint8 frames"),
    ("coarse_to_fine", ("swap",), "the stride crop and the patch grid depend on the resolution"),
    ("coarse_to_fine", ("seamless",), "neither the resize nor the join wraps"),
    ("coarse_to_fine", ("mst",), "its clustering side runs its own level chain"),
]

# (option, the options of which it needs one)
NEEDS = [
    ("mask_feather", ("content_mask",)),
    ("style_masks", ("content_mask", "content_weights")),
]


def check(active, vocab):
    """ValueError for the first rule of ``EXCLUDES`` / ``NEEDS`` that the set of canonical option names ``active`` breaks,
    naming the options as ``vocab`` (``API``, ``ENGINE`` or ``CLI``) spells them."""
    for a, others, why in EXCLUDES:
        if a in active:
            for b in others:
                if b in active:
                    raise ValueError("%s does not combine with %s: %s" % (vocab[a], vocab[b], why))
    for a, wants in NEEDS:
        if a in active and not active.intersection(wants):
            raise ValueError("%s needs %s" % (vocab[a], " or ".join(vocab[w] for w in wants)))


def check_mst(K, lam, names=("mst", "mst_smooth")):
    """(K, lambda) of an MST call: K an integer in 1..8, lambda finite and >= 0; ValueError otherwise."""
    if isinstance(K, bool) or not isinstance(K, (int, np.integer)) or not 1 <= K <= 8:
        raise ValueError("%s must be a number of clusters in 1..8, got %r" % (names[0], K))
    try:
        lam_f = float(lam)
    except (TypeError, ValueError):
        raise ValueError("%s must be a number, got %r" % (names[1], lam))
    if not np.isfinite(lam_f) or lam_f < 0:
        raise ValueError("%s must be finite and >= 0, got %r" % (names[1], lam))
    return int(K), lam_f


def _label_map(a, name, counts):
    """One uint8 label map [Hm,Wm] or stack [n,Hm,Wm] with n in ``counts``, numpy or torch; returned as [n,Hm,Wm]."""
    if not (hasattr(a, "dtype") and hasattr(a, "shape") and hasattr(a, "ndim")):
        a = np.asarray(a)
    if str(a.dtype) not in ("uint8", "torch.uint8"):
        raise ValueError("%s must be uint8 labels, got %s" % (name, a.dtype))
    if a.ndim == 2:
        a = a[None]
    if a.ndim != 3 or a.shape[0] not in counts:
        raise ValueError("%s must be [Hm,Wm] or [N,Hm,Wm] with N = %s, got shape %s"
                         % (name, " or ".join(str(c) for c in sorted(set(counts))), tuple(a.shape)))
    if a.shape[1] < 1 or a.shape[2] < 1:
        raise ValueError("%s must not be empty, got %s" % (name, tuple(a.shape)))
    return a


def check_swap_labels(swap_labels, swap, n_frames, n_styles=1, names=("swap_labels", "swap5 / swap_targets")):
    """The label maps of a labelled style swap (DESIGN.md §3.3.13): a pair (content labels [Hm,Wm] or [N,Hm,Wm], style
    labels [Hm',Wm'], or [N,Hm',Wm'] with one style per frame), uint8, numpy or torch.  ``swap``: whether the call swaps at
    any level.  Returns (content [1|N,Hm,Wm], style [1|Ns,Hm',Wm']) as given, with the frame axis added; ValueError
    otherwise, before any device work."""
    if not swap:
        raise ValueError("%s needs %s: the labels steer the style swap" % names)
    if not isinstance(swap_labels, (tuple, list)) or len(swap_labels) != 2:
        raise ValueError("%s must be a pair (content labels, style labels)" % names[0])
    content = _label_map(swap_labels[0], names[0] + " content labels", (1, n_frames))
    style = _label_map(swap_labels[1], names[0] + " style labels", (1, n_styles))
    return content, style


def check_ss_temperature(t, swap, vocab=API):
    """The temperature of the softmax swap (DESIGN.md §3.3.17): None (the hard swap), or a finite number > 0 that is a
    normal float32, and only with the style swap (``swap``: whether the call swaps at any level).  Returns it as a float
    or None; ValueError otherwise, naming the options as ``vocab`` spells them."""
    name = "--ss-temperature" if vocab is CLI else "ss_temperature"
    if t is None:
        return None
    if isinstance(t, bool) or not isinstance(t, (int, float, np.integer, np.floating)) or not np.isfinite(t) or not t > 0:
        raise ValueError("%s must be a finite number > 0, got %r" % (name, t))
    # the device takes tau as a float32 and divides by it: a value that rounds to 0, a subnormal or inf has no finite 1/tau
    f32 = np.finfo(np.float32)
    if not float(f32.tiny) <= float(t) <= float(f32.max):
        raise ValueError("%s must lie in float32's normal range [%g, %g], got %r" % (name, f32.tiny, f32.max, t))
    if not swap:
        raise ValueError("%s needs %s: the temperature is the style swap's" % (name, vocab["swap"]))
    return float(t)


def check_ss_balance(T, temperature, vocab=API):
    """The Sinkhorn iterations of the balanced swap (DESIGN.md §3.3.18): an integer in 0..256, and above 0 only with the
    softmax swap (``temperature``: its checked temperature, or None).  Returns it as an int; ValueError otherwise, naming
    the options as ``vocab`` spells them."""
    name, tname = ("--ss-balance", "--ss-temperature") if vocab is CLI else ("ss_balance", "ss_temperature")
    if isinstance(T, bool) or not isinstance(T, (int, np.integer)) or not 0 <= T <= 256:
        raise ValueError("%s must be an integer in 0..256, got %r" % (name, T))
    if T and temperature is None:
        raise ValueError("%s needs %s: the iterations balance the softmax swap" % (name, tname))
    return int(T)


def check_efdm_slices(K, efdm, vocab=API):
    """The number of rotated bases of sliced distribution matching (DESIGN.md §3.3.14): an integer in 0..32, and above 0
    only with ``efdm``.  Returns it as an int; ValueError otherwise, naming the options as ``vocab`` spells them (``--efdm``
    becomes ``--efdm-slices`` in the CLI's)."""
    name = "--efdm-slices" if vocab is CLI else "efdm_slices"
    if isinstance(K, bool) or not isinstance(K, (int, np.integer)) or not 0 <= K <= 32:
        raise ValueError("%s must be an integer in 0..32, got %r" % (name, K))
    if K and not efdm:
        raise ValueError("%s needs %s: the slices are steps of EFDM" % (name, vocab["efdm"]))
    return int(K)


def check_levels(levels, relu_targets, name="levels"):
    """A subset of the model's ``relu_targets`` (in the model's order) that a call runs: a non-empty sequence of its
    targets, none repeated.  Returns them as a tuple in the model's order; ValueError otherwise."""
    if isinstance(levels, str):
        levels = [levels]
    levels = [str(r) for r in levels]
    if not levels:
        raise ValueError("%s must name at least one relu target" % name)
    for r in levels:
        if r not in relu_targets:
            raise ValueError("%s: %s is not a relu target of this model (%s)" % (name, r, ", ".join(relu_targets)))
    if len(set(levels)) != len(levels):
        raise ValueError("%s names a relu target more than once: %s" % (name, ", ".join(levels)))
    return tuple(r for r in relu_targets if r in levels)


# the levels that carry texture and strokes rather than layout (DESIGN.md §3.3.5): the default fine stage
FINE_TARGETS = ("relu3_1", "relu2_1", "relu1_1")


def check_coarse_to_fine(f, fine_targets, relu_targets, vocab=API):
    """(f, fine levels) of a coarse-to-fine call (DESIGN.md §3.3.16): ``f`` an integer in 2..16, and ``fine_targets`` a
    subset of ``relu_targets`` (``check_levels``; None: the model's targets among relu3_1, relu2_1 and relu1_1), returned
    as a tuple in the model's order.  ValueError otherwise, for ``fine_targets`` without ``f``, and for a model with no
    default fine level, naming the options as ``vocab`` spells them."""
    name = vocab["coarse_to_fine"]
    fine_name = "--fine-targets" if vocab is CLI else "fine_targets"
    if f is None:
        raise ValueError("%s needs %s" % (fine_name, name))
    if isinstance(f, bool) or not isinstance(f, (int, np.integer)) or not 2 <= f <= 16:
        raise ValueError("%s must be an integer factor in 2..16, got %r" % (name, f))
    if fine_targets is None:
        fine = tuple(r for r in relu_targets if r in FINE_TARGETS)
        if not fine:
            raise ValueError("%s: the model has none of the default fine targets (%s); give %s"
                             % (name, ", ".join(FINE_TARGETS), fine_name))
        return int(f), fine
    return int(f), check_levels(fine_targets, relu_targets, fine_name)


def check_tile_size(tile_size, name="tile_size"):
    """The tile edge of a tiled call: a positive multiple of 16 (tile boundaries on the pooling grid of every level);
    ValueError otherwise."""
    if isinstance(tile_size, bool) or not isinstance(tile_size, (int, np.integer)) or tile_size <= 0 or tile_size % 16:
        raise ValueError("%s must be a positive multiple of 16, got %r" % (name, tile_size))
    return int(tile_size)


def check_mask_feather(sigma, name="mask_feather"):
    """The feathering sigma in mask pixels: a finite number in (0, 1024]; ValueError otherwise."""
    if isinstance(sigma, bool) or not isinstance(sigma, (int, float, np.integer, np.floating)) \
            or not np.isfinite(sigma) or not 0 < sigma <= 1024:
        raise ValueError("%s must be a finite sigma in (0, 1024] mask pixels, got %r" % (name, sigma))
    return float(sigma)


def check_temporal_strength(strength, name="temporal strength"):
    """The weight beta of the warped previous output: in [0, 1); ValueError otherwise."""
    strength = float(strength)
    if not 0.0 <= strength < 1.0:
        raise ValueError("%s must be in [0, 1), got %r" % (name, strength))
    return strength
