#!/usr/bin/env python
"""Command line front end with the flag surface of the reference's stylize.py (flags at stylize.py:14-37, the
content x style loop at stylize.py:70-119, output naming ``<content>_<style><ext>``): the TF session behind
``WCT.predict`` is replaced by the H100 engine.

  python stylize.py --checkpoints DIR5 DIR4 ... --relu-targets relu5_1 relu4_1 ... --vgg-path vgg_normalised.t7 \
      --content-path IN --style-path STYLE --out-path OUT --alpha 0.8

Spatial control: ``--content-mask MASK --mask-styles S0 S1 ...`` splits the content by an 8-bit grayscale mask (gray value
v -> region v*R // 256 for R styles: a black/white mask with two styles gives background / foreground) and region r takes
style r; the output is ``<content>_<s0>+<s1>...<ext>``.  ``--style-masks M0 M1 ...`` (one per style, quantised the same
way) gives each style a label map too: region r then takes only the pixels of style r in region r, so painting both
masks with the same grey levels links the regions ("the sky of the photo takes the sky of the painting").  A path given
twice is loaded once; one painting with one mask for every region is encoded once.

Style interpolation: ``--interp-styles S0 S1 ... --interp-weights w0 w1 ...`` stylises with the weighted blend of 1..8
styles (weights >= 0, normalised to sum 1; WCT or ``--adain``); the output is ``<content>_<s0>-<w0>+<s1>-<w1>...<ext>``
with the normalised weights.

Texture synthesis: ``--noise [--noise-size H W] [--noise-count K] [--noise-seed S]`` replaces ``--content-path`` by K frames of
seeded uniform noise made on the device (default one 512x512 frame, seed 0), stylised in one batch per style, blend or mask;
the outputs are named as above with the content ``noise<S>-<i>.png``, e.g. ``noise0-3_starry.png``.

Prepared styles: ``--style-path``, ``--interp-styles`` and ``--mask-styles`` also take ``.wctstyle`` files written by
``prepare_styles.py`` (in a folder, the entries ending in ``.wctstyle``).  Each is read once per run and reused for every
content, pass and noise batch.  A run's styles are all prepared or all images, and prepared styles take no ``--style-size``,
``--crop-size`` or ``--keep-colors`` (their size and crop were fixed when they were prepared).

Tiled stylisation: ``--tile-size T`` (a multiple of 16; 0: off) runs every level on T x T tiles widened by a halo, so device
memory follows the tile and not the image, with each level's statistics taken over the whole image (DESIGN.md §3.3.7).
``--keep-colors``, ``--concat``, ``--content-size``, ``--passes`` and ``--noise`` work on the whole image as without it.

Optimal-transport transform: ``--ost`` maps each level's content feature Gaussian onto the style's by the Monge map, the
covariance-matching map that moves the features least, instead of WCT (DESIGN.md §3.3.8); it keeps more of the content's
structure at the same ``--alpha``.  Output names are unchanged.

Seamless stylisation: ``--seamless {x,y,xy}`` pads every conv of the content path circularly along those axes (DESIGN.md
§3.3.9), so the result's opposite edges meet: ``x`` for 360° equirectangular panoramas, ``xy`` for tileable textures
(``--noise --seamless xy``).  Each wrapped side must be a multiple of 2^P, P the pools up to the deepest relu target (16
for relu5_1).  Output names are unchanged.

Multimodal style transfer: ``--mst K [--mst-smooth LAMBDA]`` clusters each level's style features into K (1..8) modes and
matches every content pixel to the mode it resembles, with a Potts smoothness of weight LAMBDA (default 0.05), so regions
of the content pair up with modes of the painting without masks (DESIGN.md §3.3.10).  Output names are unchanged.

Exact feature distribution matching: ``--efdm`` gives every channel of each level the whole value distribution of the same
channel of the style, by rank, instead of matching only its covariance (DESIGN.md §3.3.12): sparse bright strokes and an
even wash with the same statistics stylise differently.  It suits ``--noise`` texture synthesis.  Output names are
unchanged.

Sliced distribution matching: ``--efdm-slices K`` (0..32, with ``--efdm``) first runs EFDM in K random rotations of each
level's channels, each on the previous one's output, so that how the channels go together is matched too and not only
each channel's own values (DESIGN.md §3.3.14).  0 is plain ``--efdm``.  Output names are unchanged.

Softmax swap: ``--ss-temperature T`` (T > 0, with ``--swap5`` / ``--swap-targets``) rebuilds every content patch from a
blend of style patches weighted by a softmax of their scores at temperature T, instead of its single best patch (DESIGN.md
§3.3.17).  Small T approaches the hard swap; larger T blends more patches, which softens the seams between neighbouring
patches (about 0.003 blends a few patches per anchor at relu3_1).  Output names are unchanged.

Balanced swap: ``--ss-balance T`` (1..256, with ``--ss-temperature``) runs T Sinkhorn iterations on the softmax swap's
weights, so that the style patches are used about evenly instead of a few of them covering large regions (DESIGN.md
§3.3.18).  Each iteration costs about one more pass over the patch scores.  0 is the softmax swap.  Output names are
unchanged.

Labelled style swap (neural doodle): ``--swap-labels CONTENT_MAP STYLE_MAP`` with ``--swap5`` / ``--swap-targets`` gives
the content and the style each a flat-colour label map (RGB or grey PNG, any resolution); every content patch is then
rebuilt only from style patches of the same colour, or from all of them where the style has none (DESIGN.md §3.3.13).  The
distinct colours of both maps together, sorted by their packed 24-bit value, are the labels.  It takes one style file and
one content file or ``--noise`` (every noise frame shares the map), and no ``--crop-size``.  Output names are unchanged.

Colour preservation: ``--luminance-only`` stylises the luminance only and puts the content's own colours back on the
result, so the output keeps the content's palette and takes brightness and texture from the style (DESIGN.md §3.3.15).
It combines with the options above; not with ``--keep-colors`` or ``--noise``, and a ``.wctstyle`` style must have been
prepared with ``prepare_styles.py --luminance-only``.  ``--passes`` then run in one call and the colours are merged once,
after the last.  Output names are unchanged.

Scale control: ``--coarse-to-fine F`` (2..16; 0 is off) stylises a copy of the content at about 1/F of its size at every
level first, puts that result's low band into the content, and then runs only the fine levels (``--fine-targets``; default
those of relu3_1, relu2_1 and relu1_1 among ``--relu-targets``) at full size (DESIGN.md §3.3.16).  The style's large
structures then come out about F times larger on a large image while its fine texture keeps its own scale, and the deep
levels run on 1/F^2 of the pixels.  Not with the style swap, ``--seamless`` or ``--mst``.  Output names are unchanged.

Which of these options combine is decided by one table, ``wct_tf_b200/options.py``; a rejected combination is a parser error
naming both flags.

``--checkpoints`` are TF1 checkpoint directories or ``.npz`` bundles, ``--vgg-path`` a Torch7 ``.t7`` or ``.npz`` file
(wct_tf_b200.weights.load_weights); ``--synthetic-weights SEED`` runs with seeded random weights when the published
models are not on disk (offline build).
"""
from __future__ import division, print_function

import argparse
import os
import time

import numpy as np

# (flags, kwargs) -- names and defaults follow the reference one to one (tests/test_cli.py pins them)
_FLAGS = [
    (("--checkpoints",), dict(nargs="+", type=str, help="one decoder checkpoint (TF dir or .npz) per entry of --relu-targets")),
    (("--relu-targets",), dict(nargs="+", type=str, required=True, help="reluX_1 levels in pipeline order, paired with --checkpoints")),
    (("--vgg-path",), dict(type=str, default="models/vgg_normalised.t7", help="normalised VGG19 encoder (.t7 or .npz)")),
    (("--content-path",), dict(type=str, dest="content_path", help="content image, or a folder of them")),
    (("--style-path",), dict(type=str, dest="style_path", help="style image, or a folder of them")),
    (("--out-path",), dict(type=str, dest="out_path", help="folder that receives <content>_<style>.<ext>")),
    (("--keep-colors",), dict(action="store_true", default=False, help="CORAL: give the style the content's colours first")),
    (("--device",), dict(type=str, default="/gpu:0", help="/gpu:N (TF spelling), cuda:N or N")),
    (("--style-size",), dict(type=int, default=0, help="short side of the style before cropping (0: keep)")),
    (("--crop-size",), dict(type=int, default=0, help="centre-crop the style to a square of this size (0: off)")),
    (("--content-size",), dict(type=int, default=0, help="short side of the content (0: keep)")),
    (("--passes",), dict(type=int, default=1, help="feed the result back as content this many times")),
    (("-r", "--random"), dict(type=int, default=0, help="use a random subset of this many styles from the style folder")),
    (("--alpha",), dict(type=float, default=1, help="stylised / content feature blend")),
    (("--concat",), dict(action="store_true", default=False, help="write [style | result] side by side")),
    (("--adain",), dict(action="store_true", default=False, help="AdaIN statistics matching instead of WCT")),
    (("--swap5",), dict(action="store_true", default=False, help="style swap at relu5_1 (patch 3, stride 1)")),
    (("--swap-targets",), dict(nargs="+", type=str, default=None, metavar="RELU",
                               help="style swap at these --relu-targets levels (e.g. relu3_1 for brush strokes); not with --swap5")),
    (("--ss-alpha",), dict(type=float, default=0.6, help="blend of the style-swapped feature")),
    (("--ss-temperature",), dict(type=float, default=None, metavar="T",
                                 help="with --swap5 / --swap-targets: softmax swap, each content patch a blend of style patches "
                                      "weighted by a softmax of their scores at temperature T > 0 (not in the reference)")),
    (("--ss-balance",), dict(type=int, default=None, metavar="T",
                             help="with --ss-temperature: balanced swap, T in 1..256 Sinkhorn iterations that spread the "
                                  "softmax swap's use of the style patches evenly; 0 is the softmax swap (not in the reference)")),
    (("--ss-patch-size",), dict(type=int, default=3)),
    (("--ss-stride",), dict(type=int, default=1)),
    # not in the reference
    (("--synthetic-weights",), dict(type=int, default=None, help="seeded random weights (no model files needed)")),
    (("--semantics",), dict(type=str, default="tf", choices=["tf", "np"], help="wct_tf (the reference graph) or wct_np eps/blend rules")),
    (("--content-mask",), dict(type=str, default=None, help="8-bit grayscale region mask: gray v -> region v*R//256 (R = #--mask-styles)")),
    (("--mask-styles",), dict(nargs="+", type=str, default=None, help="one style image per mask region (with --content-mask)")),
    (("--style-masks",), dict(nargs="+", type=str, default=None,
                              help="one 8-bit grayscale mask per --mask-styles entry: region r takes the pixels of style r in region r")),
    (("--interp-styles",), dict(nargs="+", type=str, default=None, help="1..8 style images to blend (with --interp-weights)")),
    (("--interp-weights",), dict(nargs="+", type=float, default=None, help="one weight >= 0 per --interp-styles entry (normalised)")),
    (("--ost",), dict(action="store_true", default=False,
                      help="optimal-transport (Monge) map between the feature Gaussians instead of WCT")),
    (("--tile-size",), dict(type=int, default=0, metavar="T",
                            help="stylise in T x T tiles (a multiple of 16) in bounded device memory, with every level's "
                                 "statistics over the whole image (0: off)")),
    (("--seamless",), dict(type=str, default=None, choices=["x", "y", "xy"],
                           help="wrap-around padding along x, y or both: panoramas (x) and tileable textures (xy)")),
    (("--mst",), dict(type=int, default=None, metavar="K",
                      help="multimodal style transfer: cluster each level's style into K modes (1..8) and match the content to them")),
    (("--mst-smooth",), dict(type=float, default=None, metavar="LAMBDA",
                             help="with --mst: Potts smoothness of the content labelling, finite and >= 0 (default 0.05)")),
    (("--efdm",), dict(action="store_true", default=False,
                       help="exact feature distribution matching: give every channel the style's whole value distribution")),
    (("--efdm-slices",), dict(type=int, default=0, metavar="K",
                              help="with --efdm: match in K random channel rotations first, then per channel (0..32, "
                                   "default 0)")),
    (("--strength-map",), dict(type=str, default=None, metavar="PATH",
                               help="8-bit grayscale map of the per-pixel stylisation strength (gray v -> v/255)")),
    (("--mask-feather",), dict(type=float, default=None, metavar="SIGMA",
                               help="with --content-mask: feather the region edges by a Gaussian of SIGMA mask pixels")),
    (("--mask-weights",), dict(nargs="+", type=str, default=None, metavar="W",
                               help="one 8-bit grayscale soft weight map per --mask-styles entry, in place of --content-mask")),
    (("--luminance-only",), dict(action="store_true", default=False,
                                 help="stylise the luminance only and keep the content's colours (not with --keep-colors)")),
    (("--coarse-to-fine",), dict(type=int, default=0, metavar="F",
                                 help="scale control: stylise a 1/F copy at every level, then the --fine-targets at full size "
                                      "(2..16; 0: off)")),
    (("--fine-targets",), dict(nargs="+", type=str, default=None, metavar="RELU",
                               help="with --coarse-to-fine: the levels run at full size (default: relu3_1 relu2_1 relu1_1 "
                                    "among --relu-targets)")),
    (("--swap-labels",), dict(nargs=2, type=str, default=None, metavar=("CONTENT_MAP", "STYLE_MAP"),
                              help="with --swap5 / --swap-targets: flat-colour label maps of the content and the style; each "
                                   "content patch takes only style patches of its own colour")),
    # webcam.py:38; the three --noise-* flags are not in the reference.  Their defaults are filled in by parse_args, so that
    # giving one without --noise can be told from leaving it out.
    (("--noise",), dict(action="store_true", default=False, help="Synthesize textures from noise images")),
    (("--noise-size",), dict(nargs=2, type=int, default=None, metavar=("H", "W"), help="size of the noise frames (default 512 512)")),
    (("--noise-count",), dict(type=int, default=None, metavar="K", help="noise frames, one texture each (default 1)")),
    (("--noise-seed",), dict(type=int, default=None, metavar="S", help="seed of the noise frames, 0 .. 2^64-1 (default 0)")),
]
_NOISE_DEFAULTS = [("noise_size", [512, 512]), ("noise_count", 1), ("noise_seed", 0)]

# flags of the one-style mode that the multi-style modes (--content-mask / --mask-weights, --interp-styles) take no part of
_MULTI_EXCLUDES = [("style_path", "--style-path"), ("random", "-r/--random"), ("concat", "--concat")]


def build_parser():
    parser = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    for names, kw in _FLAGS:
        parser.add_argument(*names, **kw)
    return parser


def parse_args(argv=None):
    parser = build_parser()
    args = parser.parse_args(argv)
    check_swap_flags(parser, args)
    check_interp_flags(parser, args)
    check_values(parser, args)
    check_options(parser, args)
    check_luminance_flags(parser, args)
    if args.content_mask is not None:
        if not args.mask_styles:
            parser.error("--content-mask needs --mask-styles")
    elif args.mask_weights is not None:
        if not args.mask_styles or len(args.mask_weights) != len(args.mask_styles):
            parser.error("--mask-weights needs one map per --mask-styles entry")
    elif args.mask_styles:
        parser.error("--mask-styles needs --content-mask")
    if args.mask_styles and len(args.mask_styles) > 8:
        parser.error("--mask-styles takes at most 8 styles")
    mode = "--content-mask" if args.content_mask is not None else "--mask-weights" if args.mask_weights is not None else None
    for attr, flag in _MULTI_EXCLUDES if mode else []:
        if getattr(args, attr):
            parser.error("%s takes no %s" % (mode, flag))
    check_style_mask_flags(parser, args)
    check_noise_flags(parser, args)
    check_prepared_flags(parser, args)
    check_swap_label_flags(parser, args)
    return args


def check_swap_flags(parser, args):
    """--swap-targets: levels of --relu-targets, not with --swap5 (which is --swap-targets relu5_1)."""
    if args.swap_targets is None:
        return
    if args.swap5:
        parser.error("give --swap5 or --swap-targets, not both (--swap5 is --swap-targets relu5_1)")
    for relu in args.swap_targets:
        if relu not in (args.relu_targets or []):
            parser.error("--swap-targets: %s is not one of --relu-targets (%s)" % (relu, " ".join(args.relu_targets or [])))


MST_SMOOTH_DEFAULT = 0.05


def read_label_maps(content_map, style_map):
    """Two flat-colour label map files -> uint8 labels (content [H,W], style [H',W']): the distinct colours of both maps
    together, sorted by their packed 24-bit RGB value, become labels 0..K-1.  ValueError for more than 256 colours."""
    from PIL import Image
    packed = []
    for path in (content_map, style_map):
        rgb = np.asarray(Image.open(path).convert("RGB"), dtype=np.uint32)
        packed.append((rgb[..., 0] << 16) | (rgb[..., 1] << 8) | rgb[..., 2])
    colours, inverse = np.unique(np.concatenate([p.ravel() for p in packed]), return_inverse=True)
    if len(colours) > 256:
        raise ValueError("%d colours in the two label maps, at most 256: label maps must be flat colours (PNG, not JPEG)"
                         % len(colours))
    labels = inverse.astype(np.uint8)
    n = packed[0].size
    return labels[:n].reshape(packed[0].shape), labels[n:].reshape(packed[1].shape)


def check_swap_label_flags(parser, args):
    """--swap-labels CONTENT_MAP STYLE_MAP: needs --swap5 / --swap-targets, one --style-path file (image or .wctstyle; no
    folder, no -r), one --content-path file or --noise, and no --crop-size (a crop would cut the style but not its map).
    The maps are read here (``read_label_maps``) into ``args.swap_label_maps``."""
    if args.swap_labels is None:
        return
    if not (args.swap5 or args.swap_targets is not None):
        parser.error("--swap-labels needs --swap5 or --swap-targets")
    if not args.style_path or os.path.isdir(args.style_path) or args.random:
        parser.error("--swap-labels needs one --style-path file (no folder, no -r/--random)")
    if not args.noise and (not args.content_path or os.path.isdir(args.content_path)):
        parser.error("--swap-labels needs one --content-path file or --noise")
    if args.crop_size:
        parser.error("--swap-labels takes no --crop-size")
    try:
        args.swap_label_maps = read_label_maps(*args.swap_labels)
    except (OSError, ValueError) as e:
        parser.error("--swap-labels: %s" % e)


def check_values(parser, args):
    """The values of --tile-size (0: off), --mst / --mst-smooth (which needs --mst and defaults to 0.05 here),
    --mask-feather, --efdm-slices, --coarse-to-fine / --fine-targets and --temporal (stylize_video.py), as
    wct_tf_b200/options.py checks them."""
    from wct_tf_b200 import options
    try:
        if getattr(args, "tile_size", 0):
            options.check_tile_size(args.tile_size, "--tile-size")
        if args.mst is None and args.mst_smooth is not None:
            raise ValueError("--mst-smooth needs --mst")
        if args.mst is not None:
            if args.mst_smooth is None:
                args.mst_smooth = MST_SMOOTH_DEFAULT
            options.check_mst(args.mst, args.mst_smooth, ("--mst", "--mst-smooth"))
        if getattr(args, "mask_feather", None) is not None:
            options.check_mask_feather(args.mask_feather, "--mask-feather")
        options.check_efdm_slices(args.efdm_slices, args.efdm, options.CLI)
        options.check_ss_temperature(args.ss_temperature, args.swap5 or args.swap_targets is not None, options.CLI)
        if args.ss_balance is not None:
            options.check_ss_balance(args.ss_balance, args.ss_temperature, options.CLI)
        if getattr(args, "coarse_to_fine", 0) or getattr(args, "fine_targets", None) is not None:
            options.check_coarse_to_fine(args.coarse_to_fine or None, args.fine_targets, args.relu_targets or [], options.CLI)
        if hasattr(args, "temporal"):
            options.check_temporal_strength(args.temporal, "--temporal")
    except ValueError as e:
        parser.error(str(e))


def check_options(parser, args):
    """The combinations of the stylising flags that wct_tf_b200/options.py rejects, as parser errors naming both flags."""
    from wct_tf_b200 import options
    style_path = getattr(args, "style_path", None)
    on = dict(adain=args.adain, ost=args.ost, efdm=args.efdm, mst=args.mst is not None,
              swap=args.swap5 or args.swap_targets is not None, content_mask=getattr(args, "content_mask", None) is not None,
              style_masks=getattr(args, "style_masks", None) is not None, style_weights=args.interp_styles is not None,
              content_weights=getattr(args, "mask_weights", None) is not None,
              mask_feather=getattr(args, "mask_feather", None) is not None, strength_map=args.strength_map is not None,
              tile_size=bool(getattr(args, "tile_size", 0)), seamless=args.seamless is not None,
              temporal=bool(getattr(args, "temporal", 0)), luminance_only=getattr(args, "luminance_only", False),
              coarse_to_fine=bool(getattr(args, "coarse_to_fine", 0)),
              prepared=bool(style_path) and (is_prepared(style_path) or (os.path.isdir(style_path)
                                                                         and any(is_prepared(f) for f in os.listdir(style_path)))))
    try:
        options.check({name for name, v in on.items() if v}, options.CLI)
    except ValueError as e:
        parser.error(str(e))


def check_luminance_flags(parser, args):
    """--luminance-only: not with --keep-colors (both decide the output's colours) or --noise (noise has no colours to
    keep).  A .wctstyle style must have been prepared with prepare_styles.py --luminance-only; the model checks that when
    it reads the file."""
    if not getattr(args, "luminance_only", False):
        return
    if args.keep_colors:
        parser.error("--luminance-only does not combine with --keep-colors: both decide the colours")
    if getattr(args, "noise", False):
        parser.error("--luminance-only takes no --noise: noise frames have no colours to keep")


def run_passes(model, content_dev, styles, args, kw):
    """stylize.py:100-104: --passes calls, each on the previous result.  With --luminance-only the passes run in one call
    on the grey frames and the colours are merged once, after the last (the style swap then acts in the first pass)."""
    if getattr(args, "luminance_only", False):
        return model.predict_batch(content_dev, styles, luminance_only=True, passes=args.passes, **kw)
    result = model.predict_batch(content_dev, styles, **kw)
    for _ in range(args.passes - 1):
        result = model.predict_batch(result, styles, **kw)
    return result


def read_grey(path):
    """8-bit grayscale map file -> uint8 [H, W] (read as v/255 by the soft spatial-control options)."""
    from PIL import Image
    return np.asarray(Image.open(path).convert("L"), dtype=np.uint8)


def scale_kw(args):
    """predict_batch options of scale control (--coarse-to-fine, --fine-targets) from the parsed flags."""
    if not getattr(args, "coarse_to_fine", 0):
        return {}
    return dict(coarse_to_fine=args.coarse_to_fine, fine_targets=args.fine_targets)


def soft_kw(args):
    """predict_batch options of soft spatial control from the parsed flags."""
    kw = {}
    if getattr(args, "strength_map", None):
        kw["strength_map"] = read_grey(args.strength_map)
    if getattr(args, "mask_feather", None) is not None:
        kw["mask_feather"] = float(args.mask_feather)
    if getattr(args, "mask_weights", None):
        kw["content_weights"] = np.stack([read_grey(p) for p in args.mask_weights])
    return kw


def check_style_mask_flags(parser, args):
    """--style-masks: one mask per --mask-styles entry, with --content-mask; not with --crop-size (a crop moves the style
    off its mask) or prepared styles (they keep no feature maps to mask).  --style-size scales style and mask alike."""
    if args.style_masks is None:
        return
    if args.content_mask is None and getattr(args, "mask_weights", None) is None:
        parser.error("--style-masks needs --content-mask (or --mask-weights)")
    if len(args.style_masks) != len(args.mask_styles):
        parser.error("--style-masks needs one mask per --mask-styles entry (%d masks, %d styles)"
                     % (len(args.style_masks), len(args.mask_styles)))
    if args.crop_size:
        parser.error("--style-masks takes no --crop-size")
    if any(is_prepared(p) for p in args.mask_styles):
        parser.error("--style-masks takes no prepared styles (.wctstyle)")


PREPARED_EXT = ".wctstyle"


def is_prepared(path):
    return str(path).endswith(PREPARED_EXT)


def style_listing(path, io):
    """A style path as a list: a file, or a folder's images (imageio.get_files) and its ``.wctstyle`` files."""
    if not os.path.isdir(path):
        return [path]
    prepared = sorted(os.path.join(path, f) for f in os.listdir(path) if is_prepared(f))
    return [p for p in io.get_files(path) if not is_prepared(p)] + prepared


def check_prepared_flags(parser, args, flags=("style_size", "crop_size", "keep_colors")):
    """A run's styles are all prepared (.wctstyle) or all images; prepared styles were sized and cropped when they were
    prepared, and CORAL (--keep-colors) changes the style per content."""
    from wct_tf_b200 import imageio as io
    paths = []
    if getattr(args, "style_path", None):
        paths += style_listing(args.style_path, io) if os.path.isdir(args.style_path) else [args.style_path]
    paths += list(getattr(args, "interp_styles", None) or []) + list(getattr(args, "mask_styles", None) or [])
    kinds = set(is_prepared(p) for p in paths)
    if True not in kinds:
        return
    if len(kinds) > 1:
        parser.error("prepared styles (.wctstyle) and style images do not mix in one run")
    for attr in flags:
        if getattr(args, attr, None):
            parser.error("prepared styles (.wctstyle) take no --%s" % attr.replace("_", "-"))


class PreparedStyles(object):
    """Reads each ``.wctstyle`` file once per run (``model.load_style``) and hands out the same prepared style after."""

    def __init__(self, model):
        self.model, self.cache = model, {}

    def get(self, path):
        if path not in self.cache:
            self.cache[path] = self.model.load_style(path)
        return self.cache[path]


def check_noise_flags(parser, args):
    """--noise replaces the content images; the --noise-* flags need it, and get their defaults here."""
    if not args.noise:
        for attr, _ in _NOISE_DEFAULTS:
            if getattr(args, attr) is not None:
                parser.error("--%s needs --noise" % attr.replace("_", "-"))
        return
    if args.content_path is not None or args.content_size or args.keep_colors:
        parser.error("--noise takes no --content-path, --content-size or --keep-colors")
    for attr, default in _NOISE_DEFAULTS:
        if getattr(args, attr) is None:
            setattr(args, attr, default)
    if min(args.noise_size) < 1:
        parser.error("--noise-size must be positive")
    if args.noise_count < 1:
        parser.error("--noise-count must be >= 1")
    if not 0 <= args.noise_seed < 2 ** 64:
        parser.error("--noise-seed must be in 0 .. 2^64-1")


def check_interp_flags(parser, args, excludes=_MULTI_EXCLUDES):
    """--interp-styles / --interp-weights: each needs the other, one weight per style, 1..8 styles, valid weights."""
    if args.interp_styles is None and args.interp_weights is None:
        return
    if args.interp_styles is None:
        parser.error("--interp-weights needs --interp-styles")
    if args.interp_weights is None:
        parser.error("--interp-styles needs --interp-weights")
    if len(args.interp_styles) != len(args.interp_weights):
        parser.error("--interp-styles and --interp-weights must have the same length")
    if len(args.interp_styles) > 8:
        parser.error("--interp-styles takes at most 8 styles")
    for attr, flag in excludes:
        if getattr(args, attr, None):
            parser.error("--interp-styles takes no %s" % flag)
    try:
        normalized_weights(args.interp_weights)
    except ValueError as e:
        parser.error("--interp-weights: %s" % e)


def normalized_weights(weights):
    """One weight row -> float64 weights that sum to 1 (WCT.normalize_weights: finite, >= 0, positive sum)."""
    from wct_tf_b200.wct import WCT
    return WCT.normalize_weights(weights, 1, len(weights), dtype=np.float64)[0]


def interp_label(style_paths, weights):
    """``<s0>-<w0>+<s1>-<w1>...`` with the normalised weights printed with %g."""
    return "+".join("{}-{:g}".format(os.path.splitext(os.path.basename(p))[0], w)
                    for p, w in zip(style_paths, normalized_weights(weights)))


def interp_output_name(content_path, style_paths, weights):
    stem, ext = os.path.splitext(os.path.basename(content_path))
    return "{}_{}{}".format(stem, interp_label(style_paths, weights), ext)


def read_mask(path, R):
    """8-bit grayscale mask file -> uint8 region labels: gray value v -> region v*R // 256."""
    from PIL import Image
    gray = np.asarray(Image.open(path).convert("L"), dtype=np.int64)
    return ((gray * R) // 256).astype(np.uint8)


def mask_output_name(content_path, style_paths):
    stem, ext = os.path.splitext(os.path.basename(content_path))
    return "{}_{}{}".format(stem, "+".join(os.path.splitext(os.path.basename(p))[0] for p in style_paths), ext)


def _listing(path, io):
    return io.get_files(path) if os.path.isdir(path) else [path]


def noise_names(seed, count):
    """Content names of the --noise frames: ``noise<S>-<i>.png``."""
    return ["noise{}-{}.png".format(seed, i) for i in range(count)]


def _contents(args, io, dimg, device):
    """Yields (names, content on the device): each image of --content-path alone ([its path], HxWx3), or with --noise the
    K noise frames as one batch (``noise_names``, [K,H,W,3]) so that they are stylised in one call per style."""
    if args.noise:
        H, W = args.noise_size
        yield noise_names(args.noise_seed, args.noise_count), dimg.noise_u8(args.noise_count, H, W, seed=args.noise_seed,
                                                                           device=device)
        return
    for content_path in _listing(args.content_path, io):
        content_dev = dimg.to_device(io.get_img(content_path), device)
        if args.content_size > 0:
            content_dev = dimg.resize_to(content_dev, args.content_size)
        yield [content_path], content_dev


def _prepare_style(path, args, io, dimg, content_dev, device, prepared=None):
    """stylize.py:86-95 on the device: decode on the host, then resize / crop / CORAL without leaving the GPU.  A
    ``.wctstyle`` file gives its prepared style (``prepared``: the run's PreparedStyles)."""
    if is_prepared(path):
        return prepared.get(path)
    img = dimg.to_device(io.get_img(path), device)
    if args.style_size > 0:
        img = dimg.resize_to(img, args.style_size)
    if args.crop_size > 0:
        img = dimg.center_crop(img, args.crop_size)
    if args.keep_colors:
        img = dimg.preserve_colors_np(img, content_dev)
    return img


def _stylize_pair(model, content_dev, style_dev, args):
    """stylize.py:100-104; every pass takes and returns uint8 frames on the device (no host round trip between passes)."""
    kw = dict(alpha=args.alpha, swap5=args.swap5, ss_alpha=args.ss_alpha, adain=args.adain, return_device=True)
    if args.swap_targets:
        kw["swap_targets"] = list(args.swap_targets)
    if args.ss_temperature is not None:
        kw["ss_temperature"] = args.ss_temperature
    if args.ss_balance is not None:
        kw["ss_balance"] = args.ss_balance
    if args.tile_size:
        kw["tile_size"] = args.tile_size
    if args.ost:
        kw["ost"] = True
    if args.seamless:
        kw["seamless"] = args.seamless
    if args.mst is not None:
        kw.update(mst=args.mst, mst_smooth=args.mst_smooth)
    if args.efdm:
        kw["efdm"] = True
    if args.efdm_slices:
        kw["efdm_slices"] = args.efdm_slices
    if getattr(args, "swap_labels", None):
        kw["swap_labels"] = args.swap_label_maps
    kw.update(soft_kw(args), **scale_kw(args))
    return run_passes(model, content_dev, style_dev, args, kw)


def make_model(args):
    from wct_tf_b200.wct import WCT
    weights = None
    if args.synthetic_weights is not None:
        from wct_tf_b200.weights import make_synthetic_weights
        weights = make_synthetic_weights(args.synthetic_weights, relu_targets=args.relu_targets)
    elif not args.checkpoints:
        raise SystemExit("--checkpoints is required (or --synthetic-weights SEED)")
    return WCT(checkpoints=args.checkpoints, relu_targets=args.relu_targets, vgg_path=args.vgg_path, device=args.device,
               ss_patch_size=args.ss_patch_size, ss_stride=args.ss_stride, weights=weights, semantics=args.semantics, verbose=True)


def _stylize_masked(model, content_dev, styles_dev, labels, args, style_masks=None):
    kw = dict(alpha=args.alpha, return_device=True)
    if labels is not None:
        kw["content_mask"] = labels
    kw.update(soft_kw(args), **scale_kw(args))
    if args.seamless:
        kw["seamless"] = args.seamless
    if style_masks is not None:
        kw["style_masks"] = style_masks
    return run_passes(model, content_dev, styles_dev, args, kw)


def _once_per_path(paths, load):
    """``load(path)`` once per distinct path; a repeated path gives the same object again."""
    cache = {}
    for p in paths:
        if p not in cache:
            cache[p] = load(p)
    return [cache[p] for p in paths]


def main_masked(args, model, io, dimg, t_start):
    """--content-mask: every content image, split by the mask, with region r in style r (with --style-masks, in the
    pixels of style r labelled r).  A path given twice is loaded once and passed as the same object, so that one style
    with one mask for several regions is encoded once."""
    R = len(args.mask_styles)
    labels = read_mask(args.content_mask, R) if args.content_mask is not None else None
    style_masks = _once_per_path(args.style_masks, lambda p: read_mask(p, R)) if args.style_masks else None
    os.makedirs(args.out_path, exist_ok=True)
    device = model.engine.device
    written = 0
    prepared = PreparedStyles(model)
    for names, content_dev in _contents(args, io, dimg, device):
        styles_dev = _once_per_path(args.mask_styles, lambda p: _prepare_style(p, args, io, dimg, content_dev, device, prepared))
        results = _stylize_masked(model, content_dev, styles_dev, labels, args, style_masks)
        for name, result in zip(names, results):
            target = os.path.join(args.out_path, mask_output_name(name, args.mask_styles))
            io.save_img(target, dimg.to_host(result))
            written += 1
            print("{}: Wrote stylized output image to {}".format(written, target))
    print("Finished stylizing {} outputs in {}s".format(written, time.time() - t_start))
    return written


def main_interp(args, model, io, dimg, t_start):
    """--interp-styles: every content image in the weighted blend of the styles."""
    os.makedirs(args.out_path, exist_ok=True)
    device = model.engine.device
    kw = dict(alpha=args.alpha, adain=args.adain, return_device=True, style_weights=np.asarray(args.interp_weights, np.float64),
              **scale_kw(args))
    if args.seamless:
        kw["seamless"] = args.seamless
    written = 0
    prepared = PreparedStyles(model)
    for names, content_dev in _contents(args, io, dimg, device):
        styles_dev = [_prepare_style(p, args, io, dimg, content_dev, device, prepared) for p in args.interp_styles]
        results = run_passes(model, content_dev, styles_dev, args, kw)
        for name, result in zip(names, results):
            target = os.path.join(args.out_path, interp_output_name(name, args.interp_styles, args.interp_weights))
            io.save_img(target, dimg.to_host(result))
            written += 1
            print("{}: Wrote stylized output image to {}".format(written, target))
    print("Finished stylizing {} outputs in {}s".format(written, time.time() - t_start))
    return written


def main(argv=None, model_factory=make_model, image_ops=None):
    args = parse_args(argv)
    from wct_tf_b200 import imageio as io
    if image_ops is None:
        from wct_tf_b200 import device_image as image_ops
    dimg = image_ops
    t_start = time.time()
    model = model_factory(args)
    if args.interp_styles is not None:
        return main_interp(args, model, io, dimg, t_start)
    if args.content_mask is not None or args.mask_weights is not None:
        return main_masked(args, model, io, dimg, t_start)
    styles = style_listing(args.style_path, io)
    if os.path.isdir(args.style_path) and args.random > 0:
        styles = list(np.random.choice(styles, args.random))
    os.makedirs(args.out_path, exist_ok=True)

    device = model.engine.device
    written = 0
    prepared = PreparedStyles(model)
    for names, content_dev in _contents(args, io, dimg, device):
        for style_path in styles:
            style_dev = _prepare_style(style_path, args, io, dimg, content_dev, device, prepared)
            results = _stylize_pair(model, content_dev, style_dev, args)
            for name, result in zip(names, results):
                if args.concat:
                    # a prepared style keeps its image on the host for this
                    shown = dimg.to_device(style_dev.image[0], device) if is_prepared(style_path) else style_dev
                    result = dimg.concat_with_style(shown, result)
                stem, ext = os.path.splitext(os.path.basename(name))
                target = os.path.join(args.out_path, "{}_{}{}".format(stem, os.path.splitext(os.path.basename(style_path))[0], ext))
                io.save_img(target, dimg.to_host(result))
                written += 1
                print("{}: Wrote stylized output image to {}".format(written, target))
    print("Finished stylizing {} outputs in {}s".format(written, time.time() - t_start))
    return written


if __name__ == "__main__":
    main()
