#!/usr/bin/env python
"""Prepare styles once: encode each style image and decompose it at every relu target, and write one ``<stem>.wctstyle``
per style to ``--out-path``.  ``stylize.py`` and ``stylize_video.py`` take these files wherever they take a style image.

  python prepare_styles.py --checkpoints DIR5 DIR4 ... --relu-targets relu5_1 relu4_1 ... --vgg-path vgg_normalised.t7 \\
      --style-path STYLES --out-path PREPARED [--style-size S] [--crop-size C] [--semantics tf|np]

A file holds the (resized, cropped) style image, the WCT and AdaIN statistics of every target and the relu5_1 feature (for
``--swap5``), and with ``--swap-targets reluX_1 ...`` the feature of those levels too (for ``--swap-targets``).  It serves any model with the same encoder weights and semantics, whatever its decoders, and any subset of
its targets; the model refuses it otherwise.  ``--luminance-only`` prepares the grey of each style (same file name), which
is the form ``--luminance-only`` stylisation takes.
"""
from __future__ import print_function

import argparse
import os
import time

# the model flags of stylize.py, and the style flags
_MODEL_FLAGS = ("--checkpoints", "--relu-targets", "--vgg-path", "--device", "--synthetic-weights", "--semantics")


def build_parser():
    import stylize
    parser = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    for names, kw in stylize._FLAGS:
        if names[0] in _MODEL_FLAGS:
            parser.add_argument(*names, **kw)
    parser.add_argument("--style-path", type=str, required=True, help="style image, or a folder of them")
    parser.add_argument("--style-size", type=int, default=0, help="short side of the style before cropping (0: keep)")
    parser.add_argument("--crop-size", type=int, default=0, help="centre-crop the style to a square of this size (0: off)")
    parser.add_argument("--out-path", type=str, required=True, help="folder that receives <stem>.wctstyle")
    parser.add_argument("--swap-targets", nargs="+", type=str, default=None, metavar="RELU",
                        help="also keep the style feature of these --relu-targets levels, for the style swap there")
    parser.add_argument("--luminance-only", action="store_true", default=False,
                        help="prepare the grey of each style, for stylize.py / stylize_video.py --luminance-only")
    return parser


def output_name(style_path):
    return os.path.splitext(os.path.basename(style_path))[0] + ".wctstyle"


def main(argv=None, model_factory=None, image_ops=None):
    import stylize
    parser = build_parser()
    args = parser.parse_args(argv)
    for relu in args.swap_targets or []:
        if relu not in args.relu_targets:
            parser.error("--swap-targets: %s is not one of --relu-targets (%s)" % (relu, " ".join(args.relu_targets)))
    from wct_tf_b200 import imageio as io
    if image_ops is None:
        from wct_tf_b200 import device_image as image_ops
    args.ss_patch_size, args.ss_stride = 3, 1
    model = (model_factory or stylize.make_model)(args)
    styles = [p for p in stylize.style_listing(args.style_path, io) if not stylize.is_prepared(p)]
    os.makedirs(args.out_path, exist_ok=True)
    device = model.engine.device
    t0 = time.time()
    for path in styles:
        img = image_ops.to_device(io.get_img(path), device)
        if args.style_size > 0:
            img = image_ops.resize_to(img, args.style_size)
        if args.crop_size > 0:
            img = image_ops.center_crop(img, args.crop_size)
        target = os.path.join(args.out_path, output_name(path))
        kw = dict(swap_targets=list(args.swap_targets)) if args.swap_targets else {}
        if args.luminance_only:
            kw["luminance_only"] = True
        model.prepare_style(img, **kw).save(target)
        print("Prepared {} -> {}".format(path, target))
    print("Prepared {} styles in {:.2f}s".format(len(styles), time.time() - t0))
    return len(styles)


if __name__ == "__main__":
    main()
