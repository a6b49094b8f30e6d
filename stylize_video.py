#!/usr/bin/env python
"""Video / frame-sequence driver with the reference's flags (stylize_video.py:17-42 of eridgd/WCT-TF).

The reference splits the video into PNG frames with ffmpeg, calls ``WCT.predict`` once per frame and re-encodes
(stylize_video.py:75-149).  Here frames go through ``WCT.predict_batch`` in batches that share ONE style image (the
style side of every level is computed once per batch), while a thread pool decodes the next batch and writes the
previous one, so the GPU never waits for PNG I/O.  ``--in-path`` may also be a directory of frames (then no ffmpeg is
needed and the stylised frames are left in ``--out-path``); ffmpeg is used only when it is installed.
Additions: ``--batch``, ``--synthetic-weights``, ``--adain``.

Style interpolation: ``--interp-styles S0 S1 ...`` with ``--interp-weights w0 w1 ...`` stylises every frame with one fixed
blend (output ``<clip>_<s0>-<w0>+<s1>-<w1>...``), and with ``--morph`` sweeps piecewise-linearly from S0 to the last style
across the clip (``morph_weights``; output ``<clip>_morph_<s0>+<s1>...``).  A frame's weights depend on its index in the
clip only, so ``--batch`` does not change a frame.

Temporal stabilisation: ``--temporal STRENGTH`` (in [0, 1); default 0 = off) blends each stylised frame with its stabilised
predecessor, warped by the optical flow of the content frames, where that flow is confident (``WCT.temporal_state``,
DESIGN.md §3.3.6).  This reduces the flicker of frame-by-frame WCT.  Each (clip, style) run has one state, carried across
batches and through the frame-by-frame path, so ``--batch`` does not change a frame; ``--concat`` comes after it.

Optimal-transport transform: ``--ost`` uses the Monge map between the feature Gaussians instead of WCT at every level
(DESIGN.md §3.3.8), on the batched and the frame-by-frame path alike.

Seamless stylisation: ``--seamless {x,y,xy}`` pads the content path circularly (DESIGN.md §3.3.9), e.g. ``x`` for 360°
clips, on both paths.

Multimodal style transfer: ``--mst K [--mst-smooth LAMBDA]`` matches the content to K modes of the style at every level
(DESIGN.md §3.3.10), on both paths.

Exact feature distribution matching: ``--efdm`` gives every channel of each level the style's whole value distribution
(DESIGN.md §3.3.12), on both paths; ``--efdm-slices K`` first matches in K random channel rotations (§3.3.14).

Colour preservation: ``--luminance-only`` stylises the luminance and keeps each frame's own colours (DESIGN.md §3.3.15).
Unlike ``--keep-colors``, which makes every frame its own style, frames of one size stay in batches, and each frame is a
function of its own content only.  All passes run in one call; the colours are merged after the last.

Scale control: ``--coarse-to-fine F`` with ``--fine-targets`` stylises each frame coarse to fine (DESIGN.md §3.3.16), on
both paths.

Which of these options combine is decided by one table, ``wct_tf_b200/options.py``, as for stylize.py.
"""
from __future__ import division, print_function

import argparse
import os
import random
import shutil
import subprocess
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np


# video-specific flags; the stylisation flags are shared with stylize.py (same names and defaults as the reference,
# stylize_video.py:17-42)
_VIDEO_FLAGS = [
    (("--in-path",), dict(type=str, required=True, help="video file, or a directory of frames")),
    (("--out-path",), dict(type=str, required=True, help="folder for the encoded videos / stylised frames")),
    (("--style-path",), dict(type=str, default=None, help="style image, or a folder of them (or --interp-styles)")),
    (("--morph",), dict(action="store_true", default=False,
                        help="with --interp-styles: sweep piecewise-linearly from the first style to the last across the clip")),
    (("--tmp-dir",), dict(type=str, dest="tmp_dir", default=None, help="where ffmpeg unpacks the frames")),
    (("--keep-tmp",), dict(action="store_true", default=False, help="keep the unpacked frames")),
    (("--batch",), dict(type=int, default=15, help="frames per predict_batch call (not in the reference)")),
    (("--fps",), dict(type=int, default=30, help="frame rate of the encoded video (not in the reference: fixed 30 there)")),
    (("--temporal",), dict(type=float, default=0.0, metavar="STRENGTH",
                           help="temporal stabilisation strength in [0, 1): blend each frame with its flow-warped stabilised "
                                "predecessor (default 0: off)")),
]
_SHARED = ("--checkpoints", "--relu-targets", "--vgg-path", "--keep-colors", "--style-size", "--crop-size", "--content-size",
           "--passes", "--device", "--alpha", "--concat", "--swap5", "--ss-alpha", "--ss-temperature", "--ss-balance",
           "--ss-patch-size", "--ss-stride", "--adain", "--synthetic-weights", "--interp-styles", "--interp-weights", "--swap-targets",
           "--ost", "--seamless",
           "--mst", "--mst-smooth", "--strength-map", "--efdm", "--efdm-slices", "--luminance-only", "--coarse-to-fine",
           "--fine-targets")
# flags of the one-style mode that --interp-styles takes no part of
_INTERP_EXCLUDES = [("style_path", "--style-path"), ("concat", "--concat")]


def build_parser():
    import stylize
    parser = argparse.ArgumentParser(description="stylise a video or a frame sequence")
    for names, kw in stylize._FLAGS:
        if names[-1] in _SHARED:
            parser.add_argument(*names, **kw)
    for names, kw in _VIDEO_FLAGS:
        parser.add_argument(*names, **kw)
    return parser


def parse_args(argv=None):
    """One of --style-path or --interp-styles; with --interp-styles either --interp-weights (a fixed blend) or --morph."""
    import stylize
    parser = build_parser()
    args = parser.parse_args(argv)
    stylize.check_swap_flags(parser, args)
    if args.morph:
        if args.interp_styles is None:
            parser.error("--morph needs --interp-styles")
        if args.interp_weights is not None:
            parser.error("--morph takes no --interp-weights")
        if not 2 <= len(args.interp_styles) <= 8:
            parser.error("--morph needs 2..8 --interp-styles")
        for attr, flag in _INTERP_EXCLUDES:
            if getattr(args, attr):
                parser.error("--interp-styles takes no %s" % flag)
    else:
        if args.interp_styles is not None and args.interp_weights is None:
            parser.error("--interp-styles needs --interp-weights or --morph")
        stylize.check_interp_flags(parser, args, _INTERP_EXCLUDES)
    if args.interp_styles is None and args.style_path is None:
        parser.error("--style-path (or --interp-styles) is required")
    stylize.check_prepared_flags(parser, args)
    stylize.check_values(parser, args)
    stylize.check_options(parser, args)
    stylize.check_luminance_flags(parser, args)
    return args


def morph_weights(T, K):
    """Weights [T, K] of a piecewise-linear sweep from style 0 to style K-1 over T frames (float64): frame t sits at
    p = t (K-1) / (T-1) (0 when T = 1), between styles i = min(floor(p), K-2) and i+1 with w_i = 1 - f, w_i+1 = f, f = p - i."""
    if K < 2:
        raise ValueError("a morph needs at least 2 styles")
    w = np.zeros((T, K), np.float64)
    for t in range(T):
        p = t * (K - 1) / (T - 1) if T > 1 else 0.0
        i = min(int(np.floor(p)), K - 2)
        f = p - i
        w[t, i] = 1.0 - f
        w[t, i + 1] = f
    return w


def frame_key(name):
    """frame_12.png sorts after frame_2.png (the reference iterates os.listdir order; ffmpeg numbers the frames)."""
    digits = ''.join(ch if ch.isdigit() else ' ' for ch in os.path.basename(name)).split()
    return (int(digits[-1]) if digits else -1, name)


def batches(seq, n):
    for i in range(0, len(seq), n):
        yield seq[i:i + n]


def stylize_frames(wct_model, in_files, out_files, style_img, args, io, pool, dimg, device, weights=None, temporal=None):
    """All frames of one clip with one style (a uint8 CUDA tensor, already resized / cropped).  Frames of equal size are
    batched; the decode of batch i+1 and the PNG writes of batch i-1 overlap the GPU work of batch i.  Resize
    (``--content-size``), CORAL (``--keep-colors``), every pass and the ``--concat`` thumbnail run on the device
    (wct_tf_b200.device_image); a frame crosses PCIe once in each direction.

    Style interpolation: ``style_img`` is a list of K styles and ``weights`` a float64 [K] blend for every frame or [T, K],
    row t for frame t of the clip, so a frame's weights do not depend on the batching.

    ``temporal``: the clip's temporal state (--temporal), passed to every predict_batch call in frame order."""
    def finish(out_f, frame_u8):
        io.save_img(out_f, frame_u8)

    def prep(frames_dev):
        return dimg.resize_to(frames_dev, args.content_size) if args.content_size > 0 else frames_dev

    def interp_kw(lo, hi):
        if weights is None:
            return {}
        return dict(style_weights=weights if weights.ndim == 1 else weights[lo:hi])

    temporal_kw = {} if temporal is None else dict(temporal=temporal)
    # --ost, --seamless, --mst, --efdm, --efdm-slices, --luminance-only and --coarse-to-fine, on both paths
    import stylize
    opt_kw = dict(ost=True) if getattr(args, "ost", False) else {}
    opt_kw.update(stylize.scale_kw(args))
    if getattr(args, "luminance_only", False):
        opt_kw["luminance_only"] = True
    if getattr(args, "efdm", False):
        opt_kw["efdm"] = True
    if getattr(args, "efdm_slices", 0):
        opt_kw["efdm_slices"] = args.efdm_slices
    if getattr(args, "seamless", None):
        opt_kw["seamless"] = args.seamless
    if getattr(args, "mst", None) is not None:
        opt_kw.update(mst=args.mst, mst_smooth=args.mst_smooth)
    if getattr(args, "strength_map", None):
        opt_kw["strength_map"] = stylize.read_grey(args.strength_map)   # one map for every frame

    def coral(style, fr):
        if isinstance(style, list):
            return [dimg.preserve_colors_np(s, fr) for s in style]
        return dimg.preserve_colors_np(style, fr)

    step = max(1, args.batch)
    todo = list(batches(list(zip(in_files, out_files)), step))
    pending_loads = [pool.submit(io.get_img, f) for f, _ in todo[0]] if todo else []
    writes, count = [], 0
    for bi, group in enumerate(todo):
        frames = [f.result() for f in pending_loads]
        pending_loads = [pool.submit(io.get_img, f) for f, _ in todo[bi + 1]] if bi + 1 < len(todo) else []
        same = all(fr.shape == frames[0].shape for fr in frames) and not args.keep_colors
        first = bi * step                                      # clip index of the batch's first frame
        if same and len(frames) > 1:
            x = prep(dimg.to_device(np.stack(frames), device))
            # --passes (stylize_video.py:119-121) run back to back on the device; a style swap acts in the first pass and
            # swaps the whole batch against the one style in one call
            swap_kw = dict(swap5=True, ss_alpha=args.ss_alpha) if args.swap5 else {}
            if args.swap_targets:
                swap_kw = dict(swap_targets=list(args.swap_targets), ss_alpha=args.ss_alpha)
            if args.ss_temperature is not None:
                swap_kw["ss_temperature"] = args.ss_temperature
            if args.ss_balance is not None:
                swap_kw["ss_balance"] = args.ss_balance
            one = weights is not None or not hasattr(style_img, "shape")   # a list of styles, or a prepared style
            out = wct_model.predict_batch(x, style_img if one else style_img[None], alpha=args.alpha,
                                          adain=args.adain, passes=args.passes, return_device=True,
                                          **dict(interp_kw(first, first + len(frames)), **swap_kw, **temporal_kw, **opt_kw))
            results = [(out[i], style_img) for i in range(len(frames))]
        else:                                                  # per-frame styles (CORAL) or ragged sizes
            results = []
            for j, fr in enumerate(frames):
                fr = prep(dimg.to_device(fr, device))
                style_rgb = coral(style_img, fr) if args.keep_colors else style_img
                kw = dict(alpha=args.alpha, ss_alpha=args.ss_alpha, adain=args.adain, return_device=True,
                          **interp_kw(first + j, first + j + 1), **opt_kw)
                swap_kw = dict(swap_targets=list(args.swap_targets)) if args.swap_targets else {}
                if args.ss_temperature is not None:
                    swap_kw["ss_temperature"] = args.ss_temperature
                if args.ss_balance is not None:
                    swap_kw["ss_balance"] = args.ss_balance
                if temporal is not None or "luminance_only" in opt_kw:   # stabilised / merged after the last pass
                    o = wct_model.predict_batch(fr, style_rgb, swap5=args.swap5, passes=args.passes,
                                                **dict(kw, **swap_kw, **temporal_kw))
                else:
                    o = wct_model.predict_batch(fr, style_rgb, swap5=args.swap5, **dict(kw, **swap_kw))
                    for _ in range(args.passes - 1):
                        o = wct_model.predict_batch(o, style_rgb, swap5=False, **kw)
                results.append((o[0], style_rgb))
        for (_, out_f), (o, srgb) in zip(group, results):
            if args.concat:                                    # stylize_video.py:125-128
                if getattr(srgb, "image", None) is not None:   # a prepared style keeps its image on the host
                    srgb = dimg.to_device(srgb.image[0], device)
                o = dimg.concat_with_style(srgb, o)
            writes.append(pool.submit(finish, out_f, dimg.to_host(o)))
            count += 1
    for w in writes:
        w.result()
    return count


def have_ffmpeg():
    return shutil.which('ffmpeg') is not None


def main(argv=None, wct_factory=None, image_ops=None):
    """``wct_factory`` / ``image_ops`` let the tests drive the frame logic with stand-ins for the engine and for
    wct_tf_b200.device_image; the CLI always uses the real ones."""
    args = parse_args(argv)
    from wct_tf_b200 import imageio as io
    if image_ops is None:
        from wct_tf_b200 import device_image as image_ops
    dimg = image_ops
    start = time.time()
    if wct_factory is None:
        from wct_tf_b200.wct import WCT
        weights = None
        if args.synthetic_weights is not None:
            from wct_tf_b200.weights import make_synthetic_weights
            weights = make_synthetic_weights(args.synthetic_weights, relu_targets=args.relu_targets)
        elif not args.checkpoints:
            raise SystemExit("--checkpoints is required (or --synthetic-weights SEED)")
        wct_model = WCT(checkpoints=args.checkpoints, relu_targets=args.relu_targets, vgg_path=args.vgg_path,
                        device=args.device, ss_patch_size=args.ss_patch_size, ss_stride=args.ss_stride, weights=weights)
    else:
        wct_model = wct_factory(args)

    import stylize
    prepared = stylize.PreparedStyles(wct_model)
    if args.interp_styles is not None:
        style_files = [None]                                   # one run with the blend of every --interp-styles image
    else:
        style_files = stylize.style_listing(args.style_path, io)
    os.makedirs(args.out_path, exist_ok=True)
    from_dir = os.path.isdir(args.in_path)
    tmp_dir = args.tmp_dir or os.path.join(args.out_path, '_____fns_frames_%s' % random.randint(0, 99999))
    if from_dir:
        in_files = sorted(io.get_files(args.in_path), key=frame_key)
    else:
        if not have_ffmpeg():
            raise SystemExit("ffmpeg is not installed: pass a directory of frames as --in-path")
        in_dir = os.path.join(tmp_dir, 'input')
        os.makedirs(in_dir, exist_ok=True)
        subprocess.check_call(['ffmpeg', '-i', args.in_path, os.path.join(in_dir, 'frame_%d.png')])   # stylize_video.py:75-81
        in_files = sorted([os.path.join(in_dir, x) for x in os.listdir(in_dir)], key=frame_key)
    clip = os.path.basename(os.path.normpath(os.path.splitext(args.in_path)[0] if not from_dir else args.in_path))
    ext = '.mp4' if from_dir else os.path.splitext(args.in_path)[1]

    total = 0
    with ThreadPoolExecutor(max_workers=8) as pool:
        for style_fullpath in style_files:                     # stylize_video.py:97
            device = wct_model.engine.device if hasattr(wct_model, "engine") else None

            def load_style(path):
                if stylize.is_prepared(path):
                    return prepared.get(path)                  # read once per run
                img = dimg.to_device(io.get_img(path), device)
                if args.style_size > 0:
                    img = dimg.resize_to(img, args.style_size)
                if args.crop_size > 0:
                    img = dimg.center_crop(img, args.crop_size)
                return img
            weights = None
            if style_fullpath is None:
                style_img = [load_style(p) for p in args.interp_styles]
                if args.morph:
                    weights = morph_weights(len(in_files), len(args.interp_styles))
                    style_prefix = "morph_" + "+".join(os.path.splitext(os.path.basename(p))[0] for p in args.interp_styles)
                else:
                    weights = np.asarray(args.interp_weights, np.float64)     # normalised by WCT.predict_batch
                    style_prefix = stylize.interp_label(args.interp_styles, args.interp_weights)
            else:
                style_img = load_style(style_fullpath)
                style_prefix = os.path.basename(os.path.splitext(style_fullpath)[0])
            out_v = os.path.join(args.out_path, '{}_{}{}'.format(clip, style_prefix, ext))
            frames_dir = os.path.join(args.out_path if from_dir else tmp_dir, '{}_{}_frames'.format(clip, style_prefix))
            if os.path.isfile(out_v):                          # stylize_video.py:108-110
                print("SKIP", out_v)
                continue
            os.makedirs(frames_dir, exist_ok=True)
            out_files = [os.path.join(frames_dir, os.path.splitext(os.path.basename(f))[0] + '.png') for f in in_files]
            temporal = wct_model.temporal_state(args.temporal) if args.temporal > 0 else None    # one per (clip, style) run
            n = stylize_frames(wct_model, in_files, out_files, style_img, args, io, pool, dimg, device, weights, temporal)
            total += n
            print("Stylized {} frames with {} -> {}".format(n, style_prefix, frames_dir))
            # stylize_video.py:137-149 re-encodes "frame_%d.png".  Frames extracted by ffmpeg carry that name; a user-supplied
            # directory of frames keeps its own basenames, so it is only re-encoded when they follow the same pattern
            named_like_ffmpeg = all(os.path.basename(f) == 'frame_%d.png' % (i + 1) for i, f in enumerate(out_files))
            if have_ffmpeg() and named_like_ffmpeg:
                pattern = os.path.join(frames_dir, 'frame_%d.png')
                subprocess.check_call(['ffmpeg', '-y', '-i', pattern, '-f', 'mp4', '-q:v', '0', '-vcodec', 'mpeg4',
                                       '-r', str(args.fps), out_v])
                print('Video at: %s' % out_v)
    if not from_dir and not args.keep_tmp and len(style_files) == 1:
        shutil.rmtree(tmp_dir, ignore_errors=True)
    dt = time.time() - start
    print('Processed {} frames in: {:.2f}s ({:.1f} frames/s incl. PNG I/O)'.format(total, dt, total / max(dt, 1e-9)))
    return total


if __name__ == '__main__':
    main()
