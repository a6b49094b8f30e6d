"""``WCT`` -- drop-in for the reference inference wrapper (wct.py:14-106).

Same constructor and ``predict`` signature; the TF session is replaced by the
sm_90a engine (engine.py -> libwctb200.so).  Differences, all explicit:
  * ``checkpoints`` / ``vgg_path`` may be file paths (``.npz`` bundles, see
    weights.py) OR ``weights=`` may pass an in-memory weights dict (the offline
    build has no .t7 / TF checkpoints, so benchmarks use synthetic weights);
  * ``device`` accepts the reference's TF strings ('/gpu:0') and torch strings;
  * ``swap5=True`` (style-swap at relu5_1, ops.py:145-278) honours ``ss_patch_size`` / ``ss_stride``; with a stride the
    content is centre-cropped so that the patches tile its relu5_1 encoding, as wct.py:84-90 does;
  * ``swap_targets`` is new: the style swap at any relu levels (relu3_1 carries brush strokes, relu5_1 semantic parts);
  * ``predict_batch`` is new: a batch of frames per call (frames are independent);
  * ``content_mask`` is new: spatial control (WCT paper, section 4), a label map whose region r takes style r;
    ``style_masks`` restricts style r to its pixels labelled r;
  * ``style_weights`` is new: style interpolation (WCT paper, section 4), a weighted blend of 1..8 styles, shared by
    every frame or one row per frame;
  * ``synthesize`` is new: texture synthesis (WCT paper, section 4), the pipeline run on seeded noise made on the device;
  * ``prepare_style`` / ``load_style`` are new: the style side computed once (or read from a ``.wctstyle`` file) and
    accepted wherever a style image is (wct_tf_b200/prepared.py);
  * ``temporal_state`` / ``predict_batch(temporal=)`` are new: temporal stabilisation of a clip's frames with the optical
    flow of the content (wct_tf_b200/temporal.py);
  * ``ost`` is new: the optimal-transport transform (Lu et al., ICCV 2019), the Monge map between the content and style
    feature Gaussians, in place of WCT at every level;
  * ``seamless`` is new: circular padding of every conv of the content path along x, y or both, for 360° panoramas and
    tileable textures;
  * ``mst`` is new: multimodal style transfer (Zhang, Zhu & Zhu, ICCV 2019), each level's style clustered into K modes
    and every content pixel matched to one, so regions pair up without masks;
  * ``efdm`` is new: exact feature distribution matching (Zhang et al., CVPR 2022), every channel's values given the
    style's by rank;
  * ``swap_labels`` is new: the labelled style swap (neural doodle, Champandard 2016), each content patch matched only to
    style patches of its own label;
  * ``luminance_only`` is new: colour preservation (Gatys et al., CVPR 2017, §5), the luminance stylised and the content's
    colours kept;
  * ``ss_temperature`` is new: the softmax swap, each content patch rebuilt from a softmax-weighted blend of style
    patches instead of its single best one;
  * ``ss_balance`` is new: the balanced swap, Sinkhorn iterations that spread the softmax swap's use of the style
    patches evenly;
  * ``coarse_to_fine`` is new: scale control (Gatys et al., CVPR 2017, §6), the call run on a downscaled content and its
    result joined into the content's low band before the fine levels run at full size.
"""
from __future__ import annotations

import re
import time

import numpy as np
import torch

from . import options
from .engine import Engine, SEMANTICS
from .model import RELU_CHANNELS, seamless_axes
from .prepared import PreparedStyle


def _to_dev(a, dev):
    """uint8 image(s) [H,W,3] or [n,H,W,3], numpy or torch, host or device -> contiguous cuda uint8 [n,H,W,3]."""
    if isinstance(a, np.ndarray):
        a = torch.from_numpy(np.array(a, copy=True, order="C"))    # own, writable, contiguous
    if a.dim() == 3:
        a = a.unsqueeze(0)
    if a.dtype != torch.uint8:
        a = a.clamp(0, 255).to(torch.uint8)   # the reference feeds arrays "in [0,255]" (wct.py:74)
    return a.to(dev, non_blocking=True).contiguous()


def _style_list(styles):
    """The styles of a mask / interpolation call as a list (one image or one prepared style stands for a list of one)."""
    if isinstance(styles, PreparedStyle) or (isinstance(styles, (np.ndarray, torch.Tensor)) and styles.ndim == 3):
        return [styles]
    return list(styles)


def _torch_device(device):
    """'/gpu:0' (stylize.py:23) -> 'cuda:0'."""
    if isinstance(device, int):
        return "cuda:%d" % device
    if isinstance(device, str):
        m = re.match(r"^/?(?:device:)?gpu:(\d+)$", device.strip().lower())
        if m:
            return "cuda:%s" % m.group(1)
        if re.match(r"^\d+$", device.strip()):          # a bare ordinal, as the CLI help advertises
            return "cuda:%s" % device.strip()
        if device.strip().lower() in ("/cpu:0", "cpu"):
            raise ValueError("the CUDA engine has no CPU path (device=%r)" % (device,))
    return device


class WCT(object):
    '''Stylize images with the multi-level WCT pipeline (mirror of wct.py:14)'''

    def __init__(self, checkpoints=None, relu_targets=None, vgg_path=None, device='/gpu:0',
                 ss_patch_size=3, ss_stride=1, weights=None, semantics="tf", verbose=False):
        if relu_targets is None:
            raise ValueError("relu_targets is required")
        self.ss_patch_size = ss_patch_size
        self.ss_stride = ss_stride
        self.verbose = verbose
        if weights is None:
            from .weights import load_weights
            weights = load_weights(vgg_path, checkpoints, relu_targets)   # pairs checkpoints[i] <-> relu_targets[i] (wct.py:47)
        self.engine = Engine(weights, relu_targets, device=_torch_device(device), semantics=semantics)
        self.engine.groups = 2                  # batches >= 2 frames run as two interleaved stream pairs
        self.engine.group_priorities = True
        self.model = self.engine.model

    @staticmethod
    def preprocess(image):
        """wct.py:60-64"""
        if len(image.shape) == 3:
            image = np.expand_dims(image, 0)
        return image / 255.

    @staticmethod
    def postprocess(image):
        """wct.py:66-68"""
        return np.uint8(np.clip(image, 0, 1) * 255)

    @staticmethod
    def check_mask(content_mask, n_frames, styles):
        """Host-side validation of a spatial-control call: uint8 mask [Hm,Wm] (shared) or [N,Hm,Wm], and a list of
        1..8 uint8 [Hs,Ws,3] style images (one per region, any sizes).  Returns (mask as uint8 [1|N,Hm,Wm], styles)."""
        m = content_mask.cpu() if isinstance(content_mask, torch.Tensor) else torch.from_numpy(np.asarray(content_mask))
        if m.dtype != torch.uint8:
            raise ValueError("content_mask must be uint8, got %s" % (m.dtype,))
        if m.dim() == 2:
            m = m.unsqueeze(0)
        if m.dim() != 3 or m.shape[0] not in (1, n_frames) or m.shape[1] < 1 or m.shape[2] < 1:
            raise ValueError("content_mask must be [Hm,Wm] or [N,Hm,Wm] with N = %d frames, got %s" % (n_frames, tuple(m.shape)))
        return m.contiguous(), WCT.check_region_styles(styles)

    @staticmethod
    def check_region_styles(styles):
        """A list of 1..8 region styles: uint8 [Hs,Ws,3] images or prepared styles of one style each; ValueError else."""
        styles = _style_list(styles)
        if not 1 <= len(styles) <= 8:
            raise ValueError("a content mask needs 1..8 region styles, got %d" % len(styles))
        for s in styles:
            if isinstance(s, PreparedStyle):
                if s.n != 1:
                    raise ValueError("each region style must be one style, got a prepared style of %d" % s.n)
                continue
            if s.dtype not in (np.uint8, torch.uint8) or s.ndim not in (3, 4) or s.shape[-1] != 3 or (s.ndim == 4 and s.shape[0] != 1):
                raise ValueError("each region style must be one uint8 [Hs,Ws,3] image")
        return styles

    @staticmethod
    def check_soft_map(a, n_frames, name, planes=None):
        """Host-side validation of a soft spatial-control map (DESIGN.md §3.3.11): [Hm,Wm] or [N,Hm,Wm] (``planes`` = K:
        [K,Hm,Wm] or [N,K,Hm,Wm]), float in [0,1] or uint8 read as v/255.  Returns float32 [1|N,(K,)Hm,Wm]; soft weights
        whose sum over K exceeds 1 at a pixel are divided by that sum."""
        t = a.detach().cpu() if isinstance(a, torch.Tensor) else torch.from_numpy(np.asarray(a))
        if t.dtype == torch.uint8:
            t = t.to(torch.float64) / 255.0
        elif t.dtype.is_floating_point:
            t = t.to(torch.float64)
        else:
            raise ValueError("%s must be float in [0,1] or uint8, got %s" % (name, t.dtype))
        rank = 2 if planes is None else 3
        if t.dim() == rank:
            t = t.unsqueeze(0)
        ok = t.dim() == rank + 1 and t.shape[0] in (1, n_frames) and t.shape[-1] >= 1 and t.shape[-2] >= 1
        if ok and planes is not None:
            ok = t.shape[1] == planes
        if not ok:
            want = "[Hm,Wm] or [N,Hm,Wm]" if planes is None else "[K,Hm,Wm] or [N,K,Hm,Wm] with K = %d styles" % planes
            raise ValueError("%s must be %s with N = %d frames, got %s" % (name, want, n_frames, tuple(t.shape)))
        if not bool(torch.isfinite(t).all()) or bool((t < 0).any()) or bool((t > 1).any()):
            raise ValueError("%s must hold finite values in [0, 1]" % name)
        if planes is not None:
            tot = t.sum(dim=1, keepdim=True)
            t = torch.where(tot > 1, t / tot.clamp(min=1), t)
        return t.to(torch.float32).contiguous()

    @staticmethod
    def check_style_masks(style_masks, styles):
        """Host-side validation of the style masks of a spatial-control call: a list of one entry per region style (the
        ``styles`` of ``check_mask``), each None (the whole style) or a uint8 label map [Hm',Wm'] of any resolution, and no
        mask on a prepared style.  Returns the list with every map as a uint8 tensor; entries that were the same object
        stay the same object, so that they share one encode and one masked prepare."""
        if not isinstance(style_masks, (list, tuple)):
            raise ValueError("style_masks must be a list with one entry (None or a mask) per region style")
        if len(style_masks) != len(styles):
            raise ValueError("%d style masks for %d region styles: give one entry (None or a mask) per style"
                             % (len(style_masks), len(styles)))
        out, seen = [], {}
        for s, m in zip(styles, style_masks):
            if m is None:
                out.append(None)
                continue
            if isinstance(s, PreparedStyle):
                raise ValueError("a prepared style has no feature maps to mask: give the style image with its mask")
            if id(m) not in seen:
                t = m if isinstance(m, torch.Tensor) else torch.from_numpy(np.asarray(m))
                if t.dtype != torch.uint8 or t.dim() != 2 or t.shape[0] < 1 or t.shape[1] < 1:
                    raise ValueError("each style mask must be a uint8 label map [Hm,Wm], got %s %s" % (t.dtype, tuple(t.shape)))
                seen[id(m)] = (m, t.contiguous())
            out.append(seen[id(m)][1])
        return out

    @staticmethod
    def normalize_weights(style_weights, n_frames, K, dtype=np.float32):
        """Host-side validation of interpolation weights: [K] (shared by every frame) or [N,K], finite, >= 0, every row with a
        positive sum.  Each row is divided by its sum in float64 (a one-hot row stays exact), then cast to ``dtype``.
        Returns [1|N, K]."""
        w = style_weights.cpu().numpy() if isinstance(style_weights, torch.Tensor) else np.asarray(style_weights)
        if w.dtype.kind not in "biuf":
            raise ValueError("style_weights must be numeric, got %s" % (w.dtype,))
        w = w.astype(np.float64)
        if w.ndim == 1:
            w = w[None]
        if w.ndim != 2 or w.shape[1] != K or w.shape[0] not in (1, n_frames):
            raise ValueError("style_weights must be [K] or [N,K] with K = %d styles and N = %d frames, got %s"
                             % (K, n_frames, tuple(np.shape(style_weights))))
        if not np.isfinite(w).all() or (w < 0).any():
            raise ValueError("style_weights must be finite and >= 0")
        s = w.sum(axis=1, keepdims=True)
        if (s <= 0).any():
            raise ValueError("every row of style_weights needs a positive sum")
        return (w / s).astype(dtype)

    @staticmethod
    def check_interp(style_weights, n_frames, styles):
        """Host-side validation of an interpolation call: a list of 1..8 uint8 [Hs,Ws,3] style images (any sizes) and their
        weights (``normalize_weights``).  Returns (float32 weights [1|N, K], styles)."""
        styles = _style_list(styles)
        if not 1 <= len(styles) <= 8:
            raise ValueError("style interpolation needs 1..8 styles, got %d" % len(styles))
        for s in styles:
            if isinstance(s, PreparedStyle):
                if s.n != 1:
                    raise ValueError("each interpolated style must be one style, got a prepared style of %d" % s.n)
                continue
            if s.dtype not in (np.uint8, torch.uint8) or s.ndim not in (3, 4) or s.shape[-1] != 3 or (s.ndim == 4 and s.shape[0] != 1):
                raise ValueError("each interpolated style must be one uint8 [Hs,Ws,3] image")
        return WCT.normalize_weights(style_weights, n_frames, len(styles)), styles

    def swap_fit(self, contents, swap5, swap_targets, to_dev):
        """wct.py:84-90 for the swap levels: with ``ss_stride`` > 1 the patches may not tile the encoding of the swap level;
        centre-crop the content (on the device) so that they do.  One swap level at most with a stride (the crops of two
        levels generally differ).  Returns the content frames.

        ``swap5`` keeps the reference's rule (utils.swap_filter_fit on the relu5_1 encoding of the content).  For
        ``swap_targets`` the encoding is the one the swap level actually sees: each earlier level of n pools decodes to
        ceil(size / 2^n) 2^n, and the swap level reluK_1 pools K - 1 times.  The crop is the largest size <= the content's
        whose encoding the patches tile; ValueError naming the level and the sizes when there is none."""
        if self.ss_stride == 1 or not (swap5 or swap_targets is not None):
            return contents
        from .device_image import center_crop_to
        from .imageio import swap_filter_fit
        levels = ("relu5_1",) if swap_targets is None else self.engine.swap_levels(False, swap_targets)
        if len(levels) > 1:
            raise ValueError("ss_stride %d with %d swap levels (%s): a strided swap works at one level, whose encoding the "
                             "content is cropped to" % (self.ss_stride, len(levels), ", ".join(levels)))
        contents = to_dev(contents)
        H, W = contents.shape[1], contents.shape[2]
        if swap_targets is None:
            refit, Ht, Wt = swap_filter_fit(H, W, self.ss_patch_size, self.ss_stride)
            return center_crop_to(contents, Ht, Wt) if refit else contents
        P, S = self.ss_patch_size, self.ss_stride
        order = [l.relu_target for l in self.model.levels]
        pools = [int(r[4]) - 1 for r in order[:order.index(levels[0]) + 1]]      # reluK_1 sits after K - 1 poolings

        def encoding(x):
            for n in pools[:-1]:
                x = -(-x // 2 ** n) * 2 ** n
            return -(-x // 2 ** pools[-1])

        def fit(x):
            while x >= 1 and (encoding(x) < P or (encoding(x) - P) % S):
                x -= 1
            return x
        Ht, Wt = fit(H), fit(W)
        if Ht < 1 or Wt < 1:
            raise ValueError("the style swap at %s: patch %d / stride %d tiles the %s encoding of no crop of a %dx%d content"
                             % (levels[0], P, S, levels[0], H, W))
        return center_crop_to(contents, Ht, Wt) if (Ht, Wt) != (H, W) else contents

    def predict_batch(self, contents, styles, alpha=1, adain=False, return_float=False, out=None, swap5=False, ss_alpha=1,
                      passes=1, return_device=False, content_mask=None, style_weights=None, style_masks=None,
                      swap_targets=None, temporal=None, tile_size=None, ost=False, seamless=None, mst=None, mst_smooth=0.05,
                      strength_map=None, content_weights=None, mask_feather=None, efdm=False, swap_labels=None,
                      efdm_slices=0, luminance_only=False, coarse_to_fine=None, fine_targets=None, ss_temperature=None,
                      ss_balance=0):
        """contents: uint8 [N,H,W,3]; styles: uint8 [1|N,Hs,Ws,3] (numpy or torch; host buffers --
        ideally pinned -- or device tensors).  Returns uint8 [N,H',W',3] on the host: a numpy array,
        or ``out`` (a pinned uint8 torch tensor of the right shape) filled in place.  The call is
        synchronous like the reference's ``sess.run`` (wct.py:97).

        ``passes`` > 1 repeats the stylisation on the previous OUTPUT like stylize.py:102-104 (``--passes``), but keeps the
        intermediate frames on the device: each pass still ends in the uint8 quantisation of wct.py:66-68 and restarts from
        /255 (wct.py:60-64), so the result is bit-identical to calling predict once per pass; style swap only acts in the
        first pass, as in stylize_video.py:117-121.  ``return_device=True`` returns the uint8 cuda tensor instead of a host copy.

        Which of the options below combine is decided by one table, ``wct_tf_b200/options.py``; a call it rejects raises a
        ValueError naming both options before any device work.

        ``content_mask`` (spatial control): uint8 label map [Hm,Wm] shared by every frame, or [N,Hm,Wm]; ``styles`` is then
        a list of R (1..8) uint8 [Hs,Ws,3] images of any sizes, and region r of each frame takes style r.  The mask may have
        any resolution: every level samples it to its feature grid.  Labels >= R leave that region unstyled.

        ``style_masks`` (with ``content_mask``): a list of R entries, each None or a uint8 label map [Hm',Wm'] of style r,
        of any resolution.  Region r of every frame then takes the statistics of the pixels of style r labelled r ("the sky
        of the photo takes the sky of the painting"); None takes the whole style.  Where the style region has fewer than 2
        pixels at a level, region r keeps its content feature there.  Entries that are the same (style, mask) pair of
        objects share one encode and one masked prepare, so one painting with one segmentation is encoded once.  Not with
        prepared styles as masked entries.

        ``style_weights`` (style interpolation): ``styles`` is then a list of K (1..8) uint8 [Hs,Ws,3] images of any sizes
        and ``style_weights`` their weights, [K] for every frame or [N,K] (row n for frame n); finite, >= 0, each row with a
        positive sum, normalised to sum 1.  Frame n is stylised with the blend of the K styles, which equals the blend of
        the K single-style results at every level.

        ``swap_targets`` (style swap at any level): a list of relu targets at which the style swap replaces WCT / AdaIN in
        the first pass, with ``ss_alpha`` and the model's ``ss_patch_size`` / ``ss_stride``.  ``swap5=True`` is
        ``swap_targets=["relu5_1"]``; giving both is a ValueError, as is a level that is not a target.  With a stride
        there is one swap level, and the content is cropped so that the patches tile its encoding.

        ``temporal`` (a ``temporal_state``): the N frames are the next N frames of that clip.  They are stylised exactly as
        without it; after the last pass each frame is blended with its stabilised predecessor, warped by the optical flow of
        the content frames, where that flow is confident (DESIGN.md §3.3.6), and the state moves on.  The first frame of a
        clip, and a frame whose size differs from its predecessor's, come back unchanged.

        ``tile_size`` (tiled stylisation, DESIGN.md §3.3.7): a positive multiple of 16; None or 0 is off.  Every level runs
        in tiles of that edge with crops widened by a halo, so device memory follows the tile, not the image, and images
        too large for one pass (above about 11 600^2 pixels) can be stylised.  Each level's statistics are still those of
        the whole image: the result equals the untiled one up to the order of their summation, and byte for byte when one
        tile covers the image.  The frames of the batch run one after another.

        ``ost`` (optimal-transport transform, DESIGN.md §3.3.8): each level maps the content's feature Gaussian onto the
        style's by the Monge map, the covariance-matching map that moves the features least, instead of WCT's whitening
        and colouring; it keeps more of the content's structure at the same ``alpha``.  The style side is WCT's, so image
        and prepared styles work unchanged; with the style swap, the swap levels swap and the others use OST.

        ``seamless`` (seamless stylisation, DESIGN.md §3.3.9): "x" wraps the width (360° equirectangular panoramas), "y"
        the height, "xy" both (tileable textures, e.g. with ``synthesize``).  Every conv of the content path -- encoder,
        decoders, and the clip between levels -- pads the wrapped axes circularly, so the output equals, exactly, that of
        the infinitely tiled content and its opposite edges meet without a seam.  Each wrapped axis must be a multiple of
        2^P, P the pools up to the deepest target (16 for relu5_1).  The style side is unchanged.

        ``mst`` (multimodal style transfer, DESIGN.md §3.3.10): K in 1..8.  At every level the style's features are
        clustered into K modes (spherical k-means on their directions), every content pixel is labelled with the mode it
        resembles, the labelling is smoothed by a Potts term of weight ``mst_smooth`` (finite, >= 0; default 0.05), and
        content region k takes the WCT statistics of style mode k.  A painting with several distinct modes is then not
        averaged into one.  K = 1 is the plain WCT call, byte for byte; ``mst=None`` changes nothing.  ``styles`` is one
        style image, clustered once per call however many ``passes``.

        Soft spatial control (DESIGN.md §3.3.11).  ``strength_map``: [Hm,Wm] or [N,Hm,Wm], float in [0,1] or uint8 read as
        v/255, the per-pixel strength s of the call, out = s T(x) + (1 - s) x (in ``np`` semantics towards the unmodified
        feature x).
        ``content_weights``: [K,Hm,Wm] or [N,K,Hm,Wm] soft weights of the K region styles given in ``styles`` as for
        ``content_mask`` (divided by their sum where it exceeds 1); region k's statistics are weighted by plane k and each
        pixel blends the K transforms, the rest keeping the content.  ``mask_feather`` = sigma > 0 (with ``content_mask``):
        the label map feathered by a Gaussian of sigma mask pixels into such weights.  None for all three changes nothing.

        ``efdm`` (exact feature distribution matching, DESIGN.md §3.3.12): at every level each channel of each frame takes
        the whole value distribution of the same channel of its style, not only its mean and variance or covariance: the
        content values are ranked, value rank r takes the style's quantile at r, and equal values take the mean of their
        ranks' quantiles.  Sparse bright strokes and an even wash with the same statistics then stylise differently.
        ``efdm=False`` changes nothing.  The style is sorted once per call however many ``passes``; with the style swap,
        the swap levels swap in the first pass and the others use EFDM.

        ``efdm_slices`` = K in 0..32 (sliced distribution matching, DESIGN.md §3.3.14; with ``efdm``): before the plain EFDM
        step, each level runs EFDM in K random orthonormal bases of its channels, each on the previous step's output, so the
        joint distribution of the channels (their correlations, and the shape of their mixtures) moves towards the style's
        and not only each channel's own.  Every channel still ends with EFDM's marginal.  K = 0 changes nothing.

        ``swap_labels`` (labelled style swap, DESIGN.md §3.3.13; with ``swap5`` / ``swap_targets``): a pair (content
        labels, style labels) of uint8 label maps, numpy or torch, host or device: content [Hm,Wm] or [N,Hm,Wm]; style
        [Hm',Wm'] for a shared style, or with one style per frame [Hm',Wm'] or [N,Hm',Wm'].  At every swap level each content
        patch draws only on the style patches with its own label ("water here, trees there"); where the style has no patch
        of that label it draws on all of them.  Maps of any resolution are sampled onto each level's feature grids.  With a
        stride the content is cropped as for the swap, and a content map of exactly the content's size is cropped with it
        (any other size is stretched over the image as stylised).  Labels act in the first pass only, like the swap.

        ``ss_temperature`` = tau > 0 (softmax swap, DESIGN.md §3.3.17; with ``swap5`` / ``swap_targets``): each content
        patch is rebuilt from a blend of style patches, weighted by a softmax of their scores at temperature tau, instead of
        its single best patch.  Small tau approaches the hard swap, large tau the mean of the allowed patches; the useful
        range is small (with synthetic weights at relu3_1 of a 512^2 style, about 2 to 3 patches per anchor at tau = 0.003
        and hundreds at 0.01, tools/softmax_swap_bench.py; trained weights may differ), and blending a few close matches softens the seams between neighbouring patches.
        With ``swap_labels``
        the blend is over the patches of the anchor's label.  It acts in the first pass only, like the swap.  None is the
        hard swap.

        ``ss_balance`` = T in 1..256 (balanced swap, DESIGN.md §3.3.18; with ``ss_temperature``): T Sinkhorn iterations
        turn the softmax swap's per-anchor weights into a plan whose columns are balanced too, so that every style patch is
        used about as much as the uniform blend would use it, instead of a few bland patches covering large regions.
        Each iteration costs about one more pass over the patch scores.  It acts in the first pass only, like the swap.
        0 is the softmax swap.

        ``luminance_only`` (colour preservation, DESIGN.md §3.3.15): stylise the luminance only and keep the content's
        colours.  The content frames (after a stride swap's crop) are made grey with the style's luminance mean and spread
        (``device_image.luminance_match``), the call runs with every other option on them against the grey of each style
        (``luminance_grey``; a prepared style must have been prepared grey, ``prepare_style(luminance_only=True)``), and
        after the last pass the stylised luminance, mapped back to the content's mean and spread, replaces the content's
        luminance in all three channels (``luminance_merge``): the output has the content's YIQ chrominance up to uint8
        rounding.  With several styles the style statistics are those of their mixture: per frame under ``style_weights``,
        pooled over the distinct region styles with a content mask or weights.  ``temporal`` stabilises the merged frames.
        False changes nothing.

        ``coarse_to_fine`` = f in 2..16 (scale control, DESIGN.md §3.3.16): each pass first stylises, at every level, the
        content D resized to about 1/f of its size (``model.coarse_size``: sides rounded to multiples of 2^pools, at least
        one), joins the uint8 result S into the content's low band, J = clip(rint(C + U(S - D))) (``device_image.coarse_join``),
        and stylises J at full size at ``fine_targets`` only (relu targets; default the model's among relu3_1, relu2_1 and
        relu1_1).  The style keeps its own size in both stages, so the fine texture keeps the style's pixel scale while the
        coarse structures come out about f times larger; the deep levels also run on 1/f^2 of the pixels.  Both stages apply
        one style side, made once per call.  ``return_float`` returns the fine stage's float output.  None changes nothing."""
        call = dict(locals()) if luminance_only else None     # every keyword, re-issued on the grey frames
        prepared = isinstance(styles, PreparedStyle)
        per_frame = not prepared and (isinstance(styles, (list, tuple)) or np.ndim(styles) not in (3, 4)
                                      or (np.ndim(styles) == 4 and styles.shape[0] != 1))
        options.check({name for name, on in (
            ("adain", adain), ("ost", ost), ("efdm", efdm), ("mst", mst is not None), ("swap", swap5 or swap_targets is not None),
            ("content_mask", content_mask is not None), ("style_masks", style_masks is not None),
            ("style_weights", style_weights is not None), ("content_weights", content_weights is not None),
            ("mask_feather", mask_feather is not None), ("strength_map", strength_map is not None),
            ("tile_size", tile_size is not None and tile_size != 0), ("seamless", seamless is not None),
            ("temporal", temporal is not None), ("return_float", return_float), ("prepared", prepared),
            ("per_frame_styles", per_frame), ("luminance_only", luminance_only),
            ("coarse_to_fine", coarse_to_fine is not None)) if on}, options.API)
        ctf = None
        if coarse_to_fine is not None or fine_targets is not None:
            ctf = options.check_coarse_to_fine(coarse_to_fine, fine_targets, self.model.relu_targets)
        efdm_slices = options.check_efdm_slices(efdm_slices, efdm)
        ss_temperature = options.check_ss_temperature(ss_temperature, swap5 or swap_targets is not None)
        ss_balance = options.check_ss_balance(ss_balance, ss_temperature)
        if mask_feather is not None:
            options.check_mask_feather(mask_feather)
        if mst is not None:
            mst, mst_smooth = options.check_mst(mst, mst_smooth)
        seamless_axes(seamless)                              # ValueError for a value other than None, "x", "y", "xy"
        if tile_size is not None and tile_size != 0:
            options.check_tile_size(tile_size)
        else:
            tile_size = None
        eng = self.engine
        dev = eng.device
        n = 1 if np.ndim(contents) == 3 else contents.shape[0]
        eng.swap_levels(swap5, swap_targets)                 # ValueError for both, or a level that is not a target
        if swap_labels is not None:
            n_sty = styles.n if prepared else (len(styles) if isinstance(styles, (list, tuple))
                                               else 1 if np.ndim(styles) == 3 else styles.shape[0])
            swap_labels = options.check_swap_labels(swap_labels, swap5 or swap_targets is not None, n, n_sty)
        if style_weights is not None:
            weights, interp_styles = self.check_interp(style_weights, n, styles)
        if content_mask is not None:
            mask, region_styles = self.check_mask(content_mask, n, styles)
            if style_masks is not None:
                style_masks = self.check_style_masks(style_masks, region_styles)
        if content_weights is not None:
            region_styles = self.check_region_styles(styles)
            cweights = self.check_soft_map(content_weights, n, "content_weights", planes=len(region_styles))
            mask = torch.zeros((1, 1, 1), dtype=torch.uint8)     # soft weights take the place of the label map
            if style_masks is not None:
                style_masks = self.check_style_masks(style_masks, region_styles)
            content_mask = mask
        smap = self.check_soft_map(strength_map, n, "strength_map") if strength_map is not None else None
        if luminance_only:
            call["swap_labels"] = swap_labels
            return self._predict_luminance(contents, styles, call, n)
        soft_kw = {}

        def to_dev(a):
            return _to_dev(a, dev)

        once = int(passes) > 1 or ctf is not None           # the style side is applied more than once

        def style_dev(a):
            """A style image on the device, or a prepared style as it is.  With several passes, or two coarse-to-fine
            stages, an image is prepared once here, and every pass and stage applies it."""
            if isinstance(a, PreparedStyle):
                return a
            a = to_dev(a)
            return (eng.prepare_call(a, adain=adain, swap5=swap5, swap_targets=swap_targets, efdm=efdm, efdm_slices=efdm_slices)
                    if once else a)

        # wct.py:84-90: with a stride the filter may not fit; centre-crop the content (on the device) to a size it tiles
        Hc0, Wc0 = contents.shape[-3], contents.shape[-2]
        with torch.cuda.device(dev):
            contents = self.swap_fit(contents, swap5, swap_targets, to_dev)
        with torch.cuda.device(dev):
            c = to_dev(contents)
            lab_dev = None
            if swap_labels is not None:
                cl, sl = (t if isinstance(t, torch.Tensor) else torch.from_numpy(np.array(t, copy=True, order="C"))
                          for t in swap_labels)
                cl = self._crop_labels(cl, (Hc0, Wc0), c.shape[1:3])
                lab_dev = (cl.to(dev, non_blocking=True).contiguous(), sl.to(dev, non_blocking=True).contiguous())
            if smap is not None:
                soft_kw["strength_map"] = smap.to(dev, non_blocking=True)
            if content_weights is not None:
                soft_kw["content_weights"] = cweights.to(dev, non_blocking=True)
            elif mask_feather is not None:
                soft_kw["mask_feather"] = float(mask_feather)
            s, style_kw = None, {}
            if style_weights is not None:
                w_dev = torch.from_numpy(weights).to(dev, non_blocking=True)
                style_kw = dict(interp_styles=[style_dev(x) for x in interp_styles], interp_weights=w_dev)
            elif content_mask is not None and style_masks is not None:
                lab = mask.to(dev, non_blocking=True)
                # the same object stays the same object on the device: the engine shares its side
                on_dev = {}
                for x in region_styles:
                    if id(x) not in on_dev:
                        on_dev[id(x)] = x if isinstance(x, PreparedStyle) else to_dev(x)
                for m in style_masks:
                    if m is not None and id(m) not in on_dev:
                        on_dev[id(m)] = m.to(dev, non_blocking=True).contiguous()
                rs = [on_dev[id(x)] for x in region_styles]
                sm = [None if m is None else on_dev[id(m)] for m in style_masks]
                if once:
                    rs, sm = eng.prepare_regions_call(rs, eng.check_region_masks(sm, rs)), None
                style_kw = dict(labels=None if content_weights is not None else lab, region_styles=rs, region_masks=sm)
            elif content_mask is not None:
                lab = mask.to(dev, non_blocking=True)
                style_kw = dict(labels=None if content_weights is not None else lab,
                             region_styles=[style_dev(x) for x in region_styles])
            elif mst is not None:
                s = to_dev(styles)
                if int(passes) > 1:
                    s = eng.prepare_mst_call(s, mst)
                style_kw = dict(mst=mst, mst_smooth=mst_smooth)
            else:
                s = style_dev(styles)
            # the style swap acts in the first pass only (stylize_video.py:117-121).  A shared style swaps the whole batch
            # in one call; with one style per frame the engine swaps frame by frame.
            first_only = dict(swap5=swap5, swap_targets=swap_targets, swap_labels=lab_dev, ss_temperature=ss_temperature,
                              ss_balance=ss_balance)
            later = dict(swap5=False, swap_targets=None, swap_labels=None, ss_temperature=None, ss_balance=0)

            def one_pass(x, first, levels=None):
                if tile_size is not None:
                    return eng.stylize_tiled(x, s, alpha=alpha, adain=adain, tile_size=tile_size, ost=ost, seamless=seamless,
                                             levels=levels)
                return eng.stylize(x, s, alpha=alpha, adain=adain, ost=ost, efdm=efdm, efdm_slices=efdm_slices, seamless=seamless,
                                   levels=levels, ss_alpha=ss_alpha, ss_patch_size=self.ss_patch_size, ss_stride=self.ss_stride,
                                   **style_kw, **soft_kw, **(first_only if first else later))
            if ctf is not None:
                whole = one_pass

                def one_pass(x, first):
                    return self._coarse_to_fine(x, first, whole, *ctf)
            out_f = one_pass(c, True)
            out_dev = eng.to_u8(out_f)
            for _ in range(int(passes) - 1):
                out_f = one_pass(out_dev, False)
                out_dev = eng.to_u8(out_f)
            if temporal is not None:
                from .temporal import stabilize_
                stabilize_(temporal, c, out_dev)
            if return_device:
                eng.check_device()            # synchronises; raises WctB200Error if a kernel recorded a pipeline time-out
                return (out_dev, out_f) if return_float else out_dev
            out_u8 = self._to_host(out_dev, out)
        if return_float:
            return out_u8, out_f.cpu().numpy()
        return out_u8

    def _coarse_to_fine(self, x, first, one_pass, f, fine):
        """One coarse-to-fine pass (DESIGN.md §3.3.16) of the uint8 frames ``x`` [N,H,W,3]: ``one_pass(D, first)`` at every
        level on the coarse content D, the join J of its uint8 result into x's low band, and ``one_pass(J, first, fine)``
        at full size.  Returns the fine stage's float output."""
        from .device_image import coarse_join, imresize
        from .model import RELU_LEVEL, coarse_size
        g = 2 ** (RELU_LEVEL[self.model.deepest_target] - 1)
        d = imresize(x, coarse_size(x.shape[1], x.shape[2], f, g))
        s = self.engine.to_u8(one_pass(d, first))
        return one_pass(coarse_join(x, d, s), first, fine)

    @staticmethod
    def _crop_labels(cl, hw0, hw):
        """A content label map [n,Hm,Wm] of exactly the content's size ``hw0`` cropped with the content to ``hw``
        (center_crop_to's window); any other map as it is."""
        if tuple(cl.shape[1:]) == tuple(hw0) and tuple(hw) != tuple(hw0):
            y0, x0 = (hw0[0] - hw[0]) // 2, (hw0[1] - hw[1]) // 2
            cl = cl[:, y0:y0 + hw[0], x0:x0 + hw[1]]
        return cl

    def _to_host(self, out_dev, out):
        """The uint8 frames ``out_dev`` copied into ``out`` (a pinned uint8 tensor) or into a new numpy array."""
        if out is not None:
            out.copy_(out_dev, non_blocking=True)
            out_u8 = out
        else:
            out_u8 = torch.empty(out_dev.shape, dtype=torch.uint8, pin_memory=True)
            out_u8.copy_(out_dev, non_blocking=True)
        # the call is synchronous like sess.run (wct.py:97); a device-side time-out would otherwise leave every
        # later frame silently wrong (kernels skip their stores once the error word is set)
        self.engine.check_device()
        if out is None:
            out_u8 = out_u8.numpy().copy()
        return out_u8

    @staticmethod
    def check_grey_prepared(ps):
        """ValueError unless the prepared style ``ps`` was prepared from a grey image (R = G = B everywhere), which is
        what luminance-only transfer takes: its statistics come from that image."""
        img = ps.image
        if img is None or not ((img[..., 0] == img[..., 1]).all() and (img[..., 1] == img[..., 2]).all()):
            raise ValueError("luminance_only takes a prepared style only when it was prepared grey: prepare it with "
                             "prepare_style(style, luminance_only=True) (prepare_styles.py --luminance-only)")

    def _predict_luminance(self, contents, styles, call, n):
        """predict_batch(luminance_only=True) for a call that has passed predict_batch's checks (DESIGN.md §3.3.15)."""
        from . import device_image as D
        from .temporal import stabilize_
        listed = any(call[k] is not None for k in ("style_weights", "content_mask", "content_weights"))
        entries = _style_list(styles) if listed else [styles]
        for x in entries:
            if isinstance(x, PreparedStyle):
                self.check_grey_prepared(x)
        dev = self.engine.device
        with torch.cuda.device(dev):
            full = _to_dev(contents, dev)
            c = self.swap_fit(full, call["swap5"], call["swap_targets"], lambda a: _to_dev(a, dev))
            if call["swap_labels"] is not None:
                cl, sl = call["swap_labels"]
                call["swap_labels"] = (self._crop_labels(cl, full.shape[1:3], c.shape[1:3]), sl)
            mean_c, sd_c = D.luminance_stats(c)
            # one grey, and the exact luminance moments of that grey, per distinct style object (the same object stays
            # the same object, so that style masks keep sharing its side)
            grey, moments = {}, {}
            for x in entries:
                if id(x) not in grey:
                    img = _to_dev(x.image, dev) if isinstance(x, PreparedStyle) else D.luminance_grey(_to_dev(x, dev))
                    grey[id(x)] = x if isinstance(x, PreparedStyle) else img
                    moments[id(x)] = D.luminance_moments(img)
            if call["style_weights"] is not None:
                w = self.normalize_weights(call["style_weights"], n, len(entries), dtype=np.float64)      # [1|N, K]
                st = np.array([D.luminance_stats_from_moments(m[0], m[1][0], m[2][0])
                               for m in (moments[id(x)] for x in entries)])                               # [K, 2]
                mean_s = w @ st[:, 0]
                sd_s = np.sqrt(np.maximum(w @ (st[:, 1] ** 2 + st[:, 0] ** 2) - mean_s ** 2, 0.0))
            elif listed:
                npix = sum(m[0] for m in moments.values())
                mean_s, sd_s = D.luminance_stats_from_moments(npix, sum(m[1][0] for m in moments.values()),
                                                              sum(m[2][0] for m in moments.values()))
            else:
                mean_s, sd_s = D.luminance_stats_from_moments(*moments[id(styles)])
            (k, b), (k_inv, b_merge) = D.luminance_params(mean_c, sd_c, mean_s, sd_s)
            # the grey has the cropped content's size, which the call below does not crop again
            g = D.luminance_match(c, k, b)
            inner = dict(call, luminance_only=False, temporal=None, out=None, return_device=True)
            del inner["self"], inner["contents"], inner["styles"]
            s = self.predict_batch(g, [grey[id(x)] for x in entries] if listed else grey[id(styles)], **inner)
            if tuple(s.shape[1:3]) != tuple(c.shape[1:3]):        # odd sizes: the decoders round the size up
                c = D.imresize(c, s.shape[1:3])
            out_dev = D.luminance_merge(c, s, k_inv, b_merge)
            if call["temporal"] is not None:
                stabilize_(call["temporal"], c, out_dev)
            if call["return_device"]:
                self.engine.check_device()
                return out_dev
            return self._to_host(out_dev, call["out"])

    @staticmethod
    def temporal_state(strength):
        """The temporal state of one clip for ``predict_batch(temporal=)``: ``strength`` in [0, 1) is the weight beta of the
        warped previous output (0 leaves every frame as it is); ValueError outside that range.  ``reset()`` starts the clip
        again."""
        from .temporal import TemporalState
        return TemporalState(strength)

    def prepare_style(self, style, swap_targets=None, luminance_only=False):
        """Prepare ``style`` (uint8 [H,W,3] or [n,H,W,3]; numpy or torch, host or device) once, for any number of calls.

        Returns a ``PreparedStyle`` of n styles holding, per relu target, the WCT state for this model's semantics and the
        AdaIN moments; the relu5_1 style feature when relu5_1 is a target (the style swap is prepared from it on first use);
        and the style image on the host (``--concat``).  It is accepted wherever a style image is: ``predict_batch`` /
        ``predict`` / ``synthesize`` with n in {1, N}, and as an entry (n = 1) of the style lists of ``style_weights`` and
        ``content_mask``, with ``adain``, ``passes`` and ``swap5``.  The results are byte-identical to the image's.
        ``swap_targets`` (relu targets) keeps the style feature of those levels too, for ``predict_batch(swap_targets=)``;
        ``save`` stores them.  ``luminance_only=True`` prepares the grey of the style (``device_image.luminance_grey``), the
        form ``predict_batch(luminance_only=True)`` takes; used without that option it is simply a grey style."""
        if isinstance(style, PreparedStyle):
            return style
        if style.dtype not in (np.uint8, torch.uint8) or style.ndim not in (3, 4) or style.shape[-1] != 3:
            raise ValueError("a style must be uint8 [H,W,3] or [n,H,W,3]")
        eng = self.engine
        with torch.cuda.device(eng.device):
            s = _to_dev(style, eng.device)
            if luminance_only:
                from .device_image import luminance_grey
                s = luminance_grey(s)
            ps = eng.prepare(s, swap_targets or ())
            ps.image = s.cpu().numpy()
            ps.fingerprints = dict(eng.fingerprints())
        return ps

    def load_style(self, path):
        """Read a ``.wctstyle`` file written by ``PreparedStyle.save``.  The file serves this model when its semantics
        are this model's and it holds every relu target of this model with the same encoder weights up to that relu;
        decoders do not matter.  Otherwise ValueError, naming the field: ``version``, ``eps_cov`` / ``eps_eig`` /
        ``thresh``, ``targets`` or ``<relu>/fingerprint``."""
        from . import prepared as P
        eng = self.engine
        data = P.read_file(path)
        sem = SEMANTICS[eng.semantics]
        taps = list(dict.fromkeys(self.model.style_taps))
        P.check_file(data, path, sem, taps, eng.fingerprints())
        image = data["image"]
        ps = PreparedStyle(image.shape[0], {k: sem[k] for k in P.SEMANTIC_KEYS}, taps)
        ps.image = image
        ps.fingerprints = {relu: str(data["%s/fingerprint" % relu]) for relu in taps}
        dev = eng.device
        with torch.cuda.device(dev):
            for relu in taps:
                ps.wct[relu] = P.pack_wct_state(eng.lib, data["%s/wct_mean" % relu], data["%s/wct_cs" % relu], data["%s/wct_k" % relu], dev)
                ps.adain[relu] = P.pack_adain_state(eng.lib, data["%s/adain_mean" % relu], data["%s/adain_var" % relu], dev)
            for relu in taps:
                # relu5_1 is always stored; another level only when the style was prepared to swap there
                if relu != "relu5_1" and "%s/feat" % relu not in data:
                    continue
                C = RELU_CHANNELS[relu]
                raw = data["%s/feat" % relu]                                    # float16 [2, n, Hs+2, Ws+2, C]
                if raw.dtype != np.float16 or raw.ndim != 5 or raw.shape[:2] != (2, ps.n) or raw.shape[4] != C:
                    raise ValueError("%s: %s/feat: bad shape %s" % (path, relu, raw.shape))
                act = eng._act(ps.n, raw.shape[2] - 2, raw.shape[3] - 2, C)
                flat = torch.from_numpy(np.ascontiguousarray(raw).view(np.uint8).reshape(-1)).to(dev)
                act.buf[:flat.numel()] = flat
                ps.feats[relu] = act
            main = torch.cuda.current_stream(dev)
            ps.side = main
            for relu in taps:
                ev = torch.cuda.Event()
                ev.record(main)
                ps.events[relu] = ev
        return ps

    def synthesize(self, styles, size, count=1, seed=0, first_index=0, **kw):
        """Texture synthesis (WCT paper, section 4; the reference's ``--noise``, webcam.py:191-192): stylise ``count`` frames
        of uniform noise made on the device into textures of the style.  ``size`` is (H, W) or one integer for a square.

        Defined as ``predict_batch(noise_u8(count, H, W, seed, first_index), styles, **kw)`` and equal to it byte for byte;
        ``kw`` is any ``predict_batch`` option (``alpha``, ``adain``, ``passes``, ``swap5`` / ``ss_alpha``, ``style_weights``
        for texture mixing, ``content_mask`` for texture painting, ``return_device``, ``out``, ``return_float``), with the
        same rules and rejections.

        Texture i depends only on the seed, ``first_index + i`` and the size, the styles and options, and the weights: not
        on ``count``, on how a run is cut into calls, or on the engine's sub-batch groups (the pipeline is batch-invariant,
        tests/test_gpu_invariance.py).  ``synthesize(count=5)`` equals ``synthesize(count=2)`` followed by
        ``synthesize(count=3, first_index=2)``.  ``luminance_only`` is rejected: noise has no colours to keep."""
        if kw.get("luminance_only"):
            raise ValueError("synthesize takes no luminance_only: noise frames have no colours to keep")
        from .device_image import noise_u8
        H, W = (size, size) if isinstance(size, (int, np.integer)) else size
        noise = noise_u8(count, H, W, seed=seed, first_index=first_index, device=self.engine.device)
        return self.predict_batch(noise, styles, **kw)

    def predict(self, content, style, alpha=1, swap5=False, ss_alpha=1, adain=False, content_mask=None, style_weights=None,
                style_masks=None, swap_targets=None, tile_size=None, ost=False, seamless=None, mst=None, mst_smooth=0.05,
                strength_map=None, content_weights=None, mask_feather=None, efdm=False, swap_labels=None, efdm_slices=0,
                luminance_only=False, coarse_to_fine=None, fine_targets=None, ss_temperature=None, ss_balance=0):
        '''Stylize a single content/style pair (wct.py:70-106).  With ``content_mask`` (uint8 [Hm,Wm] label map), ``style``
        is a list of R region styles and region r of the content takes style r (with ``style_masks``, the pixels of style r
        labelled r).  With ``style_weights`` ([K]), ``style`` is a list of K styles and the content takes their weighted
        blend.  ``tile_size`` stylises in tiles, ``ost`` uses the optimal-transport transform, ``seamless`` pads the content
        path circularly, ``mst`` = K matches the content to K modes of the style and ``efdm`` matches every channel's whole
        value distribution to the style's (first in ``efdm_slices`` rotated bases); ``strength_map``, ``content_weights``
        ([K,Hm,Wm], with ``style`` a list of K region styles) and ``mask_feather`` are soft spatial control
        (``predict_batch``); ``swap_labels`` = (content labels [Hm,Wm], style labels [Hm',Wm']) steers the style swap and
        ``ss_temperature`` makes it the softmax swap, ``ss_balance`` the balanced swap; ``luminance_only`` stylises the luminance and keeps the content's colours; ``coarse_to_fine`` = f stylises a 1/f
        copy at every level first and ``fine_targets`` at full size (scale control).'''
        s = time.time()
        seen = {}

        def host(x):
            # one host array per object: a style given twice stays one object (style_masks share its side)
            if id(x) not in seen:
                seen[id(x)] = x if isinstance(x, PreparedStyle) else np.asarray(x)
            return seen[id(x)]
        if style_weights is not None or content_mask is not None or content_weights is not None:
            style = [host(x) for x in _style_list(style)]
        else:
            style = host(style)
        out = self.predict_batch(np.asarray(content), style, alpha=alpha, swap5=swap5, ss_alpha=ss_alpha, adain=adain,
                                 content_mask=content_mask, style_weights=style_weights, style_masks=style_masks,
                                 swap_targets=swap_targets, tile_size=tile_size, ost=ost, seamless=seamless, mst=mst,
                                 mst_smooth=mst_smooth, strength_map=strength_map, content_weights=content_weights,
                                 mask_feather=mask_feather, efdm=efdm, swap_labels=swap_labels, efdm_slices=efdm_slices,
                                 luminance_only=luminance_only, coarse_to_fine=coarse_to_fine, fine_targets=fine_targets,
                                 ss_temperature=ss_temperature, ss_balance=ss_balance)
        if self.verbose:
            print("Stylized in:", time.time() - s)   # wct.py:104
        return out[0]
