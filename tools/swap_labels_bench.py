"""Cost of the labelled style swap against the unlabelled one (512x512 content and style, patch 3, stride 1, synthetic
weights).

  python tools/swap_labels_bench.py [--runs 5] [--json OUT]

  levels   per level relu5_1 / relu4_1 / relu3_1 at Nc = 1 and 15: the apply per frame unlabelled, and labelled with 2 and 8
           labels (block maps of 512^2 on the content and the style, every label present in both), with the workspace the
           engine gives it
  pipeline five-level frames/s of one 15-frame step (WCT.predict_batch, one shared style) with the swap at relu3_1,
           unlabelled and with 8 labels
The variants of a case run alternately, one after another in every run; times are medians of ``--runs`` runs, each ended by
a device synchronise, after a warm-up of every variant.  The card name and power limit are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.swap_levels_bench import card, chunks      # noqa: E402
from wct_tf_b200.model import RELU_CHANNELS          # noqa: E402
from wct_tf_b200.wct import WCT                       # noqa: E402
from wct_tf_b200.weights import make_synthetic_weights  # noqa: E402

ALL = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]


def blocks(k, seed, size=512, cells=8):
    """A size x size label map of cells x cells blocks carrying each of the k labels at least once."""
    rng = np.random.default_rng(seed)
    grid = np.concatenate([np.arange(k), rng.integers(0, k, cells * cells - k)]).astype(np.uint8)
    grid = rng.permutation(grid).reshape(cells, cells)
    idx = np.arange(size) * cells // size
    return np.ascontiguousarray(grid[idx][:, idx])


def alternate(fns, runs):
    """Median seconds of each of ``fns`` (a dict), run alternately ``runs`` times after one warm-up each."""
    for fn in fns.values():
        fn()
    ts = {name: [] for name in fns}
    for _ in range(runs):
        for name, fn in fns.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts[name].append(e0.elapsed_time(e1) / 1e3)
    return {name: float(np.median(v)) for name, v in ts.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    wct = WCT(relu_targets=ALL, weights=make_synthetic_weights(42))
    eng, lib = wct.engine, wct.engine.lib
    dev = eng.device
    style_u8 = torch.from_numpy(rng.integers(0, 256, (1, 512, 512, 3), dtype=np.uint8)).to(dev)
    clip_u8 = torch.from_numpy(rng.integers(0, 256, (15, 512, 512, 3), dtype=np.uint8)).to(dev)
    maps = {k: (torch.from_numpy(blocks(k, 1)).to(dev)[None], torch.from_numpy(blocks(k, 2)).to(dev)[None]) for k in (2, 8)}
    out = dict(card=card(), workload="synthetic weights, 512x512 content and style, patch 3 stride 1; block label maps",
               levels=[], pipeline={})
    print(out["card"])

    def f32(u8):
        x = torch.empty(u8.shape, dtype=torch.float32, device=dev)
        eng._call("u8_to_f32", 1, lib.wctb200_image_u8_to_f32, u8.data_ptr(), u8.numel(), x.data_ptr(), eng._stream())
        return x

    _, sfeats = eng.encode(f32(style_u8), "relu5_1", taps=ALL)
    for relu in ("relu5_1", "relu4_1", "relu3_1"):
        sf = sfeats[relu]
        C = RELU_CHANNELS[relu]
        state = eng.swap_prepare(sf, 3, 1)
        for nc in (1, 15):
            cf, _ = eng.encode(f32(clip_u8[:nc]), relu)
            nbytes, nchunks, npat = chunks(lib, C, nc, cf.H, cf.W, sf.H, sf.W, 3, 1)
            fns = {"unlabelled": lambda: eng.swap_apply(cf, state, (sf.H, sf.W), 0.6)}
            for k, (cl, sl) in maps.items():
                fns["labels_%d" % k] = (lambda cl=cl, sl=sl: eng.swap_apply(cf, state, (sf.H, sf.W), 0.6, labels=(cl, sl)))
            t = alternate(fns, args.runs)
            r = dict(relu=relu, C=C, Nc=nc, map=[cf.H, cf.W], patches=npat, chunks=nchunks, workspace_bytes=nbytes,
                     **{name + "_ms_per_frame": 1e3 * v / nc for name, v in t.items()})
            out["levels"].append(r)
            print("%s C %d Nc %2d map %dx%d: %6d patches, %d chunk(s): apply ms/frame unlabelled %8.2f, 2 labels %8.2f, "
                  "8 labels %8.2f" % (relu, C, nc, cf.H, cf.W, npat, nchunks, r["unlabelled_ms_per_frame"],
                                      r["labels_2_ms_per_frame"], r["labels_8_ms_per_frame"]))
            del cf, fns
        del state
    torch.cuda.empty_cache()

    cl8, sl8 = (t[0] for t in maps[8])
    kw = dict(swap_targets=["relu3_1"], ss_alpha=0.6, return_device=True)
    t = alternate({"swap_relu3_1": lambda: wct.predict_batch(clip_u8, style_u8, **kw),
                   "swap_relu3_1_labels_8": lambda: wct.predict_batch(clip_u8, style_u8, swap_labels=(cl8, sl8), **kw)},
                  args.runs)
    for name, v in t.items():
        out["pipeline"][name] = 15 / v
        print("pipeline %-22s %8.2f frames/s (15 frames per step)" % (name, 15 / v))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
