"""Cost of style masks: 512x512 five-level frames/s of spatial control with masks on the content only and on the style too.

One process measures, alternating the three cases run by run, with a batch of 30 frames as two sub-batch groups:
  a  content mask R = 2 (left / right halves), two distinct 512x512 styles: the style side of each is the whole style
  b  the same content mask, ONE 512x512 style with a style mask (top / bottom) shared by both regions: one encode and one
     masked prepare per level
  c  content mask R = 4 (quadrants), one style with a style mask of 4 quadrants shared by the 4 regions
Each case reports the median frames/s of the runs, and, from one profiled step per case, the style-side time per step: the
CUDA-event time of every C-ABI call enqueued for the style side (u8 -> f32, encoder, label resizes and prepares), which
runs on the style stream next to the content work.  The card's name and power limit are read in the same call.

  python tools/style_masks_bench.py [--steps 5] [--warmup 3] [--reps 3] [--out FILE.json]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.regions_bench import card  # noqa: E402

TARGETS = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]
SIZE, BATCH, ALPHA = 512, 30, 0.8


def masks(size):
    h = w = size
    c2 = np.zeros((h, w), np.uint8)
    c2[:, w // 2:] = 1
    s2 = np.zeros((h, w), np.uint8)
    s2[h // 2:] = 1
    q = (np.arange(h)[:, None] >= h // 2).astype(np.uint8) * 2 + (np.arange(w)[None, :] >= w // 2).astype(np.uint8)
    return dict(c2=c2, s2=s2, c4=q, s4=q.T.copy())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()

    import torch
    from wct_tf_b200.weights import make_synthetic_weights
    from wct_tf_b200.wct import WCT

    result = card()
    wct = WCT(relu_targets=TARGETS, weights=make_synthetic_weights(42), semantics="tf")
    eng = wct.engine
    rng = np.random.default_rng(1000)
    content = torch.from_numpy(rng.integers(0, 256, (BATCH, SIZE, SIZE, 3), dtype=np.uint8)).cuda()
    styles = [torch.from_numpy(rng.integers(0, 256, (1, SIZE, SIZE, 3), dtype=np.uint8)).cuda() for _ in range(2)]
    m = {k: torch.from_numpy(v).cuda() for k, v in masks(SIZE).items()}
    cases = {
        "a_content_mask_R2_two_styles": lambda: eng.stylize(content, None, alpha=ALPHA, labels=m["c2"], region_styles=styles),
        "b_style_mask_R2_one_style": lambda: eng.stylize(content, None, alpha=ALPHA, labels=m["c2"], region_styles=[styles[0]] * 2,
                                                         region_masks=[m["s2"]] * 2),
        "c_style_mask_R4_one_style": lambda: eng.stylize(content, None, alpha=ALPHA, labels=m["c4"], region_styles=[styles[0]] * 4,
                                                         region_masks=[m["s4"]] * 4),
    }

    def step(name):
        return eng.to_u8(cases[name]())

    fps = {k: [] for k in cases}
    for k in cases:
        for _ in range(args.warmup):
            step(k)
    torch.cuda.synchronize()
    for _ in range(args.reps):
        for k in cases:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                step(k)
            e1.record()
            torch.cuda.synchronize()
            fps[k].append(BATCH * args.steps / (e0.elapsed_time(e1) / 1e3))
    eng.check_device()
    result["frames_per_s"] = {k: dict(median=round(float(np.median(v)), 2), runs=[round(x, 2) for x in v]) for k, v in fps.items()}

    # style-side time: one profiled step per case (CUDA events around each C-ABI call tagged "style")
    style_ms, style_launches = {}, {}
    for k in cases:
        eng.profile = {}
        step(k)
        torch.cuda.synchronize()
        recs = [rec for key, rec in eng.profile.items() if key.startswith("style:")]
        style_ms[k] = round(sum(a.elapsed_time(b) for rec in recs for a, b in rec["events"]), 3)
        style_launches[k] = sum(rec["launches"] for rec in recs)
        eng.profile = None
    result["style_side_ms_per_step"] = style_ms
    result["style_side_launches_per_step"] = style_launches
    print(json.dumps(result, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
