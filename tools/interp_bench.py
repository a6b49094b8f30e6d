"""Cost of style interpolation: 512x512 five-level frames/s, the plain single-style path vs blends of K styles.

One process measures, alternating the four cases run by run:
  plain     one style for the whole batch (Engine.stylize)
  K2        two styles, one weight row shared by every frame
  K2_morph  two styles, one weight row per frame (a morph across the 30 frames of a step)
  K4_morph  four styles, one weight row per frame
with a batch of 30 frames resident on the device as two sub-batch groups (bench.py's default), the same images in every
case.  Then one profiled step per case gives per-level CUDA-event times of the transform call (wct_apply for the plain path,
wct_apply_blend otherwise) and of the style side.  The card name and power limit are read in the same call.

  python tools/interp_bench.py [--steps 5] [--warmup 3] [--reps 3] [--out FILE.json]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from regions_bench import card  # noqa: E402
from stylize_video import morph_weights  # noqa: E402

TARGETS = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]
SIZE, BATCH, ALPHA = 512, 30, 0.8


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
    styles = [torch.from_numpy(rng.integers(0, 256, (1, SIZE, SIZE, 3), dtype=np.uint8)).cuda() for _ in range(4)]
    weights = {"K2": torch.tensor([[0.3, 0.7]], dtype=torch.float32).cuda(),
               "K2_morph": torch.from_numpy(morph_weights(BATCH, 2).astype(np.float32)).cuda(),
               "K4_morph": torch.from_numpy(morph_weights(BATCH, 4).astype(np.float32)).cuda()}

    def step(mode):
        if mode == "plain":
            out = eng.stylize(content, styles[0], alpha=ALPHA)
        else:
            w = weights[mode]
            out = eng.stylize(content, None, alpha=ALPHA, interp_styles=styles[:w.shape[1]], interp_weights=w)
        return eng.to_u8(out)

    modes = ["plain", "K2", "K2_morph", "K4_morph"]
    fps = {m: [] for m in modes}
    for m in modes:
        for _ in range(args.warmup):
            step(m)
    torch.cuda.synchronize()
    for _ in range(args.reps):
        for m in modes:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                step(m)
            e1.record()
            torch.cuda.synchronize()
            fps[m].append(BATCH * args.steps / (e0.elapsed_time(e1) / 1e3))
    eng.check_device()
    result["frames_per_s"] = {m: dict(median=float(np.median(v)), runs=[round(x, 2) for x in v]) for m, v in fps.items()}
    result["ratio_vs_plain"] = {m: result["frames_per_s"][m]["median"] / result["frames_per_s"]["plain"]["median"] for m in modes}

    # per-level transform time and style-side time: one profiled step per case (CUDA events around each C-ABI call)
    per_level, style_ms = {}, {}
    for m in modes:
        eng.profile = {}
        step(m)
        torch.cuda.synchronize()
        for key, rec in eng.profile.items():
            lvl, _, name = key.partition(":")
            t = sum(a.elapsed_time(b) for a, b in rec["events"])
            if lvl == "style":
                style_ms[m] = round(style_ms.get(m, 0.0) + t, 3)
            elif name.startswith("wct_level") or name.startswith("wct_blend"):
                per_level.setdefault(lvl, {})[m] = round(t, 3)
        eng.profile = None
    result["transform_ms_per_step"] = per_level
    result["style_side_ms_per_step"] = style_ms
    print(json.dumps(result, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
