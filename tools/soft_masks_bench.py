"""Cost of soft spatial control (DESIGN.md §3.3.11) on 512x512 five-level frames.

One process measures, alternating the five cases run by run, with a batch of 30 frames per step in two groups and one
512x512 style per region:
  a  plain WCT
  b  a left-to-right strength ramp
  c  a hard R = 2 mask of two halves
  d  the same mask with mask_feather = 16
  e  feathered (sigma = 16) R = 4 blobs
Each case reports the median frames/s of the runs and the launches per step; the card's name and power limit are read in
the same call.

  python tools/soft_masks_bench.py [--steps 5] [--warmup 3] [--reps 3] [--out FILE.json]
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
SIZE, BATCH, ALPHA, SIGMA = 512, 30, 0.8, 16.0


def blobs(size, R, seed=7):
    rng = np.random.default_rng(seed)
    m = np.zeros((size, size), np.uint8)
    yy, xx = np.mgrid[:size, :size]
    for r in range(1, R):
        cy, cx, rad = rng.integers(0, size, 2).tolist() + [int(rng.integers(size // 6, size // 3))]
        m[(yy - cy) ** 2 + (xx - cx) ** 2 < rad * rad] = r
    return m


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
    eng.groups = 2
    rng = np.random.default_rng(1000)
    content = torch.from_numpy(rng.integers(0, 256, (BATCH, SIZE, SIZE, 3), dtype=np.uint8)).cuda()
    styles = [torch.from_numpy(rng.integers(0, 256, (1, SIZE, SIZE, 3), dtype=np.uint8)).cuda() for _ in range(4)]
    ramp = torch.linspace(0, 1, SIZE, device="cuda").view(1, 1, SIZE).expand(1, SIZE, SIZE).contiguous()
    halves = torch.zeros((1, SIZE, SIZE), dtype=torch.uint8, device="cuda")
    halves[..., SIZE // 2:] = 1
    four = torch.from_numpy(blobs(SIZE, 4)).cuda()
    cases = {
        "a_plain": lambda: eng.stylize(content, styles[0], alpha=ALPHA),
        "b_strength_ramp": lambda: eng.stylize(content, styles[0], alpha=ALPHA, strength_map=ramp),
        "c_hard_R2": lambda: eng.stylize(content, None, alpha=ALPHA, labels=halves, region_styles=styles[:2]),
        "d_feather_R2": lambda: eng.stylize(content, None, alpha=ALPHA, labels=halves, region_styles=styles[:2], mask_feather=SIGMA),
        "e_feather_R4": lambda: eng.stylize(content, None, alpha=ALPHA, labels=four, region_styles=styles, mask_feather=SIGMA),
    }

    def step(name):
        return eng.to_u8(cases[name]())

    fps = {k: [] for k in cases}
    launches = {}
    for k in cases:
        for _ in range(args.warmup):
            step(k)
        n0 = eng.launches
        step(k)
        launches[k] = eng.launches - n0
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
    med = {k: float(np.median(v)) for k, v in fps.items()}
    result["frames_per_s"] = {k: dict(median=round(med[k], 2), runs=[round(x, 2) for x in v]) for k, v in fps.items()}
    result["launches_per_step"] = launches
    result["ratios"] = {"b_over_a": round(med["b_strength_ramp"] / med["a_plain"], 3),
                        "d_over_c": round(med["d_feather_R2"] / med["c_hard_R2"], 3)}
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
