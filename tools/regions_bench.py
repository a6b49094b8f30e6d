"""Cost of spatial control: 512x512 five-level frames/s, unmasked vs a label map with R = 2 and R = 4 regions.

One process measures, alternating the three modes run by run:
  plain  one style for the whole batch (Engine.stylize)
  R2     left / right halves, two styles
  R4     random blobs for regions 1..3 over region 0, plus an unlabelled strip (label 4) that keeps the content
with a batch of 30 frames as two sub-batch groups (bench.py's default), the same style images in every mode.
Then one profiled step per mode gives per-level CUDA-event times of wct_apply (plain) and wct_apply_regions, and the
tiles each level processes (covariance 32x2 tiles x block pairs summed over the regions present, apply 128-position
passes) next to the unmasked count; those counts come from the mask alone (--counts-only runs them without a GPU).
The card name and power limit are read in the same call.

  python tools/regions_bench.py [--steps 5] [--warmup 3] [--reps 3] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests.regions_ref import resize_labels  # noqa: E402

TARGETS = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]
LEVEL_SIZE = {"relu1_1": (1, 64), "relu2_1": (2, 128), "relu3_1": (4, 256), "relu4_1": (8, 512), "relu5_1": (16, 512)}
SIZE, BATCH, ALPHA = 512, 30, 0.8


def masks(size):
    h = w = size
    m2 = np.zeros((h, w), np.uint8)
    m2[:, w // 2:] = 1
    rng = np.random.default_rng(11)
    m4 = np.zeros((h, w), np.uint8)
    yy, xx = np.mgrid[:h, :w]
    for r in range(1, 4):
        cy, cx, rad = rng.integers(0, h), rng.integers(0, w), rng.integers(h // 6, h // 3)
        m4[(yy - cy) ** 2 + (xx - cx) ** 2 < rad * rad] = r
    m4[h - h // 8:, :] = 4
    return {"R2": (m2, 2), "R4": (m4, 4)}


def tile_counts(mask, R, size):
    """Per level: (covariance tiles x block pairs, apply passes) for the mask and for the unmasked path."""
    rows = {}
    for relu, (down, C) in LEVEL_SIZE.items():
        H = W = size // down
        lab = resize_labels(mask, H, W).astype(np.int64)
        cnt = np.bincount(lab.ravel(), minlength=R + 1)[:R]
        npairs = 1 if C == 64 else (C // 128) * (C // 128 + 1) // 2
        ty, tx = (H + 1) // 2, (W + 31) // 32
        padt = np.full((ty * 2, tx * 32), 255, np.int64)
        padt[:H, :W] = lab
        tiles = padt.reshape(ty, 2, tx, 32).transpose(0, 2, 1, 3).reshape(ty * tx, 64)
        cov = sum(int((tiles == r).any(axis=1).sum()) for r in range(R)) * npairs
        eff = np.where((lab < R) & (cnt[np.minimum(lab, R - 1)] >= 2), lab, R)
        padded = np.full((H + 2, W + 2), -1, np.int64)
        padded[1:-1, 1:-1] = eff
        flat = padded.ravel()
        n_at = -(-flat.size // 128)
        flat = np.concatenate([flat, np.full(n_at * 128 - flat.size, -1)]).reshape(n_at, 128)
        passes = sum(int((flat == r).any(axis=1).sum()) for r in range(R))      # mainloop + epilogue passes
        copies = int((flat == R).any(axis=1).sum())                              # tiles that copy kept pixels
        rows[relu] = dict(cov_tiles=cov, cov_tiles_unmasked=ty * tx * npairs, apply_passes=passes, apply_copy_tiles=copies,
                          apply_tiles_unmasked=n_at)
    return rows


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                           stderr=subprocess.STDOUT, timeout=30).stdout.decode().strip().splitlines()[0]
        name, plim = [s.strip() for s in q.split(",")]
        return dict(gpu=name, power_limit=plim)
    except Exception as e:      # the measurement is still reported, with the card unknown
        return dict(gpu="unknown (%s)" % e, power_limit="unknown")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", type=str, default=None)
    ap.add_argument("--counts-only", action="store_true", help="print the per-level tile counts (no GPU needed)")
    args = ap.parse_args()
    ms = masks(SIZE)
    result = dict(tiles={k: tile_counts(m, R, SIZE) for k, (m, R) in ms.items()})
    if args.counts_only:
        print(json.dumps(result, indent=1))
        return

    import torch
    from wct_tf_b200.weights import make_synthetic_weights
    from wct_tf_b200.wct import WCT

    result.update(card())
    wct = WCT(relu_targets=TARGETS, weights=make_synthetic_weights(42), semantics="tf")
    eng = wct.engine
    rng = np.random.default_rng(1000)
    content = torch.from_numpy(rng.integers(0, 256, (BATCH, SIZE, SIZE, 3), dtype=np.uint8)).cuda()
    styles = [torch.from_numpy(rng.integers(0, 256, (1, SIZE, SIZE, 3), dtype=np.uint8)).cuda() for _ in range(4)]
    labels = {k: torch.from_numpy(m).cuda() for k, (m, _) in ms.items()}

    def step(mode):
        if mode == "plain":
            out = eng.stylize(content, styles[0], alpha=ALPHA)
        else:
            R = ms[mode][1]
            out = eng.stylize(content, None, alpha=ALPHA, labels=labels[mode], region_styles=styles[:R])
        return eng.to_u8(out)

    modes = ["plain", "R2", "R4"]
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

    # per-level transform time: one profiled step per mode (CUDA events around each C-ABI call)
    per_level = {}
    for m in modes:
        eng.profile = {}
        step(m)
        torch.cuda.synchronize()
        for key, rec in eng.profile.items():
            lvl, _, name = key.partition(":")
            if name.startswith("wct_level") or name.startswith("wct_regions"):
                t = sum(a.elapsed_time(b) for a, b in rec["events"])
                per_level.setdefault(lvl, {})[m] = round(t, 3)
        eng.profile = None
    result["transform_ms_per_step"] = per_level
    print(json.dumps(result, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
