"""Cost and effect of seamless stylisation (``predict_batch(seamless=)``, ``--seamless``, DESIGN.md §3.3.9): 512x512
five-level frames/s of 30 resident frames per step in two sub-batch groups (bench.py's default), one shared prepared style,
for seamless None, "x" and "xy" in alternating runs (median of --reps); the time of one 4096x2048 "x" panorama per call;
and, per mode, the seam figure of a 512x512 frame: the mean |out[:, :, 0] - out[:, :, -1]| (the columns that meet when the
image is tiled) against the mean difference of neighbouring interior columns, and the same for rows.  The card name and
power limit are read in the same call.

  python tools/seamless_bench.py [--reps 3] [--steps 3] [--out FILE.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from regions_bench import card  # noqa: E402

TARGETS = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]
FRAMES, SIZE, ALPHA, GROUPS = 30, 512, 0.8, 2
MODES = (None, "x", "xy")


def seam(img):
    """(mean |first - last column|, mean |neighbouring interior columns|, the same for rows) of float images [N,H,W,3]."""
    img = img.astype(np.float64)
    return dict(col_seam=float(np.abs(img[:, :, 0] - img[:, :, -1]).mean()),
                col_interior=float(np.abs(np.diff(img, axis=2)).mean()),
                row_seam=float(np.abs(img[:, 0] - img[:, -1]).mean()),
                row_interior=float(np.abs(np.diff(img, axis=1)).mean()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3, help="timed steps of FRAMES frames per run")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from wct_tf_b200.weights import make_synthetic_weights
    from wct_tf_b200.wct import WCT

    wct = WCT(checkpoints=None, relu_targets=TARGETS, vgg_path=None, weights=make_synthetic_weights(42, relu_targets=TARGETS))
    eng = wct.engine
    dev = eng.device
    rng = np.random.default_rng(0)
    contents = torch.from_numpy(rng.integers(0, 256, (FRAMES, SIZE, SIZE, 3), dtype=np.uint8)).to(dev)
    ps = wct.prepare_style(rng.integers(0, 256, (SIZE, SIZE, 3), dtype=np.uint8))
    res = dict(card(), frames_per_step=FRAMES, size=SIZE, groups=GROUPS, alpha=ALPHA)

    def run(mode, steps):
        eng.groups = GROUPS
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            eng.stylize(contents, ps, alpha=ALPHA, seamless=mode)
        torch.cuda.synchronize()
        return FRAMES * steps / (time.perf_counter() - t0)

    for m in MODES:
        run(m, 1)                                                     # warm-up of every shape and workspace
    fps = {str(m): [] for m in MODES}
    for _ in range(a.reps):
        for m in MODES:
            fps[str(m)].append(run(m, a.steps))
    med = {k: float(np.median(v)) for k, v in fps.items()}
    res["fps"] = med
    res["fps_runs"] = fps
    res["fps_over_reflect"] = {k: v / med["None"] for k, v in med.items()}
    launches = {}
    for m in MODES:
        n0 = eng.launches
        eng.stylize(contents, ps, alpha=ALPHA, seamless=m)
        launches[str(m)] = eng.launches - n0
    res["launches_per_step"] = launches

    pano = torch.from_numpy(rng.integers(0, 256, (1, 2048, 4096, 3), dtype=np.uint8)).to(dev)
    eng.groups = 1
    eng.stylize(pano, ps, alpha=ALPHA, seamless="x")
    torch.cuda.synchronize()
    t = []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        eng.stylize(pano, ps, alpha=ALPHA, seamless="x")
        torch.cuda.synchronize()
        t.append(time.perf_counter() - t0)
    res["panorama_4096x2048_x_s"] = float(np.median(t))
    del pano

    res["seam"] = {}
    for m in MODES:
        out = wct.predict_batch(contents[:2], ps, alpha=ALPHA, seamless=m)
        res["seam"][str(m)] = seam(out)
    eng.check_device()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
