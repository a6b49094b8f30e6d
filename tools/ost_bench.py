"""Cost of the optimal-transport transform (``predict_batch(ost=True)``, ``--ost``, DESIGN.md §3.3.8): 512x512 five-level
frames/s of 30 resident frames per step in two sub-batch groups (bench.py's default), WCT against OST in alternating runs,
for (i) one shared prepared style and (ii) one prepared style per frame.  Then, per level, the transform's milliseconds per
frame (CUDA events around each ``wct_apply`` / ``ost_apply`` call in a run of its own, one group, so that an event pair
times the call and not its overlap with the other group), and the share of frames whose B^1/2 took the Newton-Schulz fast
path (k_out).  The card name and power limit are read in the same call.

  python tools/ost_bench.py [--reps 3] [--steps 3] [--out FILE.json]
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
    styles = rng.integers(0, 256, (FRAMES, SIZE, SIZE, 3), dtype=np.uint8)
    cases = {"shared_style": wct.prepare_style(styles[0]), "style_per_frame": wct.prepare_style(styles)}
    res = dict(card(), frames_per_step=FRAMES, size=SIZE, groups=GROUPS, alpha=ALPHA, cases={})
    for name, ps in cases.items():
        def run(ost, steps):
            eng.groups = GROUPS
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                eng.stylize(contents, ps, alpha=ALPHA, ost=ost)
            torch.cuda.synchronize()
            return FRAMES * steps / (time.perf_counter() - t0)

        run(False, 1), run(True, 1)                                   # warm-up of every shape and workspace
        wct_fps, ost_fps = [], []
        for _ in range(a.reps):
            wct_fps.append(run(False, a.steps))
            ost_fps.append(run(True, a.steps))
        levels = {}
        eng.groups = 1
        for ost in (False, True):
            eng.stylize(contents, ps, alpha=ALPHA, ost=ost)          # warm-up of the one-group workspaces
            torch.cuda.synchronize()
            eng.profile = {}
            eng.stylize(contents, ps, alpha=ALPHA, ost=ost)
            torch.cuda.synchronize()
            for key, rec in eng.profile.items():
                relu, _, call = key.partition(":")
                if call.startswith("wct_level") or call.startswith("ost_level"):
                    ms = sum(e0.elapsed_time(e1) for e0, e1 in rec["events"]) / FRAMES
                    levels.setdefault(relu, {})["ost_ms_per_frame" if ost else "wct_ms_per_frame"] = ms
            eng.profile = None
        eng.stylize(contents, ps, alpha=ALPHA, ost=True, want_info=True)
        for relu, k in zip(TARGETS, eng.last_info):
            k = k.cpu().numpy()
            levels[relu]["b_root_newton_schulz_share"] = float(k[3 * FRAMES:4 * FRAMES].mean())
            levels[relu]["w_c_newton_schulz_share"] = float(k[2 * FRAMES:3 * FRAMES].mean())
        med = lambda v: float(np.median(v))  # noqa: E731
        res["cases"][name] = dict(wct_fps=med(wct_fps), ost_fps=med(ost_fps), wct_fps_runs=wct_fps, ost_fps_runs=ost_fps,
                                  ost_over_wct=med(ost_fps) / med(wct_fps), levels=levels)
    eng.check_device()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
