"""Cost of temporal stabilisation (``predict_batch(temporal=)``, ``stylize_video.py --temporal``): five-level frames/s of
two 30-frame synthetic clips, 512x512 and 1920x1080, in batches of 15 (the CLI's default ``--batch``), with and without
strength 0.8, alternating run by run; and the flow + confidence + blend time per frame from CUDA events around the
stabilisation of the same batches.  The card name and power limit are read in the same call.

  python tools/temporal_bench.py [--reps 3] [--out FILE.json]
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
FRAMES, BATCH, ALPHA, STRENGTH = 30, 15, 0.8, 0.8
SIZES = [(512, 512), (1080, 1920)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from tests import temporal_ref as R
    from wct_tf_b200.temporal import stabilize_
    from wct_tf_b200.weights import make_synthetic_weights
    from wct_tf_b200.wct import WCT

    wct = WCT(checkpoints=None, relu_targets=TARGETS, vgg_path=None, weights=make_synthetic_weights(42, relu_targets=TARGETS))
    dev = wct.engine.device
    style = torch.from_numpy(R.texture(512, 512, 77)).to(dev)
    res = dict(card(), frames=FRAMES, batch=BATCH, strength=STRENGTH, sizes={})
    for H, W in SIZES:
        clip = torch.from_numpy(R.translating_clip(FRAMES, H, W, d=(1.5, 0.5), seed=3)).to(dev)

        def run(temporal):
            st = wct.temporal_state(STRENGTH) if temporal else None
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(0, FRAMES, BATCH):
                kw = dict(temporal=st) if temporal else {}
                wct.predict_batch(clip[i:i + BATCH], style, alpha=ALPHA, return_device=True, **kw)
            torch.cuda.synchronize()
            return FRAMES / (time.perf_counter() - t0)

        def stab_ms():
            outs = [wct.predict_batch(clip[i:i + BATCH], style, alpha=ALPHA, return_device=True) for i in range(0, FRAMES, BATCH)]
            st = wct.temporal_state(STRENGTH)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            with torch.cuda.device(dev):
                e0.record()
                for j, o in enumerate(outs):
                    stabilize_(st, clip[j * BATCH:(j + 1) * BATCH], o)
                e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / FRAMES

        run(False), run(True), stab_ms()                      # warm-up of every shape
        plain, temporal, ms = [], [], []
        for _ in range(a.reps):
            plain.append(run(False))
            temporal.append(run(True))
            ms.append(stab_ms())
        med = lambda v: float(np.median(v))  # noqa: E731
        r = dict(plain_fps=med(plain), temporal_fps=med(temporal), plain_fps_runs=plain, temporal_fps_runs=temporal,
                 stabilise_ms_per_frame=med(ms), stabilise_ms_runs=ms, stylise_ms_per_frame=1000.0 / med(plain))
        r["overhead_pct"] = 100.0 * r["stabilise_ms_per_frame"] / r["stylise_ms_per_frame"]
        res["sizes"]["%dx%d" % (W, H)] = r
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
