"""What prepared styles save: image styles against prepared styles (WCT.prepare_style) on the workloads of DESIGN §6.

  python tools/prepared_bench.py [--runs 3] [--json OUT]

Cases (synthetic weights, five levels relu5_1 .. relu1_1, WCT tf unless noted; one 512x512 style):
  single     one 512x512 content per call, ms per call
  passes2    the same with passes=2, ms per call
  video      15-frame batches of one 30-frame 512x512 clip with one style (stylize_video --batch 15), frames/s
  swap5      30 frames of 512x512 with swap5 (patch 3, stride 1): 30 single-frame calls against one batched call, frames/s
  prepare    prepare_style of the style, and load_style of its file, ms
Every case is warmed up first; the image and prepared variants alternate, each run three times; the median and the spread
(max - min) are printed.  The card name and power limit are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from wct_tf_b200.wct import WCT                       # noqa: E402
from wct_tf_b200.weights import make_synthetic_weights  # noqa: E402

ALL = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    wct = WCT(relu_targets=ALL, weights=make_synthetic_weights(42))
    dev = wct.engine.device
    style = torch.from_numpy(rng.integers(0, 256, (512, 512, 3), dtype=np.uint8)).to(dev)
    one = torch.from_numpy(rng.integers(0, 256, (1, 512, 512, 3), dtype=np.uint8)).to(dev)
    clip = torch.from_numpy(rng.integers(0, 256, (30, 512, 512, 3), dtype=np.uint8)).to(dev)
    ps = wct.prepare_style(style)

    def single(s, passes=1):
        return lambda: wct.predict_batch(one, s, return_device=True, passes=passes)

    def video(s):
        return lambda: [wct.predict_batch(clip[i:i + 15], s, return_device=True) for i in (0, 15)]

    def swap_single(s):
        return lambda: [wct.predict_batch(clip[i:i + 1], s, swap5=True, ss_alpha=0.6, return_device=True) for i in range(30)]

    def swap_batch(s):
        return lambda: wct.predict_batch(clip, s, swap5=True, ss_alpha=0.6, return_device=True)

    cases = [  # name, unit, per-run work (frames or calls), {variant: fn}
        ("single", "ms/call", 1, {"image": single(style), "prepared": single(ps)}),
        ("passes2", "ms/call", 1, {"image": single(style, 2), "prepared": single(ps, 2)}),
        ("video", "frames/s", 30, {"image": video(style), "prepared": video(ps)}),
        ("swap5", "frames/s", 30, {"single_image": swap_single(style), "batched_image": swap_batch(style),
                                   "batched_prepared": swap_batch(ps)}),
    ]
    tmp = tempfile.mkdtemp()
    path = os.path.join(tmp, "style.wctstyle")
    ps.save(path)
    cases.append(("prepare", "ms", 1, {"prepare_style": lambda: wct.prepare_style(style), "load_style": lambda: wct.load_style(path)}))
    out = dict(card=card(), workload="synthetic weights, 5 levels relu5_1..relu1_1, WCT tf, 512x512 content and style", cases={})
    print(out["card"])
    for name, unit, work, fns in cases:
        for fn in fns.values():                          # warm-up: workspaces, streams, swap state
            fn()
            fn()
        times = {k: [] for k in fns}
        for _ in range(args.runs):                        # alternate the variants
            for k, fn in fns.items():
                times[k].append(timed(fn))
        res = {}
        for k, ts in times.items():
            vals = np.array([work / t if unit == "frames/s" else 1e3 * t / work for t in ts])
            res[k] = dict(median=float(np.median(vals)), spread=float(vals.max() - vals.min()), runs=[float(v) for v in vals])
            print("%-8s %-17s %9.2f %s  (spread %.2f)" % (name, k, res[k]["median"], unit, res[k]["spread"]))
        out["cases"][name] = dict(unit=unit, **res)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
