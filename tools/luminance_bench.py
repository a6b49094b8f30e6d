"""Cost of luminance-only transfer (``predict_batch(luminance_only=True)``, ``--luminance-only``, DESIGN.md §3.3.15).

  1. 512x512 five-level frames/s of 30 frames per step (``WCT.predict_batch`` with device input and output), with and
     without ``luminance_only``, with a shared style and with one style per frame; the two settings alternate within each
     repetition, medians of --reps.
  2. CUDA events (medians of --reps) around the batched moments, the match and the merge of one 30-frame step, with their
     bytes per second from the shapes (moments read 3 B/pixel; match reads 3 and writes 3; merge reads 6 and writes 3).
The card name and power limit are read in the same call.

  python tools/luminance_bench.py [--reps 5] [--steps 2] [--out FILE.json]
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
FRAMES, SIZE, ALPHA = 30, 512, 0.8


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=2, help="timed steps of FRAMES frames per run")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from wct_tf_b200 import device_image as D
    from wct_tf_b200.wct import WCT
    from wct_tf_b200.weights import make_synthetic_weights

    wct = WCT(relu_targets=TARGETS, weights=make_synthetic_weights(42, relu_targets=TARGETS))
    dev = wct.engine.device
    rng = np.random.default_rng(0)
    contents = torch.from_numpy(rng.integers(0, 256, (FRAMES, SIZE, SIZE, 3), dtype=np.uint8)).to(dev)
    styles = torch.from_numpy(rng.integers(0, 256, (FRAMES, SIZE, SIZE, 3), dtype=np.uint8)).to(dev)
    res = dict(card(), frames_per_step=FRAMES, size=SIZE, alpha=ALPHA)
    med = lambda v: float(np.median(v))  # noqa: E731

    # 1. frames/s
    def run(lum, shared, steps):
        sty = styles[:1] if shared else styles
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            wct.predict_batch(contents, sty, alpha=ALPHA, return_device=True, luminance_only=lum)
        torch.cuda.synchronize()
        return FRAMES * steps / (time.perf_counter() - t0)

    fps = {}
    for shared in (True, False):
        tag = "shared" if shared else "per_frame"
        for lum in (False, True):                                     # warm-up of every shape and workspace
            run(lum, shared, 1)
        runs = {False: [], True: []}
        for _ in range(a.reps):
            for lum in (False, True):
                runs[lum].append(run(lum, shared, a.steps))
        off, on = med(runs[False]), med(runs[True])
        fps[tag] = dict(off=off, on=on, overhead_pct=100.0 * (off / on - 1.0), runs_off=runs[False], runs_on=runs[True])
    res["fps"] = fps

    # 2. the three pixel steps of one step
    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        fn()
        ms = []
        for _ in range(a.reps):
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        return med(ms)

    lib = D._capi.load()
    npf = SIZE * SIZE
    sums = torch.empty((FRAMES, 9), dtype=torch.int64, device=dev)
    kb = torch.tensor([[1.1, -3.0]] * FRAMES, dtype=torch.float32, device=dev)
    grey = torch.empty_like(contents)
    merged = torch.empty_like(contents)
    st = D._stream()
    c, s = contents.data_ptr(), styles.data_ptr()
    check = D._capi.check
    moments = timed(lambda: check(lib.wctb200_rgb_moments_batch_u8(c, FRAMES, npf, sums.data_ptr(), st)))
    match = timed(lambda: check(lib.wctb200_luminance_match_u8(c, FRAMES, npf, kb.data_ptr(), grey.data_ptr(), st)))
    merge = timed(lambda: check(lib.wctb200_luminance_merge_u8(c, s, FRAMES, npf, kb.data_ptr(), merged.data_ptr(), st)))
    px = FRAMES * npf
    res["kernels"] = {name: dict(ms=ms, bytes=b * px, gb_per_s=b * px / (ms * 1e6))
                      for name, ms, b in (("moments", moments, 3), ("match", match, 6), ("merge", merge, 9))}
    wct.engine.check_device()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
