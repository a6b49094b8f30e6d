"""Cost of coarse-to-fine stylisation (``predict_batch(coarse_to_fine=f)``, ``--coarse-to-fine``, DESIGN.md §3.3.16).

  1. Seconds per frame and ``torch.cuda.max_memory_allocated`` of one five-level WCT frame (device input and output, a
     prepared 512x512 style) at full resolution against f = 2 and f = 4: 2048^2 and 4096^2 untiled, 12288^2 with
     T = 2048.  The three settings alternate within each repetition; medians of --reps.  Beside them, the conv-MAC share
     that the issue's arithmetic predicts (``mac_share``, from ``model.encoder_plan`` / ``decoder_plan``).
  2. CUDA events (medians of --reps) around the join kernel at 4096^2 from 1024^2 and 12288^2 from 3072^2, with bytes/s
     over the compulsory 6 B per output pixel (3 read, 3 written) and over all bytes it touches (plus the two coarse
     images once).
The card name and power limit are read in the same call.

  python tools/coarse_bench.py [--reps 3] [--out FILE.json]
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
FINE = ("relu3_1", "relu2_1", "relu1_1")
CASES = [(2048, None), (4096, None), (12288, 2048)]


def level_macs(relu):
    """Conv MACs per full-resolution pixel of one level: its encoder and its decoder."""
    from wct_tf_b200.model import decoder_plan, encoder_plan
    macs, scale = 0.0, 1.0
    for op in encoder_plan(relu):
        if op.kind == "pool":
            scale /= 4.0
        else:
            macs += 9.0 * op.cin * op.cout * scale
    for op in decoder_plan(relu):
        if op.kind == "up":
            scale *= 4.0
        else:
            macs += 9.0 * op.cin * op.cout * scale
    return macs


def mac_share(f):
    """Conv work of a coarse-to-fine call over a full-resolution five-level call: every level on 1/f^2 of the pixels, and
    the fine levels again at full size."""
    total = sum(level_macs(r) for r in TARGETS)
    return (total / f ** 2 + sum(level_macs(r) for r in FINE)) / total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from wct_tf_b200 import device_image as D
    from wct_tf_b200.wct import WCT
    from wct_tf_b200.weights import make_synthetic_weights

    wct = WCT(relu_targets=TARGETS, weights=make_synthetic_weights(42, relu_targets=TARGETS))
    dev = wct.engine.device
    rng = np.random.default_rng(0)
    style = wct.prepare_style(rng.integers(0, 256, (512, 512, 3), dtype=np.uint8))
    res = dict(card(), style=512, reps=a.reps, mac_share={f: mac_share(f) for f in (2, 4, 8)})
    med = lambda v: float(np.median(v))  # noqa: E731

    # 1. seconds per frame and peak memory
    def run(c, f, tile):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated(dev)
        torch.cuda.reset_peak_memory_stats(dev)
        t0 = time.perf_counter()
        out = wct.predict_batch(c, style, return_device=True, coarse_to_fine=f, tile_size=tile)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        peak = torch.cuda.max_memory_allocated(dev) - base
        del out
        return dt, peak

    calls = {}
    for size, tile in CASES:
        # smooth gradients with noise: a content with structure at every scale
        t = np.arange(size, dtype=np.float32) / size
        y, x = t[:, None], t[None, :]
        img = np.empty((1, size, size, 3), np.uint8)
        for ch, plane in enumerate((128 + 100 * np.sin(9 * x + 2) + 0 * y, 128 + 100 * np.cos(7 * y) + 0 * x,
                                    128 + 90 * np.sin(5 * (x + y)))):
            plane = plane + 8 * rng.standard_normal((size, size), dtype=np.float32)
            img[0, :, :, ch] = np.clip(plane, 0, 255)
        c = torch.from_numpy(img).to(dev)
        del img
        settings = (None, 2, 4)
        for f in settings:                                  # warm-up of every shape and workspace
            run(c, f, tile)
        runs = {f: [] for f in settings}
        for _ in range(a.reps):
            for f in settings:
                runs[f].append(run(c, f, tile))
        row = {}
        for f in settings:
            row["full" if f is None else "f%d" % f] = dict(s_per_frame=med([r[0] for r in runs[f]]),
                                                           peak_gb=max(r[1] for r in runs[f]) / 1e9,
                                                           runs=[r[0] for r in runs[f]])
        for f in (2, 4):
            row["f%d" % f]["time_ratio"] = row["f%d" % f]["s_per_frame"] / row["full"]["s_per_frame"]
        calls["%d%s" % (size, "" if tile is None else "_T%d" % tile)] = row
        del c
        torch.cuda.empty_cache()
    res["calls"] = calls

    # 2. the join kernel
    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        fn()
        ms = []
        for _ in range(a.reps):
            e0.record()
            for _ in range(10):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1) / 10)
        return med(ms)

    lib = D._capi.load()
    joins = {}
    for H, h in ((4096, 1024), (12288, 3072)):
        c = torch.from_numpy(rng.integers(0, 256, (1, H, H, 3), dtype=np.uint8)).to(dev)
        d = torch.from_numpy(rng.integers(0, 256, (1, h, h, 3), dtype=np.uint8)).to(dev)
        s = torch.from_numpy(rng.integers(0, 256, (1, h, h, 3), dtype=np.uint8)).to(dev)
        out = torch.empty_like(c)
        st = D._stream()
        ms = timed(lambda: D._capi.check(lib.wctb200_coarse_join_u8(c.data_ptr(), d.data_ptr(), s.data_ptr(), 1, H, H, h, h,
                                                                    out.data_ptr(), st)))
        compulsory = 6.0 * H * H
        touched = compulsory + 6.0 * h * h
        joins["%d_from_%d" % (H, h)] = dict(ms=ms, compulsory_bytes=compulsory, gb_per_s=compulsory / (ms * 1e6),
                                            gb_per_s_touched=touched / (ms * 1e6))
        del c, d, s, out
        torch.cuda.empty_cache()
    res["join"] = joins
    wct.engine.check_device()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
