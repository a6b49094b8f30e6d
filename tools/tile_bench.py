"""Cost of tiled stylisation (``predict_batch(tile_size=)``, ``stylize.py --tile-size``, DESIGN.md §3.3.7): seconds per
five-level frame and peak allocated device memory at 2048^2 and 4096^2, untiled and at T in {512, 1024, 2048}, the runs of
one size alternating; then one 12288^2 frame tiled (the untiled call rejects it).  WCT, 512^2 style prepared once,
synthetic weights.  The card name and power limit are read in the same call.

  python tools/tile_bench.py [--reps 3] [--big-tile 2048] [--out FILE.json]
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
ALPHA = 0.8


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--big-tile", type=int, default=2048)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from wct_tf_b200.engine import Engine
    from wct_tf_b200.weights import make_synthetic_weights

    eng = Engine(make_synthetic_weights(42, relu_targets=TARGETS), TARGETS)
    dev = eng.device
    rng = np.random.default_rng(1)
    ps = eng.prepare_call(torch.from_numpy(rng.integers(0, 256, (1, 512, 512, 3), dtype=np.uint8)).to(dev))
    torch.cuda.synchronize()

    def run(content, T):
        """(seconds, peak bytes allocated above what was allocated before the call) of one frame."""
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        out = eng.stylize(content, ps, alpha=ALPHA) if T == 0 else eng.stylize_tiled(content, ps, alpha=ALPHA, tile_size=T)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        peak = torch.cuda.max_memory_allocated() - base
        del out
        return dt, peak

    res = dict(card(), sizes={})
    for S in (2048, 4096):
        content = torch.from_numpy(rng.integers(0, 256, (1, S, S, 3), dtype=np.uint8)).to(dev)
        modes = [0, 512, 1024, 2048]
        for T in modes:
            run(content, T)                                   # warm-up of every shape
        times = {T: [] for T in modes}
        peaks = {}
        for _ in range(a.reps):
            for T in modes:
                dt, peaks[T] = run(content, T)
                times[T].append(dt)
        res["sizes"]["%d" % S] = {("untiled" if T == 0 else "T%d" % T): dict(s_per_frame=float(np.median(times[T])), runs=times[T],
                                                                            peak_gb=peaks[T] / 1e9) for T in modes}
        u = res["sizes"]["%d" % S]["untiled"]["s_per_frame"]
        for k, v in res["sizes"]["%d" % S].items():
            v["vs_untiled"] = v["s_per_frame"] / u
        del content
    S = 12288
    content = torch.from_numpy(rng.integers(0, 256, (1, S, S, 3), dtype=np.uint8)).to(dev)
    dt, peak = run(content, a.big_tile)
    res["sizes"]["%d" % S] = {"T%d" % a.big_tile: dict(s_per_frame=dt, peak_gb=peak / 1e9)}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
