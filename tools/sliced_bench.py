"""Cost of sliced distribution matching (``predict_batch(efdm=True, efdm_slices=K)``, ``--efdm-slices``, DESIGN.md §3.3.14).

  1. 512x512 five-level frames/s of 30 frames per step in two sub-batch groups, at K = 0 (plain EFDM), 1, 4 and 8, with a
     shared style and with one style per frame; the K values alternate within each repetition, medians of --reps.  The
     peak device memory of each configuration is reported beside it.
  2. Per level and per step, CUDA events (medians of --reps) around one rotated style prepare (rotate + sort + decode of
     30 styles), one sliced step (rotate + sort + runs of 30 frames: half of a K = 1 chain) and one plain EFDM apply
     (keys + sort + runs): the step minus the apply is what the rotation adds.
The card name and power limit are read in the same call.

  python tools/sliced_bench.py [--reps 3] [--steps 2] [--out FILE.json]
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
SLICES = (0, 1, 4, 8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=2, help="timed steps of FRAMES frames per run")
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
    styles = torch.from_numpy(rng.integers(0, 256, (FRAMES, SIZE, SIZE, 3), dtype=np.uint8)).to(dev)
    res = dict(card(), frames_per_step=FRAMES, size=SIZE, groups=GROUPS, alpha=ALPHA)
    med = lambda v: float(np.median(v))  # noqa: E731
    for K in SLICES:                                                  # the bases, made once per process (host numpy)
        if K:
            for C in (64, 128, 256, 512):
                eng.sliced_matrices(C, K)

    # 1. frames/s
    def run(K, shared, steps):
        eng.groups = GROUPS
        sty = styles[:1] if shared else styles
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            eng.stylize(contents, sty, alpha=ALPHA, efdm=True, efdm_slices=K)
        torch.cuda.synchronize()
        return FRAMES * steps / (time.perf_counter() - t0)

    fps = {}
    for shared in (True, False):
        tag = "shared" if shared else "per_frame"
        for K in SLICES:                                              # warm-up of every shape and workspace
            run(K, shared, 1)
        runs = {K: [] for K in SLICES}
        peak = {}
        for _ in range(a.reps):
            for K in SLICES:
                torch.cuda.reset_peak_memory_stats(dev)
                runs[K].append(run(K, shared, a.steps))
                peak[K] = torch.cuda.max_memory_allocated(dev) / 2 ** 30
        fps[tag] = {str(K): dict(fps=med(runs[K]), runs=runs[K], peak_gib=peak[K]) for K in SLICES}
    res["fps"] = fps
    eng.groups = 1

    # 2. per level and step
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

    def feats_of(u8):
        x = torch.empty(u8.shape, dtype=torch.float32, device=dev)
        x.copy_(u8.float() / 255)
        return eng.encode(x, eng.model.deepest_target, taps=eng.model.style_taps)[1]

    cf, sf = feats_of(contents), feats_of(styles)
    levels = {}
    for relu in TARGETS:
        c, s = cf[relu], sf[relu]
        st = dict(eng.efdm_prepare(s), slices=1, rot=None)
        R = eng.sliced_matrices(c.C, 1)[0][0]
        rot_prep = timed(lambda: eng.efdm_prepare(s, R))
        plain = timed(lambda: eng.efdm_apply(c, st, FRAMES, 1.0))
        st["rot"] = [eng.efdm_prepare(s, R)["state"]]
        # K = 1: two steps, each a rotation, the sort and the runs (the second rotates back and blends)
        step_ms = timed(lambda: eng.efdm_sliced_apply(c, st, FRAMES, 1.0)) / 2
        rot_ms = step_ms - plain
        levels[relu] = dict(C=c.C, positions=c.H * c.W, rotated_style_prepare_ms=rot_prep, plain_apply_ms=plain,
                            sliced_step_ms=step_ms, rotation_ms=rot_ms,
                            rotation_gflop_per_s=2.0 * c.C * c.C * c.H * c.W * FRAMES / max(rot_ms, 1e-6) / 1e6)
    res["levels"] = levels
    eng.check_device()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
