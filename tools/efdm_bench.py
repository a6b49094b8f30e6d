"""Cost of exact feature distribution matching (``predict_batch(efdm=True)``, ``--efdm``, DESIGN.md §3.3.12).

  1. 512x512 five-level frames/s of 30 frames per step, one style image per frame, two sub-batch groups (bench.py's
     default): WCT against EFDM in alternating runs, medians of --reps.
  2. Per level, CUDA events around ``efdm_prepare`` (30 styles) and ``efdm_apply`` (30 frames) on the encoder's features of
     the same images, medians of --reps, with the bytes the kernels must move (from shapes, below) over that time against
     the 3.35 TB/s of the H100 SXM data sheet.
  3. One 4096x4096 frame, the few-long-segments case: WCT and EFDM five-level stylisation, and the relu1_1 apply alone.
The card name and power limit are read in the same call.

Bytes per value, from the kernels' loads and stores: the content apply builds keys (4 B of SPF16 read, 4 B written), sorts
(key, index) pairs in four passes (each a 4 B histogram read and an 8 B read + 8 B write), writes the fp64 prefix (8 B),
reads keys, indices and two prefixes and scatters one fp32 (24 B), and transposes (4 B read, 4 B written): 120 B.  The
style prepare builds keys (8 B), sorts keys alone in four passes of 12 B and writes the fp32 values (8 B): 64 B.

  python tools/efdm_bench.py [--reps 3] [--steps 3] [--out FILE.json]
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
FRAMES, SIZE, ALPHA, GROUPS, BIG = 30, 512, 0.8, 2, 4096
APPLY_BYTES, PREPARE_BYTES, HBM = 120.0, 64.0, 3.35e12


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
    styles = torch.from_numpy(rng.integers(0, 256, (FRAMES, SIZE, SIZE, 3), dtype=np.uint8)).to(dev)
    res = dict(card(), frames_per_step=FRAMES, size=SIZE, groups=GROUPS, alpha=ALPHA)
    med = lambda v: float(np.median(v))  # noqa: E731

    # 1. frames/s
    def run(efdm, steps):
        eng.groups = GROUPS
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            eng.stylize(contents, styles, alpha=ALPHA, efdm=efdm)
        torch.cuda.synchronize()
        return FRAMES * steps / (time.perf_counter() - t0)

    run(False, 1), run(True, 1)                                       # warm-up of every shape and workspace
    wct_fps, efdm_fps = [], []
    for _ in range(a.reps):
        wct_fps.append(run(False, a.steps))
        efdm_fps.append(run(True, a.steps))
    res.update(wct_fps=med(wct_fps), efdm_fps=med(efdm_fps), wct_fps_runs=wct_fps, efdm_fps_runs=efdm_fps,
               efdm_over_wct=med(efdm_fps) / med(wct_fps))
    eng.groups = 1

    # 2. per level
    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        fn()                                                          # warm-up (workspace growth)
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
        state = eng.efdm_prepare(s)
        prep_ms = timed(lambda: eng.efdm_prepare(s))
        apply_ms = timed(lambda: eng.efdm_apply(c, state, FRAMES, 1.0))
        wct_ms = timed(lambda: eng.transform(c, s, 1.0, False))
        nc, ns = c.N * c.C * c.H * c.W, s.N * s.C * s.H * s.W
        levels[relu] = dict(values_per_call=nc, prepare_ms=prep_ms, apply_ms=apply_ms, wct_level_ms=wct_ms,
                            apply_ms_per_frame=apply_ms / FRAMES, prepare_ms_per_frame=prep_ms / FRAMES,
                            apply_bytes_per_s=APPLY_BYTES * nc / (apply_ms * 1e-3),
                            apply_share_of_hbm=APPLY_BYTES * nc / (apply_ms * 1e-3) / HBM,
                            prepare_bytes_per_s=PREPARE_BYTES * ns / (prep_ms * 1e-3),
                            prepare_share_of_hbm=PREPARE_BYTES * ns / (prep_ms * 1e-3) / HBM)
    res["levels"] = levels
    del cf, sf, contents, styles
    torch.cuda.empty_cache()

    # 3. one 4096^2 frame
    big = torch.from_numpy(rng.integers(0, 256, (1, BIG, BIG, 3), dtype=np.uint8)).to(dev)
    bstyle = torch.from_numpy(rng.integers(0, 256, (1, 1024, 1024, 3), dtype=np.uint8)).to(dev)

    def once(efdm):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        eng.stylize(big, bstyle, alpha=ALPHA, efdm=efdm)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    once(False), once(True)
    w_s, e_s = [], []
    for _ in range(a.reps):
        w_s.append(once(False))
        e_s.append(once(True))
    x = torch.empty(big.shape, dtype=torch.float32, device=dev)
    x.copy_(big.float() / 255)
    c1 = eng.encode(x, "relu1_1")[0]
    s1 = eng.efdm_prepare(feats_of(bstyle)["relu1_1"])
    r11 = timed(lambda: eng.efdm_apply(c1, s1, 1, 1.0))
    n1 = c1.N * c1.C * c1.H * c1.W
    res["frame_4096"] = dict(wct_s=med(w_s), efdm_s=med(e_s), wct_s_runs=w_s, efdm_s_runs=e_s, relu1_1_apply_ms=r11,
                             relu1_1_apply_bytes_per_s=APPLY_BYTES * n1 / (r11 * 1e-3),
                             relu1_1_apply_share_of_hbm=APPLY_BYTES * n1 / (r11 * 1e-3) / HBM)
    eng.check_device()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
