"""Cost of the style swap at each relu level (512x512 content and style, patch 3, stride 1, synthetic weights).

  python tools/swap_levels_bench.py [--runs 3] [--json OUT]

  levels   per level relu5_1 / relu4_1 / relu3_1 at Nc = 1 and 15, and relu2_1 at Nc = 1: the swap prepare (the style side:
           whitening, tap norms, patch filters) and the apply per frame, with the workspace the engine gives it
           (engine.SWAP_WORKSPACE_BYTES), its chunk count, and the peak device memory of the apply
  pipeline five-level frames/s of one 30-frame step (WCT.predict_batch, one shared style): no swap, swap5, and the swap at
           relu3_1
Every case is warmed up; times are medians of ``--runs`` runs, each ended by a device synchronise.  The card name and power
limit are read in the same run."""
from __future__ import annotations

import argparse
import ctypes
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from wct_tf_b200 import engine as engine_mod          # noqa: E402
from wct_tf_b200.model import RELU_CHANNELS          # noqa: E402
from wct_tf_b200.wct import WCT                       # noqa: E402
from wct_tf_b200.weights import make_synthetic_weights  # noqa: E402

ALL = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, runs):
    ts = []
    for _ in range(runs):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def chunks(lib, C, nc, h, w, hs, ws_, p, s):
    """(workspace bytes the engine gives the apply, chunk count), from the library's sizes and layout."""
    full = lib.wctb200_style_swap_apply_workspace_bytes(C, nc, h, w, hs, ws_, p, s)
    least = lib.wctb200_style_swap_apply_min_workspace_bytes(C, nc, h, w, hs, ws_, p, s)
    nbytes = min(full, max(least, engine_mod.SWAP_WORKSPACE_BYTES))
    lay = (ctypes.c_longlong * 11)()
    lib.wctb200_debug_style_swap_layout(C, nc, h, w, hs, ws_, p, s, lay)
    cout_pad, scores = int(lay[1]), int(lay[8])
    bn = 128 if cout_pad % 128 == 0 else 64
    col = 2 * 2 * nc * (h + 2) * (w + 2)
    cols = cout_pad if nbytes >= full else (nbytes - scores) // col // bn * bn
    return nbytes, math.ceil(cout_pad / cols), int(lay[0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    wct = WCT(relu_targets=ALL, weights=make_synthetic_weights(42))
    eng, lib = wct.engine, wct.engine.lib
    dev = eng.device
    style_u8 = torch.from_numpy(rng.integers(0, 256, (1, 512, 512, 3), dtype=np.uint8)).to(dev)
    clip_u8 = torch.from_numpy(rng.integers(0, 256, (30, 512, 512, 3), dtype=np.uint8)).to(dev)
    out = dict(card=card(), workload="synthetic weights, 512x512 content and style, patch 3 stride 1", levels=[], pipeline={})
    print(out["card"])

    def f32(u8):
        x = torch.empty(u8.shape, dtype=torch.float32, device=dev)
        eng._call("u8_to_f32", 1, lib.wctb200_image_u8_to_f32, u8.data_ptr(), u8.numel(), x.data_ptr(), eng._stream())
        return x

    _, sfeats = eng.encode(f32(style_u8), "relu5_1", taps=ALL)
    for relu, ncs in (("relu5_1", (1, 15)), ("relu4_1", (1, 15)), ("relu3_1", (1, 15)), ("relu2_1", (1,))):
        sf = sfeats[relu]
        C = RELU_CHANNELS[relu]
        state = eng.swap_prepare(sf, 3, 1)
        t_prep = timed(lambda: eng.swap_prepare(sf, 3, 1), args.runs)
        for nc in ncs:
            cf, _ = eng.encode(f32(clip_u8[:nc]), relu)
            nbytes, nchunks, npat = chunks(lib, C, nc, cf.H, cf.W, sf.H, sf.W, 3, 1)
            eng.swap_apply(cf, state, (sf.H, sf.W), 0.6)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            base = torch.cuda.memory_allocated(dev)
            t_apply = timed(lambda: eng.swap_apply(cf, state, (sf.H, sf.W), 0.6), args.runs)
            peak = torch.cuda.max_memory_allocated(dev)
            r = dict(relu=relu, C=C, Nc=nc, map=[cf.H, cf.W], patches=npat, prepare_ms=1e3 * t_prep,
                     apply_ms_per_frame=1e3 * t_apply / nc, workspace_bytes=nbytes, chunks=nchunks,
                     peak_device_bytes=peak, apply_peak_above_base_bytes=peak - base)
            out["levels"].append(r)
            print("%s C %d Nc %2d map %dx%d: %6d patches, prepare %8.2f ms, apply %8.2f ms/frame, %2d chunk(s) in %.2f GB, "
                  "peak %.2f GB (%.2f GB above the resident buffers)"
                  % (relu, C, nc, cf.H, cf.W, npat, r["prepare_ms"], r["apply_ms_per_frame"], nchunks, nbytes / 1e9, peak / 1e9,
                     (peak - base) / 1e9))
            del cf
        del state
    torch.cuda.empty_cache()

    cases = {"no_swap": {}, "swap5": dict(swap5=True, ss_alpha=0.6), "swap_relu3_1": dict(swap_targets=["relu3_1"], ss_alpha=0.6)}
    for name, kw in cases.items():
        def step():
            wct.predict_batch(clip_u8, style_u8, return_device=True, **kw)
        step()
        step()
        t = timed(step, args.runs)
        out["pipeline"][name] = 30 / t
        print("pipeline %-13s %8.2f frames/s (30 frames per step)" % (name, 30 / t))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
