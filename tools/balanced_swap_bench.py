"""Cost and effect of the balanced style swap (512x512 content and style, patch 3, stride 1, tau 0.05, synthetic weights).

  python tools/balanced_swap_bench.py [--runs 5] [--json OUT]

  levels    per level relu5_1 / relu4_1 / relu3_1 at Nc = 1 and 15: the apply per frame for T = 0 (the softmax swap),
            1, 4 and 16 Sinkhorn iterations, with the workspace the engine gives it, its launch count and chunk count,
            alternated; the added ms per iteration
  breakdown where the device time of one T = 4 apply at relu3_1, Nc = 15 goes, by kernel (torch.profiler)
  balance   at relu3_1 and relu4_1, Nc = 1, tau 0.05 and 0.003: max |S_n - c_n| / max c_n of the final plan's column
            sums against T
  patch use at the same levels and tau: exp(entropy) of the normalised column sums, and the fraction of the patches that
            carry half the mass, for the hard swap (from its indices), the softmax swap and the balanced swap
The variants of a case run alternately; times are medians of ``--runs`` runs after a warm-up of every variant.  The card
name and power limit are read in the same run.  With synthetic weights the patch-use numbers say nothing about trained
models."""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.swap_labels_bench import alternate                     # noqa: E402
from tools.softmax_swap_bench import kernel_events               # noqa: E402
from tools.swap_levels_bench import card                          # noqa: E402
from wct_tf_b200 import engine as engine_mod                      # noqa: E402
from wct_tf_b200.model import RELU_CHANNELS                       # noqa: E402
from wct_tf_b200.wct import WCT                                   # noqa: E402
from wct_tf_b200.weights import make_synthetic_weights            # noqa: E402

ALL = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]
TAU = 0.05
ITERS = (0, 1, 4, 16)


def use_stats(mass):
    """(exp(entropy) of the normalised mass, fraction of the entries that carry half of it)."""
    p = np.sort(np.asarray(mass, np.float64))[::-1]
    p = p / p.sum()
    nz = p[p > 0]
    k = int(np.searchsorted(np.cumsum(p), 0.5) + 1)
    return float(np.exp(-(nz * np.log(nz)).sum())), k / p.size


def breakdown(fn):
    """Device ms of one call of ``fn`` by kernel (the tensor-core convs together), largest first."""
    out = {}
    for name, ms in kernel_events(fn):
        key = "conv_tc (correlations, fold, whitening / colouring)" if "conv_tc2_kernel" in name else \
            name.split("(")[0].split("<")[0].replace("void ", "").replace("wctb::", "")
        out[key] = out.get(key, 0.0) + ms
    return dict(sorted(out.items(), key=lambda kv: -kv[1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    wct = WCT(relu_targets=ALL, weights=make_synthetic_weights(42))
    eng, lib = wct.engine, wct.engine.lib
    dev = eng.device
    sem = engine_mod.SEMANTICS["tf"]
    style_u8 = torch.from_numpy(rng.integers(0, 256, (1, 512, 512, 3), dtype=np.uint8)).to(dev)
    clip_u8 = torch.from_numpy(rng.integers(0, 256, (15, 512, 512, 3), dtype=np.uint8)).to(dev)
    out = dict(card=card(), workload="synthetic weights, 512x512 content and style, patch 3 stride 1, tau %g" % TAU,
               levels=[], balance={}, patch_use={})
    print(out["card"])

    def f32(u8):
        x = torch.empty(u8.shape, dtype=torch.float32, device=dev)
        eng._call("u8_to_f32", 1, lib.wctb200_image_u8_to_f32, u8.data_ptr(), u8.numel(), x.data_ptr(), eng._stream())
        return x

    _, sfeats = eng.encode(f32(style_u8), "relu5_1", taps=ALL)
    for relu in ("relu5_1", "relu4_1", "relu3_1"):
        sf = sfeats[relu]
        C = RELU_CHANNELS[relu]
        state = eng.swap_prepare(sf, 3, 1)
        for nc in (1, 15):
            cf, _ = eng.encode(f32(clip_u8[:nc]), relu)
            geom = (C, nc, cf.H, cf.W, sf.H, sf.W, 3, 1)
            full = lib.wctb200_style_swap_balanced_workspace_bytes(*geom)
            nbytes = min(full, max(lib.wctb200_style_swap_balanced_min_workspace_bytes(*geom), engine_mod.SWAP_WORKSPACE_BYTES))
            lay = (ctypes.c_longlong * 11)()
            lib.wctb200_debug_style_swap_layout(*geom, lay)
            fns = {T: (lambda T=T: eng.swap_apply(cf, state, (sf.H, sf.W), 0.6, temperature=TAU, balance=T)) for T in ITERS}
            t = alternate(fns, args.runs)
            one = lib.wctb200_style_swap_balanced_launches(*geom, full, 0, 1, 0) - lib.wctb200_style_swap_balanced_launches(
                *geom, full, 0, 0, 0)
            r = dict(relu=relu, C=C, Nc=nc, map=[cf.H, cf.W], patches=int(lay[0]), workspace_bytes=int(nbytes),
                     one_chunk=bool(nbytes >= full),
                     launches={str(T): lib.wctb200_style_swap_balanced_launches(*geom, nbytes, 0, T, 0) for T in ITERS},
                     launches_per_iteration_one_chunk=one,
                     ms_per_frame={str(T): 1e3 * v / nc for T, v in t.items()},
                     ms_per_frame_per_iteration=1e3 * (t[16] - t[0]) / 16 / nc)
            out["levels"].append(r)
            print("%s C %d Nc %2d map %dx%d: %6d patches, %s; ms/frame " % (relu, C, nc, cf.H, cf.W, r["patches"],
                                                                          "one chunk" if r["one_chunk"] else "chunked")
                  + ", ".join("T %s %.2f" % kv for kv in r["ms_per_frame"].items())
                  + "; +%.3f ms/frame per iteration" % r["ms_per_frame_per_iteration"])
            if relu == "relu3_1" and nc == 15:
                b = breakdown(lambda: eng.swap_apply(cf, state, (sf.H, sf.W), 0.6, temperature=TAU, balance=4))
                out["breakdown_relu3_1_nc15_T4"] = b
                print("  T = 4 apply, relu3_1 Nc 15, device ms by kernel: " + ", ".join("%s %.2f" % kv for kv in b.items()))
            if nc == 1 and relu in ("relu4_1", "relu3_1"):
                npat, na = int(lay[0]), int(lay[2]) * int(lay[3])
                ws = torch.empty(full, dtype=torch.uint8, device=dev)
                o = eng._act(1, cf.H, cf.W, C)
                col = torch.empty(npat, dtype=torch.float32, device=dev)
                bal, use = {}, {}
                for tau in (TAU, 0.003):
                    for T in (0, 1, 4, 16, 64, 256):
                        eng._call("swap", 1, lib.wctb200_style_swap_apply_balanced, cf.ptr, 1, cf.H, cf.W, C,
                                  state.data_ptr(), sf.H, sf.W, 3, 1, 0.6, sem["eps_cov"], sem["thresh"], tau, T, None, 0, 0,
                                  0, None, 0, 0, o.ptr, None, col.data_ptr(), ws.data_ptr(), ws.numel(), None, 0, eng._stream())
                        S = col.cpu().numpy().astype(np.float64)
                        c = na / npat
                        bal["tau %g T %d" % (tau, T)] = float(np.abs(S - c).max() / c)
                        use["tau %g %s" % (tau, "softmax" if T == 0 else "balanced T=%d" % T)] = use_stats(S)
                hws = torch.empty(lib.wctb200_style_swap_apply_workspace_bytes(*geom), dtype=torch.uint8, device=dev)
                eng._call("swap", 1, lib.wctb200_style_swap_apply, cf.ptr, 1, cf.H, cf.W, C, state.data_ptr(), sf.H, sf.W, 3, 1,
                          0.6, sem["eps_cov"], sem["thresh"], o.ptr, None, hws.data_ptr(), hws.numel(), eng._stream())
                idx = hws[int(lay[9]):int(lay[9]) + 4 * na].view(torch.int32).cpu().numpy()
                use["hard"] = use_stats(np.bincount(idx, minlength=npat))
                torch.cuda.synchronize()
                out["balance"][relu] = bal
                out["patch_use"][relu] = {k: dict(effective_patches=v[0], half_mass_fraction=v[1], patches=npat)
                                          for k, v in use.items()}
                print("  column error max|S - c| / max c: " + ", ".join("%s %.2e" % kv for kv in bal.items()))
                print("  patch use (exp entropy of %d, fraction carrying half the mass): " % npat
                      + ", ".join("%s %.0f / %.3f" % (k, v[0], v[1]) for k, v in use.items()))
                del ws, hws
            del cf, fns
        del state
    torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
