"""Cost of the softmax style swap against the hard swap (512x512 content and style, patch 3, stride 1, synthetic weights).

  python tools/softmax_swap_bench.py [--runs 5] [--json OUT]

  levels    per level relu5_1 / relu4_1 / relu3_1 at Nc = 1 and 15: the apply per frame, hard and softmax (tau = 0.05), with
            the workspace the engine gives each, their chunk counts and the peak device memory of one apply
  fold      the fold's executed TFLOP/s (MACs from the shapes: the padded weight map's positions x C x P*P*B per block)
            and the correlation's, from torch.profiler kernel times of a one-chunk softmax apply at Nc = 1
  pipeline  five-level frames/s of one 15-frame step (WCT.predict_batch, one shared style) with the swap at relu3_1, hard
            and softmax
  breakdown where the device time of one softmax apply at relu3_1, Nc = 15 goes, by kernel (torch.profiler)
  entropy   the effective number of patches per anchor, exp(entropy of w), at relu3_1 for a few tau (1024 anchors of
            the first frame, from the device's own whitened features)
The variants of a case run alternately; times are medians of ``--runs`` runs after a warm-up of every variant.  The card
name and power limit are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.swap_labels_bench import alternate                     # noqa: E402
from tools.swap_levels_bench import card, chunks                  # noqa: E402
from wct_tf_b200 import engine as engine_mod                      # noqa: E402
from wct_tf_b200.model import RELU_CHANNELS                       # noqa: E402
from wct_tf_b200.wct import WCT                                   # noqa: E402
from wct_tf_b200.weights import make_synthetic_weights            # noqa: E402

ALL = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]
TAU = 0.05
BLOCK = 256                                                       # wct.cu: SOFTMAX_SWAP_BLOCK


def softmax_chunks(lib, C, nc, h, w, hs, ws_, p, s, cout_pad):
    """(workspace bytes the engine gives the softmax apply, chunk count)."""
    full = lib.wctb200_style_swap_softmax_workspace_bytes(C, nc, h, w, hs, ws_, p, s)
    least = lib.wctb200_style_swap_softmax_min_workspace_bytes(C, nc, h, w, hs, ws_, p, s)
    nbytes = min(full, max(least, engine_mod.SWAP_WORKSPACE_BYTES))
    B = min(BLOCK, cout_pad)
    if nbytes >= full:
        return nbytes, 1
    cols = B + (nbytes - least) // (2 * 2 * nc * (h + 2) * (w + 2)) // B * B
    return nbytes, -(-cout_pad // cols)


def peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def kernel_events(fn):
    """(name, device ms) of every kernel one call of ``fn`` launches, in launch order."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type.name == "CUDA"]
    ev.sort(key=lambda e: e.time_range.start)
    return [(e.name, (e.device_time if hasattr(e, "device_time") else e.cuda_time) / 1e3) for e in ev]


def conv_kernel_ms(fn):
    """Device times (ms) of the tensor-core conv kernels one call of ``fn`` launches, in launch order."""
    return [ms for name, ms in kernel_events(fn) if "conv_tc2_kernel" in name]


def breakdown(fn):
    """Device ms of one call of ``fn`` per stage: conv kernels split into the correlations and the folds by their launch
    order (whitening apply first, colouring apply last), the other kernels by name."""
    ev = kernel_events(fn)
    conv = [i for i, (name, _) in enumerate(ev) if "conv_tc2_kernel" in name]
    out = {}
    for i, (name, ms) in enumerate(ev):
        if "conv_tc2_kernel" in name:
            key = "conv: whitening / colouring apply" if i in (conv[0], conv[-1]) else "conv: correlation + fold"
        elif "k_softmax_swap_" in name:
            key = "k_softmax_swap_" + name.split("k_softmax_swap_")[1].split("<")[0].split("(")[0]
        else:
            key = "other (mean/cov, eigensolver, blend, memsets)"
        out[key] = out.get(key, 0.0) + ms
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    wct = WCT(relu_targets=ALL, weights=make_synthetic_weights(42))
    eng, lib = wct.engine, wct.engine.lib
    dev = eng.device
    style_u8 = torch.from_numpy(rng.integers(0, 256, (1, 512, 512, 3), dtype=np.uint8)).to(dev)
    clip_u8 = torch.from_numpy(rng.integers(0, 256, (15, 512, 512, 3), dtype=np.uint8)).to(dev)
    out = dict(card=card(), workload="synthetic weights, 512x512 content and style, patch 3 stride 1, tau %g" % TAU,
               levels=[], fold=[], pipeline={}, entropy={})
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
            nb_h, ch_h, npat = chunks(lib, C, nc, cf.H, cf.W, sf.H, sf.W, 3, 1)
            cout_pad = -(-npat // 64) * 64
            nb_s, ch_s = softmax_chunks(lib, C, nc, cf.H, cf.W, sf.H, sf.W, 3, 1, cout_pad)
            fns = {"hard": lambda: eng.swap_apply(cf, state, (sf.H, sf.W), 0.6),
                   "softmax": lambda: eng.swap_apply(cf, state, (sf.H, sf.W), 0.6, temperature=TAU)}
            t = alternate(fns, args.runs)
            mem = {name: peak(fn) for name, fn in fns.items()}
            r = dict(relu=relu, C=C, Nc=nc, map=[cf.H, cf.W], patches=npat, hard_chunks=ch_h, softmax_chunks=ch_s,
                     hard_workspace_bytes=nb_h, softmax_workspace_bytes=nb_s,
                     **{name + "_ms_per_frame": 1e3 * v / nc for name, v in t.items()},
                     **{name + "_peak_bytes": int(v) for name, v in mem.items()})
            out["levels"].append(r)
            print("%s C %d Nc %2d map %dx%d: %6d patches; hard %8.2f ms/frame (%d chunks, peak %.2f GB), softmax %8.2f "
                  "ms/frame (%d chunks, peak %.2f GB)" % (relu, C, nc, cf.H, cf.W, npat, r["hard_ms_per_frame"], ch_h,
                                                          mem["hard"] / 1e9, r["softmax_ms_per_frame"], ch_s,
                                                          mem["softmax"] / 1e9))
            if nc == 1:
                # one chunk: conv kernels are [whitening apply, correlation, fold x nblk, colouring apply]
                saved = engine_mod.SWAP_WORKSPACE_BYTES
                engine_mod.SWAP_WORKSPACE_BYTES = 1 << 40
                try:
                    ms = conv_kernel_ms(lambda: eng.swap_apply(cf, state, (sf.H, sf.W), 0.6, temperature=TAU))
                finally:
                    engine_mod.SWAP_WORKSPACE_BYTES = saved
                B = min(BLOCK, cout_pad)
                nblk = -(-cout_pad // B)
                assert len(ms) == 3 + nblk, (len(ms), nblk)
                corr_mac = (cf.H + 2) * (cf.W + 2) * cout_pad * 9 * C
                fold_mac = (cf.H + 4) * (cf.W + 4) * C * 9 * B * nblk
                corr_ms, fold_ms = ms[1], sum(ms[2:-1])
                f = dict(relu=relu, corr_ms=corr_ms, corr_tflops=2 * corr_mac / corr_ms / 1e9, fold_ms=fold_ms,
                         fold_tflops=2 * fold_mac / fold_ms / 1e9, blocks=nblk)
                out["fold"].append(f)
                print("  one chunk, Nc 1: correlation %.3f ms (%.0f TFLOP/s executed), fold %.3f ms over %d blocks "
                      "(%.0f TFLOP/s executed)" % (corr_ms, f["corr_tflops"], fold_ms, nblk, f["fold_tflops"]))
            if relu == "relu3_1" and nc == 15:
                b = breakdown(lambda: eng.swap_apply(cf, state, (sf.H, sf.W), 0.6, temperature=TAU))
                out["breakdown_relu3_1_nc15"] = b
                print("  softmax apply, relu3_1 Nc 15, device ms per apply by stage: " +
                      ", ".join("%s %.2f" % kv for kv in sorted(b.items(), key=lambda kv: -kv[1])))
            if relu == "relu3_1" and nc == 1:
                # effective patches per anchor from the device's whitened content and the state's filters
                aws = torch.empty(lib.wctb200_style_swap_softmax_workspace_bytes(C, 1, cf.H, cf.W, sf.H, sf.W, 3, 1),
                                  dtype=torch.uint8, device=dev)
                o = eng._act(1, cf.H, cf.W, C)
                sem = engine_mod.SEMANTICS["tf"]
                eng._call("swap", 1, lib.wctb200_style_swap_apply_softmax, cf.ptr, 1, cf.H, cf.W, C, state.data_ptr(), sf.H,
                          sf.W, 3, 1, 0.6, sem["eps_cov"], sem["thresh"], TAU, None, 0, 0, 0, None, 0, 0, o.ptr, None,
                          aws.data_ptr(), aws.numel(), None, 0, eng._stream())
                torch.cuda.synchronize()
                import ctypes
                lay = (ctypes.c_longlong * 11)()
                lib.wctb200_debug_style_swap_layout(C, 1, cf.H, cf.W, sf.H, sf.W, 3, 1, lay)
                npl = (cf.H + 2) * (cf.W + 2) * C
                pl = aws[int(lay[7]):int(lay[7]) + 4 * npl].view(torch.float16).view(2, cf.H + 2, cf.W + 2, C).float()
                wc = (pl[0] + pl[1])[1:-1, 1:-1]
                K = 9 * C
                wsp = state[int(lay[6]):int(lay[6]) + 4 * cout_pad * K].view(torch.float16).view(2, cout_pad, K).float()
                filt = (wsp[0] + wsp[1])[:npat]
                win = wc.unfold(0, 3, 1).unfold(1, 3, 1).permute(0, 1, 3, 4, 2).reshape(-1, K)
                sel = torch.from_numpy(np.random.default_rng(1).choice(win.shape[0], 1024, replace=False)).to(dev)
                x = win[sel]
                z = (x @ filt.T) / (x.norm(dim=1, keepdim=True) * float(np.sqrt(K / npat))).clamp_min(1e-30)
                for tau in (0.003, 0.01, 0.03, 0.05, 0.1, 0.3, 1.0):
                    w = torch.softmax(z.double() / tau, dim=1)
                    ent = -(w * torch.log(w.clamp_min(1e-300))).sum(dim=1)
                    out["entropy"][str(tau)] = float(torch.exp(ent).median())
                print("  effective patches per anchor (median of 1024 anchors): " +
                      ", ".join("tau %s: %.1f" % kv for kv in out["entropy"].items()))
                del aws
            del cf, fns
        del state
    torch.cuda.empty_cache()

    kw = dict(swap_targets=["relu3_1"], ss_alpha=0.6, return_device=True)
    t = alternate({"hard": lambda: wct.predict_batch(clip_u8, style_u8, **kw),
                   "softmax": lambda: wct.predict_batch(clip_u8, style_u8, ss_temperature=TAU, **kw)}, args.runs)
    for name, v in t.items():
        out["pipeline"][name] = 15 / v
        print("pipeline swap at relu3_1, %-8s %8.2f frames/s (15 frames per step)" % (name, 15 / v))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
