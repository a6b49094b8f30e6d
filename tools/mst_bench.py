"""Cost and effect of multimodal style transfer (MST, DESIGN.md §3.3.10) on 512x512 five-level frames.

One process measures, alternating the three cases run by run, with a batch of 30 frames per step and one 512x512 style:
  a  plain WCT
  b  spatial control with fixed 3-region masks: a content mask of 3 vertical stripes and one style with a style mask of 3
     horizontal stripes shared by the 3 regions (one encode and one masked prepare per level)
  c  MST with K = 3, lambda = 0.05: the same regions apply, with labels made on the device
Each case reports the median frames/s of the runs and the launches per step.  One profiled MST step gives the CUDA-event
time per level of the style clustering (once per call), the data term (with its achieved bytes/s against the H100 SXM's
3.35 TB/s) and the smoothing.  For lambda in {0, 0.05, 0.2} one frame's content labels give the number of 4-connected
label components per level: the regions apply runs one pass per region present in a 128-position tile, so fewer, larger
components make it cheaper.  The card's name and power limit are read in the same call.

  python tools/mst_bench.py [--steps 5] [--warmup 3] [--reps 3] [--out FILE.json]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.regions_bench import card  # noqa: E402

TARGETS = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]
SIZE, BATCH, ALPHA, K, LAM = 512, 30, 0.8, 3, 0.05
HBM_BYTES_PER_S = 3.35e12


def stripes(size, axis):
    lab = (np.arange(size) * 3 // size).astype(np.uint8)
    return np.repeat(lab[None, :], size, 0) if axis == 1 else np.repeat(lab[:, None], size, 1)


def components(lab):
    """4-connected components of a label map, summed over its labels."""
    from scipy import ndimage
    return int(sum(ndimage.label(lab == v)[1] for v in np.unique(lab)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()

    import torch
    from wct_tf_b200.weights import make_synthetic_weights
    from wct_tf_b200.wct import WCT

    result = card()
    wct = WCT(relu_targets=TARGETS, weights=make_synthetic_weights(42), semantics="tf")
    eng = wct.engine
    rng = np.random.default_rng(1000)
    content = torch.from_numpy(rng.integers(0, 256, (BATCH, SIZE, SIZE, 3), dtype=np.uint8)).cuda()
    style = torch.from_numpy(rng.integers(0, 256, (1, SIZE, SIZE, 3), dtype=np.uint8)).cuda()
    cmask = torch.from_numpy(stripes(SIZE, 1)).cuda()
    smask = torch.from_numpy(stripes(SIZE, 0)).cuda()
    cases = {
        "a_plain_wct": lambda: eng.stylize(content, style, alpha=ALPHA),
        "b_masks_R3": lambda: eng.stylize(content, None, alpha=ALPHA, labels=cmask, region_styles=[style] * 3,
                                          region_masks=[smask] * 3),
        "c_mst_K3": lambda: eng.stylize(content, style, alpha=ALPHA, mst=K, mst_smooth=LAM),
    }

    def step(name):
        return eng.to_u8(cases[name]())

    fps = {k: [] for k in cases}
    launches = {}
    for k in cases:
        for _ in range(args.warmup):
            step(k)
        n0 = eng.launches
        step(k)
        launches[k] = eng.launches - n0
    torch.cuda.synchronize()
    for _ in range(args.reps):
        for k in cases:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                step(k)
            e1.record()
            torch.cuda.synchronize()
            fps[k].append(BATCH * args.steps / (e0.elapsed_time(e1) / 1e3))
    eng.check_device()
    result["frames_per_s"] = {k: dict(median=round(float(np.median(v)), 2), runs=[round(x, 2) for x in v]) for k, v in fps.items()}
    result["launches_per_step"] = launches

    # the MST kernels of one step, per level (CUDA events around each C-ABI call)
    eng.profile = {}
    step("c_mst_K3")
    torch.cuda.synchronize()
    kernels = {}
    for key, rec in sorted(eng.profile.items()):
        if "mst_" not in key:
            continue
        ms = sum(a.elapsed_time(b) for a, b in rec["events"])
        row = dict(ms=round(ms, 4), launches=rec["launches"])
        if "mst_data_term" in key:
            row["bytes_per_s"] = rec["bytes"] / (ms / 1e3)
            row["share_of_3.35TB/s"] = round(row["bytes_per_s"] / HBM_BYTES_PER_S, 3)
        kernels[key] = row
    eng.profile = None
    result["mst_kernels_per_step"] = kernels

    # label components of frame 0 per level for three smoothness weights
    comps = {}
    for lam in (0.0, 0.05, 0.2):
        cap = {}
        eng.stylize(content[:1], style, alpha=ALPHA, capture=cap, mst=K, mst_smooth=lam)
        comps[str(lam)] = {relu: components(lab.cpu().numpy()[0]) for relu, lab in zip(TARGETS, cap["mst_content_labels"])}
    result["content_label_components_frame0"] = comps
    print(json.dumps(result, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
