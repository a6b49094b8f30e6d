"""Cost of texture synthesis: 512x512 five-level frames/s with the content taken from resident images, from noise made on
the device, or from noise made on the host; and the noise kernel alone.

One process measures, alternating the three cases run by run (30 frames per step, one shared 512x512 style, WCT tf,
``return_device=True`` so that no case copies its results back):
  images       WCT.predict_batch over 30 image frames already on the device
  synthesize   WCT.synthesize(count=30): wctb200_noise_u8, then the same predict_batch
  host_noise   numpy.random.default_rng(...).integers(0, 256, ...) on the host, then predict_batch (which copies it over)
Each case reports the median frames/s of its runs.  The host generator is also timed alone.

The noise kernel alone: CUDA events around 1000 launches after warm-up, once as back-to-back launches from Python (host launch
cost included) and once replayed from a CUDA graph (device time), at 30x512x512x3 and 30x1024x1024x3 bytes; GB/s is set against
the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s).  The card name, power limit and SM clock are read in the same call.

  python tools/texture_bench.py [--steps 5] [--warmup 3] [--reps 3] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from regions_bench import card  # noqa: E402

TARGETS = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]
SIZE, BATCH, ALPHA = 512, 30, 0.8
HBM_DATASHEET_GBS = 3350.0
LAUNCHES = 1000


def sm_clock():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE,
                           stderr=subprocess.STDOUT, timeout=30).stdout.decode().strip().splitlines()[0]
        return [s.strip() for s in q.split(",")]
    except Exception as e:      # the measurement is still reported, with the clock unknown
        return ["unknown (%s)" % e, "unknown"]


def kernel_time(lib, _capi, torch, n, h, w):
    """Microseconds per wctb200_noise_u8 launch: back-to-back launches, and the same launches replayed from a CUDA graph."""
    out = torch.empty((n, h, w, 3), dtype=torch.uint8, device="cuda")

    def launch(stream):
        _capi.check(lib.wctb200_noise_u8(out.data_ptr(), n, h, w, 3, 1, 0, stream))

    st = torch.cuda.current_stream().cuda_stream
    for _ in range(50):
        launch(st)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(LAUNCHES):
        launch(st)
    e1.record()
    torch.cuda.synchronize()
    stream_us = e0.elapsed_time(e1) * 1e3 / LAUNCHES

    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(100):
            launch(torch.cuda.current_stream().cuda_stream)
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(LAUNCHES // 100):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    graph_us = e0.elapsed_time(e1) * 1e3 / LAUNCHES
    nbytes = n * h * w * 3
    _capi.check(lib.wctb200_check_device(st))
    return dict(bytes=nbytes, stream_us=round(stream_us, 2), graph_us=round(graph_us, 2),
                graph_GBs=round(nbytes / graph_us / 1e3, 1), graph_share_of_datasheet=round(nbytes / graph_us / 1e3 / HBM_DATASHEET_GBS, 3),
                stream_GBs=round(nbytes / stream_us / 1e3, 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()

    import torch
    from wct_tf_b200 import _capi
    from wct_tf_b200.weights import make_synthetic_weights
    from wct_tf_b200.wct import WCT

    result = card()
    wct = WCT(relu_targets=TARGETS, weights=make_synthetic_weights(42), semantics="tf")
    rng = np.random.default_rng(1000)
    images = torch.from_numpy(rng.integers(0, 256, (BATCH, SIZE, SIZE, 3), dtype=np.uint8)).cuda()
    style = torch.from_numpy(rng.integers(0, 256, (1, SIZE, SIZE, 3), dtype=np.uint8)).cuda()
    host_rng = np.random.default_rng(7)
    counter = [0]

    def step(mode):
        counter[0] += 1
        if mode == "images":
            return wct.predict_batch(images, style, alpha=ALPHA, return_device=True)
        if mode == "synthesize":
            return wct.synthesize(style, SIZE, count=BATCH, seed=counter[0], alpha=ALPHA, return_device=True)
        noise = host_rng.integers(0, 256, (BATCH, SIZE, SIZE, 3), dtype=np.uint8)
        return wct.predict_batch(noise, style, alpha=ALPHA, return_device=True)

    modes = ["images", "synthesize", "host_noise"]
    fps, clocks = {m: [] for m in modes}, []
    for m in modes:
        for _ in range(args.warmup):
            step(m)
    torch.cuda.synchronize()
    for _ in range(args.reps):
        for m in modes:
            t0 = time.perf_counter()
            for _ in range(args.steps):
                step(m)                 # return_device=True ends in a synchronising device check
            fps[m].append(BATCH * args.steps / (time.perf_counter() - t0))
            clocks.append(sm_clock())
    result["sm_clock_after_each_run"] = clocks
    result["frames_per_s"] = {m: dict(median=round(float(np.median(v)), 2), runs=[round(x, 2) for x in v]) for m, v in fps.items()}
    result["ratio_vs_images"] = {m: round(result["frames_per_s"][m]["median"] / result["frames_per_s"]["images"]["median"], 4)
                                 for m in modes}

    t = []
    for _ in range(5):
        t0 = time.perf_counter()
        host_rng.integers(0, 256, (BATCH, SIZE, SIZE, 3), dtype=np.uint8)
        t.append(time.perf_counter() - t0)
    result["host_rng_ms_per_step"] = dict(median=round(float(np.median(t)) * 1e3, 2), runs=[round(x * 1e3, 2) for x in t])

    lib = _capi.load()
    result["noise_kernel"] = {"30x512x512x3": kernel_time(lib, _capi, torch, BATCH, 512, 512),
                              "30x1024x1024x3": kernel_time(lib, _capi, torch, BATCH, 1024, 1024)}
    result["sm_clock_end"] = sm_clock()
    print(json.dumps(result, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
