"""GPU experiment (TEST INFRASTRUCTURE, run by hand under gpurun): which part of the encoder's excess over fp32 noise
is the SPF16 storage and which is the tensor-core path?  Runs the shared encoder to relu5_1 / relu4_1 three ways and
compares each with the fp64 oracle on the same image:
  tc     the product path (wgmma split-fp16 x3, chunked register accumulation)
  ref    wctb200_conv3x3_ref: plain fp32 FFMA on CUDA cores, same SPF16 storage between layers
  cpu32  the oracle in fp32 (torch-CPU), the reference's arithmetic
Usage: python tests/noise_split_gpu.py [size]"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import nets  # noqa: E402
from wct_tf_b200 import _capi  # noqa: E402
from wct_tf_b200.engine import Engine  # noqa: E402
from wct_tf_b200.model import encoder_plan  # noqa: E402
from wct_tf_b200.weights import make_synthetic_weights  # noqa: E402


def encode_ref(eng, img, target, vgg):
    """Engine.encode with every 3x3 conv replaced by the fp32 CUDA-core validation kernel."""
    lib, st = eng.lib, eng._stream()
    N, H, W, _ = img.shape
    x = eng._act(N, H, W, 64)
    _capi.check(lib.wctb200_conv_head(img.data_ptr(), N, H, W, eng.head_w.data_ptr(), eng.head_b.data_ptr(), x.ptr, st))
    keep = []
    for op in encoder_plan(target)[1:]:
        if op.kind == "conv":
            y = eng._act(N, x.H, x.W, op.cout)
            k = torch.from_numpy(np.ascontiguousarray(np.transpose(vgg[op.name]["weight"], (2, 3, 1, 0)))).cuda()
            b = torch.from_numpy(np.asarray(vgg[op.name]["bias"])).cuda()
            keep += [k, b]
            _capi.check(lib.wctb200_conv3x3_ref(x.ptr, N, x.H, x.W, op.cin, k.data_ptr(), b.data_ptr(), op.cout, _capi.RELU, y.ptr, st))
            x = y
        else:
            y = eng._act(N, (x.H + 1) // 2, (x.W + 1) // 2, x.C)
            _capi.check(lib.wctb200_maxpool2(x.ptr, N, x.H, x.W, x.C, y.ptr, st))
            x = y
    torch.cuda.synchronize()
    return x


def main():
    size = int(sys.argv[1]) if len(sys.argv) > 1 else 128
    w = make_synthetic_weights(42)
    vgg = {l["name"]: l for l in w["vgg"]}
    print("encoder output max-abs error vs the fp64 oracle, %dx%d random images" % (size, size))
    print("%-5s %-8s %-10s %-10s %-10s" % ("seed", "target", "tc", "ref", "cpu32"))
    rows = []
    for seed in range(3):
        rng = np.random.default_rng(100 + seed)
        img8 = rng.integers(0, 256, (1, size, size, 3), dtype=np.uint8)
        x64 = nets.preprocess(img8).astype(np.float64)
        for target in ("relu4_1", "relu5_1"):
            eng = Engine(w, [target])
            img = torch.from_numpy(x64.astype(np.float32)).cuda()
            t64 = nets.encode(x64, w, [target], np.float64)[target]
            c32 = nets.encode(x64.astype(np.float32), w, [target], np.float32)[target]
            a, _ = eng.encode(img, target)
            tc = eng.act_to_f32(a).cpu().numpy()
            rf = eng.act_to_f32(encode_ref(eng, img, target, vgg)).cpu().numpy()
            eng.check_device()
            e = [float(np.abs(v - t64).max()) for v in (tc, rf, c32)]
            rows.append(e)
            print("%-5d %-8s %-10.2e %-10.2e %-10.2e" % (seed, target, *e))
    rows = np.array(rows)
    print("%-14s %-10.2e %-10.2e %-10.2e" % ("gmean", *[np.exp(np.log(rows[:, i]).mean()) for i in range(3)]))


if __name__ == "__main__":
    main()
