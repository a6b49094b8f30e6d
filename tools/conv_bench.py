"""Per-layer conv micro-benchmark: every conv shape of the 512x512 pipeline (3x3 layers and the UP2 layers that absorbed an
UpSampling2D), default dispatch vs fused MMA off.  TFLOP/s = EXECUTED algorithmic flops (2*taps*Cin*Cout per output pixel).

  python tools/conv_bench.py [BATCH] [--fixed] [--products N] [--digest]

--fixed: the per-tile cost that does not scale with K = 9*Cin (epilogue, tile hand-over, pipeline fill), from pairs of
3x3 convs with the same output shape and Cout whose Cin differs by 2x: they run the same tiles and the same epilogue, and
the second has twice the k-iterations, so  fixed = 2 t(Cin) - t(2 Cin)  and  mainloop(Cin) = t(2 Cin) - t(Cin).  Both are
turned into SM-microseconds per 128 x BN tile (time x #SMs / tiles) and into SM clocks at the clock read after timing.

--products N: split-fp16 products per MAC (wctb200_debug_set_conv_products: 3 = default, 1 = a_hi b_hi only).  N = 1 cuts
the tensor work 3x and leaves the operand traffic as it is, so the ratio of the two times tells a feed-bound mainloop from a
tensor-bound one.

--digest: seeded inputs, and a SHA-256 of each shape's default-dispatch output bytes (both planes, halo included), so that
two builds can be compared output for output."""
import hashlib, os, subprocess, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from wct_tf_b200 import _capi
from tests import gpu_util as U

FIXED = "--fixed" in sys.argv
DIGEST = "--digest" in sys.argv
PRODUCTS = int(sys.argv[sys.argv.index("--products") + 1]) if "--products" in sys.argv else 3
ARGS = [a for i, a in enumerate(sys.argv[1:]) if not a.startswith("--") and sys.argv[i] != "--products"]
B = int(ARGS[0]) if ARGS else 8
# (output H=W, Cin, Cout, up2)
SHAPES = [(512, 64, 64, 0), (256, 64, 128, 0), (256, 128, 128, 0), (256, 128, 64, 0), (128, 128, 256, 0), (128, 256, 256, 0),
          (128, 256, 128, 0), (64, 256, 512, 0), (64, 512, 512, 0), (64, 512, 256, 0), (32, 512, 512, 0),
          (64, 512, 512, 1), (128, 256, 256, 1), (256, 128, 128, 1), (512, 64, 64, 1)]
CFGS = [("default", -1), ("nofuse", 0), ("fuse", 1)]
# --fixed: (output H=W, Cin, Cout); each shape is timed at Cin and at 2*Cin
FIXED_PAIRS = [(512, 64, 64), (256, 64, 128), (256, 128, 64), (128, 256, 256)]
lib = U.lib()
assert lib.wctb200_debug_set_conv_products(PRODUCTS) == PRODUCTS, "--products takes 1, 2 or 3"


def conv_ms(hw, cin, cout, reps=20):
    """CUDA-event time of one default-dispatch 3x3 conv (+ReLU) at batch B, random ReLU'd input."""
    x = torch.randn(B, hw, hw, cin, device="cuda").relu_()
    xin = torch.empty(lib.wctb200_act_bytes(B, hw, hw, cin), dtype=torch.uint8, device="cuda")
    _capi.check(lib.wctb200_act_from_f32(x.data_ptr(), B, hw, hw, cin, xin.data_ptr(), U.stream()))
    del x
    k = (torch.randn(3, 3, cin, cout, device="cuda") * (2.0 / (9 * cin)) ** 0.5).contiguous()
    bias = torch.zeros(cout, device="cuda")
    ws = torch.empty(lib.wctb200_conv_weight_bytes(9, cin, cout), dtype=torch.uint8, device="cuda")
    _capi.check(lib.wctb200_prep_conv_weights(k.data_ptr(), 9, cin, cout, ws.data_ptr(), U.stream()))
    out = torch.empty(lib.wctb200_act_bytes(B, hw, hw, cout), dtype=torch.uint8, device="cuda")
    def run():
        _capi.check(lib.wctb200_conv3x3(xin.data_ptr(), B, hw, hw, cin, ws.data_ptr(), bias.data_ptr(), cout, 1, out.data_ptr(), U.stream()))
    for _ in range(3): run()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): run()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def sm_clock_mhz():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return float("nan")


if FIXED:
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print("%-20s %9s %9s %7s %10s %10s %9s %9s %7s   (batch %d, %d SMs, 3x3 + ReLU, default dispatch)" % (
        "HxW Cin->Cout", "t(Cin)", "t(2Cin)", "tiles", "fixed/tile", "main/tile", "fixed clk", "main clk", "fixed%",
        B, sms))
    for hw, cin, cout in FIXED_PAIRS:
        t1 = conv_ms(hw, cin, cout)
        t2 = conv_ms(hw, 2 * cin, cout)
        mhz = sm_clock_mhz()
        bn = 128 if cout % 128 == 0 else 64
        tiles = -(-(B * (hw + 2) * (hw + 2)) // 128) * (cout // bn)
        fixed_us = (2 * t1 - t2) * 1e3 * sms / tiles       # SM-microseconds per tile
        main_us = (t2 - t1) * 1e3 * sms / tiles
        print("%-20s %7.1fus %7.1fus %7d %8.3fus %8.3fus %9.0f %9.0f %6.1f%%   (SM clock %.0f MHz after timing)" % (
            "%dx%d %d->%d" % (hw, hw, cin, cout), t1 * 1e3, t2 * 1e3, tiles, fixed_us, main_us, fixed_us * mhz,
            main_us * mhz, 100.0 * (2 * t1 - t2) / t1, mhz), flush=True)
    _capi.check(lib.wctb200_check_device(U.stream()))
    sys.exit(0)

print("%-24s" % "HxW Cin->Cout" + "".join("%18s" % c[0] for c in CFGS) + "   (executed TFLOP/s, batch %d, %d products)" % (
    B, PRODUCTS))
for si, (hw, cin, cout, up2) in enumerate(SHAPES):
    if DIGEST:
        torch.manual_seed(1000 + si)
    hin = hw // 2 if up2 else hw
    x = torch.randn(B, hin, hin, cin, device="cuda").relu_()
    xin = torch.empty(lib.wctb200_act_bytes(B, hin, hin, cin), dtype=torch.uint8, device="cuda")
    _capi.check(lib.wctb200_act_from_f32(x.data_ptr(), B, hin, hin, cin, xin.data_ptr(), U.stream()))
    k = (torch.randn(3, 3, cin, cout, device="cuda") * (2.0 / (9 * cin)) ** 0.5).contiguous()
    bias = torch.zeros(cout, device="cuda")
    ws = torch.empty(lib.wctb200_conv_weight_bytes(16 if up2 else 9, cin, cout), dtype=torch.uint8, device="cuda")
    if up2:
        _capi.check(lib.wctb200_prep_conv_weights_up2(k.data_ptr(), cin, cout, ws.data_ptr(), U.stream()))
    else:
        _capi.check(lib.wctb200_prep_conv_weights(k.data_ptr(), 9, cin, cout, ws.data_ptr(), U.stream()))
    out = torch.zeros(lib.wctb200_act_bytes(B, hw, hw, cout), dtype=torch.uint8, device="cuda")
    flops = 2.0 * (4 if up2 else 9) * cin * cout * B * hw * hw
    row = "%-24s" % ("%dx%d %d->%d%s" % (hw, hw, cin, cout, " up2" if up2 else ""))
    for name, fuse in CFGS:
        lib.wctb200_debug_set_conv_fuse(fuse)
        fn = lib.wctb200_conv3x3_up2 if up2 else lib.wctb200_conv3x3
        def run():
            _capi.check(fn(xin.data_ptr(), B, hin, hin, cin, ws.data_ptr(), bias.data_ptr(), cout, 1, out.data_ptr(), U.stream()))
        for _ in range(3): run()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10): run()
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        row += "%10.0f (%5.0fus)" % (flops / ms / 1e9, ms * 1e3)
        if DIGEST and fuse == -1:
            digest = hashlib.sha256(out.cpu().numpy().tobytes()).hexdigest()[:16]
    if DIGEST:
        row += "   sha256 %s" % digest
    print(row, flush=True)
lib.wctb200_debug_set_conv_fuse(-1)
lib.wctb200_debug_set_conv_products(3)
_capi.check(lib.wctb200_check_device(U.stream()))
