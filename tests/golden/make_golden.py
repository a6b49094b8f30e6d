"""Generate the committed golden vectors (run in the BUILD container only).

  python tests/golden/make_golden.py

* wct_np_*.npz : inputs + outputs of the REFERENCE's own ``ops.wct_np``
  (/root/reference/ops.py:92-140, imported with TensorFlow/Keras stubbed, see
  oracle/ref_ops.load_reference_ops) in float32, plus the float64 run of the same
  reference code, k_c/k_s and the eigenvalue spectra.  Every vector asserts the
  spectral-gap condition of SURVEY 8c (no covariance eigenvalue in [1e-6, 1e-4]).
* Feature distribution: relu(N(0,1) @ M + 0.3) with a seeded mixing matrix M
  (SURVEY 8d), small shapes so the files stay small; `dead` zeroes some channels
  exactly (dead ReLU channels -> exact zero eigenvalues).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_ops  # noqa: E402

CASES = [
    # name, C, (Hc,Wc), (Hs,Ws), alpha, dead channels, seed
    ("c64_a10", 64, (24, 20), (16, 28), 1.0, 0, 1),
    ("c64_a06", 64, (24, 20), (16, 28), 0.6, 0, 2),
    ("c128_a08_dead", 128, (20, 20), (24, 18), 0.8, 9, 3),
    ("c256_a08", 256, (14, 14), (13, 16), 0.8, 0, 4),        # sizes keep every file under 1 MB
    ("c512_a08_dead", 512, (10, 10), (9, 12), 0.8, 40, 5),
]


def features(rng, c, hw, dead):
    h, w = hw
    m = rng.standard_normal((c, c)) / np.sqrt(c)
    x = np.maximum(rng.standard_normal((h * w, c)) @ m + 0.3, 0.0)
    if dead:
        x[:, rng.choice(c, dead, replace=False)] = 0.0
    return x.reshape(1, h, w, c).astype(np.float32)


def main(only=None):
    ref = ref_ops.load_reference_ops()
    assert ref is not None, "the reference's ops.py was not found"
    for name, c, hwc, hws, alpha, dead, seed in CASES:
        if only and name not in only:
            continue
        rng = np.random.default_rng(seed)
        content = features(rng, c, hwc, dead)
        style = features(rng, c, hws, 0)
        out32 = ref.wct_np(content, style, alpha)
        out64 = ref.wct_np(content.astype(np.float64), style.astype(np.float64), alpha)  # fp64 math, fp32 store
        _, info = ref_ops.wct_np(content.astype(np.float64), style.astype(np.float64), alpha, return_info=True)
        assert ref_ops.spectral_gap_ok(info["wc"]) and ref_ops.spectral_gap_ok(info["ws"]), name
        np.savez_compressed(os.path.join(HERE, "wct_np_%s.npz" % name), content=content, style=style,
                            alpha=np.float64(alpha), out_ref_fp32=out32, out_ref_fp64=out64,
                            k_c=info["k_c"], k_s=info["k_s"], wc=info["wc"], ws=info["ws"])
        print(name, "k", info["k_c"], info["k_s"], "ref fp32-vs-fp64 %.2e" % np.abs(out32 - out64).max(),
              "range", float(out64.min()), float(out64.max()))


def coral_golden():
    """--keep-colors: the reference's own utils.preserve_colors_np -> coral.coral_numpy (pure NumPy, imported unmodified)."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("_ref_coral", "/root/reference/coral.py")
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    rng = np.random.default_rng(21)
    style = np.uint8(rng.random((20, 26, 3)) * np.array([250, 90, 160]))
    content = np.uint8(rng.random((18, 22, 3)) * np.array([60, 220, 120]) + 20)
    coraled = ref.coral_numpy(style / 255., content / 255.)
    out = np.uint8(np.clip(coraled, 0, 1) * 255.)                       # utils.py:88-90
    np.savez_compressed(os.path.join(HERE, "coral_keep_colors.npz"), style=style, content=content, coraled=coraled, out=out)
    print("coral golden", out.shape, out.mean())


def t7_golden():
    """What the reference's torchfile.py (force_8bytes_long=True, vgg_normalised.py:16) reads back from the .t7 that
    tests/t7_writer.py writes for make_synthetic_weights(5, relu_targets=["relu3_1"]): module names, shapes, sums and the
    first 64 values of every convolution's weight and bias."""
    import importlib.util
    import tempfile
    from tests.t7_writer import write_vgg_t7
    from wct_tf_b200 import weights as W
    ref_dir = os.environ.get("WCT_TF_REFERENCE", "reference")          # a checkout of eridgd/WCT-TF
    spec = importlib.util.spec_from_file_location("_ref_torchfile", os.path.join(ref_dir, "torchfile.py"))
    tf = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tf)
    w = W.make_synthetic_weights(5, relu_targets=["relu3_1"])
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "vgg_normalised.t7")
        write_vgg_t7(path, w["vgg"])
        net = tf.load(path, force_8bytes_long=True)
    convs = [m for m in net.modules if m._typename == b"nn.SpatialConvolution"]
    out = {"names": np.array([m.name.decode() if m.name is not None else "" for m in convs])}
    for i, m in enumerate(convs):
        wt, b = np.asarray(m.weight), np.asarray(m.bias)
        out["w%d_shape" % i], out["w%d_sum" % i], out["w%d_head" % i] = np.array(wt.shape), np.float64(wt.astype(np.float64).sum()), wt.reshape(-1)[:64]
        out["b%d_sum" % i], out["b%d_head" % i] = np.float64(b.astype(np.float64).sum()), b.reshape(-1)[:64]
    np.savez_compressed(os.path.join(HERE, "t7_reference_parse.npz"), **out)
    print("t7 golden", len(convs), "convolutions")


if __name__ == "__main__":
    # python tests/golden/make_golden.py [case names...]: regenerate only those wct_np cases
    main(sys.argv[1:])
    if len(sys.argv) == 1:
        coral_golden()
        t7_golden()
