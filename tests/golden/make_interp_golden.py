"""Generate the style-interpolation golden vector (run in the BUILD container only).

  python tests/golden/make_interp_golden.py

* interp_wct_np_c128_a08.npz : sum_k w_k * wct_np(content, style_k) for K = 3 styles and one weight row, computed with the
  REFERENCE's own, unmodified ``ops.wct_np`` (/root/reference/ops.py:92-140, imported as in make_golden.py) in float32 and
  in float64 math, plus k_c and k_s.  Every vector asserts the spectral-gap condition of SURVEY 8c.  Features are drawn
  like make_golden.py's.  The name does not match ``wct_np_*.npz``, the single-style golden set of
  tests/test_gpu_transform.py.  Only this file is written: the other fixtures are not regenerated.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)
from make_golden import features  # noqa: E402
from oracle import ref_ops  # noqa: E402


def main():
    ref = ref_ops.load_reference_ops()
    assert ref is not None, "the reference's ops.py was not found"
    c, alpha, seed = 128, 0.8, 6
    rng = np.random.default_rng(seed)
    content = features(rng, c, (16, 18), 0)
    styles = np.stack([features(rng, c, hw, 0)[0] for hw in ((14, 20), (14, 20), (14, 20))])     # [K, Hs, Ws, C]
    weights = np.array([0.5, 0.3, 0.2])
    out32 = np.zeros(content.shape, np.float32)
    out64 = np.zeros(content.shape, np.float64)
    k_s = []
    for k in range(len(styles)):
        s = styles[k][None]
        out32 += np.float32(weights[k]) * ref.wct_np(content, s, alpha)
        out64 += weights[k] * ref.wct_np(content.astype(np.float64), s.astype(np.float64), alpha).astype(np.float64)
        _, info = ref_ops.wct_np(content.astype(np.float64), s.astype(np.float64), alpha, return_info=True)
        assert ref_ops.spectral_gap_ok(info["wc"]) and ref_ops.spectral_gap_ok(info["ws"]), k
        k_s.append(info["k_s"])
    np.savez_compressed(os.path.join(HERE, "interp_wct_np_c128_a08.npz"), content=content, styles=styles,
                        weights=weights, alpha=np.float64(alpha), out_ref_fp32=out32, out_ref_fp64=out64,
                        k_c=info["k_c"], k_s=np.array(k_s))
    print("interp k_c", info["k_c"], "k_s", k_s, "ref fp32-vs-fp64 %.2e" % np.abs(out32 - out64).max())


if __name__ == "__main__":
    main()
