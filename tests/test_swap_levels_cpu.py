"""The oracle of the style swap at any level (tests/swap_levels_ref.py) on the CPU."""
import glob
import os

import numpy as np
import pytest

from oracle import nets
from tests.swap_levels_ref import pipeline_levels
from tests.test_oracle import load_pipeline_fixture, swap_kwargs

SWAP5 = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "pipeline_swap5_*.npz")))


@pytest.mark.parametrize("path", SWAP5, ids=[os.path.basename(p)[9:-4] for p in SWAP5])
def test_swap_targets_relu5_1_is_swap5(path):
    """swap_targets=["relu5_1"] gives the arrays of swap5=True on the inputs of the swap5 fixtures."""
    g, targets, w = load_pipeline_fixture(path)
    kw = swap_kwargs(g)
    assert kw.pop("swap5")
    a, ia = nets.pipeline(g["content"], g["style"], w, targets, alpha=float(g["alpha"]), dtype=np.float64, return_info=True,
                          swap5=True, **kw)
    b, ib = pipeline_levels(g["content"], g["style"], w, targets, alpha=float(g["alpha"]), dtype=np.float64, return_info=True,
                            swap_targets=["relu5_1"], **kw)
    assert np.array_equal(a, b)
    assert [(i["k_c"], i["k_s"]) for i in ia] == [(i["k_c"], i["k_s"]) for i in ib]


def test_default_is_nets_pipeline_and_rejections():
    from wct_tf_b200.weights import make_synthetic_weights
    targets = ["relu2_1", "relu1_1"]
    w = make_synthetic_weights(3, relu_targets=targets)
    rng = np.random.default_rng(0)
    c, s = rng.integers(0, 256, (1, 24, 24, 3), dtype=np.uint8), rng.integers(0, 256, (1, 24, 24, 3), dtype=np.uint8)
    assert np.array_equal(pipeline_levels(c, s, w, targets, alpha=0.7), nets.pipeline(c, s, w, targets, alpha=0.7))
    swapped = pipeline_levels(c, s, w, targets, alpha=0.7, dtype=np.float64, swap_targets=["relu2_1"])
    assert np.isfinite(swapped).all()
    with pytest.raises(ValueError):
        pipeline_levels(c, s, w, targets, swap5=True, swap_targets=["relu2_1"])
    with pytest.raises(ValueError):
        pipeline_levels(c, s, w, targets, swap_targets=["relu3_1"])
