"""Style masks on the CPU: the oracle's algebra (tests/style_masks_ref.py) and host-side validation."""
import numpy as np
import pytest
import torch

from oracle import ref_ops
from tests.regions_ref import wct_regions
from tests.style_masks_ref import restrict_style, wct_style_masks
from wct_tf_b200.prepared import PreparedStyle
from wct_tf_b200.wct import WCT


def _feats(h, w, c, seed):
    rng = np.random.default_rng(seed)
    return np.maximum(rng.standard_normal((1, h, w, c)) @ rng.standard_normal((c, c)) / np.sqrt(c) + 0.2, 0)


def _content_labels():
    lab = np.zeros((9, 10), np.uint8)
    lab[:, 5:] = 1
    lab[8, :] = 4                                                   # labels >= R: unstyled strip
    return lab


@pytest.mark.parametrize("sem", ["tf", "np"])
def test_no_style_masks_and_uniform_masks_are_the_regions_oracle(sem):
    cf = _feats(9, 10, 16, 1)
    styles = [_feats(8, 8, 16, 2), _feats(7, 9, 16, 3)]
    lab = _content_labels()
    ref, rinf = wct_regions(cf, styles, lab, 0.8, sem, return_info=True)
    got, ginf = wct_style_masks(cf, styles, lab, [None, None], 0.8, sem, return_info=True)
    assert np.array_equal(got, ref)
    uniform = [np.full((8, 8), 0, np.uint8), np.full((7, 9), 1, np.uint8)]
    got_u, uinf = wct_style_masks(cf, styles, lab, uniform, 0.8, sem, return_info=True)
    # the same pixels, read as a 1 x 1 x m map: equal up to the order of the sums
    assert np.allclose(got_u, ref, rtol=0, atol=1e-5)
    assert [(i["k_c"], i["k_s"]) for i in uinf] == [(i["k_c"], i["k_s"]) for i in rinf] == [(i["k_c"], i["k_s"]) for i in ginf]


def test_masked_region_is_the_transform_against_the_cropped_style():
    """Mean and covariance do not depend on where the pixels sit: a rectangle of the style mask is the style cropped."""
    cf = _feats(9, 10, 16, 4)
    painting = _feats(12, 14, 16, 5)
    smask = np.zeros((12, 14), np.uint8)
    smask[:5] = 1                                                   # sky on top, sea below
    smask[5:, 10:] = 7                                              # labels >= R: in no style region
    lab = _content_labels()
    got, info = wct_style_masks(cf, [painting, painting], lab, [smask, smask], 0.9, "tf", return_info=True)
    ref = wct_regions(cf, [painting[:, 5:, :10], painting[:, :5]], lab, 0.9, "tf")
    assert np.allclose(got, ref, rtol=0, atol=1e-5)
    assert info[0]["k_s"] > 0 and info[1]["k_s"] > 0
    sub = cf[0][lab == 1][None, None]
    assert np.allclose(got[0][lab == 1], ref_ops.wct_tf(sub, painting[:, :5], 0.9)[0, 0], rtol=0, atol=1e-5)


def test_empty_style_region_keeps_the_content():
    cf = _feats(9, 10, 16, 6)
    styles = [_feats(8, 8, 16, 7), _feats(8, 8, 16, 8)]
    smask = np.zeros((8, 8), np.uint8)
    smask[3, 3] = 1                                                 # style region 1: one pixel -> empty
    lab = _content_labels()
    got, info = wct_style_masks(cf, styles, lab, [None, smask], 0.9, "np", return_info=True)
    assert np.array_equal(got[0][lab == 1], cf[0][lab == 1])
    assert np.array_equal(got[0][lab == 4], cf[0][lab == 4])
    assert not np.allclose(got[0][lab == 0], cf[0][lab == 0])
    assert (info[1]["k_c"], info[1]["k_s"]) == (-1, -1) and info[0]["k_c"] > 0
    assert restrict_style(styles[1], smask, 1) is None and restrict_style(styles[1], None, 1) is styles[1]


def test_check_style_masks_validation():
    s = np.zeros((5, 5, 3), np.uint8)
    m = np.zeros((4, 6), np.uint8)
    out = WCT.check_style_masks([m, None, m], [s, s, s])
    assert out[1] is None and out[0] is out[2] and out[0].dtype == torch.uint8 and tuple(out[0].shape) == (4, 6)
    with pytest.raises(ValueError):
        WCT.check_style_masks([m], [s, s])                                  # one entry per style
    with pytest.raises(ValueError):
        WCT.check_style_masks(m, [s])                                       # a list
    with pytest.raises(ValueError):
        WCT.check_style_masks([m.astype(np.int32)], [s])                    # uint8
    with pytest.raises(ValueError):
        WCT.check_style_masks([np.zeros((1, 4, 6), np.uint8)], [s])         # 2-D
    ps = PreparedStyle(1, {}, [])
    with pytest.raises(ValueError):
        WCT.check_style_masks([m], [ps])                                    # a prepared style has no features to mask
    assert WCT.check_style_masks([None], [ps]) == [None]
