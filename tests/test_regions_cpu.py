"""Spatial control on the CPU: the label-resize rule, the region oracle, and host-side validation."""
import numpy as np
import pytest

from oracle import ref_ops
from tests.regions_ref import mask_regions, resize_labels, wct_regions
from wct_tf_b200.wct import WCT


@pytest.mark.parametrize("hm,wm,hf,wf", [(7, 5, 3, 4), (100, 37, 13, 6), (5, 9, 11, 23), (64, 64, 8, 8), (3, 3, 3, 3)])
def test_label_resize_rule(hm, wm, hf, wf):
    rng = np.random.default_rng(hm * wm + hf)
    mask = rng.integers(0, 9, (2, hm, wm), dtype=np.uint8)
    got = resize_labels(mask, hf, wf)
    assert got.shape == (2, hf, wf)
    for y in range(hf):
        for x in range(wf):
            sy, sx = ((2 * y + 1) * hm) // (2 * hf), ((2 * x + 1) * wm) // (2 * wf)
            assert np.array_equal(got[:, y, x], mask[:, sy, sx])
    assert np.array_equal(resize_labels(mask, hm, wm), mask)          # same size: identity


def test_label_resize_centres_of_downsampled_blocks():
    mask = np.arange(64, dtype=np.uint8).reshape(8, 8)
    assert np.array_equal(resize_labels(mask, 4, 4), mask[1::2, 1::2])
    assert np.array_equal(resize_labels(mask, 16, 16), mask.repeat(2, 0).repeat(2, 1))


def test_mask_file_quantisation():
    v = np.arange(256, dtype=np.uint8)
    assert np.array_equal(np.unique(mask_regions(v, 2)), [0, 1])
    assert mask_regions(v, 2)[127] == 0 and mask_regions(v, 2)[128] == 1
    assert np.array_equal(np.bincount(mask_regions(v, 4)), [64] * 4)
    assert mask_regions(v, 3).max() == 2


def _feats(h, w, c, seed):
    rng = np.random.default_rng(seed)
    return np.maximum(rng.standard_normal((1, h, w, c)) @ rng.standard_normal((c, c)) / np.sqrt(c) + 0.2, 0)


@pytest.mark.parametrize("sem", ["tf", "np"])
def test_one_region_everywhere_is_the_plain_transform(sem):
    cf, sf = _feats(9, 7, 16, 1), _feats(6, 11, 16, 2)
    got, info = wct_regions(cf, [sf], np.zeros((9, 7), np.uint8), 0.7, sem, return_info=True)
    fn = ref_ops.wct_tf if sem == "tf" else ref_ops.wct_np
    ref, rinf = fn(cf, sf, 0.7, return_info=True)
    assert np.array_equal(got, ref.astype(got.dtype) if sem == "np" else ref)
    assert (info[0]["k_c"], info[0]["k_s"]) == (rinf["k_c"], rinf["k_s"])


def test_unlabelled_and_single_pixel_regions_keep_the_content():
    cf = _feats(8, 8, 16, 3)
    styles = [_feats(5, 5, 16, 4), _feats(6, 6, 16, 5), _feats(7, 7, 16, 6)]
    lab = np.zeros((8, 8), np.uint8)
    lab[:, 4:] = 1
    lab[0, 0] = 2                # region 2: a single pixel -> skipped
    lab[7, :] = 5                # labels >= R: unstyled strip
    got, info = wct_regions(cf, styles, lab, 0.9, "tf", return_info=True)
    keep = (lab >= 3) | (lab == 2)
    assert np.array_equal(got[0][keep], cf[0][keep])
    assert not np.allclose(got[0][lab == 0], cf[0][lab == 0])
    assert info[2]["k_c"] == -1 and info[0]["k_c"] > 0 and info[1]["k_c"] > 0
    # a region is transformed on its own: the other regions' pixels do not enter its statistics
    sub = cf[0][lab == 1][None, None]
    assert np.array_equal(got[0][lab == 1], ref_ops.wct_tf(sub, styles[1], 0.9)[0, 0])


def test_check_mask_validation():
    s = np.zeros((5, 5, 3), np.uint8)
    m, styles = WCT.check_mask(np.zeros((4, 6), np.uint8), 3, [s, s])
    assert m.shape == (1, 4, 6) and len(styles) == 2
    with pytest.raises(ValueError):
        WCT.check_mask(np.zeros((4, 6), np.int32), 1, [s])
    with pytest.raises(ValueError):
        WCT.check_mask(np.zeros((2, 4, 6), np.uint8), 3, [s])              # 2 masks for 3 frames
    with pytest.raises(ValueError):
        WCT.check_mask(np.zeros((4, 6), np.uint8), 1, [s] * 9)               # R > 8
    with pytest.raises(ValueError):
        WCT.check_mask(np.zeros((4, 6), np.uint8), 1, [np.zeros((5, 5, 3), np.float32)])
