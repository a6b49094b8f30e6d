"""Soft spatial control, the float64 oracle's algebra (tests/soft_masks_ref.py)."""
import numpy as np
import pytest

from tests.soft_masks_ref import apply_soft, feather, kish_record, record_stats, resize_area, weighted_stats


def test_feathered_planes_sum_to_one():
    rng = np.random.default_rng(0)
    lab = rng.integers(0, 4, (2, 23, 31)).astype(np.uint8)           # label 3 = keep (R = 3)
    f = feather(lab, 4, 2.5)
    assert np.allclose(f.sum(1), 1.0, atol=1e-12)
    assert (f >= 0).all()
    assert feather(lab, 3, 2.5).sum(1).max() <= 1.0 + 1e-12


def test_area_resample_identity_and_constant():
    rng = np.random.default_rng(1)
    m = rng.random((2, 3, 17, 29)).astype(np.float32)       # fp32 maps: the integer-weighted fp64 sums are exact
    assert np.array_equal(resize_area(m, 17, 29), m)
    for hf, wf in [(5, 7), (40, 61), (1, 1), (17, 3)]:
        assert np.allclose(resize_area(np.full((1, 17, 29), 0.37), hf, wf), 0.37, atol=1e-15)
    # downsampling by an integer factor is the block mean
    b = rng.random((8, 12))
    assert np.allclose(resize_area(b, 4, 3), b.reshape(4, 2, 3, 4).mean((1, 3)), atol=1e-15)


def test_zero_one_weights_are_region_statistics():
    rng = np.random.default_rng(2)
    x = rng.standard_normal((9, 11, 5))
    w = (rng.random((9, 11)) < 0.4).astype(np.float64)
    m, cov, n = weighted_stats(x, w)
    sel = x.reshape(-1, 5)[w.reshape(-1) > 0]
    assert n == sel.shape[0]
    assert np.allclose(m, sel.mean(0), atol=1e-12)
    assert np.allclose(cov, np.cov(sel.T), atol=1e-12)


def test_constant_weight_is_frame_statistics():
    rng = np.random.default_rng(3)
    x = rng.standard_normal((7, 13, 4))
    m, cov, n = weighted_stats(x, np.full((7, 13), 0.3))
    f = x.reshape(-1, 4)
    assert np.isclose(n, f.shape[0])
    assert np.allclose(m, f.mean(0), atol=1e-12)
    assert np.allclose(cov, np.cov(f.T), atol=1e-10)


@pytest.mark.parametrize("shift", [0.0, 3.0])
def test_kish_record_is_the_weighted_covariance(shift):
    rng = np.random.default_rng(4)
    x = rng.standard_normal((10, 12, 6)) + 5.0
    w = rng.random((10, 12)) ** 2
    m, cov, n = weighted_stats(x, w)
    t = np.full(6, shift)
    n2, s, S = kish_record(x, w, t)
    m2, cov2 = record_stats(n2, t, s, S)
    assert np.isclose(n, n2)
    assert np.allclose(m2, m, atol=1e-10)
    assert np.allclose(cov2, cov, atol=1e-10)


def test_soft_apply_limits():
    rng = np.random.default_rng(5)
    x = rng.standard_normal((6, 7, 3))
    Ms, bs = rng.standard_normal((2, 3, 3)), rng.standard_normal((2, 3))
    zero = np.zeros((2, 6, 7))
    assert np.array_equal(apply_soft(x, Ms, bs, zero), x)
    onehot = np.zeros((2, 6, 7))
    onehot[0, :, :3] = 1
    onehot[1, :, 3:] = 1
    out = apply_soft(x, Ms, bs, onehot)
    assert np.allclose(out[:, :3], x[:, :3] @ Ms[0].T + bs[0])
    assert np.allclose(out[:, 3:], x[:, 3:] @ Ms[1].T + bs[1])


@pytest.mark.parametrize("sem", ["tf", "np"])
def test_transform_from_stats_is_the_reference(sem):
    from oracle import ref_ops
    from tests.soft_masks_ref import frame_stats, transform_from_stats
    rng = np.random.default_rng(6)
    x = rng.standard_normal((1, 9, 10, 6)) * np.array([1, 2, 3, 0.5, 1, 4]) + 2.0
    st = rng.standard_normal((1, 7, 8, 6)) + 1.0
    M, b, _, _ = transform_from_stats(*frame_stats(x), *frame_stats(st), 0.7, sem)
    p = dict(tf=dict(eps_cov=1e-8, eps_eig=0.0, readd_content_mean=True), np=dict(eps_cov=0.0, eps_eig=1e-5, readd_content_mean=False))
    ref = ref_ops.wct_generic(x, st, 0.7, **p[sem])               # in float64 (wct_np casts its result to float32)
    assert np.abs((x[0] @ M.T + b) - ref[0]).max() <= 1e-10


@pytest.mark.parametrize("sem", ["tf", "np"])
def test_zero_one_weights_reproduce_wct_regions(sem):
    from tests.regions_ref import wct_regions
    from tests.soft_masks_ref import wct_soft
    rng = np.random.default_rng(7)
    x = rng.standard_normal((1, 12, 14, 5)) + 1.0
    styles = [rng.standard_normal((1, 6, 7, 5)) * (k + 1) for k in range(3)]
    lab = rng.integers(0, 4, (12, 14))
    lab[0, 0] = 2
    lab[lab == 2] = 3
    lab[0, 0] = 2                                  # region 2 holds one pixel: skipped; label 3 keeps the content
    w = np.stack([(lab == k).astype(np.float64) for k in range(3)])
    tol = 1e-10 if sem == "tf" else 1e-5                           # wct_np's result is cast to float32
    assert np.abs(wct_soft(x, styles, w, None, 0.8, sem) - wct_regions(x, styles, lab, 0.8, sem)).max() <= tol


@pytest.mark.parametrize("sem", ["tf", "np"])
def test_constant_weights_are_style_interpolation(sem):
    from tests.interp_ref import wct_interp
    from tests.soft_masks_ref import wct_soft
    rng = np.random.default_rng(8)
    x = rng.standard_normal((1, 11, 13, 5)) + 0.5
    styles = [rng.standard_normal((1, 6, 9, 5)) * (k + 1) + k for k in range(3)]
    c = np.array([0.5, 0.3, 0.2])
    w = c[:, None, None] * np.ones((3, 11, 13))
    tol = 1e-10 if sem == "tf" else 1e-5                           # wct_np's result is cast to float32
    assert np.abs(wct_soft(x, styles, w, None, 0.9, sem) - wct_interp(x, styles, c, 0.9, sem)).max() <= tol
