"""The EFDM oracle (tests/efdm_ref.py) has the properties its definition promises (DESIGN.md §3.3.12).  No GPU needed."""
import numpy as np
import pytest

from tests import efdm_ref as E


def _rng(seed):
    return np.random.default_rng(seed)


def test_equal_sizes_distinct_content_takes_the_style_multiset():
    rng = _rng(0)
    x, s = rng.standard_normal((2, 9, 11, 5)), rng.standard_normal((1, 9, 11, 5)) * 3 + 1
    out = E.efdm(x, s, 1.0)
    for n in range(2):
        for c in range(5):
            assert np.allclose(np.sort(out[n, ..., c].ravel()), np.sort(s[0, ..., c].ravel()), rtol=0, atol=1e-12)


@pytest.mark.parametrize("shape", [(1, 7, 13, 3), (2, 4, 4, 2)])
@pytest.mark.parametrize("ms", [(5, 5), (20, 31), (1, 3)])
def test_output_is_monotone_in_x(shape, ms):
    rng = _rng(1)
    x = np.round(np.maximum(rng.standard_normal(shape), 0) * 16) / 16          # ties and a zero run
    s = rng.standard_normal((1, ms[0], ms[1], shape[3]))
    out = E.efdm(x, s, 1.0)
    for n in range(shape[0]):
        for c in range(shape[3]):
            xo, yo = x[n, ..., c].ravel(), out[n, ..., c].ravel()
            order = np.argsort(xo, kind="stable")
            assert np.all(np.diff(yo[order]) >= -1e-12)


def test_tie_runs_take_their_mean_rank_value():
    rng = _rng(2)
    x = np.round(rng.uniform(0, 1, (1, 6, 10, 1)) * 4) / 4                      # five values, long runs
    s = rng.standard_normal((1, 6, 10, 1))
    out = E.efdm(x, s, 1.0)[0, ..., 0].ravel()
    xv = x[0, ..., 0].ravel()
    Q = np.sort(s.ravel())
    r0 = 0
    for v in np.unique(xv):
        members = xv == v
        assert np.unique(out[members]).size == 1
        k = int(members.sum())
        assert np.isclose(out[members][0], Q[r0:r0 + k].mean(), rtol=0, atol=1e-12)
        r0 += k


def test_alpha_zero_is_the_identity():
    rng = _rng(3)
    x, s = rng.standard_normal((2, 5, 6, 4)), rng.standard_normal((2, 7, 3, 4))
    assert np.array_equal(E.efdm(x, s, 0.0), x)


def test_alpha_blends_linearly():
    rng = _rng(4)
    x, s = rng.standard_normal((1, 5, 6, 2)), rng.standard_normal((1, 5, 6, 2))
    assert np.allclose(E.efdm(x, s, 0.3), 0.3 * E.efdm(x, s, 1.0) + 0.7 * x, rtol=0, atol=1e-12)


def test_single_content_value_and_single_style_value():
    rng = _rng(5)
    s = rng.standard_normal((1, 4, 5, 3))
    one = E.efdm(np.full((1, 1, 1, 3), 0.25), s, 1.0)           # Nc = 1: the median rank, the mean of Q at u = (Ms-1)/2
    Q = np.sort(s.reshape(-1, 3), axis=0)
    assert np.allclose(one[0, 0, 0], 0.5 * (Q[9] + Q[10]), rtol=0, atol=1e-12)
    x = rng.standard_normal((2, 3, 4, 3))
    out = E.efdm(x, np.full((1, 1, 1, 3), -1.5), 1.0)           # Ms = 1: every value takes the style's one value
    assert np.array_equal(out, np.full_like(x, -1.5))


@pytest.mark.parametrize("zeros", [0.0, 0.6])
def test_style_mean_is_kept_when_sizes_are_equal(zeros):
    rng = _rng(6)
    x = np.round(rng.standard_normal((1, 12, 10, 3)) * 8) / 8
    x[rng.random(x.shape) < zeros] = 0.0
    s = rng.standard_normal((1, 10, 12, 3))
    out = E.efdm(x, s, 1.0)
    assert np.allclose(out.reshape(-1, 3).mean(0), s.reshape(-1, 3).mean(0), rtol=0, atol=1e-12)


def test_output_does_not_depend_on_spatial_order():
    rng = _rng(7)
    x = np.round(np.maximum(rng.standard_normal((1, 8, 9, 2)), 0) * 8) / 8
    s = rng.standard_normal((1, 5, 7, 2))
    perm = rng.permutation(72)
    xp = x.reshape(1, 72, 2)[:, perm].reshape(1, 8, 9, 2)
    want = E.efdm(x, s, 1.0).reshape(1, 72, 2)[:, perm]
    assert np.array_equal(E.efdm(xp, s, 1.0).reshape(1, 72, 2), want)


def test_rank_quantiles_interpolate_the_style():
    Q = np.array([0.0, 1.0, 2.0, 3.0])
    assert np.array_equal(E.rank_quantiles(Q, 4), Q)
    assert np.allclose(E.rank_quantiles(Q, 2), [0.5, 2.5])                     # u = 0.5, 2.5
    assert np.allclose(E.rank_quantiles(Q, 8), [0.0, 0.25, 0.75, 1.25, 1.75, 2.25, 2.75, 3.0])   # u = r/2 - 1/4, clamped


def test_w1_of_efdm_is_below_that_of_the_content():
    rng = _rng(8)
    x = np.maximum(rng.standard_normal((1, 16, 16, 4)), 0)
    s = rng.exponential(2.0, (1, 12, 20, 4))
    assert np.all(E.w1(E.efdm(x, s, 1.0), s) < E.w1(x, s))
    assert np.all(E.floor_w1(x, s) >= 0)
