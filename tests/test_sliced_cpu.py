"""Sliced distribution matching (DESIGN.md §3.3.14) on the CPU: the bases of ``wct_tf_b200.sliced``, the float64 oracle
``tests/sliced_ref.py`` and its properties, the distribution distance it is for, and the value check of ``efdm_slices``."""
import zlib

import numpy as np
import pytest

from oracle import ref_ops
from tests import efdm_ref as E
from tests import sliced_ref as SR
from wct_tf_b200 import options, sliced


def _mixture(rng, n, m, c, scale=1.0):
    """ReLU'd mixture of two correlated Gaussians [n, m, c]: exact zeros, correlated channels, far from Gaussian."""
    A = rng.standard_normal((c, c)) / np.sqrt(c)
    z = rng.standard_normal((n, m, c)) @ A.T
    z[:, : m // 2] += 1.5 * rng.standard_normal(c)
    return scale * np.maximum(z, 0)


@pytest.mark.parametrize("c", [8, 64, 512])
def test_rotations_orthonormal_distinct_deterministic(c):
    Rs = sliced.rotations(c, 3)
    for R in Rs:
        assert R.dtype == np.float32 and R.shape == (c, c)
        err = np.abs(R.astype(np.float64) @ R.T.astype(np.float64) - np.eye(c)).max()
        assert err <= 8 * np.sqrt(c) * 2.0 ** -24, err
    assert not np.allclose(Rs[0], Rs[1]) and not np.allclose(Rs[1], Rs[2])
    assert sliced.rotations(c, 2)[1].tobytes() == Rs[1].tobytes()       # a chain of K is a prefix of one of K + 1
    sliced._rotation.cache_clear()
    assert sliced.rotations(c, 3)[2].tobytes() == Rs[2].tobytes()


def test_rotation_bytes_pinned():
    assert zlib.crc32(sliced.rotations(64, 1)[0].tobytes()) == 0x673D303E
    assert zlib.crc32(sliced.rotations(512, 2)[1].tobytes()) == 0xB4DB92C8


def test_step_matrices():
    c, K = 64, 3
    Rs, Gs = sliced.rotations(c, K), sliced.step_matrices(c, K)
    assert len(Gs) == K + 1
    assert Gs[0].tobytes() == Rs[0].tobytes()
    for k in range(1, K):
        want = (Rs[k].astype(np.float64) @ Rs[k - 1].astype(np.float64).T).astype(np.float32)
        assert np.abs(Gs[k] - want).max() <= 2.0 ** -23
    assert np.array_equal(Gs[K], Rs[K - 1].T)
    with pytest.raises(ValueError):
        sliced.step_matrices(c, 0)


def test_k0_is_efdm():
    rng = np.random.default_rng(1)
    x = _mixture(rng, 2, 120, 16).reshape(2, 10, 12, 16)
    y = _mixture(rng, 1, 90, 16).reshape(1, 9, 10, 16)
    for alpha in (1.0, 0.6):
        assert np.array_equal(SR.sliced_efdm(x, y, 0, alpha), E.efdm(x, y, alpha))


def test_steps_match_projected_marginals_and_final_is_efdm():
    """Each step's output has, in its own basis, the style's projected marginals; the final output's sorted values per
    channel are EFDM's, and with Nc = Ms and distinct values the style's own multiset."""
    rng = np.random.default_rng(2)
    c, m, K = 16, 200, 3
    x = _mixture(rng, 1, m, c)[0]
    y = _mixture(rng, 1, m, c, 1.5)[0] + 1e-3 * rng.standard_normal((m, c))     # distinct values
    trace = []
    out = SR.sliced_frame(x, y, K, 1.0, trace)
    Ss = SR.style_states(y, K)
    Gs = sliced.step_matrices(c, K)
    for k, (v, mk) in enumerate(trace):
        yk = v @ Gs[k].astype(np.float64).T
        want = np.stack([E.efdm_channel(yk[:, j], Ss[k][:, j]) for j in range(c)], 1)
        np.testing.assert_allclose(np.sort(mk, 0), np.sort(want, 0), rtol=0, atol=1e-12)
        np.testing.assert_allclose(np.sort(mk, 0), np.sort(Ss[k], 0), rtol=0, atol=1e-12)
    np.testing.assert_allclose(np.sort(out, 0), np.sort(y, 0), rtol=0, atol=1e-12)


def test_permutation_blend_and_frames():
    rng = np.random.default_rng(3)
    c, m, K = 8, 150, 2
    x = _mixture(rng, 2, m, c)
    y = _mixture(rng, 2, 130, c, 1.3)
    out = SR.sliced_frame(x[0], y[0], K)
    perm = rng.permutation(m)
    np.testing.assert_allclose(SR.sliced_frame(x[0][perm], y[0], K), out[perm], rtol=0, atol=1e-12)
    a = 0.35
    np.testing.assert_allclose(SR.sliced_frame(x[0], y[0], K, a), a * out + (1 - a) * x[0], rtol=0, atol=1e-12)
    assert np.array_equal(SR.sliced_frame(x[0], y[0], K, 0.0), x[0])
    both = SR.sliced_efdm(x.reshape(2, 10, 15, c), y.reshape(2, 10, 13, c), K)
    for n in range(2):
        np.testing.assert_array_equal(both[n].reshape(-1, c), SR.sliced_frame(x[n], y[n], K))


def test_sliced_w1_falls_with_k_and_beats_efdm_and_wct():
    """Held-out sliced-W1 to the style (256 directions drawn apart from the transform's bases), C = 32, 2048 content and
    2560 style points of ReLU'd correlated mixtures.  Measured with this oracle: content 0.7567, K = 0 (EFDM) 0.2311,
    K = 4 0.1325, K = 16 0.0683, WCT (``wct_np`` at alpha = 1) 0.0812."""
    rng = np.random.default_rng(20261018)
    c = 32
    x = _mixture(rng, 1, 2048, c)[0]
    y = _mixture(np.random.default_rng(7), 1, 2560, c, 1.7)[0]
    dirs = SR.held_out_directions(c, 256)
    d = {K: SR.sliced_w1(SR.sliced_frame(x, y, K), y, dirs) for K in (0, 4, 16)}
    wct = np.asarray(ref_ops.wct_np(x.reshape(1, -1, c), y.reshape(1, -1, c), alpha=1.0)).reshape(-1, c)
    d_wct = SR.sliced_w1(wct, y, dirs)
    print("held-out sliced-W1: content %.4f  K=0 %.4f  K=4 %.4f  K=16 %.4f  wct %.4f"
          % (SR.sliced_w1(x, y, dirs), d[0], d[4], d[16], d_wct))
    assert d[16] < d[4] < d[0]
    assert d[16] < d_wct and d[16] < d[0]


@pytest.mark.parametrize("bad", [-1, 33, 2.5, True, "3", None])
def test_check_efdm_slices(bad):
    with pytest.raises(ValueError, match="efdm_slices"):
        options.check_efdm_slices(bad, True)


def test_check_efdm_slices_values():
    assert options.check_efdm_slices(0, False) == 0
    assert options.check_efdm_slices(np.int64(32), True) == 32
    with pytest.raises(ValueError, match="efdm_slices needs efdm"):
        options.check_efdm_slices(4, False)
    with pytest.raises(ValueError, match="--efdm-slices needs --efdm"):
        options.check_efdm_slices(4, False, options.CLI)
