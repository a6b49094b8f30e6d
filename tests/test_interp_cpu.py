"""Style interpolation on the CPU: weight validation and normalisation, the morph schedule, and the algebra behind the
engine's blend of style statistics, checked on the reference-code fixture (tests/golden/interp_wct_np_c128_a08.npz)."""
import os

import numpy as np
import pytest

from oracle import ref_ops
from stylize_video import morph_weights
from tests.interp_ref import adain_interp, wct_interp
from wct_tf_b200.wct import WCT

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "interp_wct_np_c128_a08.npz")


def test_normalize_weights_rows_sum_to_one():
    w = WCT.normalize_weights([1, 3], 5, 2)
    assert w.dtype == np.float32 and w.shape == (1, 2)
    assert np.array_equal(w, np.float32([[0.25, 0.75]]))
    rows = np.array([[2.0, 1.0, 1.0], [0.1, 0.2, 0.7], [5.0, 0.0, 5.0]])
    w = WCT.normalize_weights(rows, 3, 3)
    assert w.shape == (3, 3)
    assert np.array_equal(w, (rows / rows.sum(1, keepdims=True)).astype(np.float32))      # float64 division, then cast
    assert np.abs(w.astype(np.float64).sum(1) - 1).max() <= 1e-7


def test_normalize_weights_one_hot_rows_stay_exact():
    rows = np.array([[0, 7.5, 0], [3, 0, 0], [0, 0, 1e-30]])
    w = WCT.normalize_weights(rows, 3, 3)
    assert np.array_equal(w, np.eye(3, dtype=np.float32)[[1, 0, 2]])
    assert np.array_equal(WCT.normalize_weights([4.0], 2, 1), np.ones((1, 1), np.float32))


@pytest.mark.parametrize("bad", [[1, -0.5], [np.nan, 1], [np.inf, 1], [0, 0], [[1, 1], [0, 0], [1, 0]], [1, 1, 1],
                                 [[1, 1]] * 2, [[[1, 1]]], ["a", "b"]])
def test_normalize_weights_rejects(bad):
    with pytest.raises(ValueError):
        WCT.normalize_weights(np.array(bad) if not isinstance(bad[0], str) else bad, 3, 2)


def test_check_interp_validation():
    s = np.zeros((5, 6, 3), np.uint8)
    w, styles = WCT.check_interp([1, 1], 4, [s, np.zeros((1, 9, 7, 3), np.uint8)])
    assert w.shape == (1, 2) and len(styles) == 2
    w, styles = WCT.check_interp([2], 1, s)                                 # one image: K = 1
    assert np.array_equal(w, [[1.0]]) and len(styles) == 1
    with pytest.raises(ValueError):
        WCT.check_interp([1] * 9, 1, [s] * 9)                               # K > 8
    with pytest.raises(ValueError):
        WCT.check_interp([], 1, [])
    with pytest.raises(ValueError):
        WCT.check_interp([1, 1], 1, [s, s.astype(np.float32)])
    with pytest.raises(ValueError):
        WCT.check_interp([1, 1], 1, [s, np.zeros((2, 5, 5, 3), np.uint8)])
    with pytest.raises(ValueError):
        WCT.check_interp([1, 1, 1], 1, [s, s])                              # one weight per style


@pytest.mark.parametrize("T,K", [(1, 2), (2, 2), (7, 2), (10, 3), (31, 4), (5, 8), (3, 5)])
def test_morph_weights_schedule(T, K):
    w = morph_weights(T, K)
    assert w.shape == (T, K) and w.dtype == np.float64
    assert np.abs(w.sum(1) - 1).max() <= 1e-15 and (w >= 0).all()
    assert np.array_equal(w[0], np.eye(K)[0])
    if T > 1:
        assert np.array_equal(w[-1], np.eye(K)[K - 1])
    for t in range(T):                                                      # at most two neighbouring styles per frame
        nz = np.nonzero(w[t])[0]
        assert len(nz) <= 2 and (len(nz) < 2 or nz[1] == nz[0] + 1)
    # every style's weight rises to its peak and falls after it (piecewise monotone)
    for k in range(K):
        d = np.diff(w[:, k])
        peak = int(w[:, k].argmax())
        assert (d[:peak] >= 0).all() and (d[peak:] <= 0).all()


def test_morph_weights_rule():
    w = morph_weights(5, 3)                                                 # p = 0, 0.5, 1, 1.5, 2
    assert np.array_equal(w, [[1, 0, 0], [0.5, 0.5, 0], [0, 1, 0], [0, 0.5, 0.5], [0, 0, 1]])
    with pytest.raises(ValueError):
        morph_weights(4, 1)


def _operator_blend(content, styles, weights, alpha, eps_cov, eps_eig, readd, thresh=ref_ops.THRESH):
    """The engine's form in float64: whiten once, colour with C_w = sum w_k C_sk, shift by m_w = sum w_k m_sk."""
    fcx, shape = ref_ops._flat(content)
    mc = fcx.mean(axis=1, keepdims=True)
    fc = fcx - mc
    cov = fc @ fc.T / (fcx.shape[1] - 1) + eps_cov * np.eye(fc.shape[0])
    e, v = np.linalg.eigh(cov)
    keep = e > thresh
    Wc = (v[:, keep] * (e[keep] + eps_eig) ** -0.5) @ v[:, keep].T
    Cw, mw = 0.0, 0.0
    for s, w in zip(styles, weights):
        fsx, _ = ref_ops._flat(s)
        ms = fsx.mean(axis=1, keepdims=True)
        fs = fsx - ms
        cs = fs @ fs.T / (fsx.shape[1] - 1) + eps_cov * np.eye(fs.shape[0])
        es, vs = np.linalg.eigh(cs)
        ks = es > thresh
        Cw = Cw + w * ((vs[:, ks] * np.sqrt(es[ks] + eps_eig)) @ vs[:, ks].T)
        mw = mw + w * ms
    out = alpha * (Cw @ Wc @ fc + mw) + (1 - alpha) * (fc + mc if readd else fc)
    return ref_ops._unflat(out, shape)


def test_fixture_against_output_level_oracle():
    g = np.load(GOLDEN)
    styles = [s[None] for s in g["styles"]]
    w, alpha = g["weights"], float(g["alpha"])
    assert len(styles) == 3 and abs(w.sum() - 1) < 1e-15
    got, infos = wct_interp(g["content"].astype(np.float64), [s.astype(np.float64) for s in styles], w, alpha, "np",
                            return_info=True)
    assert np.abs(got - g["out_ref_fp64"]).max() <= 1e-10
    assert np.abs(g["out_ref_fp32"] - g["out_ref_fp64"]).max() <= 1e-4
    for k, inf in enumerate(infos):
        assert ref_ops.spectral_gap_ok(inf["wc"]) and ref_ops.spectral_gap_ok(inf["ws"])
        assert inf["k_c"] == int(g["k_c"]) and inf["k_s"] == int(g["k_s"][k])


@pytest.mark.parametrize("sem", ["tf", "np"])
def test_operator_blend_equals_output_blend(sem):
    """sum_k w_k WCT_k(x) == WCT with C_s -> sum w_k C_sk, m_s -> sum w_k m_sk (weights summing to 1), in float64."""
    g = np.load(GOLDEN)
    c = g["content"].astype(np.float64)
    styles = [s[None].astype(np.float64) for s in g["styles"]]
    w, alpha = g["weights"], float(g["alpha"])
    p = dict(tf=dict(eps_cov=1e-8, eps_eig=0.0, readd=True), np=dict(eps_cov=0.0, eps_eig=1e-5, readd=False))[sem]
    out_sum = sum(wk * ref_ops.wct_generic(c, s, alpha, eps_cov=p["eps_cov"], eps_eig=p["eps_eig"], readd_content_mean=p["readd"])
                  for s, wk in zip(styles, w))
    blend = _operator_blend(c, styles, w, alpha, p["eps_cov"], p["eps_eig"], p["readd"])
    assert np.abs(blend - out_sum).max() <= 1e-10 * max(1.0, np.abs(out_sum).max())


def test_adain_blend_of_statistics_equals_output_blend():
    rng = np.random.default_rng(3)
    c = np.maximum(rng.normal(0.5, 1, (1, 9, 11, 16)), 0)
    styles = [np.maximum(rng.normal(0.2 * k, 1 + k, (1, 5 + k, 7, 16)), 0) for k in range(3)]
    w, alpha = np.array([0.2, 0.5, 0.3]), 0.7
    sig = sum(wk * np.sqrt(s.var(axis=(1, 2), keepdims=True)) for s, wk in zip(styles, w))
    mu = sum(wk * s.mean(axis=(1, 2), keepdims=True) for s, wk in zip(styles, w))
    y = (c - c.mean(axis=(1, 2), keepdims=True)) / np.sqrt(c.var(axis=(1, 2), keepdims=True) + 1e-5) * sig + mu
    assert np.abs(alpha * y + (1 - alpha) * c - adain_interp(c, styles, w, alpha)).max() <= 1e-12
