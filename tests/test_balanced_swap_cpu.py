"""The balanced style swap (DESIGN.md §3.3.18) on the CPU: the float64 oracle's plan (rows, columns, convergence, the
assignment limit), the option check, and the API's forwarding of ``ss_balance`` through a recording stub engine."""
import itertools

import numpy as np
import pytest
import torch
from scipy.optimize import linear_sum_assignment

from tests import balanced_swap_ref as BR
from tests import softmax_swap_ref as SR
from tests import swap_labels_ref as SLR
from tests.test_softmax_swap_cpu import RecordingEngine, _allowed, _imgs, _whitened, api  # noqa: F401
from wct_tf_b200 import options
from wct_tf_b200.prepared import PreparedStyle


def _case(seed, hc, hs, p=3, s=1, c=8):
    """(scores, norms, K) of the hard swap on whitened random features."""
    wc, ws = _whitened(seed, hc, hs, c)
    _, inf = SR.style_swap_softmax(wc, ws, p, s, 1.0, return_info=True)
    return inf["scores"], inf["norms"], p * p * c


def _col_err(col, c):
    return np.abs(col - c).max() / c.max()


@pytest.mark.parametrize("tau", [0.01, 0.05, 1.0])
def test_zero_iterations_are_the_softmax_weights(tau):
    scores, norms, K = _case(3, 9, 10)
    w, col, c, h, _ = BR.balanced_weights(scores, norms, K, tau, 0)
    w0, _ = SR.softmax_weights(scores, norms, K, tau)
    assert np.array_equal(w, w0)
    assert (h == 0).all()
    assert np.allclose(col, w0.reshape(-1, w0.shape[2]).sum(axis=0))


@pytest.mark.parametrize("ps", [(3, 1), (5, 2)])
@pytest.mark.parametrize("iters", [0, 1, 4, 20])
def test_rows_sum_to_one_and_vanish_outside_the_allowed_set(ps, iters):
    p, s = ps
    hc, hs = (9, 10) if p == 3 else (11, 15)
    wc, ws = _whitened(3 * p + s, hc, hs)
    allowed = _allowed(hc, hs, p, s, 3, 2)
    assert (~allowed).any()
    for mask in (None, allowed):
        _, inf = BR.style_swap_balanced(wc, ws, p, s, 0.05, iters, mask)
        w = inf["w"]
        assert np.allclose(w.sum(axis=2), 1.0, atol=1e-12)
        assert (w >= 0).all()
        if mask is not None:
            assert (w[~mask] == 0).all()


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_columns_converge_to_the_targets(seed):
    scores, norms, K = _case(seed, 9, 10)
    errs = {}
    for T in (0, 1, 20):
        _, col, c, _, _ = BR.balanced_weights(scores, norms, K, 0.05, T)
        errs[T] = _col_err(col, c)
    assert errs[20] < errs[0] and errs[20] < errs[1], errs
    _, col, c, _, _ = BR.balanced_weights(scores, norms, K, 0.05, 500)
    assert _col_err(col, c) < 1e-6
    assert np.isclose(c.sum(), scores.shape[0] * scores.shape[1])
    assert np.allclose(c, c[0])                           # without labels c_n = Na / n_p


def test_identical_rows_are_balanced_after_one_iteration():
    rng = np.random.default_rng(7)
    n, na = 12, 20
    row = rng.standard_normal(n)
    scores = np.broadcast_to(row, (4, 5, n)).copy()
    norms = np.ones((4, 5))
    w0, col0, c, _, _ = BR.balanced_weights(scores, norms, 18, 0.1, 0)
    assert _col_err(col0, c) > 0.1
    w, col, c, _, _ = BR.balanced_weights(scores, norms, 18, 0.1, 1)
    assert np.allclose(col, c, rtol=1e-12) and np.allclose(c, na / n)
    assert np.allclose(w, 1.0 / n)


def test_labelled_targets_and_convergence():
    hc, hs, p, s = 9, 10, 3, 1
    wc, ws = _whitened(5, hc, hs)
    # vertical stripes: content labels 0..2, style labels 0..1 (label 2 absent from the style: fallback anchors)
    cl = (np.arange(hc)[None, :].repeat(hc, 0) * 3 // hc).astype(np.uint8)
    sl = (np.arange(hs)[None, :].repeat(hs, 0) * 2 // hs).astype(np.uint8)
    alab, plab = SLR.anchor_labels(cl, hc, hc, p, s), SLR.patch_labels(sl, hs, hs, p, s)
    allowed = SLR.allowed(alab, plab)
    c = BR.targets(allowed)
    assert np.isclose(c.sum(), alab.size)
    # c_n = cnt(l(n)) / np(l(n)) + F / n_p
    F = (~np.isin(alab, plab)).sum()
    assert 0 < F < alab.size
    want = np.array([(alab == l).sum() / (plab == l).sum() for l in plab]) + F / plab.size
    assert np.allclose(c, want, rtol=1e-12)
    errs = []
    for T in (0, 20, 500):
        _, inf = BR.style_swap_balanced(wc, ws, p, s, 0.05, T, allowed)
        errs.append(_col_err(inf["col_sums"], inf["c"]))
    assert errs[1] < errs[0] and errs[2] < 1e-6, errs


def test_small_temperature_approaches_the_optimal_assignment():
    """Na = n_p, a unique optimum: the plan's row arg-max is the linear_sum_assignment optimum."""
    rng = np.random.default_rng(11)
    n = 6
    scores = rng.standard_normal((2, 3, n))
    norms = np.full((2, 3), np.sqrt(18 / n))             # z = scores
    _, z = SR.softmax_weights(scores, norms, 18, 1.0)
    zf = z.reshape(n, n)
    r, col = linear_sum_assignment(-zf)
    best = zf[r, col].sum()
    # unique optimum: every other assignment is worse by a clear margin
    others = sorted(zf[np.arange(n), list(q)].sum() for q in itertools.permutations(range(n)))
    assert np.isclose(others[-1], best) and others[-1] - others[-2] > 0.05
    w, cs, c, _, _ = BR.balanced_weights(scores, norms, 18, 0.003, 3000)
    assert np.array_equal(w.reshape(n, n).argmax(axis=1), col)
    assert _col_err(cs, c) < 1e-3
    assert np.array_equal(SR.softmax_weights(scores, norms, 18, 0.003)[0].reshape(n, n).argmax(axis=1), zf.argmax(axis=1))


@pytest.mark.parametrize("T", [0, 1, 16, 256, np.int64(3), np.int32(0)])
def test_check_ss_balance_accepts(T):
    assert options.check_ss_balance(T, 0.05) == int(T)
    assert type(options.check_ss_balance(T, 0.05)) is int


def test_check_ss_balance_zero_needs_nothing():
    assert options.check_ss_balance(0, None) == 0


@pytest.mark.parametrize("T", [-1, 257, 1.0, 2.5, "3", None, True, False, float("nan")])
def test_check_ss_balance_rejects_values(T):
    with pytest.raises(ValueError, match="ss_balance must be an integer in 0..256"):
        options.check_ss_balance(T, 0.05)
    with pytest.raises(ValueError, match="--ss-balance must be an integer in 0..256"):
        options.check_ss_balance(T, 0.05, options.CLI)


def test_check_ss_balance_needs_the_temperature():
    with pytest.raises(ValueError, match="ss_balance needs ss_temperature"):
        options.check_ss_balance(4, None)
    with pytest.raises(ValueError, match="--ss-balance needs --ss-temperature"):
        options.check_ss_balance(4, None, options.CLI)
    # a parameter of the softmax swap: no entry of its own in the options table
    assert "ss_balance" not in options.SPELLINGS and "ss_balance" not in options.AROUND
    assert all("ss_balance" not in (a,) + tuple(b) for a, b, _ in options.EXCLUDES)


def test_predict_batch_forwards_the_iterations(api):  # noqa: F811
    c, s = _imgs(2, 32, 32), _imgs(1, 16, 16, 1)
    api.predict_batch(c, s, swap_targets=["relu3_1"], ss_temperature=0.05, ss_balance=4, passes=2)
    (_, kw0), (_, kw1) = api.engine.calls
    assert kw0["ss_balance"] == 4 and kw0["ss_temperature"] == 0.05
    assert kw1["ss_balance"] == 0 and kw1["ss_temperature"] is None      # the swap acts in the first pass only
    api.engine.calls.clear()
    api.predict(c[0], s[0], swap5=True, ss_temperature=2, ss_balance=np.int64(16))
    assert api.engine.calls[0][1]["ss_balance"] == 16
    api.engine.calls.clear()
    api.predict_batch(c, PreparedStyle(1, {}, ["relu5_1"]), swap5=True, ss_temperature=0.1, ss_balance=1)
    assert api.engine.calls[0][1]["ss_balance"] == 1
    api.engine.calls.clear()
    api.predict_batch(c, s, swap5=True, ss_temperature=0.1)
    assert api.engine.calls[0][1]["ss_balance"] == 0


def test_synthesize_forwards_the_iterations(api, monkeypatch):  # noqa: F811
    from wct_tf_b200 import device_image
    monkeypatch.setattr(device_image, "noise_u8", lambda n, h, w, seed=0, first_index=0, device=None: torch.zeros(
        (n, h, w, 3), dtype=torch.uint8))
    api.synthesize(_imgs(1, 16, 16), (32, 48), count=2, swap_targets=["relu3_1"], ss_temperature=0.02, ss_balance=8)
    assert api.engine.calls[0][1]["ss_balance"] == 8


@pytest.mark.parametrize("kw,match", [
    (dict(swap5=True, ss_balance=4), "ss_balance needs ss_temperature"),
    (dict(swap5=True, ss_temperature=0.05, ss_balance=-1), "integer in 0..256"),
    (dict(swap5=True, ss_temperature=0.05, ss_balance=300), "integer in 0..256"),
    (dict(swap5=True, ss_temperature=0.05, ss_balance=1.5), "integer in 0..256"),
])
def test_predict_batch_rejects_before_device_work(api, kw, match):  # noqa: F811
    with pytest.raises(ValueError, match=match):
        api.predict_batch(_imgs(2, 32, 32), _imgs(1, 16, 16), **kw)
    assert api.engine.calls == []
