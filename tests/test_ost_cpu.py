"""The fp64 oracle of the optimal-transport transform (tests/ost_ref.py) against the properties that define it: M is
symmetric PSD, pushes the content covariance onto the style's, moves the features no more than WCT, is the identity for
equal covariances, the per-channel ratio of deviations for diagonal ones, and annihilates the discarded directions."""
import numpy as np
import pytest

from tests import ost_ref as O

SIZES = [8, 16, 32, 64]


def _spd(c, rng, lo=0.2, hi=5.0, rank=None):
    q, _ = np.linalg.qr(rng.standard_normal((c, c)))
    lam = rng.uniform(lo, hi, c)
    if rank is not None:
        lam[rank:] = 0.0
    return (q * lam) @ q.T


@pytest.mark.parametrize("c", SIZES)
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_symmetric_psd(c, seed):
    rng = np.random.default_rng(seed)
    for rc, rs in ((None, None), (c // 2, None), (None, c // 3)):
        M = O.ost_map(_spd(c, rng, rank=rc), _spd(c, rng, rank=rs), eps_eig=1e-5)
        assert np.abs(M - M.T).max() <= 1e-10 * np.abs(M).max()
        assert np.linalg.eigvalsh((M + M.T) / 2).min() >= -1e-10 * np.abs(M).max()


@pytest.mark.parametrize("c", SIZES)
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_pushes_content_onto_style_at_lower_cost_than_wct(c, seed):
    rng = np.random.default_rng(10 + seed)
    A, S = _spd(c, rng), _spd(c, rng)
    M, info = O.ost_map(A, S, eps_eig=0.0, return_info=True)
    assert info["k_c"] == c and info["k_s"] == c
    Cs2 = info["Cs"] @ info["Cs"]
    assert np.linalg.norm(M @ A @ M - Cs2) <= 1e-10 * np.linalg.norm(Cs2)
    I, T = np.eye(c), info["T"]
    cost_ost = np.trace((M - I) @ A @ (M - I))
    cost_wct = np.trace((T - I) @ A @ (T - I).T)
    assert cost_ost <= cost_wct * (1 + 1e-12)


@pytest.mark.parametrize("c", SIZES)
def test_equal_covariances_give_identity(c):
    A = _spd(c, np.random.default_rng(20))
    assert np.abs(O.ost_map(A, A) - np.eye(c)).max() <= 1e-10


@pytest.mark.parametrize("c", SIZES)
def test_diagonal_pairs(c):
    rng = np.random.default_rng(30)
    sc, ss = rng.uniform(0.1, 4, c), rng.uniform(0.1, 4, c)
    M = O.ost_map(np.diag(sc), np.diag(ss))
    assert np.abs(M - np.diag(np.sqrt(ss / sc))).max() <= 1e-10


@pytest.mark.parametrize("c", SIZES)
def test_rank_deficient_content_annihilates_discarded_directions(c):
    rng = np.random.default_rng(40)
    A = _spd(c, rng, rank=c // 2)
    M, info = O.ost_map(A, _spd(c, rng), eps_eig=1e-5, return_info=True)
    assert info["k_c"] == c // 2
    lam, E = np.linalg.eigh(A)
    null = E[:, lam <= 1e-5]
    assert null.shape[1] == c - c // 2
    assert np.abs(M @ null).max() <= 1e-10 * np.abs(M).max()


def test_generic_on_features_matches_map():
    """ost_generic: the covariance of the features (with eps_cov) through ost_map, then the alpha blend of wct_generic."""
    rng = np.random.default_rng(50)
    c = 16
    x = rng.standard_normal((1, 12, 10, c)) @ rng.standard_normal((c, c)) + 1.0
    y = rng.standard_normal((1, 9, 11, c)) @ rng.standard_normal((c, c)) - 0.5
    for sem in ("tf", "np"):
        out, info = O.ost(x, y, 0.6, sem, return_info=True)
        fx, fy = x.reshape(-1, c), y.reshape(-1, c)
        eps = O.SEMANTICS[sem]["eps_cov"]
        M = O.ost_map(np.cov(fx, rowvar=False) + eps * np.eye(c), np.cov(fy, rowvar=False) + eps * np.eye(c),
                      O.SEMANTICS[sem]["eps_eig"])
        mc = fx.mean(0)
        base = fx if sem == "tf" else fx - mc
        ref = 0.6 * ((fx - mc) @ M.T + fy.mean(0)) + 0.4 * base
        assert np.abs(out.reshape(-1, c) - ref).max() <= 1e-10
