"""Multimodal style transfer on the CPU: the oracle of tests/mst_ref.py (ICM monotonicity and limits, the k-means++ draws,
the Lloyd fixed point, the data term), ``pipeline_mst`` with K = 1 against the plain pipeline, and the argument checks."""
import numpy as np
import pytest

from oracle import nets
from tests import mst_ref as M
from wct_tf_b200.engine import Engine
from wct_tf_b200.weights import make_synthetic_weights


def _D(N, H, W, K, seed, inf_cols=()):
    D = np.random.default_rng(seed).random((N, H, W, K)).astype(np.float32) * 0.2
    for k in inf_cols:
        D[..., k] = np.inf
    return D


@pytest.mark.parametrize("lam", [0.0, 0.05, 0.2, 1.0])
@pytest.mark.parametrize("shape", [(2, 13, 17, 3), (1, 1, 9, 2), (1, 8, 1, 5), (3, 6, 6, 8)])
def test_icm_energy_never_increases(shape, lam):
    D = _D(*shape, seed=sum(shape), inf_cols=(1,) if shape[-1] > 2 else ())
    hist = []
    M.icm(D, lam, history=hist)
    assert len(hist) == 1 + 2 * M.SWEEPS
    E = [M.energy(D, h, lam) for h in hist]
    for a, b in zip(E, E[1:]):
        assert b <= a + 1e-9 * max(1.0, abs(a)), (E,)


def test_icm_lambda_zero_is_argmin_and_k1_is_zero():
    D = _D(2, 9, 11, 4, seed=3)
    assert np.array_equal(M.icm(D, 0.0), np.argmin(D, -1))
    assert not M.icm(_D(2, 9, 11, 1, seed=4), 0.7).any()


def test_icm_smooths_an_isolated_pixel():
    D = np.zeros((1, 5, 5, 2), np.float32)
    D[..., 1] = 0.1
    D[0, 2, 2] = (0.1, 0.0)               # one pixel prefers label 1 by 0.1
    assert M.icm(D, 0.0)[0, 2, 2] == 1
    assert M.icm(D, 0.05)[0, 2, 2] == 0   # 4 disagreeing neighbours cost 0.2 > 0.1
    assert M.icm(D, 0.02)[0, 2, 2] == 1   # 0.08 < 0.1


def _blobs(K, P, C, seed, noise=0.05):
    rng = np.random.default_rng(seed)
    dirs = rng.standard_normal((K, C))
    lab = rng.integers(0, K, P)
    return dirs[lab] + noise * rng.standard_normal((P, C)), lab


def test_kmeanspp_draws_are_valid_and_deterministic():
    f, _ = _blobs(4, 700, 16, 1)
    u = M.unit(f)
    idx = M.kmeanspp(u, 4, level=2)
    M.check_draws(u, idx, level=2)
    assert idx == M.kmeanspp(u, 4, level=2)
    assert idx != M.kmeanspp(u, 4, level=3)
    assert len(set(idx)) == 4              # well separated: each draw lands in a new blob


def test_kmeanspp_all_equal_copies_centre_0():
    f = np.zeros((300, 8))
    f[:, 3] = 2.0                          # every direction is e_3 exactly: every d is 0
    u = M.unit(f)
    idx = M.kmeanspp(u, 3, level=0)
    assert idx[1] == idx[0] and idx[2] == idx[0]
    M.check_draws(u, idx, level=0)


def test_lloyd_recovers_blobs_and_is_a_fixed_point():
    f, truth = _blobs(3, 900, 32, 5)
    lab, c, idx, it, cnt = M.style_clusters(f.reshape(30, 30, 32), 3, level=1)
    lab = lab.reshape(-1)
    # a partition equal to the truth up to the permutation of the labels
    perm = {int(t): int(l) for t, l in zip(truth, lab)}
    assert np.array_equal(np.vectorize(perm.get)(truth), lab)
    assert it < M.LLOYD_MAX and cnt.sum() == 900
    u = M.unit(f)
    again, margin = M.assign(u, c)
    assert np.array_equal(again, lab) and margin.min() > 0
    assert np.allclose(M.update(u, lab, c), c, atol=1e-12)


def test_update_keeps_an_empty_cluster():
    u = M.unit(np.random.default_rng(0).standard_normal((50, 8)))
    c = np.eye(3, 8)
    out = M.update(u, np.zeros(50, np.int64), c)
    assert np.array_equal(out[1:], c[1:]) and not np.array_equal(out[0], c[0])


def test_data_term():
    f = np.random.default_rng(2).standard_normal((2, 5, 6, 16))
    f[0, 0, 0] = 0
    c = M.unit(np.random.default_rng(3).standard_normal((3, 16)))
    D = M.data_term(f, c, [5, 1, 9])
    assert D.shape == (2, 5, 6, 3) and np.isinf(D[..., 1]).all()
    assert np.allclose(D[0, 0, 0, [0, 2]], 1.0)
    assert (D[..., [0, 2]] >= 0).all() and (D[..., [0, 2]] <= 2).all()


def test_pipeline_mst_k1_is_the_plain_pipeline():
    targets = ["relu2_1", "relu1_1"]
    w = make_synthetic_weights(7, relu_targets=targets)
    rng = np.random.default_rng(0)
    content = rng.integers(0, 256, (24, 20, 3), dtype=np.uint8)
    style = rng.integers(0, 256, (18, 22, 3), dtype=np.uint8)
    got = M.pipeline_mst(content, style, w, targets, K=1, alpha=0.7, dtype=np.float64)
    ref = nets.pipeline(content, style, w, targets, alpha=0.7, dtype=np.float64)
    assert np.abs(got - ref).max() < 1e-9


@pytest.mark.parametrize("K,lam", [(0, 0.05), (9, 0.05), (2.0, 0.05), (True, 0.05), (None, 0.05), (3, -0.1), (3, float("nan")),
                                   (3, float("inf")), (3, "x")])
def test_check_mst_rejects(K, lam):
    with pytest.raises(ValueError):
        Engine.check_mst(K, lam)


def test_check_mst_accepts():
    assert Engine.check_mst(np.int64(8), 0) == (8, 0.0)
    assert Engine.check_mst(1, 0.05) == (1, 0.05)
