"""CPU: the float64 reference, metric and bound of tests/whitening_ref.py -- that they are exact where they must be, that
they catch each way stage B can be subtly wrong, and what a float32 one-sided Jacobi with and without the null floor
delivers on a graded kept tail."""
import math

import numpy as np
import pytest

from tests import whitening_ref as R

SPECTRA = {
    **{"graded_%g" % c: (lambda C, c=c: R.graded(C, c, seed=C + int(np.log10(c)))) for c in (1e2, 1e3, 5e3, 3e4, 1e5)},
    **{"tail_%g" % l: (lambda C, l=l: R.tail(C, l, seed=C + int(l))) for l in (1.0, 30.0, 300.0)},
    "cut": lambda C: R.cut(C, seed=C + 4),
    "cut_rank": lambda C: R.cut(C, seed=C + 5, rank=C // 2 + 3),
    "clustered": lambda C: R.clustered(C, seed=C + 6),
    **{"near_guard_%g" % f: (lambda C, f=f: R.near_guard(C, f, seed=C + 7)) for f in (0.9, 1.0, 1.02, 1.1, 2.0)},
}


def _s32(spec, C, sem="tf"):
    Q, lam = SPECTRA[spec](C)
    n, s, S = R.record_of(Q, lam)
    return R.sigma32(n, s, S, R.SEMANTICS[sem]["eps_cov"])


def test_sigma32_matches_an_independent_fp64_to_fp32_computation():
    """Random records (n, s, S), entry by entry in Python floats (IEEE double) and one fp32 rounding, eps_cov in fp32."""
    rng = np.random.default_rng(0)
    for C, eps_cov in ((16, 1e-8), (24, 0.0)):
        n = float(rng.integers(2, 5000))
        s = rng.standard_normal(C) * 30.0
        S = rng.standard_normal((C, C)) * 100.0
        S = S @ S.T + np.outer(s, s) / n
        got = R.sigma32(n, s, np.triu(S), eps_cov)
        for i in range(C):
            for j in range(C):
                a, b = min(i, j), max(i, j)
                v = np.float32((float(S[a, b]) - float(s[i]) * float(s[j]) / n) / (n - 1.0))
                if i == j:
                    v = np.float32(v + np.float32(eps_cov))
                assert got[i, j].view(np.uint32) == v.view(np.uint32), (C, i, j)


@pytest.mark.parametrize("C", [64, 256])
@pytest.mark.parametrize("sem", ["tf", "np"])
@pytest.mark.parametrize("spec", sorted(SPECTRA))
def test_metric_is_zero_for_the_exact_solution(spec, sem, C):
    """float64 W and C_s of the fp32 covariance: every entry of Ew and Ec within 1e-3 of the bound (only float64 rounding)."""
    eps_eig = R.SEMANTICS[sem]["eps_eig"]
    S32 = _s32(spec, C, sem)
    basis = R.eig(S32)
    W, Cs = R.exact_w(S32, eps_eig), R.exact_cs(S32, eps_eig)
    bw, mw = R.whitening_bound(basis[0], R.THRESH, "jacobi", np.abs(W).max())
    rw, _ = R.worst_ratio(R.whitening_error(W, S32, eps_eig, basis=basis), bw, mw)
    Ec, drop = R.colouring_error(Cs, S32, eps_eig, basis=basis)
    bc, mc, bd = R.colouring_bound(basis[0], R.THRESH, "jacobi", np.abs(Cs).max())
    rc, _ = R.worst_ratio(Ec, bc, mc)
    rd = float((drop / bd).max()) if drop.size else 0.0
    print("%s %s: exact W %.2e, exact C_s %.2e / %.2e of the bound" % (spec, sem, rw, rc, rd))
    assert max(rw, rc, rd) < 1e-3


def _cols(S32):
    """Exact Jacobi columns g_i = lam_i e_i of S32 (float64) and the basis."""
    lam, E = R.eig(S32)
    return E * lam, (lam, E)


def _variant_ratio(name, C=64):
    """Worst error / bound of one defect variant over the spectra it applies to."""
    worst = 0.0
    for spec in ("graded_100", "graded_30000", "tail_30", "clustered", "cut"):
        S32 = _s32(spec, C)
        G, basis = _cols(S32)
        lam, E = basis
        solver = "jacobi"
        if name == "unrotated_tail_pair":
            keep = np.flatnonzero(lam > R.THRESH)
            p, q = keep[0], keep[1]                    # the two smallest kept eigenvalues: one pair not diagonalised
            c, s = math.cos(0.3), math.sin(0.3)
            G = G.copy()
            G[:, p], G[:, q] = c * G[:, p] - s * G[:, q], s * G[:, p] + c * G[:, q]
            W, _ = R.from_columns(G, S32, "white")
        elif name == "d_over_norm":
            W, _ = R.from_columns(G, S32, "white", power=1)
        elif name == "transposed_Q":
            keep = lam > R.THRESH
            W = (E.T * np.where(keep, 1.0 / np.sqrt(np.abs(lam)), 0.0)) @ E
        elif name == "kept_dropped":
            keep = lam > R.THRESH
            keep[np.flatnonzero(keep)[0]] = False
            W = (E * np.where(keep, 1.0 / np.sqrt(np.abs(lam)), 0.0)) @ E.T
        elif name == "newton_schulz_two_early":
            if spec not in ("graded_100", "graded_1000"):
                continue
            W, _, _ = R.newton_schulz(S32, skip=2)
            solver = "newton_schulz"
        b, m = R.whitening_bound(lam, R.THRESH, solver, np.abs(R.exact_w(S32)).max())
        r, _ = R.worst_ratio(R.whitening_error(W, S32, basis=basis), b, m)
        worst = max(worst, r)
    return worst


@pytest.mark.parametrize("name", ["unrotated_tail_pair", "d_over_norm", "newton_schulz_two_early", "transposed_Q",
                                  "kept_dropped"])
def test_defect_variants_exceed_the_bound(name):
    r = _variant_ratio(name)
    print("defect variant %s: worst error / bound = %.3g" % (name, r))
    assert r >= 10.0


def test_newton_schulz_emulation_converges_within_the_bound():
    """The float64 iteration on spectra the guard accepts (converged within the 16-iteration budget) is inside the bound,
    with and without its trailing iteration.  Skipping that iteration (the iterate at the passing residual test) leaves an
    error of the order of the stopping residual, which is the convergence level the bound grants Newton-Schulz, so that
    defect is not detectable by this metric; stopping two iterations early is (test_defect_variants_exceed_the_bound)."""
    for spec in ("graded_100", "graded_1000", "graded_5000"):
        S32 = _s32(spec, 128)
        basis = R.eig(S32)
        for skip in (0, 1):
            W, _, it = R.newton_schulz(S32, skip=skip)
            assert it <= 16, (spec, it)
            b, m = R.whitening_bound(basis[0], R.THRESH, "newton_schulz", np.abs(W).max())
            r, _ = R.worst_ratio(R.whitening_error(W, S32, basis=basis), b, m)
            print("Newton-Schulz %s, %d updates%s: worst error / bound = %.3g" % (
                spec, it, " (trailing iteration skipped)" if skip else "", r))
            assert r <= 1.0


@pytest.mark.parametrize("C,lmax", [(64, 1.0), (64, 30.0), (64, 300.0), (128, 30.0), (128, 300.0)])
def test_float32_jacobi_null_floor_on_tail_spectra(C, lmax):
    """A graded kept tail under the null floor 3.16e-6 lambda_max (null2 = 1e-11 amax, the rule before thresh entered it):
    the float32 restatement with that floor freezes the tail pairs after sweep 0 and whitens them wrong by more than the
    bound wherever the tail reaches below it (lambda_max > 3.2).  With k_jacobi's rule (kernel_null2: below
    max(thresh / 2, 16 eps lambda_max), capped at the old floor) and with the floor off it is inside the bound.  k is
    right every way."""
    Q, lam = R.tail(C, lmax, seed=C + int(lmax))
    S32 = R.sigma32(*R.record_of(Q, lam), R.SEMANTICS["tf"]["eps_cov"])
    basis = R.eig(S32)
    k_ref = int((basis[0] > R.THRESH).sum())
    res = {}
    for floor in (1e-11, None, 0.0):
        G, sweeps = R.jacobi_f32(S32, null_floor=floor)
        W, k = R.from_columns(G, S32, "white")
        b, m = R.whitening_bound(basis[0], R.THRESH, "jacobi", np.abs(W).max())
        r, excl = R.worst_ratio(R.whitening_error(W, S32, basis=basis), b, m)
        res[floor] = r
        print("C=%d lambda_max=%g floor %s: sweeps %d, k %d (ref %d), worst error / bound %.3g (%d entries not determined "
              "by fp32)" % (C, lmax, "kernel" if floor is None else floor, sweeps, k, k_ref, r, excl))
        assert k == k_ref
    if lmax > 3.2:
        assert res[1e-11] > 1.0, "the 1e-11 floor does not show the tail defect here: %s" % res
    assert res[None] <= 1.0 and res[0.0] <= 1.0, res


def test_float32_jacobi_rank_deficient_noise_stays_below_the_kernel_floor():
    """The null columns of an exactly rank-deficient fp32 matrix (lambda_max 1 .. 1000) stay below k_jacobi's floor, so
    the sweeps do not grow against the 1e-11 rule."""
    for C, r, lmax in ((64, 40, 100.0), (128, 80, 300.0), (128, 80, 1.0)):
        Q = R.haar(C, C + r)
        lam = np.concatenate([np.geomspace(lmax, lmax * 1e-2, r), np.zeros(C - r)])
        S32 = R.sigma_of(Q, lam).astype(np.float32)
        _, s_old = R.jacobi_f32(S32, null_floor=1e-11)
        G, s_new = R.jacobi_f32(S32)
        noise = np.sort(np.linalg.norm(G.astype(np.float64), axis=0))[C - r - 1] / lmax
        print("rank %d of %d, lambda_max %g: sweeps %d (1e-11 rule %d), largest null column %.2g lambda_max" % (
            r, C, lmax, s_new, s_old, noise))
        assert noise < 16 * R.EPS and s_new <= s_old + 1
