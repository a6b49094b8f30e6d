"""Stage B of a WCT level (DESIGN.md §3.3): the whitening matrix W_c and the colouring matrix C_s, checked in float64 in the
eigenbasis of the very fp32 covariance the solvers receive.

Spectra.  Each builder returns (Q, lam): Q a seeded Haar orthogonal matrix (QR of a Gaussian with the sign fix), lam the
designed eigenvalues, so that Sigma = Q diag(lam) Q^T.  `graded` spans the Newton-Schulz budget, `tail` puts a graded run
of kept eigenvalues under the Jacobi kernel's null floor (3.16e-6 lambda_max), `cut` decides k without ambiguity,
`clustered` repeats eigenvalues 8 and 32 times, `near_guard` probes the Newton-Schulz guard's 1.01 margin.

Metric.  (lam_i, e_i) = eigh(Sigma32) in float64, P = diag(lam_i / (lam_i + eps_eig) on kept i, 0 on dropped i):
    Ew = E^T W Sigma32 W E - P                          (whitening)
    Ec_ij = (e_i^T C_s^2 e_j - (lam_i + eps_eig) [i = j kept]) / sqrt(lam_i lam_j)   on the kept block  (colouring)
    Ec_i  = |C_s e_i| / sqrt(lam_kept,min)                                           for a dropped e_i
Both are scale-free: an error along a direction that W amplifies 316x shows at full size.  ("max error / max entry" hides
exactly these errors and is not used.)

Bound, per entry (i, j), eps = 2^-24, tau the solver's convergence level:
    |E_ij| <= conv_ij + 4 eps lam_max / sqrt(lam_i lam_j) + s_ij
  * conv_ij, the solver's convergence term.
    Jacobi stops when every pair's cosine is below tau = 2 sqrt(C) eps (launch_jacobi), and W is built from the
    NORMALISED columns u_i = g_i / |g_i| (k_eig_post).  A cosine c between u_i and u_j leaves u_i = e_i + c e_j, and then
    e_i^T W Sigma W e_j = c (1 + sqrt(lam_j / lam_i)): the whitening amplifies it by the square root of the eigenvalue
    ratio.  With both cosines of the pair: conv_ij = tau (2 + sqrt(lam_i / lam_j) + sqrt(lam_j / lam_i)).
    Newton-Schulz stops one iteration after max|I - Z Y| < 2e-5 (matfun_tc.cu), and the split-fp16 products of that
    iteration round by 2^-21 of the largest entry, sqrt(C) of them per entry: tau = 2e-5 + 2^-21 sqrt(C).  That is relative to
    the iterate's largest eigenvalue, so Y = (Sigma / s)^1/2 carries an absolute error up to tau |Y|, which along e_i is
    tau sqrt(lam_max / lam_i) relative; Z = Y^-1 (I - R) inherits it, and Z Sigma Z - I collects it from both sides:
    conv_ij = tau (2 + sqrt(lam_max / lam_i) + sqrt(lam_max / lam_j)).  (This is why an entrywise residual does not
    bound the small-eigenvalue directions by itself.)
    An entry with a dropped index carries the cosine of the kept column alone: conv = 2 tau (Jacobi).
  * 4 eps lam_max / sqrt(lam_i lam_j): a rotation against the largest column updates each entry of a small column by
    x + cm1 x - s y, two roundings (the product s y and the sum) of up to eps |g|_max = eps lam_max each; that is a
    backward error of 2 eps lam_max in each of the two columns i and j, and a symmetric backward error dA reaches the
    whitening as W dA W, i.e. dA_ij / sqrt(lam_i lam_j) in the eigenbasis.  This is the part of the error that fp32
    rotation cannot remove.  (A dropped index: lam_i -> the
    kept lam_j, both dropped: lam_kept,min.)
  * s_ij = 2^-20 sqrt(C) w_max (sqrt(lam_i) + sqrt(lam_j)): the stored operand.  W is read back as M_hi + M_lo, whose
    split leaves 2^-22 of the row's max (test_gpu_apply.py) and whose fp32 products leave a few 2^-24 more, 2^-21 in all;
    it enters Ew_ij as dW_ij (sqrt(lam_i) + sqrt(lam_j)) in the eigenbasis, and the sum of C independent roundings in
    dW_ij grows as sqrt(C): 2^-20 sqrt(C) carries a factor 2 for that model.  (For C_s: w_max -> max|C_s|, and the same
    form divided by sqrt(lam_i lam_j) instead of multiplied.)
Entries whose rounding term 4 eps lam_max / sqrt(lam_i lam_j) is >= 0.1 are not determined by fp32 data and are
excluded; every excluded entry is counted and reported.  No constant above is fitted to a measurement.

A float32 NumPy restatement of one-sided Jacobi (`jacobi_f32`) with the rotation rule of rot_scalars (jacobi_common.cuh),
including its null floor and a switch for it, serves as an oracle of what fp32 rotation delivers and as a negative
control.  It runs round-robin disjoint pairs, not the kernel's schedule.
"""
import numpy as np

EPS = 2.0 ** -24
THRESH = 1e-5
NS_TOL = 2e-5
SEMANTICS = {"tf": dict(eps_cov=1e-8, eps_eig=0.0, readd=1), "np": dict(eps_cov=0.0, eps_eig=1e-5, readd=0)}


# ------------------------------------------------------------------------------------------------------------ spectra
def haar(C, seed):
    z = np.random.default_rng(seed).standard_normal((C, C))
    q, r = np.linalg.qr(z)
    return q * np.sign(np.diag(r))


def graded(C, cond, seed=0, lmax=4.0):
    """Geometric from lmax down to lmax / cond; all kept (lmax / cond >= 4 thresh for cond <= 1e5)."""
    return haar(C, seed), np.geomspace(lmax, lmax / cond, C)


def tail(C, lmax, seed=0, nt=12):
    """A bulk over two decades below lmax and a geometric tail of nt kept eigenvalues from 4 thresh up to 10x the null
    floor 3.16e-6 lmax (1e-3 when that is lower): the tail straddles the floor.  Neighbours are at least a factor 1.34
    apart (25^(1/11) for lmax <= 31.6), far more than the eps lmax a rotation rounds them by wherever the metric looks."""
    top = max(10 * 3.16e-6 * lmax, 1e-3)
    lam = np.concatenate([np.geomspace(lmax, lmax * 1e-2, C - nt), np.geomspace(top, 4 * THRESH, nt)])
    return haar(C, seed), lam


def cut(C, seed=0, rank=None):
    """Dropped eigenvalues at 0, 1e-9 and thresh/4, kept ones from 4 thresh up to 1; none in [thresh/4, 4 thresh].
    rank: exactly rank-deficient (C - rank zero eigenvalues, the rest kept)."""
    if rank is not None:
        lam = np.concatenate([np.geomspace(1.0, 4 * THRESH, rank), np.zeros(C - rank)])
    else:
        nd = C // 8
        lam = np.concatenate([np.geomspace(1.0, 4 * THRESH, C - 3 * nd), np.zeros(nd), np.full(nd, 1e-9),
                              np.full(nd, THRESH / 4)])
    return haar(C, seed), lam


def clustered(C, seed=0):
    """Multiplicities 32 (at 0.3) and 8 (at 1e-3) inside a geometric kept range 1 .. 1e-4."""
    rest = np.geomspace(1.0, 1e-4, C - 40)
    return haar(C, seed), np.concatenate([np.full(32, 0.3), np.full(8, 1e-3), rest])


def near_guard(C, factor, seed=0):
    """lam_min = factor thresh under a well-conditioned rest 0.1 .. 0.02: the Newton-Schulz guard's margin."""
    return haar(C, seed), np.concatenate([np.geomspace(0.1, 0.02, C - 1), [factor * THRESH]])


def sigma_of(Q, lam):
    return (Q * lam) @ Q.T


# ------------------------------------------------------------------------------------------------- the fp32 covariance
def sigma32(n, s, S, eps_cov):
    """The fp32 covariance the library forms from a record (n, s [C], S [C][C] upper triangle read), restated from
    cov_from_sums / k_record_cov_finalize (cov_tc.cu): fp64 (S - s_i s_j / n) / (n - 1), rounded to fp32, eps_cov added in
    fp32 on the diagonal.  No product feeds an add directly, so nvcc has nothing to contract: bit for bit."""
    S = np.triu(S) + np.triu(S, 1).T
    r = ((S - np.outer(s, s) / n) / (n - 1.0)).astype(np.float32)
    d = np.arange(len(s))
    r[d, d] = r[d, d] + np.float32(eps_cov)
    return r


def record_of(Q, lam, n=1025.0):
    """A record whose covariance is Q diag(lam) Q^T: S = (n - 1) Sigma, s = 0."""
    return n, np.zeros(len(lam)), (n - 1.0) * sigma_of(Q, lam)


# ------------------------------------------------------------------------------------------------------------ metric
def eig(S32):
    lam, E = np.linalg.eigh(np.asarray(S32, np.float64))
    return lam, E


def whitening_error(W, S32, eps_eig=0.0, thresh=THRESH, basis=None):
    lam, E = basis if basis is not None else eig(S32)
    keep = lam > thresh
    target = np.where(keep, lam / (lam + eps_eig), 0.0)
    return E.T @ np.asarray(W, np.float64) @ np.asarray(S32, np.float64) @ np.asarray(W, np.float64) @ E - np.diag(target)


def colouring_error(Cs, S32, eps_eig=0.0, thresh=THRESH, basis=None):
    """(Ec on the kept block, |C_s e_i| / sqrt(lam_kept,min) for dropped i)."""
    lam, E = basis if basis is not None else eig(S32)
    keep = lam > thresh
    Cs = np.asarray(Cs, np.float64)
    ce = Cs @ E
    G = ce.T @ ce
    lk = lam[keep]
    Ec = (G[np.ix_(keep, keep)] - np.diag(lk + eps_eig)) / np.sqrt(np.outer(lk, lk))
    drop = np.linalg.norm(ce[:, ~keep], axis=0) / np.sqrt(lk.min()) if (~keep).any() else np.zeros(0)
    return Ec, drop


def tau_of(solver, C):
    """Jacobi: the cosine tolerance.  Newton-Schulz: the stopping residual plus the rounding of the last iteration's
    split-fp16 products, 2^-21 of the largest entry summed over C terms (sqrt(C), as for the stored operand)."""
    return 2.0 * np.sqrt(C) * EPS if solver == "jacobi" else NS_TOL + 2.0 ** -21 * np.sqrt(C)


def conv_term(lam, keep, solver, C):
    """conv_ij of the module docstring over the index pairs (i, j); lam float64 [C]."""
    tau = tau_of(solver, C)
    la = np.abs(lam)
    kk = np.outer(keep, keep)
    with np.errstate(divide="ignore", invalid="ignore"):
        if solver == "jacobi":
            r = np.sqrt(la[:, None] / la[None, :])
            c = tau * (2.0 + r + 1.0 / r)
        else:
            a = np.sqrt(la.max() / la)
            c = tau * (2.0 + a[:, None] + a[None, :])
    return np.where(kk, c, 2.0 * tau)


def whitening_bound(lam, thresh, solver, op_max):
    """(bound [C][C], mask of determined entries) for Ew, module docstring; op_max = max |W| entry."""
    # An entry with a dropped index (W e_i = 0 there) is reached by the rounding of the kept column's direction into e_i,
    # eps lam_max / lam_j relative, and by the stored operand: the kept entries' form with lam_i -> lam_j (both dropped:
    # lam_kept,min) in the rounding term and |lam_i| in the storage term.
    C = len(lam)
    keep = lam > thresh
    kk = np.outer(keep, keep)
    le = np.where(keep, lam, np.inf)
    lmin = np.minimum(le[:, None], le[None, :])
    lmin = np.where(np.isinf(lmin), lam[keep].min(), lmin)
    geo = np.where(kk, np.sqrt(np.abs(np.outer(lam, lam))), lmin)
    rnd = 4.0 * EPS * lam.max() / geo
    sq = np.sqrt(np.abs(lam))
    s = 2.0 ** -20 * np.sqrt(C) * op_max * (sq[:, None] + sq[None, :])
    return conv_term(lam, keep, solver, C) + rnd + s, rnd < 0.1


def colouring_bound(lam, thresh, solver, op_max):
    """(bound on the kept block, mask, bound for the dropped |C_s e_i| / sqrt(lam_kmin)); op_max = max |C_s| entry."""
    C = len(lam)
    keep = lam > thresh
    lk = lam[keep]
    sq = np.sqrt(lk)
    rnd = 4.0 * EPS * lam.max() / np.outer(sq, sq)
    s = 2.0 ** -20 * np.sqrt(C) * op_max * (1.0 / sq[:, None] + 1.0 / sq[None, :])
    b = conv_term(lk, np.ones(len(lk), bool), solver, C) + rnd + s
    bdrop = 2.0 * tau_of(solver, C) + 4.0 * EPS * lam.max() / lk.min() + 2.0 ** -20 * np.sqrt(C) * op_max / np.sqrt(lk.min())
    return b, rnd < 0.1, bdrop


def worst_ratio(err, bound, mask):
    r = np.abs(err) / bound
    return float(np.max(np.where(mask, r, 0.0))), int((~mask).sum())


# --------------------------------------------------------------------------------------------- exact float64 solutions
def exact_w(S32, eps_eig=0.0, thresh=THRESH):
    lam, E = eig(S32)
    keep = lam > thresh
    f = np.where(keep, 1.0 / np.sqrt(np.abs(lam) + eps_eig), 0.0)
    return (E * f) @ E.T


def exact_cs(S32, eps_eig=0.0, thresh=THRESH):
    lam, E = eig(S32)
    keep = lam > thresh
    f = np.where(keep, np.sqrt(np.abs(lam) + eps_eig), 0.0)
    return (E * f) @ E.T


def from_columns(G, S32, mode, eps_eig=0.0, thresh=THRESH, power=2):
    """k_eig_post + k_outer_gemm in float64 from Jacobi columns G (column i = sigma_i u_i): Rayleigh quotients against S32,
    d = f(lam) / |g|^power (power = 2 is the library's rule), W = G diag(d) G^T."""
    G = np.asarray(G, np.float64)
    A = np.asarray(S32, np.float64)
    ss = (G * G).sum(0)
    lam = np.where(ss > 0, np.einsum("ij,ik,kj->j", G, A, G) / np.where(ss > 0, ss, 1.0), 0.0)
    sg = np.abs(lam)
    keep = sg > thresh
    f = 1.0 / np.sqrt(sg + eps_eig) if mode == "white" else np.sqrt(sg + eps_eig)
    d = np.where(keep, f / np.where(ss > 0, ss, 1.0) ** (power / 2.0), 0.0)
    return (G * d) @ G.T, int(keep.sum())


# ------------------------------------------------------------------------------------ float32 one-sided Jacobi oracle
def _rounds(C):
    idx = list(range(C))
    out = []
    for _ in range(C - 1):
        out.append((np.array(idx[:C // 2]), np.array(idx[C // 2:][::-1])))
        idx = [idx[0], idx[-1]] + idx[1:-1]
    return out


def kernel_null2(amax, thresh):
    """k_jacobi's null floor from the largest squared column norm of the previous sweep."""
    f32 = np.float32
    return min(f32(1e-11) * amax, max(f32(0.25) * f32(thresh) * f32(thresh), f32(9.1e-13) * amax))


def jacobi_f32(A, null_floor=None, thresh=THRESH, max_sweeps=40, skip_pair=None):
    """One-sided (Hestenes) Jacobi on the fp32 matrix A, float32 throughout.  Rotation rule of rot_scalars: a pair is
    rotated when g^2 > tol^2 a b with tol = 2 sqrt(C) 2^-24, unless both columns are below null2 = null_floor * max|col|^2
    of the previous sweep (0 in sweep 0).  null_floor=None: k_jacobi's rule (kernel_null2, with thresh); a number f:
    null2 = f * max|col|^2 (0 turns the floor off, 1e-11 is the rule before thresh entered it).  skip_pair=(p, q): never
    rotate that pair.  Returns (G, sweeps)."""
    f32 = np.float32
    C = A.shape[0]
    G = np.array(A, dtype=f32, copy=True)
    tol = f32(2.0 * np.sqrt(C) * EPS)
    null2 = f32(0.0)
    sweep = 0
    for sweep in range(max_sweeps):
        any_rot = False
        amax = f32(0.0)
        for p, q in _rounds(C):
            x, y = G[:, p], G[:, q]
            a = (x * x).sum(0, dtype=f32)
            b = (y * y).sum(0, dtype=f32)
            g = (x * y).sum(0, dtype=f32)
            amax = max(amax, a.max(), b.max())
            rot = (np.maximum(a, b) > null2) & (g * g > tol * tol * a * b)
            if skip_pair is not None:
                rot &= ~(((p == skip_pair[0]) & (q == skip_pair[1])) | ((p == skip_pair[1]) & (q == skip_pair[0])))
            if not rot.any():
                continue
            any_rot = True
            d = b - a
            g2 = g + g
            w = np.sqrt(d * d + g2 * g2)
            t = np.where(rot, np.where(d < 0, -g2, g2) / np.where(rot, np.abs(d) + w, f32(1)), f32(0)).astype(f32)
            c = (f32(1) / np.sqrt(f32(1) + t * t)).astype(f32)
            s = (t * c).astype(f32)
            G[:, p] = (c * x - s * y).astype(f32)
            G[:, q] = (s * x + c * y).astype(f32)
        null2 = kernel_null2(amax, thresh) if null_floor is None else f32(null_floor) * amax
        if not any_rot:
            break
    return G, sweep + 1


# ------------------------------------------------------------------------------------- float64 Newton-Schulz emulation
def newton_schulz(A, eps_eig=0.0, max_it=16, tol=NS_TOL, skip=0):
    """The coupled iteration of matfun_tc.cu in float64: Y0 = A/s, Z0 = I, T = (3I - ZY)/2, Y <- YT, Z <- TZ; the residual
    max|I - Z Y| is taken from each iteration's first product, and the iteration whose residual passes the test still
    runs its update (the trailing iteration).  skip = 1 returns the iterate at the passing test without that update
    (stopped one iteration early), skip = 2 the iterate one update before that.
    Returns (A^-1/2 estimate, A^+1/2 estimate, updates run; max_it + 1 if the test never passed)."""
    C = A.shape[0]
    A = np.asarray(A, np.float64) + eps_eig * np.eye(C)
    s = np.linalg.norm(A)
    hist = [(np.eye(C), A / s)]
    for it in range(max_it):
        Z, Y = hist[-1]
        ZY = Z @ Y
        r = np.abs(np.eye(C) - ZY).max()
        T = 0.5 * (3.0 * np.eye(C) - ZY)
        hist.append((T @ Z, Y @ T))
        if r < tol:
            Z, Y = hist[-1 - skip]
            return Z / np.sqrt(s), Y * np.sqrt(s), len(hist) - 1 - skip
    Z, Y = hist[-1]
    return Z / np.sqrt(s), Y * np.sqrt(s), max_it + 1
