"""NumPy oracle of the statistics records of tiled stylisation (DESIGN.md §3.3.7; include/wctb200.h, stats_rect /
stats_accumulate / transform_from_stats): per frame the pixel count n, the centring shift t, s = sum (x - t) and
S = sum (x - t)(x - t)^T (its diagonal for AdaIN), folded tile by tile and finalised once, all in float64."""
import numpy as np


def record(x, t, diag=False):
    """The record of the pixels ``x`` [n, C] centred on the shift ``t`` [C]."""
    x = np.asarray(x, np.float64)
    d = x - np.asarray(t, np.float64)
    S = (d * d).sum(axis=0) if diag else d.T @ d
    return dict(n=float(x.shape[0]), t=np.array(t, np.float64), s=d.sum(axis=0), S=S)


def empty(C, diag=False):
    return dict(n=0.0, t=np.zeros(C), s=np.zeros(C), S=np.zeros(C if diag else (C, C)))


def accumulate(a, b):
    """Fold record ``b`` into ``a``: b's sums re-centred on a's shift, D = t_b - t_a, then added.  An empty ``a`` takes
    ``b`` as it is."""
    if a["n"] == 0:
        return {k: np.copy(v) if isinstance(v, np.ndarray) else v for k, v in b.items()}
    D = b["t"] - a["t"]
    s = b["s"] + b["n"] * D
    if np.ndim(b["S"]) == 1:
        S = b["S"] + 2 * D * b["s"] + b["n"] * D * D
    else:
        S = b["S"] + (np.outer(D, b["s"]) + np.outer(b["s"], D)) + b["n"] * np.outer(D, D)
    return dict(n=a["n"] + b["n"], t=a["t"], s=a["s"] + s, S=a["S"] + S)


def covariance(r, eps_cov=0.0):
    """WCT finalisation (k_cov_finalize): mean = t + s / n, cov = (S - s s^T / n) / (n - 1) + eps_cov I."""
    n = r["n"]
    cov = (r["S"] - np.outer(r["s"], r["s"]) / n) / (n - 1) + eps_cov * np.eye(len(r["s"]))
    return r["t"] + r["s"] / n, cov


def moments(r):
    """AdaIN finalisation (k_moments_finalize): mean = t + s / n, biased var = S / n - (s / n)^2."""
    m = r["s"] / r["n"]
    return r["t"] + m, np.maximum(r["S"] / r["n"] - m * m, 0.0)
