"""The random bases of sliced distribution matching (DESIGN.md §3.3.14).

Step k of a chain of K rotates each level's C channels into the orthonormal basis R_k, matches every 1-D marginal there
(EFDM) and rotates back; the last step (k = K + 1) is plain EFDM in the channel basis.  R_k depends only on (C, k), so a
chain of K steps is a prefix of one of K + 1, and every frame, batch and call sees the same bases.

R_k is a Gaussian matrix drawn from PCG64([TAG, C, k]) whose rows are orthonormalised by modified Gram-Schmidt applied
twice, in float64 with elementwise products and ``np.add.reduce`` (no BLAS or LAPACK, whose summation order varies by
build), then rounded to fp32.  The step matrices fold each back-rotation into the next forward one: G_1 = R_1, G_k = fp32(R_k R_{k-1}^T)
(float64 products of the fp32 R's), G_{K+1} = R_K^T.
"""
import functools

import numpy as np

TAG = 0x5CED                 # fixed seed tag of the bases
MAX_SLICES = 32


def _mgs(A):
    """Rows of float64 A orthonormalised by modified Gram-Schmidt (on a copy)."""
    Q = np.array(A, dtype=np.float64)
    C = Q.shape[0]
    for j in range(C):
        Q[j] /= np.sqrt(np.add.reduce(Q[j] * Q[j]))
        if j + 1 < C:
            rest = Q[j + 1:]
            rest -= np.add.reduce(rest * Q[j], axis=1)[:, None] * Q[j]
    return Q


@functools.lru_cache(maxsize=None)
def _rotation(C, k):
    g = np.random.Generator(np.random.PCG64([TAG, int(C), int(k)])).standard_normal((C, C))
    R = _mgs(_mgs(g)).astype(np.float32)
    R.setflags(write=False)
    return R


def rotations(C, K):
    """R_1 .. R_K: fp32 C x C orthonormal matrices (read-only); the projections of a pixel's values v are R v."""
    return [_rotation(int(C), k) for k in range(1, int(K) + 1)]


def _product_t(A, B):
    """fp32(A B^T) of fp32 A, B, computed in float64 row by row with ``np.add.reduce``."""
    A64, B64 = A.astype(np.float64), B.astype(np.float64)
    return np.stack([np.add.reduce(A64[i][None, :] * B64, axis=1) for i in range(A.shape[0])]).astype(np.float32)


@functools.lru_cache(maxsize=None)
def _step(C, k):
    if k == 1:
        return _rotation(C, 1)
    G = _product_t(_rotation(C, k), _rotation(C, k - 1))
    G.setflags(write=False)
    return G


def step_matrices(C, K):
    """G_1 .. G_{K+1} of a chain of K >= 1 slices: fp32 C x C; step k computes y_k = G_k m_{k-1} (m_0 the content)."""
    K = int(K)
    if K < 1:
        raise ValueError("a sliced chain has K >= 1 slices, got %d" % K)
    return [_step(int(C), k) for k in range(1, K + 1)] + [np.ascontiguousarray(_rotation(int(C), K).T)]
