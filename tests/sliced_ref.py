"""CPU oracle of sliced distribution matching (DESIGN.md §3.3.14), float64.

Per frame, with content x_0 [Nc, C], style Y [Ms, C] and the step matrices G_1 .. G_{K+1} of ``wct_tf_b200.sliced``:

    S_k     = the values of R_k Y sorted per channel (S_{K+1}: of Y itself)
    y_1     = G_1 x_0;  m_k = EFDM(y_k, S_k) at alpha = 1 (``efdm_ref.efdm_channel``);  y_{k+1} = G_{k+1} m_k
    out     = alpha m_{K+1} + (1 - alpha) x_0

K = 0 is plain EFDM.  ``step`` is one step on its own, for teacher-forcing the device against the oracle.
"""
import numpy as np

from tests import efdm_ref as E
from wct_tf_b200 import sliced


def step(v, G, style_proj, alpha=1.0, blend_with=None):
    """One step of a frame: EFDM of G v against the projected style values, v [Nc, C], style_proj [Ms, C] (any order).
    ``blend_with`` [Nc, C]: return alpha m + (1 - alpha) blend_with instead of m."""
    y = np.asarray(v, np.float64) @ np.asarray(G, np.float64).T
    m = np.empty_like(y)
    for c in range(y.shape[1]):
        m[:, c] = E.efdm_channel(y[:, c], style_proj[:, c], 1.0)
    return m if blend_with is None else alpha * m + (1.0 - alpha) * np.asarray(blend_with, np.float64)


def style_states(Y, K):
    """The K + 1 projected style value sets of a frame's style Y [Ms, C]: R_k Y (fp32 R's, float64 products), then Y."""
    C = Y.shape[1]
    Y = np.asarray(Y, np.float64)
    return [Y @ R.astype(np.float64).T for R in sliced.rotations(C, K)] + [Y]


def sliced_frame(x, Y, K, alpha=1.0, trace=None):
    """out [Nc, C] of one frame; ``trace`` (a list) receives each step's input (m_{k-1}, x_0 for k = 1) and output m_k."""
    x = np.asarray(x, np.float64)
    if K == 0:
        return np.stack([E.efdm_channel(x[:, c], Y[:, c], alpha) for c in range(x.shape[1])], 1)
    C = x.shape[1]
    Gs = sliced.step_matrices(C, K)
    Ss = style_states(Y, K)
    m = x
    for k in range(K + 1):
        v, m = m, step(m, Gs[k], Ss[k])
        if trace is not None:
            trace.append((v, m))
    return alpha * m + (1.0 - alpha) * x


def sliced_efdm(content, style, K, alpha=1.0):
    """content [N,H,W,C], style [Ns,Hs,Ws,C] with Ns in {1, N}."""
    content = np.asarray(content, np.float64)
    style = np.asarray(style, np.float64)
    N, H, W, C = content.shape
    Ns = style.shape[0]
    assert Ns in (1, N) and style.shape[3] == C
    out = np.empty_like(content)
    for n in range(N):
        out[n] = sliced_frame(content[n].reshape(-1, C), style[0 if Ns == 1 else n].reshape(-1, C), K, alpha).reshape(H, W, C)
    return out


def held_out_directions(C, D, seed=20260):
    """D unit directions [D, C] drawn apart from the transform's bases."""
    U = np.random.default_rng(seed).standard_normal((D, C))
    return U / np.linalg.norm(U, axis=1, keepdims=True)


def sliced_w1(a, b, dirs):
    """Mean over the directions of the 1-D Wasserstein-1 distance between the projections of the point sets a [Na, C] and
    b [Nb, C] (quantile functions compared exactly over the union of their breakpoints)."""
    pa = np.asarray(a, np.float64) @ dirs.T
    pb = np.asarray(b, np.float64) @ dirs.T
    return float(E.w1(pa[None, :, None, :], pb[None, :, None, :]).mean())
