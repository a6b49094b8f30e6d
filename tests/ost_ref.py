"""CPU oracle of the optimal-transport transform (OST, DESIGN.md §3.3.8).

OST replaces WCT's colouring of the whitened content, T_w = C_s W_c, by the Monge map between the content Gaussian
N(m_c, A_c) and the style's (Lu et al., ICCV 2019), with the kept-eigenvalue rules of ``oracle.ref_ops.wct_generic``:

    W_c = E_k (lambda + eps_eig)^-1/2 E_k^T,   S_c = E_k (lambda + eps_eig)^+1/2 E_k^T,   C_s as in wct_generic,
    B = S_c C_s C_s S_c,   B^1/2 = V sqrt(max(mu, 0)) V^T,   M = W_c B^1/2 W_c,
    out = alpha (M (x - m_c) + m_s) + (1 - alpha) base.
"""
import numpy as np

from oracle import nets, ref_ops

SEMANTICS = {
    "tf": dict(eps_cov=1e-8, eps_eig=0.0, readd_content_mean=True),
    "np": dict(eps_cov=0.0, eps_eig=1e-5, readd_content_mean=False),
}


def _kept(cov, thresh):
    E, lam, _ = np.linalg.svd(cov)
    k = int((lam > thresh).sum())
    return E[:, :k], lam[:k], k, lam


def ost_map(cov_c, cov_s, eps_eig=0.0, thresh=ref_ops.THRESH, return_info=False):
    """M (and WCT's T_w = C_s W_c) of two covariances A_c, A_s (eps_cov already on their diagonals), in their dtype."""
    cov_c, cov_s = np.asarray(cov_c), np.asarray(cov_s)
    Ec, lc, k_c, wc = _kept(cov_c, thresh)
    Es, ls, k_s, ws = _kept(cov_s, thresh)
    Wc = (Ec * (lc + eps_eig) ** -0.5) @ Ec.T
    Sc = (Ec * (lc + eps_eig) ** 0.5) @ Ec.T
    Cs = (Es * (ls + eps_eig) ** 0.5) @ Es.T
    P = Sc @ Cs
    B = P @ P.T
    mu, V = np.linalg.eigh((B + B.T) / 2)
    Bh = (V * np.sqrt(np.maximum(mu, 0))) @ V.T
    M = Wc @ Bh @ Wc
    if return_info:
        return M, dict(T=Cs @ Wc, Wc=Wc, Sc=Sc, Cs=Cs, B=B, k_c=k_c, k_s=k_s, wc=wc, ws=ws)
    return M


def _cov(flat, eps_cov):
    mean = flat.mean(axis=1, keepdims=True)
    f = flat - mean
    cov = f @ f.T / (flat.shape[1] - 1)
    if eps_cov:
        cov = cov + np.eye(cov.shape[0], dtype=cov.dtype) * cov.dtype.type(eps_cov)
    return mean, f, cov


def ost_generic(content, style, alpha, *, eps_cov, eps_eig, thresh=ref_ops.THRESH, readd_content_mean, return_info=False):
    """OST on one 1xHxWxC content / style pair with the statistics and eigenvalue rules of wct_generic.  Like wct_generic
    it computes in the dtype of its inputs: float64 for the truth, float32 for an fp32 engine's noise."""
    fcx, shape = ref_ops._flat(content)
    fsx, _ = ref_ops._flat(style)
    mc, fc, cov_c = _cov(fcx, eps_cov)
    ms, _, cov_s = _cov(fsx, eps_cov)
    M, info = ost_map(cov_c, cov_s, eps_eig, thresh, return_info=True)
    base = fc + mc if readd_content_mean else fc
    out = ref_ops._unflat(alpha * (M @ fc + ms) + (1 - alpha) * base, shape)
    if return_info:
        return out, dict(info, M=M)
    return out


def ost(content, style, alpha, semantics="tf", return_info=False):
    return ost_generic(content, style, alpha, **SEMANTICS[semantics], return_info=return_info)


def pipeline_ost(content_u8, style_u8, weights, relu_targets, alpha=1.0, semantics="tf", dtype=np.float32, return_info=False):
    """``oracle.nets.pipeline`` with OST in place of WCT at every level, all in ``dtype``."""
    relu_targets = list(relu_targets)
    x = nets.preprocess(content_u8).astype(dtype)
    style_feats = nets.encode(nets.preprocess(style_u8).astype(dtype), weights, relu_targets, dtype)
    info = []
    for i, relu in enumerate(relu_targets):
        if i > 0:
            x = np.clip(x, 0, 1)
        cf = nets.encode(x, weights, [relu], dtype)[relu]
        f, inf = ost(cf, style_feats[relu], alpha, semantics, return_info=True)
        info.append(inf)
        x = nets.decode(np.asarray(f, dtype=dtype), weights, relu, dtype)
    if return_info:
        return x, info
    return x
