"""GPU parity: Jacobi eigensolver, WCT level (vs the reference's own wct_np golden
vectors and vs the wct_tf restatement), AdaIN -- all through the C-ABI."""
import glob
import os

import numpy as np
import pytest
import torch

from oracle import ref_ops
from wct_tf_b200 import _capi
from tests import gpu_util as U

pytestmark = pytest.mark.gpu
GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "wct_np_*.npz")))


@pytest.mark.parametrize("n", [64, 128, 256, 512])
def test_jacobi_eigh_matches_lapack(n):
    rng = np.random.default_rng(n)
    count = 3
    mats = []
    for i in range(count):
        f = np.maximum(rng.standard_normal((3 * n, n)) @ (rng.standard_normal((n, n)) / np.sqrt(n)) + 0.3, 0)
        if i == 1:
            f[:, rng.choice(n, n // 8, replace=False)] = 0.0      # dead channels -> exact zero eigenvalues
        f -= f.mean(0)
        mats.append((f.T @ f / (f.shape[0] - 1)).astype(np.float32))
    a = np.stack(mats)
    d = U.dev(a)
    sigma = torch.empty((count, n), dtype=torch.float32, device="cuda")
    sweeps = torch.zeros(count, dtype=torch.int32, device="cuda")
    _capi.check(U.lib().wctb200_jacobi_eigh(d.data_ptr(), n, count, sigma.data_ptr(), sweeps.data_ptr(), U.stream()))
    torch.cuda.synchronize()
    g = d.cpu().numpy().astype(np.float64)       # [count][col][row]: column i = sigma_i u_i
    sg = sigma.cpu().numpy().astype(np.float64)
    print("sweeps", sweeps.cpu().numpy())
    assert (sweeps.cpu().numpy() < 40).all(), "Jacobi did not converge"
    for i in range(count):
        w = np.linalg.eigvalsh(a[i].astype(np.float64))[::-1]
        got = np.sort(sg[i])[::-1]
        assert np.abs(got - np.abs(w)).max() <= 4e-5 * np.abs(w).max(), (i, np.abs(got - np.abs(w)).max())
        # reconstruct A = sum_i sigma_i u_i u_i^T over the non-null columns, u_i = the NORMALISED column i (the transform uses
        # exactly this: d_i = f(sigma_i) / |g_i|^2, k_eig_post; sigma_i is the Rayleigh quotient, and the column norms of the
        # tensor-core solver drift from sigma_i by a few 1e-5 relative -- a pure scaling of the columns)
        keep = sg[i] > 1e-6 * sg[i].max()
        gi = g[i][keep]                       # rows = columns of G
        nrm = np.linalg.norm(gi, axis=1)
        assert np.abs(nrm / sg[i][keep] - 1).max() <= 2e-4
        u = gi / nrm[:, None]
        rec = (u.T * sg[i][keep]) @ u
        assert np.abs(rec - a[i]).max() <= 5e-5 * np.abs(a[i]).max()
        assert np.abs(u @ u.T - np.eye(u.shape[0])).max() <= 2e-5


def _run_wct(content, style, alpha, sem):
    nc, hc, wc, c = content.shape
    ns, hs, ws_, _ = style.shape
    cin = U.act_from_numpy(content)
    sin = U.act_from_numpy(style)
    out = U.act_alloc(nc, hc, wc, c)
    ws = torch.empty(U.lib().wctb200_wct_workspace_bytes(c, nc, ns), dtype=torch.uint8, device="cuda")
    kbuf = torch.zeros(2 * (nc + ns), dtype=torch.int32, device="cuda")
    p = dict(tf=(1e-8, 0.0, 1), np=(0.0, 1e-5, 0))[sem]
    _capi.check(U.lib().wctb200_wct_level(cin.data_ptr(), nc, hc, wc, sin.data_ptr(), ns, hs, ws_, c, float(alpha),
                                          p[0], p[1], 1e-5, p[2], out.data_ptr(), kbuf.data_ptr(), ws.data_ptr(),
                                          ws.numel(), U.stream()))
    U.check_device()
    got = U.act_to_numpy(out, nc, hc, wc, c)
    padded = U.act_raw_padded(out, nc, hc, wc, c)
    assert np.isfinite(padded).all()
    assert np.array_equal(padded, np.pad(padded[:, 1:-1, 1:-1], ((0, 0), (1, 1), (1, 1), (0, 0)), mode="reflect"))
    return got, kbuf.cpu().numpy()


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[7:-4] for p in GOLDEN])
def test_wct_level_vs_reference_wct_np_golden(path):
    """north_star: stylised features within 1e-3 max-abs of the reference's wct_np."""
    g = np.load(path)
    got, k = _run_wct(g["content"], g["style"], float(g["alpha"]), "np")
    assert k[0] == int(g["k_c"]) and k[1] == int(g["k_s"]), (k, int(g["k_c"]), int(g["k_s"]))
    e32 = np.abs(got - g["out_ref_fp32"]).max()
    e64 = np.abs(got - g["out_ref_fp64"]).max()
    noise = np.abs(g["out_ref_fp32"] - g["out_ref_fp64"]).max()
    print("max-abs vs reference wct_np fp32 %.2e, vs its fp64 run %.2e (reference fp32-vs-fp64 %.2e), sweeps %s"
          % (e32, e64, noise, k[2:]))
    assert e32 <= 1e-3 and e64 <= 1e-3


@pytest.mark.parametrize("alpha", [1.0, 0.6])
def test_wct_level_tf_semantics_batched_shared_style(alpha):
    """wct_tf (ops.py:24-90): eps*I on the covariance, no eigenvalue eps, blend with fc+mc.
    Batch of 3 content frames sharing one style == 3 independent calls of the oracle."""
    g = np.load(GOLDEN[2])
    rng = np.random.default_rng(0)
    base = g["content"][0]
    contents = np.stack([base, np.roll(base, 3, axis=0) * 0.9 + 0.05, base[::-1].copy()]).astype(np.float32)
    style = g["style"]
    got, k = _run_wct(contents, style, alpha, "tf")
    for i in range(3):
        ref, info = ref_ops.wct_tf(contents[i:i + 1].astype(np.float64), style.astype(np.float64), alpha, return_info=True)
        assert ref_ops.spectral_gap_ok(info["wc"]) and ref_ops.spectral_gap_ok(info["ws"])
        assert k[i] == info["k_c"] and k[3] == info["k_s"]
        assert np.abs(got[i:i + 1] - ref).max() <= 1e-3, np.abs(got[i:i + 1] - ref).max()


def test_wct_level_per_frame_styles():
    g = np.load(GOLDEN[0])
    c2 = np.concatenate([g["content"], g["content"][:, ::-1]]).astype(np.float32)
    s2 = np.concatenate([g["style"], g["style"][:, :, ::-1] * 1.3]).astype(np.float32)
    got, k = _run_wct(c2, s2, 0.8, "np")
    for i in range(2):
        ref = ref_ops.wct_np(c2[i:i + 1].astype(np.float64), s2[i:i + 1].astype(np.float64), 0.8)
        assert np.abs(got[i:i + 1] - ref).max() <= 1e-3


@pytest.mark.parametrize("c", [64, 512])
@pytest.mark.parametrize("alpha", [1.0, 0.5])
def test_adain_level(c, alpha):
    rng = np.random.default_rng(c)
    content = np.maximum(rng.normal(0.5, 1, (2, 9, 11, c)), 0).astype(np.float32)
    style = np.maximum(rng.normal(0.2, 2, (1, 7, 13, c)), 0).astype(np.float32)
    cin, sin = U.act_from_numpy(content), U.act_from_numpy(style)
    out = U.act_alloc(2, 9, 11, c)
    ws = torch.empty(U.lib().wctb200_wct_workspace_bytes(c, 2, 1), dtype=torch.uint8, device="cuda")
    _capi.check(U.lib().wctb200_adain_level(cin.data_ptr(), 2, 9, 11, sin.data_ptr(), 1, 7, 13, c, alpha, 1e-5,
                                            out.data_ptr(), ws.data_ptr(), ws.numel(), U.stream()))
    got = U.act_to_numpy(out, 2, 9, 11, c)
    for i in range(2):
        ref = ref_ops.adain(U.split_repr(content[i:i + 1]), U.split_repr(style), alpha)
        assert np.abs(got[i:i + 1] - ref).max() <= 2e-5 * (1 + np.abs(ref).max())


ADAIN_MEANS = (0.3, 5.0, 30.0)
ADAIN_STDS = (1.0, 0.1, 0.03)


def _adain_features(shape, rng):
    """Channel c takes mean x std combination c % 11 of ADAIN_MEANS x ADAIN_STDS; combination 9 is a constant channel
    (var = 0: eps governs) and 10 an all-zero channel."""
    n, h, w, c = shape
    x = rng.standard_normal(shape)
    for ch in range(c):
        k = ch % 11
        if k < 9:
            x[..., ch] = ADAIN_MEANS[k // 3] + ADAIN_STDS[k % 3] * x[..., ch]
        else:
            x[..., ch] = 29.71 if k == 9 else 0.0
    return x.astype(np.float32)


@pytest.mark.parametrize("alpha", [1.0, 0.6])
@pytest.mark.parametrize("shape", [(1, 256, 256, 64), (2, 128, 128, 128), (1, 64, 64, 256), (3, 32, 32, 512), (1, 37, 53, 64)],
                         ids=lambda s: "x".join(map(str, s)))
def test_adain_level_moments_at_numeric_edges(shape, alpha):
    """AdaIN vs the two-pass float64 oracle on channels with large means and small spreads (where sum x^2 / HW - mean^2
    cancels), a constant channel and an all-zero one, at level-sized maps.  Per channel c:
        max |got - ref| <= 1e-5 max |ref_c| + 1e-4 alpha sqrt(var_s,c)
    (the SPF16 rounding of the output, plus a 1e-5-class error on the normalised part)."""
    n, h, w, c = shape
    rng = np.random.default_rng(sum(shape))
    content = _adain_features(shape, rng)
    ns = n if n == 2 else 1
    style = (rng.uniform(0.0, 3.0, c) + rng.uniform(0.2, 2.0, c) * rng.standard_normal((ns, h // 2 + 3, w // 2 + 5, c)))
    style = style.astype(np.float32)
    cin, sin = U.act_from_numpy(content), U.act_from_numpy(style)
    out = U.act_alloc(n, h, w, c)
    ws = torch.empty(U.lib().wctb200_wct_workspace_bytes(c, n, ns), dtype=torch.uint8, device="cuda")
    _capi.check(U.lib().wctb200_adain_level(cin.data_ptr(), n, h, w, sin.data_ptr(), ns, style.shape[1], style.shape[2], c, alpha,
                                            1e-5, out.data_ptr(), ws.data_ptr(), ws.numel(), U.stream()))
    U.check_device()
    got = U.act_to_numpy(out, n, h, w, c)
    worst = (0.0, None)
    for i in range(n):
        s64 = U.split_repr(style[i if ns > 1 else 0][None])
        ref = ref_ops.adain(U.split_repr(content[i:i + 1]), s64, alpha)
        err = np.abs(got[i:i + 1] - ref).max(axis=(0, 1, 2))
        tol = 1e-5 * np.abs(ref).max(axis=(0, 1, 2)) + 1e-4 * alpha * np.sqrt(s64.var(axis=(0, 1, 2)))
        r = err / tol
        if r.max() > worst[0]:
            ch = int(r.argmax())
            worst = (float(r.max()), (i, ch, ch % 11, float(err[ch]), float(tol[ch])))
    print("worst err / tol %.3g at (frame, channel, combination, err, tol) %s" % worst)
    assert worst[0] <= 1.0, worst


def test_split_style_prepare_and_apply_equals_combined_level():
    """wctb200_wct_style_prepare + wctb200_wct_apply (two-stream form) == wctb200_wct_level."""
    g = np.load(GOLDEN[3])
    content = np.concatenate([g["content"], g["content"][:, ::-1]]).astype(np.float32)
    style = g["style"].astype(np.float32)
    nc, hc, wc, c = content.shape
    ns, hs, ws_, _ = style.shape
    ref, kref = _run_wct(content, style, 0.7, "tf")
    lib = U.lib()
    cin, sin = U.act_from_numpy(content), U.act_from_numpy(style)
    out = U.act_alloc(nc, hc, wc, c)
    ws = torch.empty(lib.wctb200_wct_workspace_bytes(c, nc, ns), dtype=torch.uint8, device="cuda")
    state = torch.empty(lib.wctb200_wct_style_state_bytes(c, ns), dtype=torch.uint8, device="cuda")
    kbuf = torch.zeros(2 * (nc + ns), dtype=torch.int32, device="cuda")
    _capi.check(lib.wctb200_wct_style_prepare(sin.data_ptr(), ns, hs, ws_, c, 1e-8, 0.0, 1e-5, state.data_ptr(),
                                              ws.data_ptr(), ws.numel(), U.stream()))
    _capi.check(lib.wctb200_wct_apply(cin.data_ptr(), nc, hc, wc, c, state.data_ptr(), ns, 0.7, 1e-8, 0.0, 1e-5, 1,
                                      out.data_ptr(), kbuf.data_ptr(), ws.data_ptr(), ws.numel(), U.stream()))
    U.check_device()
    got = U.act_to_numpy(out, nc, hc, wc, c)
    assert np.array_equal(kbuf.cpu().numpy()[: nc + ns], kref[: nc + ns])
    assert np.abs(got - ref).max() <= 2e-5


@pytest.mark.parametrize("shape", [(1, 8, 32, 64), (2, 9, 40, 64), (1, 16, 33, 128), (1, 12, 20, 256), (2, 8, 8, 512),
                                   (1, 70, 130, 64), (1, 3, 2, 128)])
def test_covariance_kernels(shape):
    """Stage A of the transform (ops.py:43-45,105-108): per-channel mean and fc fc^T/(HW-1) on wgmma
    (MN-major operands, centred in shared memory)."""
    _covariance_case(shape, 0.3)


@pytest.mark.parametrize("offset", [0.3, 30.0])
@pytest.mark.parametrize("shape", [(1, 256, 256, 64), (1, 512, 512, 64)], ids=lambda s: "x".join(map(str, s)))
def test_covariance_level_sizes_with_offset(shape, offset):
    """relu1_1-sized maps (HW = 262 144 at 512 x 512: full split-K, 64 tiles per CTA) with small and large channel means: the
    sampled shift must keep S - s s^T / HW free of cancellation."""
    _covariance_case(shape, offset)


def _covariance_case(shape, offset):
    rng = np.random.default_rng(3)
    n, h, w, c = shape
    x = np.maximum(rng.standard_normal(shape) @ (rng.standard_normal((c, c)) / np.sqrt(c)) + offset, 0).astype(np.float32)
    lib = U.lib()
    buf = U.act_from_numpy(x)
    mean = torch.empty((n, c), dtype=torch.float32, device="cuda")
    cov = torch.empty((n, c, c), dtype=torch.float32, device="cuda")
    _capi.check(lib.wctb200_covariance(buf.data_ptr(), n, h, w, c, 1e-8, mean.data_ptr(), cov.data_ptr(), U.stream()))
    U.check_device()
    xs = U.split_repr(x).reshape(n, -1, c)
    for i in range(n):
        ref = np.cov(xs[i].T) + 1e-8 * np.eye(c)
        got = cov[i].cpu().numpy()
        assert np.abs(mean[i].cpu().numpy() - xs[i].mean(0)).max() <= 1e-6
        # tensor-core chunks add with truncation: ~24 adds x 2^-24 on the all-positive diagonal sums
        assert np.abs(got - ref).max() <= 1.5e-6 * max(1.0, np.abs(ref).max()), np.abs(got - ref).max()
        assert np.array_equal(got, got.T)


@pytest.mark.parametrize("sem", ["tf", "np"])
@pytest.mark.parametrize("flat", ["content", "style"])
@pytest.mark.parametrize("c", [64, 256])
def test_wct_level_constant_frame(c, flat, sem):
    """A constant map (a black video frame at relu1_1: every channel at its bias) has a zero covariance, so k = 0 on that
    side and the transform degenerates to a blend with the means.  The output must be finite, match the oracle's blend,
    and k_out must carry the oracle's counts."""
    rng = np.random.default_rng(c + (flat == "style"))
    mix = rng.standard_normal((c, c)) / np.sqrt(c)
    content = np.maximum(rng.standard_normal((1, 24, 32, c)) @ mix + 0.3, 0).astype(np.float32)
    style = np.maximum(rng.standard_normal((1, 20, 28, c)) @ mix.T + 0.3, 0).astype(np.float32)
    level = rng.uniform(0.0, 2.0, c).astype(np.float32)
    if flat == "content":
        content[:] = level
    else:
        style[:] = level
    alpha = 0.7
    got, k = _run_wct(content, style, alpha, sem)
    fn = ref_ops.wct_tf if sem == "tf" else ref_ops.wct_np
    ref, info = fn(U.split_repr(content), U.split_repr(style), alpha, return_info=True)
    assert (info["k_c"] == 0) == (flat == "content") and (info["k_s"] == 0) == (flat == "style")
    assert ref_ops.spectral_gap_ok(info["ws"] if flat == "content" else info["wc"])
    assert (k[0], k[1]) == (info["k_c"], info["k_s"]), (k, info["k_c"], info["k_s"])
    err = np.abs(got - ref).max()
    print("constant %s, %s semantics, C=%d: k %s, max-abs vs oracle %.2e" % (flat, sem, c, k[:2], err))
    assert err <= 2e-5 * (1 + np.abs(ref).max()), err


def test_jacobi_rank_deficient_null_space_stays_below_threshold():
    """HW < C (e.g. relu5_1 of a 256x256 image): 483 of 512 eigenvalues are exactly zero.  The count
    k = #(sigma > 1e-5) (ops.py:68,112) must equal what LAPACK finds on the same fp32 matrix."""
    rng = np.random.default_rng(1)
    C, hw = 512, 30
    x = np.maximum(rng.standard_normal((hw, C)) @ (rng.standard_normal((C, C)) / np.sqrt(C)) * 1.5 + 0.8, 0)
    xc = (x - x.mean(0)).astype(np.float32)
    cov = (xc.T @ xc / np.float32(hw - 1)).astype(np.float32)
    k_ref = int((np.linalg.svd(cov, compute_uv=False) > 1e-5).sum())
    assert k_ref == hw - 1
    d = U.dev(cov[None].copy())
    sigma = torch.empty((1, C), dtype=torch.float32, device="cuda")
    sweeps = torch.zeros(1, dtype=torch.int32, device="cuda")
    _capi.check(U.lib().wctb200_jacobi_eigh(d.data_ptr(), C, 1, sigma.data_ptr(), sweeps.data_ptr(), U.stream()))
    torch.cuda.synchronize()
    sg = np.sort(sigma.cpu().numpy()[0])[::-1]
    w = np.linalg.eigvalsh(cov.astype(np.float64))[::-1]
    print("lambda_max %.1f, k %d (ref %d), largest null value %.2e, sweeps %d" % (w[0], (sg > 1e-5).sum(), k_ref, sg[k_ref], int(sweeps.item())))
    assert int((sg > 1e-5).sum()) == k_ref
    assert np.abs(sg[:k_ref] - w[:k_ref]).max() <= 4e-5 * w[0]


@pytest.mark.parametrize("case", [
    # C, content HxW, style HxW, alpha, seed, patch, stride   (the swapped encoding must tile the content: (ho-1)*stride + patch == H)
    (64, (9, 11), (8, 12), 0.6, 5, 3, 1), (128, (12, 12), (13, 11), 1.0, 6, 3, 1), (512, (6, 7), (7, 6), 0.6, 7, 3, 1),
    (64, (9, 11), (11, 9), 0.6, 8, 5, 2),        # --ss-patch-size 5 --ss-stride 2
    (128, (9, 7), (10, 8), 0.7, 9, 3, 2),        # stride 2
    (64, (8, 10), (9, 9), 0.5, 10, 4, 1),        # even patch, stride 1
    (64, (7, 9), (8, 8), 0.6, 12, 1, 1),         # 1x1 patches
], ids=lambda c: "C%d_p%ds%d" % (c[0], c[5], c[6]))
def test_style_swap_level_matches_oracle(case):
    """wctb200_style_swap_level vs the NumPy restatement of ops.py:145-278 (itself pinned to the reference's own code by
    tests/golden/pipeline_swap5_*.npz).  The arg-max is discrete, so the vector must decide every position by a clear
    margin (asserted on the fp64 oracle), and then the matched patch indices must be identical."""
    C, hwc, hws, alpha, seed, patch, stride = case
    rng = np.random.default_rng(seed)

    def feat(hw):
        m = rng.standard_normal((C, C)) / np.sqrt(C)
        return np.maximum(rng.standard_normal((hw[0] * hw[1], C)) @ m + 0.3, 0.0).reshape(1, hw[0], hw[1], C).astype(np.float32)

    content, style = feat(hwc), feat(hws)
    ref, info = ref_ops.wct_style_swap(U.split_repr(content).astype(np.float64), U.split_repr(style).astype(np.float64), alpha,
                                       patch_size=patch, stride=stride, return_info=True)
    assert ref_ops.spectral_gap_ok(info["wc"]) and ref_ops.spectral_gap_ok(info["ws"]), "ill-posed vector (eigenvalue near the cut)"
    assert info["margin"].min() > 2e-3, "ill-posed vector (arg-max decided by %.1e)" % info["margin"].min()
    cin, sin = U.act_from_numpy(content), U.act_from_numpy(style)
    out = U.act_alloc(1, hwc[0], hwc[1], C)
    nbytes = U.lib().wctb200_style_swap_workspace_bytes(C, hwc[0], hwc[1], hws[0], hws[1], patch, stride)
    assert nbytes > 0
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    kbuf = torch.zeros(2, dtype=torch.int32, device="cuda")
    _capi.check(U.lib().wctb200_style_swap_level(cin.data_ptr(), hwc[0], hwc[1], sin.data_ptr(), hws[0], hws[1], C, patch, stride,
                                                 alpha, 1e-8, 1e-5, out.data_ptr(), kbuf.data_ptr(), ws.data_ptr(), ws.numel(),
                                                 U.stream()))
    U.check_device()
    got = U.act_to_numpy(out, 1, hwc[0], hwc[1], C)
    assert tuple(kbuf.cpu().tolist()) == (info["k_c"], info["k_s"])
    err = np.abs(got - ref).max()
    print("style swap C=%d patch %d stride %d: max-abs vs fp64 oracle %.2e (k %d/%d, min arg-max margin %.1e)"
          % (C, patch, stride, err, info["k_c"], info["k_s"], info["margin"].min()))
    assert err <= 1e-3
    padded = U.act_raw_padded(out, 1, hwc[0], hwc[1], C)
    assert np.array_equal(padded, np.pad(padded[:, 1:-1, 1:-1], ((0, 0), (1, 1), (1, 1), (0, 0)), mode="reflect"))


# ---------------------------------------------------------------------------
# matrix-function fast path (matfun_tc.cu): W_c = A^-1/2, C_s = A^+1/2 by coupled Newton-Schulz where k = C
# ---------------------------------------------------------------------------
def _cov_batch(C, HW, count, decay, seed, dead=0):
    out = []
    for i in range(count):
        r = np.random.default_rng(seed + i)
        X = np.maximum(r.standard_normal((C, C)) / np.sqrt(C) @ r.standard_normal((C, HW)) + 0.3, 0)
        X *= np.exp(-decay * np.arange(C) / C)[:, None]
        if dead:
            X[r.choice(C, dead, replace=False)] = 0.0
        X -= X.mean(1, keepdims=True)
        out.append((X @ X.T / (HW - 1) + 1e-8 * np.eye(C)).astype(np.float32))
    return np.stack(out)


def _matfun(A, n_first, thresh=1e-5, eps_eig=0.0):
    count, C = A.shape[0], A.shape[1]
    dA = U.dev(A)
    out = torch.full_like(dA, float("nan"))
    ok = torch.zeros(count, dtype=torch.int32, device="cuda")
    info = torch.zeros(count * 4, dtype=torch.float32, device="cuda")
    _capi.check(U.lib().wctb200_debug_matfun(dA.data_ptr(), C, count, n_first, thresh, eps_eig, out.data_ptr(), ok.data_ptr(),
                                             info.data_ptr(), U.stream()))
    U.check_device()
    return out.cpu().numpy(), ok.cpu().numpy(), info.cpu().numpy().reshape(count, 4)


@pytest.mark.parametrize("C,HW", [(128, 4096), (256, 2048), (512, 1024), (512, 4096)])
def test_matfun_fast_path_matches_float64_eigh(C, HW):
    """Well-conditioned covariances (every eigenvalue far above 1e-5): the guard accepts all of them, A^-1/2 (first half of the
    batch) and A^+1/2 (second half) agree with the float64 eigendecomposition to 2e-4 of their largest entry (measured
    3e-5 .. 6e-5), eps_eig included (wct_np semantics)."""
    for eps_eig in (0.0, 1e-5):
        A = _cov_batch(C, HW, 6, 0.0, 7 * C + HW)
        out, ok, info = _matfun(A, 3, eps_eig=eps_eig)
        assert ok.tolist() == [1] * 6, (ok, info)
        for b in range(6):
            w, v = np.linalg.eigh(A[b].astype(np.float64))
            ref = (v * (w + eps_eig) ** (-0.5 if b < 3 else 0.5)) @ v.T
            err = np.abs(out[b] - ref).max() / np.abs(ref).max()
            assert err <= 2e-4, (C, b, err)
            assert info[b, 2] > 1e-5 and info[b, 2] <= w[0] * 1.001 + eps_eig          # the bound really is a lower bound of lambda_min


@pytest.mark.parametrize("C", [128, 512])
def test_matfun_guard_leaves_hard_matrices_to_the_eigensolver(C):
    """Rank-deficient covariances (dead channels: eigenvalues at the 1e-8 regulariser), eigenvalues straddling the 1e-5 threshold and
    a degenerate all-zero matrix must NOT take the fast path; a mixed batch flags exactly the good ones."""
    good = _cov_batch(C, 4096, 2, 0.0, 11)
    dead = _cov_batch(C, 4096, 2, 0.0, 12, dead=5)
    w, v = np.linalg.eigh(good[0].astype(np.float64))
    w2 = w.copy(); w2[:3] = [4e-6, 9e-6, 2e-5]                                  # two eigenvalues below, one just above the threshold
    near = ((v * w2) @ v.T).astype(np.float32)[None]
    zero = np.zeros((1, C, C), np.float32)
    A = np.concatenate([good[:1], dead[:1], near, zero, good[1:], dead[1:]])
    out, ok, info = _matfun(A, 3)
    assert ok.tolist() == [1, 0, 0, 0, 1, 0], (ok, info)


def test_wct_level_fast_path_equals_eigensolver_path():
    """The same WCT level through the matrix-function fast path (default) and with it switched off (Jacobi eigensolver): k = C on both,
    zero sweeps reported by the fast path, stylised features within 3e-4 of each other and each within the gate of the oracle."""
    rng = np.random.default_rng(5)
    C = 256
    mix = rng.standard_normal((C, C)) / np.sqrt(C)
    content = np.maximum(rng.standard_normal((2, 24, 40, C)) @ mix + 0.3, 0).astype(np.float32)
    style = np.maximum(rng.standard_normal((2, 30, 28, C)) @ mix.T + 0.3, 0).astype(np.float32)
    lib = U.lib()
    res = {}
    for mode in (1, 0):
        lib.wctb200_debug_set_matfun(mode, 0)
        try:
            res[mode] = _run_wct(content, style, 0.7, "tf")
        finally:
            lib.wctb200_debug_set_matfun(1, 0)
    (fast, kf), (slow, ks) = res[1], res[0]
    assert kf[:4].tolist() == [C] * 4 and ks[:4].tolist() == [C] * 4
    assert kf[4:].tolist() == [0] * 4 and min(ks[4:]) > 0                         # sweeps: none on the fast path
    assert np.abs(fast - slow).max() <= 3e-4, np.abs(fast - slow).max()
    for i in range(2):
        ref = ref_ops.wct_tf(content[i:i + 1].astype(np.float64), style[i:i + 1].astype(np.float64), 0.7)
        assert np.abs(fast[i:i + 1] - ref).max() <= 1e-3 and np.abs(slow[i:i + 1] - ref).max() <= 1e-3
