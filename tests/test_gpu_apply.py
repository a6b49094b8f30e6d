"""GPU: the transform apply GEMM, out = M x + bias (CONV_APPLY of conv_tc.cu, DESIGN.md §3 "Stage D" and §3.1), against
float64 on transforms and statistics injected through the public layouts.

Every WCT, OST, blend, regions and soft-mask level ends in this GEMM, one weight set per frame.  The transforms here are
written by the test (wctb200_wct_transform_layout), or made by the library's own finalize from an injected statistics
record and style state, so each reference is exact float64 arithmetic on known operands and each bound follows from the
arithmetic of the kernel:
  * the stored operands are exact: x = x_hi + x_lo and M = M_hi + M_lo as fp16 pairs;
  * the kernel forms a_hi b_hi in chunks added with round-to-nearest, and the two cross products in one truncating
    accumulator added once (DESIGN.md §3.1); dropping a_lo b_lo costs 2^-22 sum |M||x|, the truncating chunk sums and the
    fp32 adds a few 2^-24 sum |M||x| each: together within 2^-20 (sum_j |M_ij||x_j| + |b_i|) (measured: up to ~2^-21);
  * the output is stored as an SPF16 pair: 2^-22 |out| + 2^-25 (the absolute step of a subnormal lo).
A wrong weight set, a dropped lo plane or a cross-product accumulator that is never added is off by 2^-11 sum |M||x| or
more, 2^9 times these bounds."""
import ctypes

import numpy as np
import pytest
import torch

from wct_tf_b200 import _capi
from tests import gpu_util as U

pytestmark = pytest.mark.gpu

SEMANTICS = {"tf": dict(eps_cov=1e-8, eps_eig=0.0, readd=1), "np": dict(eps_cov=0.0, eps_eig=1e-5, readd=0)}
THRESH = 1e-5


def _ws(nbytes):
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device="cuda")


# ------------------------------------------------------------------------------------------------------- layouts
def split16(m):
    """fp32 values -> (hi, lo) fp16 planes as split_f32 makes them (hi = fp16(m), lo = fp16(m - hi))."""
    m = np.asarray(m, dtype=np.float32)
    hi = m.astype(np.float16)
    lo = (m - hi.astype(np.float32)).astype(np.float16)
    return hi, lo


def transform_offsets(C, P):
    """(total bytes, [M, bias, k slot, row exponents]) of a WCT transform buffer of P problems."""
    o = [ctypes.c_size_t() for _ in range(3)]
    nbytes = U.lib().wctb200_wct_transform_layout(C, P, *[ctypes.byref(x) for x in o])
    oexp = U.lib().wctb200_wct_transform_row_exp_offset(C, P)
    assert 0 < oexp and oexp + P * C * 4 <= nbytes
    return nbytes, [x.value for x in o] + [oexp]


def row_exponents(Ms):
    """The e that puts each row's max |m| 2^e into [512, 1024) (0 for an all-zero row), as the library picks it."""
    amax = np.abs(np.asarray(Ms, np.float32)).max(-1)
    e = np.frexp(amax)[1]
    return np.where(amax > 0, np.clip(10 - e, -14, 40), 0).astype(np.int32)


def write_transform(Ms, bias, kc=None):
    """A WCT transform buffer of P = len(Ms) problems in the library's own form: row i of M [P,C,C] times 2^e_i, split into
    hi / lo fp16 planes, e in the row-exponent slot, bias fp32 [P,C], k slot [k_c x P | sweeps x P] (k_c = C unless given).
    Returns (device buffer, (M_hi + M_lo) 2^-e in float64)."""
    P, C = Ms.shape[0], Ms.shape[1]
    nbytes, (om, ob, ok, oexp) = transform_offsets(C, P)
    e = row_exponents(Ms)
    sc = np.exp2(e.astype(np.float64))
    hi, lo = split16(np.asarray(Ms, np.float32) * sc[..., None].astype(np.float32))
    kk = np.zeros(2 * P, np.int32)
    kk[:P] = C if kc is None else kc
    buf = np.zeros(nbytes, np.uint8)
    buf[om:om + P * 2 * C * C * 2] = np.stack([hi, lo], 1).reshape(-1).view(np.uint8)
    buf[ob:ob + P * C * 4] = np.asarray(bias, np.float32).reshape(-1).view(np.uint8)
    buf[ok:ok + 2 * P * 4] = kk.view(np.uint8)
    buf[oexp:oexp + P * C * 4] = e.reshape(-1).view(np.uint8)
    return U.dev(buf), (hi.astype(np.float64) + lo.astype(np.float64)) / sc[..., None]


def read_transform(tr, C, P):
    """(M = (M_hi + M_lo) 2^-e as float64 [P,C,C], bias float64 [P,C], k slot) of a transform buffer; asserts that every
    row exponent puts the row's max into [512, 1024)."""
    _, (om, ob, ok, oexp) = transform_offsets(C, P)
    b = tr.cpu().numpy()
    m = b[om:om + P * 2 * C * C * 2].view(np.float16).reshape(P, 2, C, C).astype(np.float64)
    inv = np.exp2(-b[oexp:oexp + P * C * 4].view(np.int32).reshape(P, C).astype(np.float64))
    ms = m[:, 0] + m[:, 1]
    amax = np.abs(ms).max(-1)
    assert ((amax == 0) | ((amax >= 512) & (amax < 1024))).all(), "a row's max is outside [512, 1024)"
    return ms * inv[..., None], b[ob:ob + P * C * 4].view(np.float32).reshape(P, C).astype(np.float64), \
        b[ok:ok + 2 * P * 4].view(np.int32)


def write_record(n, t, s, S):
    """A statistics record (wctb200_stats_record_layout, diag = 0): fp64 n [N], t [N][C], s [N][C], S [N][C][C]."""
    N, C = t.shape
    o = [ctypes.c_size_t() for _ in range(4)]
    nbytes = U.lib().wctb200_stats_record_layout(C, N, 0, *[ctypes.byref(x) for x in o])
    buf = np.zeros(nbytes, np.uint8)
    for off, a in zip(o, (n, t, s, S)):
        a = np.ascontiguousarray(a, np.float64).reshape(-1)
        buf[off.value:off.value + a.nbytes] = a.view(np.uint8)
    return U.dev(buf)


def write_style_state(mean_s, Cs, ks):
    """A WCT style state (wctb200_wct_style_state_layout): fp32 mean_s [Ns][C], C_s [Ns][C][C], int32 [k_s x Ns | sweeps]."""
    Ns, C = mean_s.shape
    o = [ctypes.c_size_t() for _ in range(3)]
    nbytes = U.lib().wctb200_wct_style_state_layout(C, Ns, *[ctypes.byref(x) for x in o])
    buf = np.zeros(nbytes, np.uint8)
    kk = np.zeros(2 * Ns, np.int32)
    kk[:Ns] = ks
    for off, a in zip(o, (np.asarray(mean_s, np.float32), np.asarray(Cs, np.float32), kk)):
        a = np.ascontiguousarray(a).reshape(-1)
        buf[off.value:off.value + a.nbytes] = a.view(np.uint8)
    return U.dev(buf)


# ------------------------------------------------------------------------------------------------------- operands
def features(shape, seed):
    """Level-like features: channels with a large mean and a small spread, a constant channel and an all-zero one (the
    pattern of AdaIN's moment tests), and channels whose scale decays over four decades."""
    n, h, w, c = shape
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(shape, dtype=np.float32)
    k = np.arange(c) % 5
    scale = np.exp(-9.0 * np.arange(c) / c).astype(np.float32)
    x = np.where(k == 0, 37.5 + 1e-3 * x, x)
    x = np.where(k == 1, np.float32(29.71), x)
    x = np.where(k == 2, np.float32(0.0), x)
    x = np.where(k >= 3, x * scale, x)
    return x.astype(np.float32)


def decade_matrix(C, rng):
    """Entries of both signs spanning 1e-6 .. 30, a diagonal of ~300 (W_c reaches ~300 at lambda ~ 1e-5), ~10% exact zeros
    and row 5 all zero.  (Sized so that every output stays inside the SPF16 range, |v| < 65504.)"""
    M = np.sign(rng.standard_normal((C, C))) * 10.0 ** rng.uniform(-6.0, np.log10(30.0), (C, C))
    M[np.arange(C), np.arange(C)] = np.sign(rng.standard_normal(C)) * rng.uniform(200.0, 300.0, C)
    M[rng.random((C, C)) < 0.1] = 0.0
    M[5] = 0.0
    return M.astype(np.float32)


def frame_matrices(C, P, seed):
    """P matrices that differ by far more than the bounds: a row permutation of one decade matrix each (the all-zero row
    moves with it), so that the weight set of another frame fails by a wide margin."""
    rng = np.random.default_rng(seed)
    M0 = decade_matrix(C, rng)
    return np.stack([M0[rng.permutation(C)] if p else M0 for p in range(P)])


def apply_bound(M, x, b):
    """Per output element: 2^-20 (sum_j |M_ij||x_j| + |b_i|) + SPF16 rounding of the output; M float64 [C,C], x [...,C]."""
    ref = x @ M.T + b
    mag = np.abs(x) @ np.abs(M).T + np.abs(b)
    assert np.abs(ref).max() < 65504.0, "the test's operands leave the SPF16 range"
    return ref, 2.0 ** -20 * mag + 2.0 ** -22 * np.abs(ref) + 2.0 ** -25


def reflect_pad(interior):
    """[n, h, w, c] -> [n, h+2, w+2, c], the reflect halo of the SPF16 layout (row 0 = row 1, row h+1 = row h-2)."""
    return np.pad(interior, ((0, 0), (1, 1), (1, 1), (0, 0)), mode="reflect")


def raw_planes(buf, n, h, w, c):
    torch.cuda.synchronize()
    return buf.view(torch.int16).view(2, n, h + 2, w + 2, c).cpu().numpy()


def check_layout(out, n, h, w, c, what):
    """No NaN cell left anywhere in the padded planes, and the halo is the reflection of the interior, bit for bit."""
    raw = raw_planes(out, n, h, w, c)
    assert np.isfinite(raw.view(np.float16)).all(), what + ": a cell was never written"
    for pl in range(2):
        assert np.array_equal(raw[pl], reflect_pad(raw[pl][:, 1:-1, 1:-1])), what + ": halo is not the reflected interior"


# ------------------------------------------------------------------------------------------------------ 1. apply
APPLY_CASES = [
    # C, N, H, W
    (64, 2, 512, 512),
    (64, 1, 540, 960),
    (128, 2, 256, 256),
    (256, 3, 128, 128),
    (512, 4, 64, 64),
    (512, 5, 30, 45),      # 128-position tiles straddle rows and end ragged at every frame boundary
    (512, 3, 3, 2),
    (64, 3, 37, 53),
]


@pytest.mark.parametrize("case", APPLY_CASES, ids=lambda c: "C%d_%dx%dx%d" % c)
def test_transform_apply_against_fp64(case):
    """wctb200_wct_transform_apply with a different M per frame against float64 of (M_hi + M_lo) x_stored + bias, within
    2^-20 (sum_j |M_ij||x_j| + |b_i|) + 2^-22 |out| + 2^-25 per element (module docstring); the halo is the reflected
    interior bit for bit and no poisoned cell is left."""
    C, N, H, W = case
    x = features((N, H, W, C), seed=C + H)
    Ms = frame_matrices(C, N, seed=C * 7 + N)
    rng = np.random.default_rng(C + W)
    bias = (rng.standard_normal((N, C)) * 10.0 ** rng.uniform(-3, 3, (N, C))).astype(np.float32)
    tr, Mq = write_transform(Ms, bias)
    act = U.act_from_numpy(x)
    out = U.act_alloc(N, H, W, C)
    _capi.check(U.lib().wctb200_wct_transform_apply(act.data_ptr(), N, H, W, C, tr.data_ptr(), out.data_ptr(), U.stream()))
    U.check_device()
    check_layout(out, N, H, W, C, "apply")
    xs = U.act_raw_padded(act, N, H, W, C)[:, 1:-1, 1:-1]
    got = U.act_raw_padded(out, N, H, W, C)[:, 1:-1, 1:-1]
    worst = 0.0
    for n in range(N):
        ref, bound = apply_bound(Mq[n], xs[n], bias[n].astype(np.float64))
        ratio = np.abs(got[n] - ref) / bound
        worst = max(worst, float(ratio.max()))
        if ratio.max() > 1.0:
            U.dump("fail_apply_C%d_%d" % (C, n), got=got[n], ref=ref, bound=bound)
        assert ratio.max() <= 1.0, "frame %d: worst error / bound = %.3g" % (n, ratio.max())
    print("apply C=%d %dx%dx%d: worst error / bound = %.3g" % (C, N, H, W, worst))


@pytest.mark.parametrize("C,N,H,W", [(64, 2, 37, 53), (512, 3, 3, 2), (256, 2, 40, 33)])
def test_identity_transform_returns_the_input_bits(C, N, H, W):
    """M = I and bias 0 (stored as 512 I, scale 2^-9): the products are 512 x_hi and 512 x_lo exactly, and their fp32 sum
    times 2^-9 is x_hi + x_lo.  Every stored value hi + lo of the output, halo included, equals the input's exactly.  (Its
    split may differ: where the input's lo was rounded as an fp16 subnormal, hi + lo can be a tie that fp16(hi + lo)
    rounds the other way, and a lo of -0 comes back as +0.)"""
    x = features((N, H, W, C), seed=C + N)
    tr, _ = write_transform(np.broadcast_to(np.eye(C, dtype=np.float32), (N, C, C)).copy(), np.zeros((N, C)))
    act = U.act_from_numpy(x)
    out = U.act_alloc(N, H, W, C)
    _capi.check(U.lib().wctb200_wct_transform_apply(act.data_ptr(), N, H, W, C, tr.data_ptr(), out.data_ptr(), U.stream()))
    U.check_device()
    assert np.array_equal(U.act_raw_padded(out, N, H, W, C), U.act_raw_padded(act, N, H, W, C))


# ------------------------------------------------------------------------------ 2. the operand of the library's finalize
def style_colouring(C, decay, seed):
    """C_s = A^1/2 (eigenvalues > thresh) of a covariance like the deep levels': ReLU features whose channel scales decay
    as exp(-decay c / C).  Rounded to fp32, as a state stores it."""
    r = np.random.default_rng(seed)
    HW = 4 * C
    X = np.maximum(r.standard_normal((C, C)) / np.sqrt(C) @ r.standard_normal((C, HW)) + 0.3, 0)
    X *= np.exp(-decay * np.arange(C) / C)[:, None]
    X -= X.mean(1, keepdims=True)
    lam, E = np.linalg.eigh(X @ X.T / (HW - 1))
    keep = lam > THRESH
    return ((E[:, keep] * np.sqrt(lam[keep])) @ E[:, keep].T).astype(np.float32), int(keep.sum())


def finalize(C, d, mean_c, mean_s, Cs, alpha, sem):
    """wctb200_wct_transform_from_stats of a record with covariance diag(d) and mean mean_c per frame, against a style
    state (mean_s, Cs) of one style per frame.  Returns (transform buffer, M_hi + M_lo, bias, k slot)."""
    lib = U.lib()
    Nc = mean_c.shape[0]
    s = SEMANTICS[sem]
    n = 1025.0
    S = np.zeros((Nc, C, C))
    S[:, np.arange(C), np.arange(C)] = d * (n - 1)
    rec = write_record(np.full(Nc, n), mean_c.astype(np.float64), np.zeros((Nc, C)), S)
    state = write_style_state(mean_s, Cs, C)
    ws = _ws(lib.wctb200_wct_workspace_bytes(C, Nc, 0))
    tr = torch.full((transform_offsets(C, Nc)[0],), 255, dtype=torch.uint8, device="cuda")
    _capi.check(lib.wctb200_wct_transform_from_stats(rec.data_ptr(), Nc, C, state.data_ptr(), Nc, alpha, s["eps_cov"],
                                                     s["eps_eig"], THRESH, s["readd"], tr.data_ptr(), ws.data_ptr(),
                                                     ws.numel(), U.stream()))
    U.check_device()
    return (tr,) + read_transform(tr, C, Nc)


@pytest.fixture(params=[0, 1], ids=["jacobi", "newton_schulz"])
def matfun(request):
    lib = U.lib()
    lib.wctb200_debug_set_matfun(request.param, 0)
    yield request.param
    lib.wctb200_debug_set_matfun(1, 0)


@pytest.mark.parametrize("sem", ["tf", "np"])
@pytest.mark.parametrize("alpha", [1.0, 0.6, 0.1])
@pytest.mark.parametrize("C", [64, 256, 512])
def test_finalized_operand_against_fp64(C, alpha, sem, matfun):
    """The operand and bias of the library's finalize, and their apply, against float64 on injected statistics.

    The record's covariance is diag(d), d powers of 4 spanning the kept range (4^-8 .. 4^4; 4^-2 .. 4^3 with the
    Newton-Schulz knob on, where it converges to fp32 accuracy), so W_c = diag(w), w = (d + eps)^-1/2 up to ~250,
    whichever solver runs.  First, C_s = 4 I and alpha = 1 give M = 4 W_c: its per-column relative error is
    eps_W, W_c's own error, and must stay at the fp32 level (the Newton-Schulz iteration's own convergence level).  Then, with one style per frame (frame 0 a flat spectrum,
    frame 1 one that decays as the deep levels' do), in float64:
        M_ref = alpha C_s W_c + (1 - alpha) I,   bias_ref = alpha m_s - M_ref m_c + (1 - alpha) readd m_c
        |M_hi + M_lo - M_ref| <= eps_W |M_ref| + 2^-21 max_j |M_ref,ij|       (entrywise)
        |out - M_ref x - bias_ref| <= 2^-19 (sum |M_ref||x| + |alpha m_s| + sum |M_ref||m_c| + (1 - alpha) readd |m_c|)
    The 2^-21 row term is what a split of fp32 into two normal fp16 halves leaves (2^-22 relative) plus the fp32
    products.  On the output, the GEMM's 2^-21 adds to the fp32 operand, the bias's fp32 dot product over C terms (C/32 + 5
    roundings per lane chain) and the output's rounding; a lo half that is an fp16 subnormal (|m| < 2^-3) or flushed to zero (|m| < ~3e-8) loses more than that
    wherever a row's entries are all small -- the rows of the decaying channels at small alpha."""
    s = SEMANTICS[sem]
    Nc = 2
    rng = np.random.default_rng(C + int(alpha * 10))
    ex = np.arange(C) % 13 - 8 if not matfun else np.arange(C) % 3 - 1
    d = 4.0 ** ex
    dr = (np.float32(d) + np.float32(s["eps_cov"])).astype(np.float64)     # the fp32 covariance diagonal
    w = 1.0 / np.sqrt(dr + np.float64(np.float32(s["eps_eig"])))
    mean_c = (rng.standard_normal((Nc, C)) * 5.0).astype(np.float32)
    a32 = float(np.float32(alpha))

    # eps_W: C_s = 4 I, alpha = 1 -> M = 4 W_c
    four = np.broadcast_to(4.0 * np.eye(C, dtype=np.float32), (Nc, C, C)).copy()
    _, Mw, _, kw = finalize(C, d, mean_c, np.zeros((Nc, C), np.float32), four, 1.0, sem)
    assert (kw[:Nc] == C).all(), kw
    Wref = np.diag(4.0 * w)
    eps_w = float((np.abs(Mw - Wref[None]) / (4.0 * w)[None, None, :]).max())
    print("C=%d %s matfun=%d: eps_W = %.3g (2^%.1f), sweeps %s" % (C, sem, matfun, eps_w, np.log2(max(eps_w, 1e-300)),
                                                                  kw[Nc:]))
    # Jacobi: a few fp32 roundings; Newton-Schulz stops at its own convergence level, a few 2^-20 (its accuracy is not
    # what this test is about: the bounds below take eps_W as measured)
    assert eps_w <= (2.0 ** -16 if matfun and C >= 128 else 2.0 ** -20), "W_c of a diagonal covariance is off by %.3g" % eps_w

    # the transform against per-frame styles: frame 0 flat, frame 1 decaying
    Cs = np.stack([style_colouring(C, dec, seed=C + f)[0] for f, dec in enumerate((0.0, 12.0))])
    mean_s = (rng.standard_normal((Nc, C)) * 3.0).astype(np.float32)
    tr, Mq, bq, kk = finalize(C, d, mean_c, mean_s, Cs, alpha, sem)
    assert (kk[:Nc] == C).all(), kk
    H, W = 24, 40
    x = (mean_c[:, None, None, :] + rng.standard_normal((Nc, H, W, C)) * np.sqrt(d)).astype(np.float32)
    act = U.act_from_numpy(x)
    out = U.act_alloc(Nc, H, W, C)
    _capi.check(U.lib().wctb200_wct_transform_apply(act.data_ptr(), Nc, H, W, C, tr.data_ptr(), out.data_ptr(), U.stream()))
    U.check_device()
    xs = U.act_raw_padded(act, Nc, H, W, C)[:, 1:-1, 1:-1]
    got = U.act_raw_padded(out, Nc, H, W, C)[:, 1:-1, 1:-1]
    fails = []
    for f in range(Nc):
        mc, ms = mean_c[f].astype(np.float64), mean_s[f].astype(np.float64)
        Mref = a32 * Cs[f].astype(np.float64) * w[None, :] + (1.0 - a32) * np.eye(C)
        bref = a32 * ms - Mref @ mc + ((1.0 - a32) * mc if s["readd"] else 0.0)
        ebound = eps_w * np.abs(Mref) + 2.0 ** -21 * np.abs(Mref).max(1, keepdims=True)
        er = float((np.abs(Mq[f] - Mref) / np.maximum(ebound, 1e-300)).max())
        ref = xs[f] @ Mref.T + bref
        obound = 2.0 ** -19 * (np.abs(xs[f]) @ np.abs(Mref).T + np.abs(a32 * ms) + np.abs(Mref) @ np.abs(mc)
                               + ((1.0 - a32) * np.abs(mc) if s["readd"] else 0.0))
        orr = float((np.abs(got[f] - ref) / obound).max())
        print("  frame %d (%s spectrum) alpha=%.1f: operand error / bound = %.3g, output error / bound = %.3g" % (
            f, "decaying" if f else "flat", alpha, er, orr))
        if er > 1.0 or orr > 1.0:
            fails.append((f, er, orr))
    assert not fails, "frame, operand error / bound, output error / bound: %s" % fails


# ------------------------------------------------------------------------------------------------- 3. weighted apply
@pytest.mark.parametrize("K", [1, 3, 8])
@pytest.mark.parametrize("C", [64, 256, 512])
def test_weighted_apply_against_fp64(C, K):
    """wctb200_wct_transform_apply_weighted with K injected transforms per frame, fractional weights and a strength map,
    against float64 of sum_k v_k (M_k x + b_k) + (1 - V) x, with v_k = s w_k and 1 - V as the kernel rounds them in fp32.
    Bound: the bound of the plain apply summed over k, 2^-20 (sum_k v_k (sum_j |M_k,ij||x_j| + |b_k,i|) + (1 - V)|x_i|),
    plus the output's SPF16 rounding.  Pixels where
    every v_k = 0 keep their input bytes, halo included."""
    N, H, W = 2, 19, 45
    x = features((N, H, W, C), seed=C + K)
    rng = np.random.default_rng(C * K)
    Ms = frame_matrices(C, N * K, seed=C + 3 * K)
    bias = (rng.standard_normal((N * K, C)) * 10.0 ** rng.uniform(-3, 3, (N * K, C))).astype(np.float32)
    tr, Mq = write_transform(Ms, bias)
    wts = rng.random((N, K + 1, H, W))
    wts = (wts / wts.sum(1, keepdims=True))[:, :K].astype(np.float32)
    wts[:, :, :, -3:] = 0.0                              # a band that keeps its input
    strength = np.tile(np.linspace(0.1, 1.0, W, dtype=np.float32), (N, H, 1))
    act = U.act_from_numpy(x)
    out = U.act_alloc(N, H, W, C)
    d_w, d_s = U.dev(wts), U.dev(strength)              # held until the kernel has read them
    _capi.check(U.lib().wctb200_wct_transform_apply_weighted(act.data_ptr(), N, H, W, C, tr.data_ptr(), K, d_w.data_ptr(),
                                                              d_s.data_ptr(), out.data_ptr(), U.stream()))
    U.check_device()
    check_layout(out, N, H, W, C, "weighted apply")
    xs = U.act_raw_padded(act, N, H, W, C)[:, 1:-1, 1:-1]
    got = U.act_raw_padded(out, N, H, W, C)[:, 1:-1, 1:-1]
    b64 = bias.astype(np.float64)
    worst = 0.0
    for n in range(N):
        v32 = strength[n][None] * wts[n]                  # v_k = s w_k, one fp32 product
        V32 = np.zeros((H, W), np.float32)
        for k in range(K):                                 # V and 1 - V in fp32, in k order, as the epilogue forms them
            V32 = V32 + v32[k]
        keep = (np.float32(1.0) - V32).astype(np.float64)[..., None]
        v = v32.astype(np.float64)
        ref = keep * xs[n]
        mag = keep * np.abs(xs[n])
        for k in range(K):
            z = n * K + k
            r, _ = apply_bound(Mq[z], xs[n], b64[z])
            ref += v[k][..., None] * r
            mag += v[k][..., None] * (np.abs(xs[n]) @ np.abs(Mq[z]).T + np.abs(b64[z]))
        bound = 2.0 ** -20 * mag + 2.0 ** -22 * np.abs(ref) + 2.0 ** -25
        ratio = np.abs(got[n] - ref) / bound
        worst = max(worst, float(ratio.max()))
        if ratio.max() > 1.0:
            U.dump("fail_weighted_C%d_K%d_%d" % (C, K, n), got=got[n], ref=ref, bound=bound)
        assert ratio.max() <= 1.0, "frame %d: worst error / bound = %.3g" % (n, ratio.max())
    print("weighted apply C=%d K=%d: worst error / bound = %.3g" % (C, K, worst))
    raw_in, raw_out = raw_planes(act, N, H, W, C), raw_planes(out, N, H, W, C)
    assert np.array_equal(raw_out[:, :, :, -4:, :], raw_in[:, :, :, -4:, :])   # the kept band and its halo column
