"""The style swap at the sizes it runs at: C = 512, hundreds to thousands of patches, many output-channel tiles of the
correlation, checked stage by stage against float64.

``wctb200_debug_style_swap_layout`` says where one prepare + apply leaves each stage's result, so a test reads them all
back after the call and checks each stage on the device's own inputs to it:

  filters   the per-tap norms are the fp64 norms of the device's whitened style within an fp32 sum of n_patches
            squares (n_patches * 2^-24 relative, plus 2^-21 for rsqrtf); the split filters are that style times those
            norms, emulated in fp32 and split into fp16 pairs: equal bit for bit.  Padding filters are zero.
  a. scores against fp64 dot products of the STORED operands (whitened content hi+lo, filters hi+lo; the filters' lo plane
     is an fp16 subnormal for most entries, so the stored values are the operands the tensor cores saw):
        |s - s^| <= (2^-16 + ceil(K/128) * 2^-24) * sum_k |x_k w_k| + 2^-22 |s^|
     2^-16: the tensor core's truncating accumulation inside a chunk of 128 products (DESIGN 3.1) and the dropped lo*lo
     product (2^-22); ceil(K/128) * 2^-24: one round-to-nearest add per chunk into the running sum; 2^-22: the SPF16 store
     of the score.  A dropped cross product (2^-11 relative) or a score from a wrong tile is far outside.  Every real patch
     channel is checked; the padding channels hold 0.
  b. arg-max: the first maximum of the device's own scores merged as k_swap_argmax merges them (fp32 hi + lo, ties to the
     lower index, real patches only).  Exact.
  c. agreement with the oracle: the whitened content and style within 1e-3 max-abs of the oracle's fp64 ones (the gate of
     the teacher-forced levels).  Per position, delta = max_n sum_k (|dx_k| |w_nk| + |x_k| |dw_nk|) + the bound of (a), dx
     and dw the device's stored operands minus the oracle's, bounds |device score - oracle score| for every patch.  Where
     the oracle's margin exceeds 2 delta the device must choose the oracle's patch; everywhere the oracle's score of the
     device's patch is within 2 delta of the oracle's maximum.  The positions inside that band are printed.
  d. gather: the average of the device's whitened style at the device's indices, in fp64, within an fp32 sum of <= P^2
     terms, the rounded 1/count and its product ((P^2 + 2) * 2^-24 of the mean magnitude) and the SPF16 store.
  e. output: the oracle evaluated at the device's indices, <= 1e-3 max-abs; k_c / k_s exact; every cell finite; the
     reflect halo intact.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import nets, ref_ops
from tests import gpu_util as U
from tests.test_gpu_conv_handoff import _both_grids
from tests.test_gpu_invariance import assert_bits, frame_copy, planes
from wct_tf_b200 import _capi
from wct_tf_b200.engine import Engine
from wct_tf_b200.weights import make_synthetic_weights

pytestmark = pytest.mark.gpu
C = 512                           # the swap only runs at relu5_1
TF = (1e-8, 1e-5)                 # eps_cov, thresh (the TF graph's)
ALL = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]
GATE = 1e-3


def _feats(rng, n, h, w, offset):
    """Relu-like features with channel correlations (each frame its own mix), fp32 [n,h,w,C]."""
    out = []
    for _ in range(n):
        m = rng.standard_normal((C, C)) / np.sqrt(C)
        out.append(np.maximum(rng.standard_normal((h * w, C)) @ m + offset, 0.0).reshape(h, w, C))
    return np.stack(out).astype(np.float32)


def _ws(nbytes):
    return torch.full((max(int(nbytes), 1),), 255, dtype=torch.uint8, device="cuda")   # 0xffff: an fp16 NaN, int32 -1


def _layout(nc, hc, wc, hs, ws_, p, s):
    out = (ctypes.c_longlong * 11)()
    _capi.check(U.lib().wctb200_debug_style_swap_layout(C, nc, hc, wc, hs, ws_, p, s, out))
    keys = ("n_patches", "cout_pad", "ho", "wo", "feat", "norms", "wsplit", "wc_feat", "scores", "idx", "ss_feat")
    return dict(zip(keys, [int(v) for v in out]))


def _fp16_planes(buf, off, n, h, w, c):
    nb = 2 * n * (h + 2) * (w + 2) * c * 2
    return buf[off:off + nb].view(torch.float16).view(2, n, h + 2, w + 2, c).cpu().numpy()


def _merge32(pl):
    """fp32 hi + lo, as merge_f32 forms it."""
    return pl[0].astype(np.float32) + pl[1].astype(np.float32)


def _windows(f, p, s):
    """[ho*wo, p*p*C] VALID p x p windows every s pixels of f [H,W,C], in the filters' (ky, kx, c) order."""
    v = np.lib.stride_tricks.sliding_window_view(f, (p, p), axis=(0, 1))[::s, ::s]
    return v.transpose(0, 1, 3, 4, 2).reshape(-1, p * p * f.shape[2])


def _split16(x32):
    x = np.clip(x32, np.float32(-65000), np.float32(65000)).astype(np.float32)
    hi = x.astype(np.float16)
    return hi, (x - hi.astype(np.float32)).astype(np.float16)


def _tile_bn(cout_pad, bn):
    return bn if bn and cout_pad % bn == 0 else (128 if cout_pad % 128 == 0 else 64)


def run_swap(cin, sin, nc, hc, wc, hs, ws_, p, s, alpha, bn=0):
    """prepare + apply through the C-ABI; every stage's result read back to the host."""
    lib = U.lib()
    L = _layout(nc, hc, wc, hs, ws_, p, s)
    state = _ws(lib.wctb200_style_swap_state_bytes(C, hs, ws_, p, s))
    pws = _ws(lib.wctb200_style_swap_prepare_workspace_bytes(C, hs, ws_, p, s))
    aws = _ws(lib.wctb200_style_swap_apply_workspace_bytes(C, nc, hc, wc, hs, ws_, p, s))
    out = U.act_alloc(nc, hc, wc, C)
    kout = torch.full((nc + 1,), -7, dtype=torch.int32, device="cuda")
    lib.wctb200_debug_set_conv_bn(bn)
    try:
        _capi.check(lib.wctb200_style_swap_prepare(sin.data_ptr(), hs, ws_, C, p, s, *TF, state.data_ptr(), None, pws.data_ptr(),
                                                   pws.numel(), U.stream()))
        _capi.check(lib.wctb200_style_swap_apply(cin.data_ptr(), nc, hc, wc, C, state.data_ptr(), hs, ws_, p, s, alpha, *TF,
                                                 out.data_ptr(), kout.data_ptr(), aws.data_ptr(), aws.numel(), U.stream()))
        U.check_device()
    finally:
        lib.wctb200_debug_set_conv_bn(0)
    torch.cuda.synchronize()
    npat, cp, K = L["n_patches"], L["cout_pad"], p * p * C
    nb = 2 * cp * K * 2
    return dict(
        L=L, out=out, out_bits=planes(out, nc, hc, wc, C), k=kout.cpu().numpy(),
        feat=_fp16_planes(state, L["feat"], 1, hs, ws_, C)[:, 0],
        norms=state[L["norms"]:L["norms"] + K * 4].view(torch.float32).cpu().numpy(),
        wsplit=state[L["wsplit"]:L["wsplit"] + nb].view(torch.float16).view(2, cp, K).cpu().numpy(),
        wc_feat=_fp16_planes(aws, L["wc_feat"], nc, hc, wc, C),
        scores=_fp16_planes(aws, L["scores"], nc, hc, wc, cp),
        idx=aws[L["idx"]:L["idx"] + nc * L["ho"] * L["wo"] * 4].view(torch.int32).view(nc, L["ho"], L["wo"]).cpu().numpy(),
        ss_feat=_fp16_planes(aws, L["ss_feat"], nc, hc, wc, C),
        n_patches=npat)


def check_swap(r, content64, style64, p, s, alpha, what, bn=0):
    """Checks filters and a-e of one run_swap result.  content64 [nc,hc,wc,C] / style64 [1,hs,ws,C]: the values the device
    inputs hold, in float64.  Returns per-frame (oracle info, worst output error, band count)."""
    L, npat = r["L"], r["n_patches"]
    nc, hc, wc = content64.shape[:3]
    ho, wo, cp, K = L["ho"], L["wo"], L["cout_pad"], p * p * C
    eb = 2.0 ** -16 + math.ceil(K / 128) * 2.0 ** -24
    # -- filters: norms from the device's whitened style, filters = style * norms split into fp16 pairs
    feat32 = _merge32(r["feat"])[1:-1, 1:-1]
    pat32 = _windows(feat32, p, s)
    assert pat32.shape[0] == npat
    ssq = (pat32.astype(np.float64) ** 2).sum(0)
    inv64 = 1.0 / np.sqrt(np.maximum(ssq, 1e-12))
    rel = np.abs(r["norms"] / inv64 - 1.0).max()
    assert rel <= npat * 2.0 ** -24 + 2.0 ** -21, "%s: per-tap norms off by %.2e relative" % (what, rel)
    hi, lo = _split16(pat32 * r["norms"][None, :])
    assert_bits(r["wsplit"][0, :npat].view(np.int16), hi.view(np.int16), what + " filters hi")
    assert_bits(r["wsplit"][1, :npat].view(np.int16), lo.view(np.int16), what + " filters lo")
    assert not r["wsplit"][:, npat:].any(), what + ": padding filters not zero"
    W = r["wsplit"][0, :npat].astype(np.float64) + r["wsplit"][1, :npat].astype(np.float64)
    absW = np.abs(W)
    feat64 = r["feat"][0].astype(np.float64) + r["feat"][1].astype(np.float64)
    results = []
    for i in range(nc):
        tag = "%s frame %d" % (what, i)
        # -- a. scores
        wcf = r["wc_feat"][0, i].astype(np.float64) + r["wc_feat"][1, i].astype(np.float64)
        X = _windows(wcf[1:-1, 1:-1], p, s)
        sd = _merge32(r["scores"][:, i])[1:1 + (ho - 1) * s + 1:s, 1:1 + (wo - 1) * s + 1:s].reshape(ho * wo, cp)
        assert not (sd[:, npat:] != 0).any(), tag + ": padding channels of the scores are not 0"
        sd = sd[:, :npat]
        sd64 = sd.astype(np.float64)
        shat = X @ W.T
        bound = eb * (np.abs(X) @ absW.T) + 2.0 ** -22 * np.abs(shat)
        ratio = float((np.abs(sd64 - shat) / bound).max())
        assert ratio <= 1.0, "%s: score error %.2f x its bound" % (tag, ratio)
        # -- b. arg-max of the device's own scores
        idx = r["idx"][i].reshape(-1)
        assert np.array_equal(idx, sd.argmax(axis=1)), tag + ": idx is not the first maximum of the scores"
        # -- c. agreement with the oracle (which pastes the device's patches: e is compared with the same call)
        ref, info = ref_ops.wct_style_swap(content64[i:i + 1], style64, alpha, p, s, return_info=True, idx=r["idx"][i])
        assert ref_ops.spectral_gap_ok(info["wc"]) and ref_ops.spectral_gap_ok(info["ws"]), "ill-posed vector (eigenvalue near the cut)"
        wc_o, ws_o = info["wc_feat"][0], info["ws_feat"][0]
        e_wc = np.abs(wcf[1:-1, 1:-1] - wc_o).max()
        e_ws = np.abs(feat64[1:-1, 1:-1] - ws_o).max()
        assert e_wc <= GATE and e_ws <= GATE, "%s: whitened content %.2e / style %.2e from the oracle" % (tag, e_wc, e_ws)
        Xo = _windows(wc_o, p, s)
        Po = _windows(ws_o, p, s)
        Wo = Po / np.sqrt(np.maximum((Po ** 2).sum(0, keepdims=True), 1e-12))
        so = Xo @ Wo.T
        delta = (np.abs(X - Xo) @ absW.T + np.abs(Xo) @ np.abs(W - Wo).T + bound).max(axis=1)
        top2 = np.partition(so, -2, axis=1)[:, -2:]
        best, margin = top2[:, 1], top2[:, 1] - top2[:, 0]
        decided = margin > 2 * delta
        assert np.array_equal(idx[decided], so.argmax(axis=1)[decided]), tag + ": a decided position chose another patch"
        chosen = so[np.arange(len(idx)), idx]
        assert (chosen >= best - 2 * delta).all(), tag + ": the chosen patch scores below the band"
        band = int((~decided).sum())
        # -- d. gather
        zeros = np.zeros((1, hc, wc, C))
        g = ref_ops.style_swap(zeros, feat64[None, 1:-1, 1:-1], p, s, idx=r["idx"][i])[0]
        gabs = ref_ops.style_swap(zeros, np.abs(feat64[None, 1:-1, 1:-1]), p, s, idx=r["idx"][i])[0]
        ss = r["ss_feat"][0, i].astype(np.float64) + r["ss_feat"][1, i].astype(np.float64)
        tol = (p * p + 2) * 2.0 ** -24 * gabs + 2.0 ** -22 * np.abs(g) + 2.0 ** -24
        assert (np.abs(ss[1:-1, 1:-1] - g) <= tol).all(), tag + ": gathered feature off by %.2e" % np.abs(ss[1:-1, 1:-1] - g).max()
        # -- e. output
        pad = r["out_bits"][:, i].astype(np.int16).view(np.float16).astype(np.float64)
        padded = pad[0] + pad[1]
        assert np.isfinite(padded).all(), tag + ": cells left unwritten"
        assert np.array_equal(padded, np.pad(padded[1:-1, 1:-1], ((1, 1), (1, 1), (0, 0)), mode="reflect")), tag + ": halo"
        e_out = float(np.abs(padded[1:-1, 1:-1] - ref[0]).max())
        assert (r["k"][i], r["k"][nc]) == (info["k_c"], info["k_s"]), tag + ": k_c / k_s"
        bnr = _tile_bn(cp, bn)
        print("%s: %d patches, cout_pad %d, BN %d x %d tiles, k %d/%d, score err/bound %.3g, whitened %.1e/%.1e, "
              "band %d of %d positions, output err %.2e"
              % (tag, npat, cp, bnr, cp // bnr, info["k_c"], info["k_s"], ratio, e_wc, e_ws, band, len(idx), e_out))
        assert e_out <= GATE, "%s: output %.2e from the oracle at the device's indices" % (tag, e_out)
        results.append((info, e_out, band, so))
    return results


def _synthetic(nc, hwc, hws, seed):
    rng = np.random.default_rng(seed)
    content, style = _feats(rng, nc, hwc[0], hwc[1], 0.3), _feats(rng, 1, hws[0], hws[1], 0.4)
    return content, style, U.split_repr(content), U.split_repr(style)


def _run_synthetic(nc, hwc, hws, p, s, bn=0, seed=1, alpha=0.6):
    content, style, c64, s64 = _synthetic(nc, hwc, hws, seed)
    cin, sin = U.act_from_numpy(content), U.act_from_numpy(style)
    r = run_swap(cin, sin, nc, hwc[0], hwc[1], hws[0], hws[1], p, s, alpha, bn)
    return r, check_swap(r, c64, s64, p, s, alpha, "c%dx%d s%dx%d p%ds%d" % (hwc + hws + (p, s)), bn), (cin, sin)


# ------------------------------------------------------------------------------------------------------------------------
SCALE = [  # content h x w, style h x w, patch, stride
    pytest.param((32, 32), (32, 32), 3, 1, id="512sq_900_patches"),           # 15 tiles at BN 64, fused
    pytest.param((64, 64), (32, 32), 3, 1, id="1024_content_512_style"),       # 3 844 positions
    pytest.param((33, 33), (32, 32), 5, 2, id="p5s2_196_patches"),             # cout_pad 256: two BN-128 tiles
    pytest.param((32, 32), (32, 32), 16, 1, id="p16_K131072"),                 # strips of 143 rows, 289 patches
]


@pytest.mark.parametrize("hwc,hws,p,s", SCALE)
def test_style_swap_at_scale(hwc, hws, p, s):
    r, _, _ = _run_synthetic(1, hwc, hws, p, s)
    assert r["n_patches"] == ((hws[0] - p) // s + 1) * ((hws[1] - p) // s + 1)


def test_style_swap_1024_style_both_grids():
    """3 844 patches (1024^2 style), 61 N tiles: the same bytes on a grid of one CTA per SM and on the default grid."""
    hwc, hws = (32, 32), (64, 64)
    content, style, c64, s64 = _synthetic(1, hwc, hws, 2)
    cin, sin = U.act_from_numpy(content), U.act_from_numpy(style)
    one, dflt = _both_grids(lambda: run_swap(cin, sin, 1, 32, 32, 64, 64, 3, 1, 0.6))
    for key in ("out_bits", "feat", "norms", "wsplit", "wc_feat", "scores", "idx", "ss_feat"):
        assert np.array_equal(np.asarray(one[key]).view(np.uint8), np.asarray(dflt[key]).view(np.uint8)), key
    assert dflt["L"]["cout_pad"] == 3904
    check_swap(dflt, c64, s64, 3, 1, 0.6, "c32x32 s64x64")


def test_style_swap_rank_deficient_content():
    """16 x 16 content: 256 pixels for 512 channels, so k_c < 512 and the whitened content lives in a subspace."""
    _, res, _ = _run_synthetic(1, (16, 16), (32, 32), 3, 1)
    assert res[0][0]["k_c"] <= 255


@pytest.mark.parametrize("hws,bn", [((10, 10), 64), ((3, 67), 64), ((3, 67), 128), ((10, 18), 64), ((10, 18), 128),
                                    ((3, 131), 64)], ids=lambda v: "x".join(map(str, v)) if isinstance(v, tuple) else "bn%d" % v)
def test_style_swap_last_tile_edges(hws, bn):
    """64 / 65 / 128 / 129 patches: a full last tile, a last tile with one real patch, at each tile width cout_pad allows."""
    r, _, _ = _run_synthetic(1, (24, 24), hws, 3, 1, bn=bn)
    assert r["L"]["cout_pad"] % bn == 0


@pytest.mark.parametrize("hws", [(3, 4), (3, 5)], ids=["2_patches", "3_patches"])
def test_style_swap_few_patches_negative_scores(hws):
    """2 or 3 patches: at some positions every real score is negative, where a zero padding filter would win an arg-max that
    looked past the real patches."""
    r, res, _ = _run_synthetic(1, (24, 24), hws, 3, 1)
    so = res[0][3]
    neg = int((so.max(axis=1) < 0).sum())
    print("%d patches: %d of %d positions with every real score < 0" % (r["n_patches"], neg, so.shape[0]))
    assert neg > 0
    assert r["idx"].max() < r["n_patches"]


def test_style_swap_batched_frames():
    """Four 32 x 32 frames in one apply against a 32 x 32 style: every frame passes the checks and equals
    style_swap_level on that frame alone, bit for bit."""
    nc, hw = 4, (32, 32)
    r, _, (cin, sin) = _run_synthetic(nc, hw, hw, 3, 1, seed=3)
    lib = U.lib()
    for i in range(nc):
        one = U.act_alloc(1, 32, 32, C)
        lws = _ws(lib.wctb200_style_swap_workspace_bytes(C, 32, 32, 32, 32, 3, 1))
        _capi.check(lib.wctb200_style_swap_level(frame_copy(cin, i, nc, 32, 32, C).data_ptr(), 32, 32, sin.data_ptr(), 32, 32, C,
                                                 3, 1, 0.6, *TF, one.data_ptr(), None, lws.data_ptr(), lws.numel(), U.stream()))
        assert_bits(planes(one, 1, 32, 32, C)[:, 0], r["out_bits"][:, i], "batched apply frame %d" % i)
    U.check_device()


# ------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def weights():
    return make_synthetic_weights(42)


def _act64(act):
    nbytes = U.lib().wctb200_act_bytes(act.N, act.H, act.W, act.C)
    return U.act_raw_padded(act.buf[:nbytes], act.N, act.H, act.W, act.C)[:, 1:-1, 1:-1]


def _engine_swap5(weights, csize, ssize, alpha=0.8, ss_alpha=0.6, seeds=(1000, 7)):
    """swap5 through the engine with capture: relu5_1 equals a direct prepare/apply on the captured content feature and the
    style's relu5_1 feature, which passes the stage checks; every level is teacher-forced as in test_gpu_pipeline, the
    relu5_1 oracle evaluated at the device's indices.  Returns the worst level error."""
    eng = Engine(weights, ALL, semantics="tf")
    content = np.random.default_rng(seeds[0]).integers(0, 256, (1, csize, csize, 3), dtype=np.uint8)
    style = np.random.default_rng(seeds[1]).integers(0, 256, (1, ssize, ssize, 3), dtype=np.uint8)
    d_style = torch.from_numpy(style).cuda()
    cap = {}
    eng.stylize(torch.from_numpy(content).cuda(), d_style, alpha=alpha, want_info=True, capture=cap, swap5=True,
                ss_alpha=ss_alpha)
    eng.check_device()
    cf, tf5 = cap["content_feat"][0], cap["transformed"][0]
    ps = eng.prepare_call(d_style, swap5=True)
    torch.cuda.synchronize()
    f5 = ps.feat5
    r = run_swap(cf.buf, f5.buf, 1, cf.H, cf.W, f5.H, f5.W, 3, 1, ss_alpha)
    nbytes = U.lib().wctb200_act_bytes(1, cf.H, cf.W, C)
    assert_bits(r["out_bits"], planes(tf5.buf[:nbytes], 1, cf.H, cf.W, C), "engine relu5_1 vs the direct swap")
    check_swap(r, _act64(cf), _act64(f5), 3, 1, ss_alpha, "engine %d/%d relu5_1" % (csize, ssize))
    sfe = nets.encode(nets.preprocess(style).astype(np.float64), weights, ALL, np.float64)
    worst = 0.0
    for i, relu in enumerate(ALL):
        x = cap["level_input"][i].cpu().numpy().astype(np.float64)
        if i == 0:
            assert np.abs(x - content / 255.0).max() < 1e-7
        else:
            assert x.min() >= 0 and x.max() <= 1
        cfo = nets.encode(x, weights, [relu], np.float64)[relu]
        e_enc = np.abs(eng.act_to_f32(cap["content_feat"][i]).cpu().numpy() - cfo).max()
        k = eng.last_info[i].cpu().numpy()
        if i == 0:
            f, info = ref_ops.wct_style_swap(cfo, sfe[relu], ss_alpha, 3, 1, return_info=True, idx=r["idx"][0])
            assert (k[0], k[1]) == (info["k_c"], info["k_s"])
        else:
            f, info = ref_ops.wct_tf(cfo, sfe[relu], alpha, return_info=True)
            assert (k[0], k[1]) == (info["k_c"], info["k_s"])
        assert ref_ops.spectral_gap_ok(info["wc"]) and ref_ops.spectral_gap_ok(info["ws"]), "ill-posed vector"
        e_wct = np.abs(eng.act_to_f32(cap["transformed"][i]).cpu().numpy() - f).max()
        y = nets.decode(np.asarray(f, dtype=np.float64), weights, relu, np.float64)
        if i < len(ALL) - 1:
            y = np.clip(y, 0, 1)
        e_out = np.abs(cap["level_output"][i].cpu().numpy() - y).max()
        print("swap5 %s %dx%d: encoder %.2e  transform %.2e  level output %.2e" % (relu, csize, csize, e_enc, e_wct, e_out))
        worst = max(worst, e_enc, e_wct, e_out)
    return worst


def test_engine_swap5_config2_512(weights):
    """512^2 content and style, five levels: relu5_1 maps of 32 x 32, 900 patches."""
    assert _engine_swap5(weights, 512, 512) <= GATE


def test_engine_swap5_config4_1024_content_512_style(weights):
    """1024^2 content / 512^2 style: 3 844 positions against 900 patches."""
    assert _engine_swap5(weights, 1024, 512) <= GATE
