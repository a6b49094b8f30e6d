"""The style swap at any relu level: the chunked apply and ``swap_targets``.

1. Chunk invariance through the C-ABI: every workspace from wctb200_style_swap_apply_min_workspace_bytes up gives the
   same output planes (halo included) and k_out, byte for byte, whether the correlation runs in one chunk, one N tile per
   chunk, two, three or with a ragged last chunk; cout_pad = 320 (= 64 mod 128) runs 128-wide chunks at its own N tile
   of 64.  One byte less than the minimum is WCTB200_EWS.
2. Accuracy at the finer levels' sizes: the one-chunk apply passes the stage checks of test_gpu_style_swap_scale (scores,
   the arg-max against float64 with its margin rule, the output at the device's indices) at C = 256 and 128, and a
   chunked apply equals it byte for byte.
3. The engine at 512^2: relu3_1 under the default workspace (two chunks) equals a one-chunk call.
4. The pipeline: swap_targets=["relu5_1"] is swap5; relu3_1 and relu4_1 + relu3_1 are teacher-forced level by level;
   batch, passes, prepared styles and .wctstyle files; every new ValueError.
"""
import math

import numpy as np
import pytest
import torch

import tests.test_gpu_style_swap_scale as SC
from oracle import nets, ref_ops
from tests import gpu_util as U
from tests.swap_levels_ref import pipeline_levels
from tests.test_gpu_invariance import assert_bits, planes
from wct_tf_b200 import _capi, engine as engine_mod
from wct_tf_b200.engine import Engine
from wct_tf_b200.wct import WCT
from wct_tf_b200.weights import make_synthetic_weights

pytestmark = pytest.mark.gpu
TF = (1e-8, 1e-5)
ALL = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]
GATE = 1e-3
EWS = _capi.EWS


def _ws(nbytes):
    return torch.full((max(int(nbytes), 1),), 255, dtype=torch.uint8, device="cuda")


def _align(n):
    return (n + 255) // 256 * 256


def _chunk_sizes(L, nc, hc, wc, bn):
    """Workspace sizes -> what they test: the full one, the minimum, 2 / 3 chunks and a ragged last chunk."""
    cp = L["cout_pad"]
    tiles = cp // bn
    col = 2 * 2 * nc * (hc + 2) * (wc + 2)

    def ws(cols):
        return _align(L["scores"] + cols * col)
    sizes = {"full": ws(cp), "min": ws(bn)}
    for k in (2, 3):
        if tiles >= k:
            sizes["%d_chunks" % k] = ws(math.ceil(tiles / k) * bn)
    ragged = [t for t in range(2, tiles) if tiles % t]
    if ragged:
        sizes["ragged_%d" % (ragged[0] * bn)] = ws(ragged[0] * bn)
    if bn == 64 and cp % 128 == 64:
        sizes["128_wide"] = ws(128)
    return sizes


def _apply(lib, cin, nc, hc, wc, c, state, hs, ws_, p, s, nbytes):
    aws = _ws(nbytes)
    out = U.act_alloc(nc, hc, wc, c)
    kout = torch.full((nc + 1,), -7, dtype=torch.int32, device="cuda")
    rc = lib.wctb200_style_swap_apply(cin.data_ptr(), nc, hc, wc, c, state.data_ptr(), hs, ws_, p, s, 0.6, *TF, out.data_ptr(),
                                      kout.data_ptr(), aws.data_ptr(), aws.numel(), U.stream())
    if rc:
        return rc, None, None, None
    U.check_device()
    torch.cuda.synchronize()
    return rc, planes(out, nc, hc, wc, c), kout.cpu().numpy(), aws


# content h=w, style h=w per (patch, stride): 289 patches (cout_pad 320, BN 64) or 361 (384, BN 128)
GEOM = {(3, 1): (18, 19), (5, 2): (21, 41), (16, 1): (18, 32)}


@pytest.mark.parametrize("nc", [1, 3])
@pytest.mark.parametrize("ps", list(GEOM), ids=lambda v: "p%ds%d" % v)
@pytest.mark.parametrize("c", [64, 128, 256, 512])
def test_chunked_apply_is_byte_identical(c, ps, nc):
    p, s = ps
    hc, hs = GEOM[ps]
    lib = U.lib()
    rng = np.random.default_rng(c + 7 * p + nc)
    content = np.maximum(rng.standard_normal((nc, hc, hc, c)) + 0.3, 0).astype(np.float32)
    style = np.maximum(rng.standard_normal((1, hs, hs, c)) + 0.4, 0).astype(np.float32)
    cin, sin = U.act_from_numpy(content), U.act_from_numpy(style)
    state = _ws(lib.wctb200_style_swap_state_bytes(c, hs, hs, p, s))
    pws = _ws(lib.wctb200_style_swap_prepare_workspace_bytes(c, hs, hs, p, s))
    _capi.check(lib.wctb200_style_swap_prepare(sin.data_ptr(), hs, hs, c, p, s, *TF, state.data_ptr(), None, pws.data_ptr(),
                                               pws.numel(), U.stream()))
    SC.C = c                      # the layout hook of the scale test reads the module's channel count
    try:
        L = SC._layout(nc, hc, hc, hs, hs, p, s)
    finally:
        SC.C = 512
    cp = L["cout_pad"]
    bn = 128 if cp % 128 == 0 else 64
    full = lib.wctb200_style_swap_apply_workspace_bytes(c, nc, hc, hc, hs, hs, p, s)
    least = lib.wctb200_style_swap_apply_min_workspace_bytes(c, nc, hc, hc, hs, hs, p, s)
    sizes = _chunk_sizes(L, nc, hc, hc, bn)
    assert sizes["full"] == full and sizes["min"] == least
    ref_bits, ref_k = None, None
    for name, nbytes in sizes.items():
        rc, bits, k, aws = _apply(lib, cin, nc, hc, hc, c, state, hs, hs, p, s, nbytes)
        assert rc == 0, "%s: %s" % (name, U.lib().wctb200_last_error().decode())
        if ref_bits is None:
            ref_bits, ref_k = bits, k
            idx = aws[L["idx"]:L["idx"] + nc * L["ho"] * L["wo"] * 4].view(torch.int32).cpu().numpy()
            assert idx.min() >= 0 and idx.max() < L["n_patches"]
        else:
            assert_bits(bits, ref_bits, "C %d p%d s%d Nc %d: %s workspace vs full" % (c, p, s, nc, name))
            assert np.array_equal(k, ref_k), name + ": k_out"
    rc, _, _, _ = _apply(lib, cin, nc, hc, hc, c, state, hs, hs, p, s, least - 1)
    assert rc == EWS
    print("C %d p%d s%d Nc %d: %d patches, cout_pad %d, BN %d, %s" % (c, p, s, nc, L["n_patches"], cp, bn, sorted(sizes)))


@pytest.mark.parametrize("c,hwc,hws,chunk_tiles", [(256, (64, 64), (64, 64), 20), (128, (96, 96), (64, 64), 13)],
                         ids=["C256_64sq_3844_patches", "C128_96sq_map"])
def test_accuracy_at_finer_levels(c, hwc, hws, chunk_tiles):
    """The stage checks of the scale test on the one-chunk apply, then a chunked apply equal to it byte for byte."""
    SC.C = c
    try:
        r, res, (cin, sin) = SC._run_synthetic(1, hwc, hws, 3, 1, seed=c)
        L = r["L"]
        lib = U.lib()
        state = _ws(lib.wctb200_style_swap_state_bytes(c, hws[0], hws[1], 3, 1))
        pws = _ws(lib.wctb200_style_swap_prepare_workspace_bytes(c, hws[0], hws[1], 3, 1))
        _capi.check(lib.wctb200_style_swap_prepare(sin.data_ptr(), hws[0], hws[1], c, 3, 1, *TF, state.data_ptr(), None,
                                                   pws.data_ptr(), pws.numel(), U.stream()))
        bn = 128 if L["cout_pad"] % 128 == 0 else 64
        col = 2 * 2 * (hwc[0] + 2) * (hwc[1] + 2)
        nbytes = _align(L["scores"] + chunk_tiles * bn * col)
        chunks = math.ceil(L["cout_pad"] / (chunk_tiles * bn))
        assert chunks >= 3
        rc, bits, k, aws = _apply(lib, cin, 1, hwc[0], hwc[1], c, state, hws[0], hws[1], 3, 1, nbytes)
        assert rc == 0, U.lib().wctb200_last_error().decode()
        idx = aws[L["idx"]:L["idx"] + L["ho"] * L["wo"] * 4].view(torch.int32).view(1, L["ho"], L["wo"]).cpu().numpy()
        assert np.array_equal(idx, r["idx"]), "chunked arg-max"
        assert_bits(bits, r["out_bits"], "%d chunks vs one" % chunks)
        assert np.array_equal(k, r["k"])
        print("C %d: %d patches in %d chunks of %d, band %d, output err %.2e" % (c, r["n_patches"], chunks, chunk_tiles * bn,
                                                                                res[0][2], res[0][1]))
    finally:
        SC.C = 512


# ------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def weights():
    return make_synthetic_weights(42)


@pytest.fixture(scope="module")
def wct(weights):
    return WCT(relu_targets=ALL, weights=weights)


def _imgs(n, h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, h, w, 3), dtype=np.uint8)


def test_engine_relu3_1_512_default_policy_equals_one_chunk(weights, monkeypatch):
    eng = Engine(weights, ALL, semantics="tf")
    lib = eng.lib
    full = lib.wctb200_style_swap_apply_workspace_bytes(256, 1, 128, 128, 128, 128, 3, 1)
    SC.C = 256
    try:
        L = SC._layout(1, 128, 128, 128, 128, 3, 1)
    finally:
        SC.C = 512
    col = 2 * 2 * 130 * 130
    cols = (engine_mod.SWAP_WORKSPACE_BYTES - L["scores"]) // col // 64 * 64
    assert full > engine_mod.SWAP_WORKSPACE_BYTES and math.ceil(L["cout_pad"] / cols) == 2
    c = torch.from_numpy(_imgs(1, 512, 512, 5)).cuda()
    s = torch.from_numpy(_imgs(1, 512, 512, 6)).cuda()
    two = eng.to_u8(eng.stylize(c, s, alpha=0.8, swap_targets=["relu3_1"]))
    monkeypatch.setattr(engine_mod, "SWAP_WORKSPACE_BYTES", full)
    one = eng.to_u8(eng.stylize(c, s, alpha=0.8, swap_targets=["relu3_1"]))
    eng.check_device()
    assert torch.equal(one, two)


@pytest.mark.parametrize("prepared", [False, True])
def test_swap_targets_relu5_1_is_swap5(wct, prepared):
    c, s = _imgs(3, 256, 256, 1), _imgs(1, 256, 256, 2)
    st = wct.prepare_style(s[0]) if prepared else s
    a = wct.predict_batch(c, st, swap5=True, ss_alpha=0.6, alpha=0.8)
    b = wct.predict_batch(c, st, swap_targets=["relu5_1"], ss_alpha=0.6, alpha=0.8)
    assert np.array_equal(a, b)


def _teacher_forced(weights, swap, csize=256, ssize=256, alpha=0.8, ss_alpha=0.6):
    """Every level of one engine run against the oracle on the device's own level input; at a swap level the oracle pastes
    the device's patches, which a direct C-ABI prepare + apply on the captured features (byte-equal to the engine's level)
    reads back."""
    eng = Engine(weights, ALL, semantics="tf")
    content, style = _imgs(1, csize, csize, 1000), _imgs(1, ssize, ssize, 7)
    d_style = torch.from_numpy(style).cuda()
    cap = {}
    eng.stylize(torch.from_numpy(content).cuda(), d_style, alpha=alpha, want_info=True, capture=cap, swap_targets=swap,
                ss_alpha=ss_alpha)
    eng.check_device()
    ps = eng.prepare_call(d_style, swap_targets=swap)
    torch.cuda.synchronize()
    sfe = nets.encode(nets.preprocess(style).astype(np.float64), weights, ALL, np.float64)
    worst = 0.0
    for i, relu in enumerate(ALL):
        x = cap["level_input"][i].cpu().numpy().astype(np.float64)
        cfo = nets.encode(x, weights, [relu], np.float64)[relu]
        e_enc = np.abs(eng.act_to_f32(cap["content_feat"][i]).cpu().numpy() - cfo).max()
        k = eng.last_info[i].cpu().numpy()
        if relu in swap:
            cf, tf, sf = cap["content_feat"][i], cap["transformed"][i], ps.feats[relu]
            SC.C = cf.C
            try:
                r = SC.run_swap(cf.buf, sf.buf, 1, cf.H, cf.W, sf.H, sf.W, 3, 1, ss_alpha)
            finally:
                SC.C = 512
            nbytes = U.lib().wctb200_act_bytes(1, cf.H, cf.W, cf.C)
            assert_bits(r["out_bits"], planes(tf.buf[:nbytes], 1, cf.H, cf.W, cf.C), "engine %s vs the direct swap" % relu)
            f, info = ref_ops.wct_style_swap(cfo, sfe[relu], ss_alpha, 3, 1, return_info=True, idx=r["idx"][0])
        else:
            f, info = ref_ops.wct_tf(cfo, sfe[relu], alpha, return_info=True)
        assert (k[0], k[1]) == (info["k_c"], info["k_s"]), relu
        assert ref_ops.spectral_gap_ok(info["wc"]) and ref_ops.spectral_gap_ok(info["ws"]), "ill-posed vector"
        e_t = np.abs(eng.act_to_f32(cap["transformed"][i]).cpu().numpy() - f).max()
        y = nets.decode(np.asarray(f, dtype=np.float64), weights, relu, np.float64)
        if i < len(ALL) - 1:
            y = np.clip(y, 0, 1)
        e_out = np.abs(cap["level_output"][i].cpu().numpy() - y).max()
        print("swap %s, %s: encoder %.2e  transform %.2e  level output %.2e" % (swap, relu, e_enc, e_t, e_out))
        worst = max(worst, e_enc, e_t, e_out)
    return worst


@pytest.mark.parametrize("swap", [["relu3_1"], ["relu4_1", "relu3_1"]], ids=["relu3_1", "relu4_1+relu3_1"])
def test_teacher_forced_levels(weights, swap):
    assert _teacher_forced(weights, swap) <= GATE


def test_extended_oracle_runs_at_relu3_1(weights):
    """The extended oracle itself (tests/swap_levels_ref.py) at a small size: finite, and different from plain WCT."""
    c, s = _imgs(1, 64, 64, 3), _imgs(1, 64, 64, 4)
    a = pipeline_levels(c, s, weights, ALL, alpha=0.8, dtype=np.float64, swap_targets=["relu3_1"])
    b = nets.pipeline(c, s, weights, ALL, alpha=0.8, dtype=np.float64)
    assert np.isfinite(a).all() and np.abs(a - b).max() > 1e-3


def test_batch_passes_prepared_and_file(wct, tmp_path):
    c, s = _imgs(3, 256, 256, 11), _imgs(1, 256, 256, 12)
    sw = dict(swap_targets=["relu3_1"], ss_alpha=0.6, alpha=0.8)
    batch = wct.predict_batch(c, s, **sw)
    for i in range(3):
        assert np.array_equal(wct.predict_batch(c[i:i + 1], s, **sw)[0], batch[i]), "frame %d" % i
    two = wct.predict_batch(c, s, passes=2, **sw)
    by_hand = wct.predict_batch(wct.predict_batch(c, s, **sw), s, alpha=0.8)
    assert np.array_equal(two, by_hand)
    ps = wct.prepare_style(s[0], swap_targets=["relu3_1"])
    assert np.array_equal(wct.predict_batch(c, ps, **sw), batch)
    path = str(tmp_path / "s.wctstyle")
    ps.save(path)
    loaded = wct.load_style(path)
    assert set(loaded.feats) == {"relu5_1", "relu3_1"}
    assert np.array_equal(wct.predict_batch(c, loaded, **sw), batch)
    assert np.array_equal(wct.predict_batch(c, loaded, swap5=True, ss_alpha=0.6, alpha=0.8),
                          wct.predict_batch(c, s, swap5=True, ss_alpha=0.6, alpha=0.8))


def test_rejections(weights):
    wct = WCT(relu_targets=ALL, weights=weights)
    c, s = _imgs(1, 64, 64, 1), _imgs(1, 64, 64, 2)
    with pytest.raises(ValueError, match="swap5 or swap_targets"):
        wct.predict_batch(c, s, swap5=True, swap_targets=["relu3_1"])
    with pytest.raises(ValueError, match="relu6_1 is not a relu target"):
        wct.predict_batch(c, s, swap_targets=["relu6_1"])
    sub = WCT(relu_targets=["relu4_1", "relu2_1"], weights=make_synthetic_weights(42, relu_targets=["relu4_1", "relu2_1"]))
    with pytest.raises(ValueError, match="relu3_1 is not a relu target"):
        sub.predict_batch(c, s, swap_targets=["relu3_1"])
    with pytest.raises(ValueError, match="content_mask"):
        wct.predict_batch(c, [s[0]], swap_targets=["relu3_1"], content_mask=np.zeros((8, 8), np.uint8))
    with pytest.raises(ValueError, match="style_weights"):
        wct.predict_batch(c, [s[0], s[0]], swap_targets=["relu3_1"], style_weights=[1, 1])
    with pytest.raises(ValueError, match="swap_targets"):
        wct.predict(c[0], s[0], swap_targets=["relu3_1"], style_weights=[1])
    ps = wct.prepare_style(s[0])
    with pytest.raises(ValueError, match="no relu3_1 feature"):
        wct.predict_batch(c, ps, swap_targets=["relu3_1"])
    with pytest.raises(ValueError, match="relu6_1 is not a relu target"):
        wct.prepare_style(s[0], swap_targets=["relu6_1"])
    strided = WCT(relu_targets=ALL, weights=weights, ss_patch_size=3, ss_stride=2)
    with pytest.raises(ValueError, match="2 swap levels"):
        strided.predict_batch(c, s, swap_targets=["relu4_1", "relu3_1"])
    wide = WCT(relu_targets=ALL, weights=weights, ss_patch_size=5, ss_stride=2)
    with pytest.raises(ValueError, match="relu3_1.*8x8"):
        wide.predict_batch(_imgs(1, 8, 8, 3), s, swap_targets=["relu3_1"])
    eng = wct.engine
    d = torch.from_numpy(c).cuda()
    with pytest.raises(ValueError, match="swap5 / swap_targets"):
        eng.stylize(d, None, swap_targets=["relu3_1"], interp_styles=[torch.from_numpy(s).cuda()],
                    interp_weights=torch.ones(1, 1, device="cuda"))


def test_strided_single_level_refit(weights):
    """ss_stride 3 at relu3_1 of five levels: relu5_1 and relu4_1 decode a 70^2 content to 80^2, whose relu3_1 encoding
    (20) patch 3 / stride 3 does not tile; the content is cropped to 48^2 (encoding 12).  Patch 3 / stride 2 tiles no crop
    there (every size reaches relu3_1 as a multiple of 4)."""
    wct = WCT(relu_targets=ALL, weights=weights, ss_patch_size=3, ss_stride=3)
    c, s = _imgs(2, 70, 70, 21), _imgs(1, 64, 64, 22)
    out = wct.predict_batch(c, s, swap_targets=["relu3_1"], ss_alpha=0.6)
    assert out.shape[1:3] == (48, 48)
    assert np.array_equal(out[1], wct.predict_batch(c[1:], s, swap_targets=["relu3_1"], ss_alpha=0.6)[0])
    with pytest.raises(ValueError, match="relu3_1.*70x70"):
        WCT(relu_targets=ALL, weights=weights, ss_patch_size=3, ss_stride=2).predict_batch(c, s, swap_targets=["relu3_1"])
