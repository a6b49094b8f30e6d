"""The labelled style swap (DESIGN.md §3.3.13): each content anchor matched only to the style patches of its own label.

1. C-ABI, uniform labels: wctb200_style_swap_apply_labels equals wctb200_style_swap_apply byte for byte (output planes with
   the halo, k_out) at C in {64,128,256,512}, (P,S) in {(3,1),(5,2)}, Nc in {1,3}, at every workspace size the chunk test
   of test_gpu_swap_levels picks.
2. C-ABI, block labels (3 and 8 labels, the last absent from the style): every workspace size gives the same bytes; in one
   chunk idx is the first maximum of the device's own scores over the anchor's allowed patches (the unconstrained one for
   the absent label); against float64 the margin rule of test_gpu_style_swap_scale holds restricted to the allowed
   patches; the output is the oracle's at the device's indices within 1e-3.
3. Frame i of a three-frame labelled apply equals that frame alone, bit for bit.
4. Engine and API: uniform labels = no labels (relu5_1, relu3_1); a teacher-forced pipeline; shared style = per-frame
   styles and maps; prepared styles and .wctstyle files; passes; synthesize.
"""
import math

import numpy as np
import pytest
import torch

import tests.test_gpu_style_swap_scale as SC
from oracle import nets, ref_ops
from tests import gpu_util as U
from tests import swap_labels_ref as SLR
from tests.test_gpu_invariance import assert_bits, frame_copy, planes
from tests.test_gpu_swap_levels import GEOM, _apply, _chunk_sizes, _ws
from wct_tf_b200 import _capi
from wct_tf_b200.device_image import noise_u8
from wct_tf_b200.engine import Engine
from wct_tf_b200.wct import WCT
from wct_tf_b200.weights import make_synthetic_weights

pytestmark = pytest.mark.gpu
TF = (1e-8, 1e-5)
ALL = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]
GATE = 1e-3


def _blocks(h, w, labels, seed, cells=4):
    """A label map of h x w made of cells x cells random blocks, values drawn from ``labels``."""
    rng = np.random.default_rng(seed)
    grid = rng.choice(np.asarray(labels, np.uint8), (cells, cells))
    return np.ascontiguousarray(grid[np.arange(h) * cells // h][:, np.arange(w) * cells // w])


def _setup(c, p, s, nc, seed):
    hc, hs = GEOM[(p, s)]
    lib = U.lib()
    rng = np.random.default_rng(seed)
    content = np.maximum(rng.standard_normal((nc, hc, hc, c)) + 0.3, 0).astype(np.float32)
    style = np.maximum(rng.standard_normal((1, hs, hs, c)) + 0.4, 0).astype(np.float32)
    cin, sin = U.act_from_numpy(content), U.act_from_numpy(style)
    state = _ws(lib.wctb200_style_swap_state_bytes(c, hs, hs, p, s))
    pws = _ws(lib.wctb200_style_swap_prepare_workspace_bytes(c, hs, hs, p, s))
    _capi.check(lib.wctb200_style_swap_prepare(sin.data_ptr(), hs, hs, c, p, s, *TF, state.data_ptr(), None, pws.data_ptr(),
                                               pws.numel(), U.stream()))
    SC.C = c
    try:
        L = SC._layout(nc, hc, hc, hs, hs, p, s)
    finally:
        SC.C = 512
    return dict(lib=lib, hc=hc, hs=hs, cin=cin, sin=sin, state=state, L=L, content=content, style=style)


def _apply_labels(lib, cin, nc, hc, wc, c, state, hs, ws_, p, s, nbytes, cl, sl, alpha=0.6):
    """The labelled apply with ``nbytes`` of workspace; cl: cuda uint8 [Ncl,Hm,Wm], sl: cuda uint8 [Hm',Wm']."""
    assert cl.is_contiguous() and sl.is_contiguous()
    aws = _ws(nbytes)
    lbuf = _ws(lib.wctb200_style_swap_labels_workspace_bytes(cl.shape[0], hc, wc, hs, ws_, p, s))
    out = U.act_alloc(nc, hc, wc, c)
    kout = torch.full((nc + 1,), -7, dtype=torch.int32, device="cuda")
    rc = lib.wctb200_style_swap_apply_labels(cin.data_ptr(), nc, hc, wc, c, state.data_ptr(), hs, ws_, p, s, alpha, *TF,
                                             cl.data_ptr(), cl.shape[0], cl.shape[1], cl.shape[2], sl.data_ptr(), sl.shape[-2],
                                             sl.shape[-1], out.data_ptr(), kout.data_ptr(), aws.data_ptr(), aws.numel(),
                                             lbuf.data_ptr(), lbuf.numel(), U.stream())
    if rc:
        return rc, None, None, None
    U.check_device()
    torch.cuda.synchronize()
    return rc, planes(out, nc, hc, wc, c), kout.cpu().numpy(), aws


def _sizes(d, c, nc, p, s):
    bn = 128 if d["L"]["cout_pad"] % 128 == 0 else 64
    return _chunk_sizes(d["L"], nc, d["hc"], d["hc"], bn)


# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nc", [1, 3])
@pytest.mark.parametrize("ps", [(3, 1), (5, 2)], ids=lambda v: "p%ds%d" % v)
@pytest.mark.parametrize("c", [64, 128, 256, 512])
def test_uniform_labels_equal_the_plain_apply(c, ps, nc):
    p, s = ps
    d = _setup(c, p, s, nc, c + 3 * p + nc)
    hc, hs = d["hc"], d["hs"]
    # per-frame maps for three frames, one shared map for one; neither at the feature resolution
    cl = torch.full((nc, 2 * hc + 3, hc + 1), 9, dtype=torch.uint8, device="cuda")
    sl = torch.full((5, 7), 9, dtype=torch.uint8, device="cuda")
    for name, nbytes in _sizes(d, c, nc, p, s).items():
        rc, ref, kref, _ = _apply(d["lib"], d["cin"], nc, hc, hc, c, d["state"], hs, hs, p, s, nbytes)
        assert rc == 0
        rc, got, k, _ = _apply_labels(d["lib"], d["cin"], nc, hc, hc, c, d["state"], hs, hs, p, s, nbytes, cl, sl)
        assert rc == 0, d["lib"].wctb200_last_error().decode()
        assert_bits(got, ref, "C %d p%d s%d Nc %d %s: uniform labels vs unlabelled" % (c, p, s, nc, name))
        assert np.array_equal(k, kref), name + ": k_out"
    # a label buffer one byte short
    need = d["lib"].wctb200_style_swap_labels_workspace_bytes(nc, hc, hc, hs, hs, p, s)
    out = U.act_alloc(nc, hc, hc, c)
    aws, lbuf = _ws(_sizes(d, c, nc, p, s)["full"]), _ws(need - 1)
    rc = d["lib"].wctb200_style_swap_apply_labels(d["cin"].data_ptr(), nc, hc, hc, c, d["state"].data_ptr(), hs, hs, p, s, 0.6,
                                                  *TF, cl.data_ptr(), nc, cl.shape[1], cl.shape[2], sl.data_ptr(), 5, 7,
                                                  out.data_ptr(), None, aws.data_ptr(), aws.numel(), lbuf.data_ptr(),
                                                  lbuf.numel(), U.stream())
    assert rc == _capi.EWS


def _restricted_margin_check(d, c, p, s, i, idx, allowed, alpha):
    """test_gpu_style_swap_scale's rule (c) restricted to each anchor's allowed patches, and the oracle's output at the
    device's indices.  Returns (band size, output error)."""
    L = d["L"]
    npat, K = L["n_patches"], p * p * c
    nbw = 2 * L["cout_pad"] * K * 2
    wsplit = d["state"][L["wsplit"]:L["wsplit"] + nbw].view(torch.float16).view(2, L["cout_pad"], K).cpu().numpy()
    W = wsplit[0, :npat].astype(np.float64) + wsplit[1, :npat].astype(np.float64)
    absW = np.abs(W)
    wc_pl = d["wc_feat"]
    X = SC._windows(wc_pl[0, i].astype(np.float64)[1:-1, 1:-1] + wc_pl[1, i].astype(np.float64)[1:-1, 1:-1], p, s)
    eb = 2.0 ** -16 + math.ceil(K / 128) * 2.0 ** -24
    shat = X @ W.T
    bound = eb * (np.abs(X) @ absW.T) + 2.0 ** -22 * np.abs(shat)
    c64, s64 = U.split_repr(d["content"][i:i + 1]), U.split_repr(d["style"])
    ref, info = ref_ops.wct_style_swap(c64, s64, alpha, p, s, return_info=True, idx=idx.reshape(L["ho"], L["wo"]))
    assert ref_ops.spectral_gap_ok(info["wc"]) and ref_ops.spectral_gap_ok(info["ws"]), "ill-posed vector"
    Xo, Po = SC._windows(info["wc_feat"][0], p, s), SC._windows(info["ws_feat"][0], p, s)
    Wo = Po / np.sqrt(np.maximum((Po ** 2).sum(0, keepdims=True), 1e-12))
    so = Xo @ Wo.T
    delta = (np.abs(X - Xo) @ absW.T + np.abs(Xo) @ np.abs(W - Wo).T + bound).max(axis=1)
    som = np.where(allowed, so, -np.inf)
    top2 = np.sort(som, axis=1)[:, -2:]
    best, margin = top2[:, 1], top2[:, 1] - top2[:, 0]
    decided = margin > 2 * delta
    assert np.array_equal(idx[decided], som.argmax(axis=1)[decided]), "a decided anchor chose another allowed patch"
    assert allowed[np.arange(len(idx)), idx].all(), "an anchor took a patch outside its allowed set"
    assert (so[np.arange(len(idx)), idx] >= best - 2 * delta).all(), "the chosen patch scores below the band"
    out = d["out_bits"][:, i].astype(np.int16).view(np.float16).astype(np.float64)
    e_out = float(np.abs((out[0] + out[1])[1:-1, 1:-1] - ref[0]).max())
    assert e_out <= GATE, "output %.2e from the oracle at the device's indices" % e_out
    return int((~decided).sum()), e_out


@pytest.mark.parametrize("k", [3, 8])
@pytest.mark.parametrize("ps", [(3, 1), (5, 2)], ids=lambda v: "p%ds%d" % v)
@pytest.mark.parametrize("c", [128, 512])
def test_block_labels(c, ps, k):
    p, s = ps
    nc = 3
    d = _setup(c, p, s, nc, 100 * k + c + p)
    L, hc, hs, lib = d["L"], d["hc"], d["hs"], d["lib"]
    ho, wo, npat = L["ho"], L["wo"], L["n_patches"]
    cl_np = np.stack([_blocks(3 * hc, 3 * hc, range(k), 10 * k + i) for i in range(nc)])
    sl_np = _blocks(2 * hs + 1, 2 * hs + 1, range(k - 1), 7 * k, cells=5)          # label k - 1 is absent from the style
    cl, sl = torch.from_numpy(cl_np).cuda(), torch.from_numpy(sl_np).cuda()
    sizes = _sizes(d, c, nc, p, s)
    ref = None
    for name, nbytes in sizes.items():
        rc, bits, kk, aws = _apply_labels(lib, d["cin"], nc, hc, hc, c, d["state"], hs, hs, p, s, nbytes, cl, sl)
        assert rc == 0, lib.wctb200_last_error().decode()
        if ref is None:
            assert name == "full"
            ref, kref, full_ws = bits, kk, aws
        else:
            assert_bits(bits, ref, "C %d p%d s%d k %d: %s workspace vs one chunk" % (c, p, s, k, name))
            assert np.array_equal(kk, kref)
    idx = full_ws[L["idx"]:L["idx"] + nc * ho * wo * 4].view(torch.int32).view(nc, ho * wo).cpu().numpy()
    assert idx.min() >= 0 and idx.max() < npat
    SC.C = c
    try:
        scores = SC._fp16_planes(full_ws, L["scores"], nc, hc, hc, L["cout_pad"])
        d["wc_feat"] = SC._fp16_planes(full_ws, L["wc_feat"], nc, hc, hc, c)
    finally:
        SC.C = 512
    d["out_bits"] = ref
    plab = SLR.patch_labels(sl_np, hs, hs, p, s)
    assert len(plab) == npat
    for i in range(nc):
        alab = SLR.anchor_labels(cl_np[i], hc, hc, p, s).reshape(-1)
        allowed = SLR.allowed(alab[None], plab)[0]
        sd = SC._merge32(scores[:, i])[1:1 + (ho - 1) * s + 1:s, 1:1 + (wo - 1) * s + 1:s].reshape(ho * wo, -1)[:, :npat]
        assert np.array_equal(idx[i], np.where(allowed, sd, -np.inf).argmax(axis=1)), "frame %d: masked first maximum" % i
        absent = ~np.isin(alab, plab)
        assert absent.any() and (~absent).any()
        assert np.array_equal(idx[i][absent], sd[absent].argmax(axis=1)), "frame %d: absent label" % i
        band, e_out = _restricted_margin_check(d, c, p, s, i, idx[i], allowed, 0.6)
        print("C %d p%d s%d %d labels frame %d: %d patches, %d anchors (%d absent), band %d, output err %.2e"
              % (c, p, s, k, i, npat, ho * wo, int(absent.sum()), band, e_out))


def test_frame_alone_equals_batched():
    c, p, s, nc = 256, 3, 1, 3
    d = _setup(c, p, s, nc, 5)
    hc, hs, lib = d["hc"], d["hs"], d["lib"]
    cl_np = np.stack([_blocks(40, 30, range(4), i) for i in range(nc)])
    cl, sl = torch.from_numpy(cl_np).cuda(), torch.from_numpy(_blocks(19, 19, range(3), 9)).cuda()
    full = lib.wctb200_style_swap_apply_workspace_bytes(c, nc, hc, hc, hs, hs, p, s)
    rc, bits, k, _ = _apply_labels(lib, d["cin"], nc, hc, hc, c, d["state"], hs, hs, p, s, full, cl, sl)
    assert rc == 0
    one = lib.wctb200_style_swap_apply_workspace_bytes(c, 1, hc, hc, hs, hs, p, s)
    for i in range(nc):
        rc, b1, k1, _ = _apply_labels(lib, frame_copy(d["cin"], i, nc, hc, hc, c), 1, hc, hc, c, d["state"], hs, hs, p, s, one,
                                      cl[i:i + 1].contiguous(), sl)
        assert rc == 0
        assert_bits(b1[:, 0], bits[:, i], "labelled apply frame %d alone vs batched" % i)
        assert (k1[0], k1[1]) == (k[i], k[nc])


# ------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def weights():
    return make_synthetic_weights(42)


@pytest.fixture(scope="module")
def wct(weights):
    return WCT(relu_targets=ALL, weights=weights)


def _imgs(n, h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, h, w, 3), dtype=np.uint8)


@pytest.mark.parametrize("swap", [dict(swap5=True), dict(swap_targets=["relu3_1"])], ids=["relu5_1", "relu3_1"])
def test_uniform_labels_equal_no_labels(wct, swap):
    c, s = _imgs(3, 256, 256, 1), _imgs(1, 256, 256, 2)
    kw = dict(swap, ss_alpha=0.6, alpha=0.8)
    ref = wct.predict_batch(c, s, **kw)
    got = wct.predict_batch(c, s, swap_labels=(np.full((64, 48), 4, np.uint8), np.full((9, 9), 4, np.uint8)), **kw)
    assert np.array_equal(got, ref)
    # every content label absent from the style: every anchor may take every patch
    got = wct.predict_batch(c, s, swap_labels=(np.full((3, 5, 5), 1, np.uint8), _blocks(30, 30, [0, 2, 3], 1)), **kw)
    assert np.array_equal(got, ref)


def test_teacher_forced_pipeline(weights):
    """Every level of one engine run against the oracle on the device's level input; the relu3_1 swap equals a direct
    labelled C-ABI apply on the captured features, takes only allowed patches, and the oracle evaluated at its indices."""
    eng = Engine(weights, ALL, semantics="tf")
    content, style = _imgs(1, 256, 256, 1000), _imgs(1, 256, 256, 7)
    cl_np, sl_np = _blocks(256, 256, range(4), 1), _blocks(256, 256, range(3), 2)
    d_style = torch.from_numpy(style).cuda()
    lab = (torch.from_numpy(cl_np).cuda(), torch.from_numpy(sl_np).cuda())
    cap = {}
    eng.stylize(torch.from_numpy(content).cuda(), d_style, alpha=0.8, want_info=True, capture=cap, swap_targets=["relu3_1"],
                ss_alpha=0.6, swap_labels=lab)
    eng.check_device()
    ps = eng.prepare_call(d_style, swap_targets=["relu3_1"])
    torch.cuda.synchronize()
    sfe = nets.encode(nets.preprocess(style).astype(np.float64), weights, ALL, np.float64)
    worst = 0.0
    for i, relu in enumerate(ALL):
        x = cap["level_input"][i].cpu().numpy().astype(np.float64)
        cfo = nets.encode(x, weights, [relu], np.float64)[relu]
        k = eng.last_info[i].cpu().numpy()
        if relu == "relu3_1":
            cf, tf, sf = cap["content_feat"][i], cap["transformed"][i], ps.feats[relu]
            lib = U.lib()
            state = _ws(lib.wctb200_style_swap_state_bytes(cf.C, sf.H, sf.W, 3, 1))
            pws = _ws(lib.wctb200_style_swap_prepare_workspace_bytes(cf.C, sf.H, sf.W, 3, 1))
            _capi.check(lib.wctb200_style_swap_prepare(sf.ptr, sf.H, sf.W, cf.C, 3, 1, *TF, state.data_ptr(), None,
                                                       pws.data_ptr(), pws.numel(), U.stream()))
            full = lib.wctb200_style_swap_apply_workspace_bytes(cf.C, 1, cf.H, cf.W, sf.H, sf.W, 3, 1)
            rc, bits, _, aws = _apply_labels(lib, cf.buf, 1, cf.H, cf.W, cf.C, state, sf.H, sf.W, 3, 1, full, lab[0][None],
                                             lab[1])
            assert rc == 0
            nbytes = lib.wctb200_act_bytes(1, cf.H, cf.W, cf.C)
            assert_bits(bits, planes(tf.buf[:nbytes], 1, cf.H, cf.W, cf.C), "engine relu3_1 vs the direct labelled apply")
            SC.C = cf.C
            try:
                L = SC._layout(1, cf.H, cf.W, sf.H, sf.W, 3, 1)
            finally:
                SC.C = 512
            idx = aws[L["idx"]:L["idx"] + L["ho"] * L["wo"] * 4].view(torch.int32).view(L["ho"], L["wo"]).cpu().numpy()
            alab = SLR.anchor_labels(cl_np, cf.H, cf.W, 3, 1)
            plab = SLR.patch_labels(sl_np, sf.H, sf.W, 3, 1)
            assert SLR.allowed(alab, plab)[np.arange(L["ho"])[:, None], np.arange(L["wo"])[None], idx].all()
            f, info = ref_ops.wct_style_swap(cfo, sfe[relu], 0.6, 3, 1, return_info=True, idx=idx)
        else:
            f, info = ref_ops.wct_tf(cfo, sfe[relu], 0.8, return_info=True)
        assert (k[0], k[1]) == (info["k_c"], info["k_s"]), relu
        e_t = np.abs(eng.act_to_f32(cap["transformed"][i]).cpu().numpy() - f).max()
        y = nets.decode(np.asarray(f, dtype=np.float64), weights, relu, np.float64)
        if i < len(ALL) - 1:
            y = np.clip(y, 0, 1)
        e_out = np.abs(cap["level_output"][i].cpu().numpy() - y).max()
        print("labelled swap relu3_1, %s: transform %.2e  level output %.2e" % (relu, e_t, e_out))
        worst = max(worst, e_t, e_out)
    assert worst <= GATE


def test_shared_style_equals_per_frame_styles_and_maps(wct):
    c, s = _imgs(3, 256, 256, 11), _imgs(1, 256, 256, 12)
    cl = np.stack([_blocks(256, 256, range(5), 20 + i) for i in range(3)])
    sl = _blocks(128, 128, range(4), 30)
    kw = dict(swap_targets=["relu3_1"], ss_alpha=0.6, alpha=0.8)
    shared = wct.predict_batch(c, s, swap_labels=(cl, sl), **kw)
    per = wct.predict_batch(c, np.concatenate([s] * 3), swap_labels=(cl, np.stack([sl] * 3)), **kw)
    assert np.array_equal(shared, per)
    for i in range(3):
        assert np.array_equal(wct.predict_batch(c[i:i + 1], s, swap_labels=(cl[i], sl), **kw)[0], shared[i]), "frame %d" % i
    free = wct.predict_batch(c, s, **kw)
    assert not np.array_equal(shared, free)
    # per-frame style maps: frame 1 with another map differs from the shared-map call there only
    sl2 = np.stack([sl, _blocks(128, 128, range(4), 31), sl])
    mixed = wct.predict_batch(c, np.concatenate([s] * 3), swap_labels=(cl, sl2), **kw)
    assert np.array_equal(mixed[0], shared[0]) and np.array_equal(mixed[2], shared[2])
    assert np.array_equal(mixed[1], wct.predict_batch(c[1:2], s, swap_labels=(cl[1], sl2[1]), **kw)[0])


def test_prepared_file_and_passes(wct, tmp_path):
    c, s = _imgs(2, 256, 256, 21), _imgs(1, 256, 256, 22)
    lab = (_blocks(256, 256, range(3), 3), _blocks(256, 256, range(3), 4))
    kw = dict(swap_targets=["relu3_1"], ss_alpha=0.6, alpha=0.8)
    ref = wct.predict_batch(c, s, swap_labels=lab, **kw)
    ps = wct.prepare_style(s[0], swap_targets=["relu3_1"])
    assert np.array_equal(wct.predict_batch(c, ps, swap_labels=lab, **kw), ref)
    path = str(tmp_path / "s.wctstyle")
    ps.save(path)
    assert np.array_equal(wct.predict_batch(c, wct.load_style(path), swap_labels=lab, **kw), ref)
    d_lab = tuple(torch.from_numpy(t).cuda() for t in lab)                 # device maps too
    assert np.array_equal(wct.predict_batch(c, s, swap_labels=d_lab, **kw), ref)
    two = wct.predict_batch(c, s, passes=2, swap_labels=lab, **kw)
    assert np.array_equal(two, wct.predict_batch(ref, s, alpha=0.8))
    assert np.array_equal(wct.predict(c[0], s[0], swap_labels=lab, **kw), ref[0])


def test_synthesize_equals_predict_batch_on_noise(wct):
    s = _imgs(1, 256, 256, 31)
    lab = (_blocks(128, 192, range(3), 5), _blocks(256, 256, range(3), 6))
    kw = dict(swap_targets=["relu4_1", "relu3_1"], ss_alpha=0.6, alpha=0.8, swap_labels=lab)
    got = wct.synthesize(s, (256, 384), count=2, seed=3, **kw)
    ref = wct.predict_batch(noise_u8(2, 256, 384, seed=3, device=wct.engine.device), s, **kw)
    assert np.array_equal(got, ref)
