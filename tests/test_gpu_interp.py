"""Style interpolation on the GPU: the blend entry points against wct_apply / adain_level (byte identity on one-hot rows),
per-frame rows and the five-level pipeline against the fp64 output-level oracle (tests/interp_ref.py), the reference-code
fixture, argument checks, and the Python / video front ends."""
import os

import numpy as np
import pytest
import torch
from PIL import Image

import tests.gpu_util as U
from oracle import nets, ref_ops
from tests.interp_ref import adain_interp, level_interp, pipeline_interp, wct_interp
from tests.test_gpu_pipeline import ALL, FREE_RUN_NOISE_FACTOR
from tests.test_gpu_regions import _feats, _prepare
from wct_tf_b200 import _capi
from wct_tf_b200.engine import Engine, SEMANTICS
from wct_tf_b200.weights import make_synthetic_weights
from wct_tf_b200.wct import WCT

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "interp_wct_np_c128_a08.npz")


@pytest.fixture(scope="module")
def weights():
    return make_synthetic_weights(42)


def _apply(cin, shape, state, alpha, sem="tf"):
    lib = U.lib()
    nc, hc, wc, c = shape
    sp = SEMANTICS[sem]
    out = torch.zeros(lib.wctb200_act_bytes(nc, hc, wc, c), dtype=torch.uint8, device="cuda")
    ws = torch.empty(lib.wctb200_wct_workspace_bytes(c, nc, 0), dtype=torch.uint8, device="cuda")
    kbuf = torch.zeros(2 * (nc + 1), dtype=torch.int32, device="cuda")
    _capi.check(lib.wctb200_wct_apply(cin.data_ptr(), nc, hc, wc, c, state.data_ptr(), 1, alpha, sp["eps_cov"], sp["eps_eig"],
                                      sp["thresh"], sp["readd"], out.data_ptr(), kbuf.data_ptr(), ws.data_ptr(), ws.numel(),
                                      U.stream()))
    U.check_device()
    return out, kbuf.cpu().numpy()


def _blend(cin, shape, states, w, alpha, sem="tf", K=None, ws_k=None):
    lib = U.lib()
    nc, hc, wc, c = shape
    w = np.asarray(w, np.float32)
    K = len(states) if K is None else K
    sp = SEMANTICS[sem]
    out = torch.zeros(lib.wctb200_act_bytes(nc, hc, wc, c), dtype=torch.uint8, device="cuda")
    nbytes = lib.wctb200_wct_blend_workspace_bytes(c, nc, ws_k or K, w.shape[0]) or lib.wctb200_wct_blend_workspace_bytes(c, nc, 8, nc)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    kbuf = torch.zeros(2 * (nc + max(K, 1)), dtype=torch.int32, device="cuda")
    wd = U.dev(w)
    _capi.check(lib.wctb200_wct_apply_blend(cin.data_ptr(), nc, hc, wc, c, _capi.pointer_array([s.data_ptr() if s is not None else 0
                                                                                               for s in states]),
                                            K, wd.data_ptr(), w.shape[0], alpha, sp["eps_cov"], sp["eps_eig"], sp["thresh"],
                                            sp["readd"], out.data_ptr(), kbuf.data_ptr(), ws.data_ptr(), ws.numel(), U.stream()))
    U.check_device()
    return out, kbuf.cpu().numpy()


def _adain_level(cin, shape, style, alpha):
    lib = U.lib()
    nc, hc, wc, c = shape
    sin = U.act_from_numpy(style)
    out = torch.zeros(lib.wctb200_act_bytes(nc, hc, wc, c), dtype=torch.uint8, device="cuda")
    ws = torch.empty(lib.wctb200_wct_workspace_bytes(c, nc, 1), dtype=torch.uint8, device="cuda")
    _capi.check(lib.wctb200_adain_level(cin.data_ptr(), nc, hc, wc, sin.data_ptr(), 1, style.shape[1], style.shape[2], c, alpha,
                                        1e-5, out.data_ptr(), ws.data_ptr(), ws.numel(), U.stream()))
    U.check_device()
    return out


def _adain_blend(cin, shape, styles, w, alpha, K=None, null=None):
    lib = U.lib()
    nc, hc, wc, c = shape
    w = np.asarray(w, np.float32)
    K = len(styles) if K is None else K
    sins = [U.act_from_numpy(s) for s in styles]
    ptrs = [s.data_ptr() for s in sins]
    if null is not None:
        ptrs[null] = 0
    out = torch.zeros(lib.wctb200_act_bytes(nc, hc, wc, c), dtype=torch.uint8, device="cuda")
    ws = torch.empty(lib.wctb200_adain_blend_workspace_bytes(c, nc, 8), dtype=torch.uint8, device="cuda")
    wd = U.dev(w)
    _capi.check(lib.wctb200_adain_blend(cin.data_ptr(), nc, hc, wc, c, _capi.pointer_array(ptrs),
                                        _capi.int_array([s.shape[1] for s in styles]), _capi.int_array([s.shape[2] for s in styles]),
                                        K, wd.data_ptr(), w.shape[0], alpha, 1e-5, out.data_ptr(), ws.data_ptr(), ws.numel(),
                                        U.stream()))
    U.check_device()
    return out


def _frame(buf, shape, n):
    """bytes of frame n (both planes, halo included) of an SPF16 buffer"""
    nc, hc, wc, c = shape
    return buf.view(torch.int16).view(2, nc, hc + 2, wc + 2, c)[:, n]


STYLE_SHAPES = [(1, 14, 20), (1, 11, 9), (1, 16, 16)]


# ---------------------------------------------------------------------------------------------------------- byte identity
@pytest.mark.parametrize("nc", [1, 3])
@pytest.mark.parametrize("c", [64, 128, 256, 512])
def test_one_hot_blend_is_byte_identical_to_wct_apply(c, nc):
    shape = (nc, 12, 20, c)
    content = _feats(shape, c + nc)
    styles = [_feats(s + (c,), 10 + i) for i, s in enumerate(STYLE_SHAPES)]
    states = [_prepare(s) for s in styles]
    cin = U.act_from_numpy(content)
    refs = [_apply(cin, shape, st, 0.7) for st in states]
    out, k = _blend(cin, shape, states[:1], [[1.0]], 0.7)                      # K = 1, weight 1
    assert torch.equal(out, refs[0][0])
    assert np.array_equal(k, refs[0][1])
    for j in range(3):                                                         # one shared one-hot row among K = 3
        out, k = _blend(cin, shape, states, [np.eye(3)[j]], 0.7)
        assert torch.equal(out, refs[j][0]), j
        assert np.array_equal(k[:nc], refs[j][1][:nc]) and k[nc + j] == refs[j][1][nc]
    if nc == 3:                                                                # per-frame one-hot rows
        pick = [2, 0, 1]
        out, k = _blend(cin, shape, states, np.eye(3)[pick], 0.7)
        for n, j in enumerate(pick):
            assert torch.equal(_frame(out, shape, n), _frame(refs[j][0], shape, n)), n


@pytest.mark.parametrize("nc", [1, 3])
@pytest.mark.parametrize("c", [64, 128, 256, 512])
def test_one_hot_adain_blend_is_byte_identical_to_adain_level(c, nc):
    shape = (nc, 12, 20, c)
    rng = np.random.default_rng(c * nc)
    content = np.maximum(rng.normal(0.5, 1, shape), 0).astype(np.float32)
    styles = [np.maximum(rng.normal(0.2 * i, 1 + i, s + (c,)), 0).astype(np.float32) for i, s in enumerate(STYLE_SHAPES)]
    cin = U.act_from_numpy(content)
    refs = [_adain_level(cin, shape, s, 0.6) for s in styles]
    assert torch.equal(_adain_blend(cin, shape, styles[:1], [[1.0]], 0.6), refs[0])
    for j in range(3):
        assert torch.equal(_adain_blend(cin, shape, styles, [np.eye(3)[j]], 0.6), refs[j]), j
    if nc == 3:
        pick = [1, 2, 0]
        out = _adain_blend(cin, shape, styles, np.eye(3)[pick], 0.6)
        for n, j in enumerate(pick):
            assert torch.equal(_frame(out, shape, n), _frame(refs[j], shape, n)), n


# ---------------------------------------------------------------------------------------------------------- accuracy
@pytest.mark.parametrize("sem", ["tf", "np", "adain"])
def test_per_frame_rows_match_float64_oracle(sem):
    c = 128
    shape = (3, 16, 16, c)
    content = _feats(shape, 7)
    styles = [_feats(s + (c,), 20 + i) for i, s in enumerate([(1, 14, 20), (1, 18, 16), (1, 20, 20)])]
    rows = np.random.default_rng(5).dirichlet(np.ones(3), size=3).astype(np.float32)
    cin = U.act_from_numpy(content)
    if sem == "adain":
        out = _adain_blend(cin, shape, styles, rows, 0.8)
    else:
        out, k = _blend(cin, shape, [_prepare(s, sem) for s in styles], rows, 0.8, sem)
    got = U.act_to_numpy(out, *shape)
    s64 = [U.split_repr(s) for s in styles]
    for n in range(3):
        c64 = U.split_repr(content[n:n + 1])
        w = rows[n].astype(np.float64)
        if sem == "adain":
            ref = adain_interp(c64, s64, w, 0.8)
            assert np.abs(got[n:n + 1] - ref).max() <= 2e-5 * (1 + np.abs(ref).max())
            continue
        ref, infos = wct_interp(c64, s64, w, 0.8, sem, return_info=True)
        for j, inf in enumerate(infos):
            assert ref_ops.spectral_gap_ok(inf["wc"]) and ref_ops.spectral_gap_ok(inf["ws"])
            assert k[n] == inf["k_c"] and k[3 + j] == inf["k_s"]
        err = np.abs(got[n:n + 1] - ref).max()
        print("%s frame %d: max-abs vs fp64 output-level oracle %.2e" % (sem, n, err))
        assert err <= 1e-3


def test_blend_vs_reference_golden():
    g = np.load(GOLDEN)
    content, styles = g["content"], [s[None] for s in g["styles"]]
    shape = content.shape
    states = [_prepare(s, "np") for s in styles]
    out, k = _blend(U.act_from_numpy(content), shape, states, [g["weights"]], float(g["alpha"]), "np")
    got = U.act_to_numpy(out, *shape)
    assert k[0] == int(g["k_c"]) and list(k[1:4]) == list(g["k_s"])
    e32, e64 = np.abs(got - g["out_ref_fp32"]).max(), np.abs(got - g["out_ref_fp64"]).max()
    print("max-abs vs reference interpolation fp32 %.2e, fp64 %.2e" % (e32, e64))
    assert e32 <= 1e-3 and e64 <= 1e-3


def test_bad_arguments_are_rejected():
    c = 64
    shape = (3, 8, 8, c)
    cin = U.act_from_numpy(_feats(shape, 1))
    state = _prepare(_feats((1, 8, 8, c), 2))
    styles = [_feats((1, 8, 8, c), 3)] * 9
    for states, w, K in (([], np.ones((1, 1)), 0), ([state] * 9, np.ones((1, 9)) / 9, 9), ([state] * 2, np.ones((2, 2)) / 2, 2),
                         ([state, None], np.ones((1, 2)) / 2, 2)):
        with pytest.raises(_capi.WctB200Error):
            _blend(cin, shape, states, w, 1.0, K=K, ws_k=8)
    for sts, w, K, null in ((styles[:1], np.ones((1, 1)), 0, None), (styles, np.ones((1, 9)) / 9, 9, None),
                            (styles[:2], np.ones((2, 2)) / 2, 2, None), (styles[:2], np.ones((1, 2)) / 2, 2, 1)):
        with pytest.raises(_capi.WctB200Error):
            _adain_blend(cin, shape, sts, w, 1.0, K=K, null=null)


# ---------------------------------------------------------------------------------------------------------- pipeline
def _teacher_forced_interp(weights, sem, csize, ssizes, w, alpha=0.8, seed=100):
    adain = sem == "adain"
    eng = Engine(weights, ALL, semantics="tf" if adain else sem)
    rng = np.random.default_rng(seed)
    content = rng.integers(0, 256, (1, csize, csize, 3), dtype=np.uint8)
    styles = [rng.integers(0, 256, (1, s, s, 3), dtype=np.uint8) for s in ssizes]
    w32 = np.asarray([w], np.float32)
    cap = {}
    out = eng.stylize(torch.from_numpy(content).cuda(), None, alpha=alpha, adain=adain, want_info=True, capture=cap,
                      interp_styles=[torch.from_numpy(s).cuda() for s in styles], interp_weights=torch.from_numpy(w32).cuda())
    eng.check_device()
    sfe = [nets.encode(nets.preprocess(s).astype(np.float64), weights, ALL, np.float64) for s in styles]
    worst = 0.0
    for i, relu in enumerate(ALL):
        x = cap["level_input"][i].cpu().numpy().astype(np.float64)
        cf = nets.encode(x, weights, [relu], np.float64)[relu]
        e_enc = np.abs(eng.act_to_f32(cap["content_feat"][i]).cpu().numpy() - cf).max()
        f, infos = level_interp(cf, [s[relu] for s in sfe], w32[0].astype(np.float64), alpha, sem, adain, return_info=True)
        if not adain:
            k = eng.last_info[i].cpu().numpy()
            for j, inf in enumerate(infos):
                assert ref_ops.spectral_gap_ok(inf["wc"]) and ref_ops.spectral_gap_ok(inf["ws"]), (relu, j)
                assert k[0] == inf["k_c"] and k[1 + j] == inf["k_s"], (relu, j, k, inf["k_c"], inf["k_s"])
        e_f = np.abs(eng.act_to_f32(cap["transformed"][i]).cpu().numpy() - f).max()
        y = nets.decode(np.asarray(f, dtype=np.float64), weights, relu, np.float64)
        if i < len(ALL) - 1:
            y = np.clip(y, 0, 1)
        e_out = np.abs(cap["level_output"][i].cpu().numpy() - y).max()
        print("%s %dx%d K=%d %s: encoder %.2e  transform %.2e  level output %.2e" % (relu, csize, csize, len(ssizes), sem, e_enc,
                                                                                    e_f, e_out))
        worst = max(worst, e_enc, e_f, e_out)
    assert out.shape == (1, csize, csize, 3)
    return worst


@pytest.mark.parametrize("sem", ["tf", "np", "adain"])
def test_teacher_forced_interp_128(weights, sem):
    assert _teacher_forced_interp(weights, sem, 128, [144, 96, 112], [0.5, 0.3, 0.2]) <= 1e-3


def test_teacher_forced_interp_512_tf(weights):
    assert _teacher_forced_interp(weights, "tf", 512, [512, 384], [0.35, 0.65], seed=1000) <= 1e-3


def test_free_running_interp_vs_oracle(weights):
    size = 128
    rng = np.random.default_rng(1000)
    content = rng.integers(0, 256, (1, size, size, 3), dtype=np.uint8)
    styles = [rng.integers(0, 256, (1, s, s, 3), dtype=np.uint8) for s in (128, 96)]
    w = np.float32([0.4, 0.6])
    o64 = pipeline_interp(content[0], [s[0] for s in styles], w.astype(np.float64), weights, ALL, alpha=0.8, semantics="np",
                          dtype=np.float64)
    o32 = pipeline_interp(content[0], [s[0] for s in styles], w, weights, ALL, alpha=0.8, semantics="np", dtype=np.float32)
    eng = Engine(weights, ALL, semantics="np")
    out = eng.stylize(torch.from_numpy(content).cuda(), None, alpha=0.8, interp_styles=[torch.from_numpy(s).cuda() for s in styles],
                      interp_weights=torch.from_numpy(w[None]).cuda())
    eng.check_device()
    noise = np.abs(o32 - o64).max()
    err = np.abs(out.cpu().numpy() - o64).max()
    print("free-running interpolated 5-level: engine-vs-fp64 oracle %.3e ; oracle fp32-vs-fp64 %.3e" % (err, noise))
    assert err <= max(1e-3, FREE_RUN_NOISE_FACTOR * noise)


# ---------------------------------------------------------------------------------------------------------- front ends
@pytest.mark.parametrize("adain", [False, True])
def test_predict_batch_one_hot_equals_single_style(weights, adain):
    wct = WCT(checkpoints=None, relu_targets=ALL, vgg_path=None, weights=weights)
    rng = np.random.default_rng(3)
    c = rng.integers(0, 256, (3, 96, 80, 3), dtype=np.uint8)
    s0 = rng.integers(0, 256, (70, 90, 3), dtype=np.uint8)
    s1 = rng.integers(0, 256, (64, 64, 3), dtype=np.uint8)
    plain = wct.predict_batch(c, s1, alpha=0.8, adain=adain)
    assert np.array_equal(wct.predict_batch(c, [s0, s1], alpha=0.8, adain=adain, style_weights=[0, 2]), plain)
    assert np.array_equal(wct.predict_batch(c, [s1], alpha=0.8, adain=adain, style_weights=[1]), plain)


@pytest.mark.parametrize("adain", [False, True])
def test_batch_with_per_frame_rows_equals_single_frames(weights, adain):
    wct = WCT(checkpoints=None, relu_targets=ALL, vgg_path=None, weights=weights)
    assert wct.engine.groups == 2
    rng = np.random.default_rng(4)
    c = rng.integers(0, 256, (3, 64, 96, 3), dtype=np.uint8)
    styles = [rng.integers(0, 256, (s, s, 3), dtype=np.uint8) for s in (64, 80, 48)]
    rows = np.array([[1, 0, 0], [0.2, 0.5, 0.3], [0, 0.25, 0.75]])
    batch = wct.predict_batch(c, styles, alpha=0.8, adain=adain, style_weights=rows, passes=2)
    for i in range(3):
        one = wct.predict_batch(c[i:i + 1], styles, alpha=0.8, adain=adain, style_weights=rows[i], passes=2)
        assert np.array_equal(one[0], batch[i]), i


def test_interp_rejections(weights):
    wct = WCT(checkpoints=None, relu_targets=ALL, vgg_path=None, weights=weights)
    c = np.zeros((32, 32, 3), np.uint8)
    with pytest.raises(ValueError):
        wct.predict(c, [c, c], swap5=True, style_weights=[1, 1])
    with pytest.raises(ValueError):
        wct.predict(c, [c, c], content_mask=np.zeros((32, 32), np.uint8), style_weights=[1, 1])
    for bad in ([1, -1], [np.nan, 1], [0, 0], [1, 1, 1], [[1, 1], [1, 1]]):
        with pytest.raises(ValueError):
            wct.predict(c, [c, c], style_weights=bad)


def test_video_morph_frames_equal_per_frame_calls(tmp_path):
    import stylize_video as V
    from wct_tf_b200 import imageio as io
    targets = ["relu3_1", "relu2_1", "relu1_1"]
    wct = WCT(checkpoints=None, relu_targets=targets, vgg_path=None, weights=make_synthetic_weights(7, relu_targets=targets))
    rng = np.random.default_rng(9)
    frames = tmp_path / "clip"
    frames.mkdir()
    for i in range(5):
        Image.fromarray(rng.integers(0, 256, (48, 64, 3), dtype=np.uint8)).save(str(frames / ("frame_%d.png" % (i + 1))))
    spaths = []
    for j, s in enumerate((40, 56)):
        spaths.append(str(tmp_path / ("s%d.png" % j)))
        Image.fromarray(rng.integers(0, 256, (s, s, 3), dtype=np.uint8)).save(spaths[-1])
    n = V.main(["--relu-targets"] + targets + ["--in-path", str(frames), "--out-path", str(tmp_path / "out"), "--interp-styles"]
               + spaths + ["--morph", "--batch", "2", "--alpha", "0.8"], wct_factory=lambda a: wct)
    assert n == 5
    rows = V.morph_weights(5, 2)
    styles = [io.get_img(p) for p in spaths]
    for t in range(5):
        got = io.get_img(str(tmp_path / "out" / "clip_morph_s0+s1_frames" / ("frame_%d.png" % (t + 1))))
        ref = wct.predict_batch(io.get_img(str(frames / ("frame_%d.png" % (t + 1)))), styles, alpha=0.8, style_weights=rows[t])
        assert np.array_equal(got, ref[0]), t
