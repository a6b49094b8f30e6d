"""Seamless stylisation on the device (DESIGN.md §3.3.9): the halo rewrite, the conv producers and the encoder head under
the wrap flags, the engine's encode / decode against tiled copies, parity with the wrap oracle (tests/seamless_ref.py),
shift equivariance, the combinations with the other options, and the rejections."""
import numpy as np
import pytest
import torch

from oracle import nets, ref_ops
from tests import gpu_util as U
from tests import seamless_ref as S
from tests.test_gpu_pipeline import FREE_RUN_NOISE_FACTOR
from tests.test_gpu_tiles import TF_TILED_BOUND
from wct_tf_b200 import _capi
from wct_tf_b200.engine import Act, Engine
from wct_tf_b200.model import RELU_LEVEL, tile_halos
from wct_tf_b200.wct import WCT
from wct_tf_b200.weights import make_synthetic_weights

pytestmark = pytest.mark.gpu
ALL = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]
WX, WY, EDGE, RELU, POOL2 = _capi.HALO_WRAP_X, _capi.HALO_WRAP_Y, _capi.HALO_EDGE, _capi.RELU, _capi.POOL2


@pytest.fixture(scope="module")
def weights():
    return make_synthetic_weights(42)


@pytest.fixture(scope="module")
def engine(weights):
    return Engine(weights, ALL)


def _u8(n, H, W, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, H, W, 3), dtype=np.uint8)


def _planes(buf, n, h, w, c):
    """Both planes of an SPF16 buffer as raw 16-bit words [2, n, h+2, w+2, c]."""
    torch.cuda.synchronize()
    return buf.view(torch.int16).view(2, n, h + 2, w + 2, c).cpu().numpy()


def _pad_planes(inner, flags):
    """The halo of ``flags`` around raw interior planes [2, n, h, w, c]: np.pad per axis, x first."""
    def mode(wrap):
        return "wrap" if flags & wrap else ("edge" if flags & EDGE else "reflect")
    p = np.pad(inner, ((0, 0), (0, 0), (0, 0), (1, 1), (0, 0)), mode=mode(WX))
    return np.pad(p, ((0, 0), (0, 0), (1, 1), (0, 0), (0, 0)), mode=mode(WY))


def _halo(buf, n, h, w, c, flags):
    _capi.check(U.lib().wctb200_act_halo(buf.data_ptr(), n, h, w, c, flags, U.stream()))


def _tile3(x, flags, axis_y=1, axis_x=2):
    """x tiled 3x along the wrapped axes (numpy, NHWC-like axes)."""
    reps = [1] * x.ndim
    if flags & WY:
        reps[axis_y] = 3
    if flags & WX:
        reps[axis_x] = 3
    return np.tile(x, reps)


def _centre(x, flags, h, w, axis_y=1, axis_x=2):
    sl = [slice(None)] * x.ndim
    if flags & WY:
        sl[axis_y] = slice(h, 2 * h)
    if flags & WX:
        sl[axis_x] = slice(w, 2 * w)
    return x[tuple(sl)]


# ------------------------------------------------------------------------------------------------------------- act_halo
@pytest.mark.parametrize("C", [8, 64, 512])
@pytest.mark.parametrize("hw", [(2, 2), (2, 5), (7, 3), (16, 9)])
def test_act_halo_modes_byte_exact(C, hw):
    h, w = hw
    n = 2
    x = np.random.default_rng(C + h * 31 + w).standard_normal((n, h, w, C)).astype(np.float32)
    ref = U.act_from_numpy(x)
    reflect = _planes(ref, n, h, w, C)
    assert np.array_equal(reflect, _pad_planes(reflect[:, :, 1:-1, 1:-1], 0))
    for flags in (WX, WY, WX | WY, EDGE, EDGE | WX, EDGE | WY):
        buf = ref.clone()
        _halo(buf, n, h, w, C, flags)
        got = _planes(buf, n, h, w, C)
        assert np.array_equal(got[:, :, 1:-1, 1:-1], reflect[:, :, 1:-1, 1:-1])        # the interior is not touched
        assert np.array_equal(got, _pad_planes(reflect[:, :, 1:-1, 1:-1], flags)), flags
    # flags 0 writes act_from_f32's reflect halo over a poisoned one
    buf = ref.clone()
    v = buf.view(torch.float16).view(2, n, h + 2, w + 2, C)
    v[:, :, 0] = float("nan"); v[:, :, -1] = float("nan"); v[:, :, :, 0] = float("nan"); v[:, :, :, -1] = float("nan")
    _halo(buf, n, h, w, C, 0)
    assert np.array_equal(_planes(buf, n, h, w, C), reflect)
    assert U.lib().wctb200_act_halo(buf.data_ptr(), n, h, w, C, RELU, U.stream()) == _capi.EINVAL


# ------------------------------------------------------------------------------------------------------- conv producers
def _prep(w_hwio, up2=False):
    kh, kw, cin, cout = w_hwio.shape
    lib = U.lib()
    src = U.dev(w_hwio.astype(np.float32))
    dst = torch.empty(lib.wctb200_conv_weight_bytes(16 if up2 else 9, cin, cout), dtype=torch.uint8, device="cuda")
    if up2:
        _capi.check(lib.wctb200_prep_conv_weights_up2(src.data_ptr(), cin, cout, dst.data_ptr(), U.stream()))
    else:
        _capi.check(lib.wctb200_prep_conv_weights(src.data_ptr(), 9, cin, cout, dst.data_ptr(), U.stream()))
    return dst


def _run_conv(x, wsplit, bias, cout, flags, in_flags, up2=False):
    """conv3x3 (or conv3x3_up2) of the fp32 map x [n,h,w,cin] whose halo is written in the mode of in_flags; returns the
    raw output planes."""
    n, h, w, cin = x.shape
    buf = U.act_from_numpy(x)
    if in_flags:
        _halo(buf, n, h, w, cin, in_flags)
    if up2:
        oh, ow = 2 * h, 2 * w
    elif flags & POOL2:
        oh, ow = (h + 1) // 2, (w + 1) // 2
    else:
        oh, ow = h, w
    out = U.act_alloc(n, oh, ow, cout)
    fn = U.lib().wctb200_conv3x3_up2 if up2 else U.lib().wctb200_conv3x3
    _capi.check(fn(buf.data_ptr(), n, h, w, cin, wsplit.data_ptr(), bias.data_ptr(), cout, flags, out.data_ptr(), U.stream()))
    U.check_device()
    return _planes(out, n, oh, ow, cout), (oh, ow)


@pytest.mark.parametrize("cin,cout", [(64, 64), (128, 128), (64, 128)])
@pytest.mark.parametrize("kind", ["plain", "pool", "edge", "up2"])
@pytest.mark.parametrize("wrap", [WX, WY, WX | WY], ids=["x", "y", "xy"])
def test_conv_wrap_equals_centre_of_tiled(cin, cout, kind, wrap):
    """The interior equals, bit for bit, the centre copy of the same conv without wrap flags on the input tiled 3x along
    the wrapped axes; every halo cell is a copy of the wrapped interior cell (edge on the other axis with HALO_EDGE)."""
    rng = np.random.default_rng(cin + cout)
    n, h, w = 2, 12, 10
    x = np.maximum(rng.standard_normal((n, h, w, cin)), 0).astype(np.float32)
    wt = (rng.standard_normal((3, 3, cin, cout)) * np.sqrt(2.0 / (9 * cin))).astype(np.float32)
    bias = U.dev(rng.standard_normal(cout).astype(np.float32) * 0.1)
    up2 = kind == "up2"
    ws = _prep(wt, up2)
    flags = RELU | (POOL2 if kind == "pool" else 0) | (EDGE if kind == "edge" else 0)
    in_extra = EDGE if up2 else 0                         # the input of an UP2 conv carries the edge halo
    got, (oh, ow) = _run_conv(x, ws, bias, cout, flags | wrap, in_extra | wrap, up2)
    ref, _ = _run_conv(_tile3(x, wrap), ws, bias, cout, flags, in_extra, up2)
    inner = got[:, :, 1:-1, 1:-1]
    assert np.array_equal(inner, _centre(ref[:, :, 1:-1, 1:-1], wrap, oh, ow, 2, 3))
    assert np.array_equal(got, _pad_planes(inner, (flags & EDGE) | wrap))


@pytest.mark.parametrize("wrap", [WX, WY, WX | WY], ids=["x", "y", "xy"])
@pytest.mark.parametrize("tc", [1, 0], ids=["tc", "simt"])
def test_conv_head_wrap_equals_centre_of_tiled(weights, wrap, tc):
    lib = U.lib()
    eng = Engine(weights, ["relu1_1"])
    n, h, w = 2, 18, 22
    img = np.random.default_rng(5).random((n, h, w, 3)).astype(np.float32)

    def head(x, flags):
        nn, hh, ww, _ = x.shape
        out = U.act_alloc(nn, hh, ww, 64)
        _capi.check(lib.wctb200_conv_head_flags(U.dev(x).data_ptr(), nn, hh, ww, eng.head_w.data_ptr(), eng.head_b.data_ptr(),
                                                flags, out.data_ptr(), U.stream()))
        U.check_device()
        return _planes(out, nn, hh, ww, 64)
    lib.wctb200_debug_set_conv_head_tc(tc)             # returns the previous setting
    try:
        got = head(img, wrap)
        ref = head(_tile3(img, wrap), 0)
        plain = U.act_alloc(n, h, w, 64)
        _capi.check(lib.wctb200_conv_head(U.dev(img).data_ptr(), n, h, w, eng.head_w.data_ptr(), eng.head_b.data_ptr(),
                                          plain.data_ptr(), U.stream()))
        assert np.array_equal(head(img, 0), _planes(plain, n, h, w, 64))      # flags 0 is wctb200_conv_head
    finally:
        lib.wctb200_debug_set_conv_head_tc(1)
    inner = got[:, :, 1:-1, 1:-1]
    assert np.array_equal(inner, _centre(ref[:, :, 1:-1, 1:-1], wrap, h, w, 2, 3))
    assert np.array_equal(got, _pad_planes(inner, wrap))
    out = U.act_alloc(n, h, w, 64)
    assert lib.wctb200_conv_head_flags(U.dev(img).data_ptr(), n, h, w, eng.head_w.data_ptr(), eng.head_b.data_ptr(), EDGE,
                                       out.data_ptr(), U.stream()) == _capi.EINVAL


# ------------------------------------------------------------------------------------------------- engine encode / decode
@pytest.mark.parametrize("relu", ALL)
@pytest.mark.parametrize("mode", ["x", "xy"])
def test_engine_encode_decode_equal_centre_of_tiled(engine, relu, mode):
    """Seamless encode = the centre copy of the reflect encode of the content tiled 3x (each copy at least h_A wide), and
    seamless decode = the centre copy of the reflect decode of the feature tiled 3x (each copy at least (h_B - h_A) / g
    feature pixels wide), bit for bit."""
    eng = engine
    flags = WX | (WY if mode == "xy" else 0)
    g = 2 ** (RELU_LEVEL[relu] - 1)
    h_a, h_b = tile_halos(relu)
    H, W = 96, 112
    assert W >= h_a and W // g >= (h_b - h_a) // g
    img = np.random.default_rng(3).random((1, H, W, 3)).astype(np.float32)
    f, _ = eng.encode(U.dev(img), relu, seamless=mode)
    big, _ = eng.encode(U.dev(_tile3(img, flags)), relu)
    got = _planes(f.buf, 1, f.H, f.W, f.C)[:, :, 1:-1, 1:-1]
    ref = _planes(big.buf, 1, big.H, big.W, big.C)[:, :, 1:-1, 1:-1]
    assert np.array_equal(got, _centre(ref, flags, f.H, f.W, 2, 3))
    dec = eng.decode(f, ALL.index(relu), clip=False, seamless=mode).cpu().numpy()
    # the same feature tiled 3x, raw planes and all, with the reflect halo
    tiled = _tile3(got, flags, 2, 3)
    bigf = Act(U.act_alloc(1, tiled.shape[2], tiled.shape[3], f.C), 1, tiled.shape[2], tiled.shape[3], f.C)
    bigf.buf.view(torch.int16).view(2, 1, bigf.H + 2, bigf.W + 2, f.C)[:, :, 1:-1, 1:-1] = torch.from_numpy(tiled).cuda()
    _halo(bigf.buf, 1, bigf.H, bigf.W, f.C, 0)
    decb = eng.decode(bigf, ALL.index(relu), clip=False).cpu().numpy()
    assert np.array_equal(dec.view(np.uint32), _centre(decb, flags, H, W).view(np.uint32))
    eng.check_device()


# --------------------------------------------------------------------------------------------------- parity with the oracle
def _teacher_forced(weights, mode, targets, size, adain=False, ost=False, alpha=0.8, stylize_kw=None, level_fn=None):
    eng = Engine(weights, targets)
    content = _u8(1, size[0], size[1], 100)
    style = _u8(1, 96, 112, 7)
    cap = {}
    kw = dict(stylize_kw or {})
    if "labels" not in kw and "interp_styles" not in kw:
        kw.update(adain=adain, ost=ost)
    sty = kw.pop("style", torch.from_numpy(style).cuda())
    eng.stylize(torch.from_numpy(content).cuda(), sty, alpha=alpha, capture=cap, seamless=mode, **kw)
    eng.check_device()
    sfe = nets.encode(nets.preprocess(style).astype(np.float64), weights, targets, np.float64)
    worst = 0.0
    for i, relu in enumerate(targets):
        x = cap["level_input"][i].cpu().numpy().astype(np.float64)
        cf = S.encode(x, weights, [relu], np.float64, mode)[relu]
        e_enc = np.abs(eng.act_to_f32(cap["content_feat"][i]).cpu().numpy() - cf).max()
        if level_fn:
            f = level_fn(i, relu, cf)
        else:
            f = S.transform(cf, sfe[relu], alpha, adain, ost)
            if not adain:
                _, info = ref_ops.wct_tf(cf, sfe[relu], alpha, return_info=True)
                assert ref_ops.spectral_gap_ok(info["wc"]) and ref_ops.spectral_gap_ok(info["ws"]), "ill-posed vector"

        e_tr = np.abs(eng.act_to_f32(cap["transformed"][i]).cpu().numpy() - f).max()
        y = S.decode(np.asarray(f, np.float64), weights, relu, np.float64, mode)
        if i < len(targets) - 1:
            y = np.clip(y, 0, 1)
        e_out = np.abs(cap["level_output"][i].cpu().numpy() - y).max()
        print("%s %s %s: encoder %.2e transform %.2e output %.2e" % (mode, relu, size, e_enc, e_tr, e_out))
        worst = max(worst, e_enc, e_tr, e_out)
    return worst


# A 2:1 panorama of 96 x 192: at 128 x 256 relu4_1 has exactly C = 512 pixels, and the content covariance's smallest
# eigenvalue sits at the threshold (ill-posed for any padding).
@pytest.mark.parametrize("mode,size,targets,kind", [
    ("xy", (128, 128), ALL, "wct"),
    ("x", (96, 192), ALL, "wct"),
    ("y", (96, 80), ALL[2:], "wct"),
    ("xy", (96, 96), ALL, "adain"),
    ("x", (96, 128), ALL, "ost"),
    ("xy", (72, 88), ["relu3_1", "relu1_1", "relu2_1"], "wct"),
])
def test_teacher_forced_levels_vs_wrap_oracle(weights, mode, size, targets, kind):
    assert _teacher_forced(weights, mode, targets, size, adain=kind == "adain", ost=kind == "ost") <= 1e-3


def test_teacher_forced_content_mask_and_style_weights(weights):
    from tests import interp_ref, regions_ref
    H, W = 96, 128
    styles = [_u8(1, 80, 96, 11), _u8(1, 96, 80, 12)]
    sfe = [nets.encode(nets.preprocess(s).astype(np.float64), weights, ["relu2_1"], np.float64)["relu2_1"] for s in styles]
    mask = np.zeros((H, W), np.uint8)
    mask[:, W // 2:] = 1
    lab = torch.from_numpy(mask).cuda()

    def regions(i, relu, cf):
        return regions_ref.wct_regions(cf, sfe, regions_ref.resize_labels(mask, cf.shape[1], cf.shape[2]), 0.8)
    kw = dict(labels=lab, region_styles=[torch.from_numpy(s).cuda() for s in styles])
    assert _teacher_forced(weights, "xy", ["relu2_1"], (H, W), stylize_kw=kw, level_fn=regions) <= 1e-3
    wv = np.array([[0.3, 0.7]], np.float32)

    def interp(i, relu, cf):
        return interp_ref.wct_interp(cf, sfe, wv[0].astype(np.float64), 0.8)
    kw = dict(interp_styles=[torch.from_numpy(s).cuda() for s in styles], interp_weights=torch.from_numpy(wv).cuda())
    assert _teacher_forced(weights, "x", ["relu2_1"], (H, W), stylize_kw=kw, level_fn=interp) <= 1e-3


def test_free_running_and_shift_equivariance(weights):
    """Five levels free-running against the float64 wrap oracle within FREE_RUN_NOISE_FACTOR times its own fp32 noise, and
    a circular shift of the content by (32, 48) pixels shifts the device output by the same amount, within that bound
    (only the summation order of the statistics differs); one level within 1e-3."""
    content, style = _u8(1, 128, 128, 1000), _u8(1, 128, 128, 7)
    o64 = S.pipeline(content[0], style[0], weights, ALL, alpha=0.8, dtype=np.float64, wrap="xy")
    o32 = S.pipeline(content[0], style[0], weights, ALL, alpha=0.8, dtype=np.float32, wrap="xy")
    noise = np.abs(o32 - o64).max()
    eng = Engine(weights, ALL)
    s = torch.from_numpy(style).cuda()
    got = eng.stylize(torch.from_numpy(content).cuda(), s, alpha=0.8, seamless="xy").cpu().numpy()
    err = np.abs(got - o64).max()
    rolled = np.roll(content, (32, 48), axis=(1, 2))
    got_r = eng.stylize(torch.from_numpy(rolled).cuda(), s, alpha=0.8, seamless="xy").cpu().numpy()
    e_shift = np.abs(got_r - np.roll(got, (32, 48), axis=(1, 2))).max()
    one = Engine(weights, ["relu3_1"])
    a = one.stylize(torch.from_numpy(content).cuda(), s, alpha=0.8, seamless="xy").cpu().numpy()
    b = one.stylize(torch.from_numpy(rolled).cuda(), s, alpha=0.8, seamless="xy").cpu().numpy()
    e_one = np.abs(b - np.roll(a, (32, 48), axis=(1, 2))).max()
    print("free-running 5-level xy: %.3e (oracle fp32 noise %.3e); shift 5 levels %.3e, 1 level %.3e" % (err, noise, e_shift, e_one))
    bound = max(1e-3, FREE_RUN_NOISE_FACTOR * noise)
    assert err <= bound and e_shift <= bound and e_one <= 1e-3
    eng.check_device()


# ------------------------------------------------------------------------------------------------------------ combinations
def test_synthesize_prepared_and_batch(weights):
    wct = WCT(relu_targets=ALL, weights=weights)
    style = _u8(1, 128, 144, 2)[0]
    from wct_tf_b200.device_image import noise_u8
    tex = wct.synthesize(style, (128, 192), count=3, seed=5, seamless="xy", alpha=0.8)
    noise = noise_u8(3, 128, 192, seed=5, device=wct.engine.device)
    assert np.array_equal(tex, wct.predict_batch(noise, style, seamless="xy", alpha=0.8))
    ps = wct.prepare_style(style)
    assert np.array_equal(tex, wct.synthesize(ps, (128, 192), count=3, seed=5, seamless="xy", alpha=0.8))
    frames = np.concatenate([wct.predict_batch(noise[i:i + 1], style, seamless="xy", alpha=0.8) for i in range(3)])
    assert np.array_equal(tex, frames)
    # a wrapped texture is not the reflect one
    assert not np.array_equal(tex, wct.predict_batch(noise, style, alpha=0.8))
    one = wct.predict(noise[0].cpu().numpy(), style, alpha=0.8, seamless="x")
    assert np.array_equal(one, wct.predict_batch(noise[:1], style, alpha=0.8, seamless="x")[0])


@pytest.mark.parametrize("case", ["wct", "adain", "passes2", "y"])
def test_one_tile_equals_untiled_seamless(weights, case):
    wct = WCT(relu_targets=ALL, weights=weights)
    c, s = _u8(1, 160, 192, 1), _u8(1, 128, 144, 2)
    kw = dict(alpha=0.8, adain=case == "adain", passes=2 if case == "passes2" else 1, return_float=True,
              seamless="y" if case == "y" else "xy")
    ref_u8, ref_f = wct.predict_batch(c, s, **kw)
    got_u8, got_f = wct.predict_batch(c, s, tile_size=256, **kw)
    assert np.array_equal(got_u8, ref_u8)
    assert np.array_equal(got_f.view(np.uint32), ref_f.view(np.uint32))


@pytest.mark.parametrize("H,W,T,mode", [(1024, 2048, 512, "x"), (512, 512, 256, "xy"), (1024, 512, 512, "x")])
def test_many_tiles_teacher_forced_seamless(engine, H, W, T, mode):
    """Every level of an untiled seamless run, run again tiled from the same input: wrapped axes cut into tiles take their
    crops modulo the image, a wrapped axis one tile spans is encoded with the wrap flag."""
    eng = engine
    c = torch.from_numpy(_u8(1, H, W, 5)).cuda()
    s = torch.from_numpy(_u8(1, 256, 256, 6)).cuda()
    cap = {}
    eng.stylize(c, s, alpha=0.8, capture=cap, seamless=mode)
    ps = eng.prepare_call(s)
    torch.cuda.synchronize()
    worst = {}
    for i, lvl in enumerate(eng.model.levels):
        got = eng.tiled_level(cap["level_input"][i], i, ps.wct[lvl.relu_target], 0.8, False, T, clip=i < len(ALL) - 1,
                              seamless=mode)
        ref = cap["level_output"][i]
        assert got.shape == ref.shape
        worst[lvl.relu_target] = float((got - ref).abs().max())
    print("tiled seamless %dx%d T=%d %s: %s" % (H, W, T, mode, worst))
    assert max(worst.values()) <= TF_TILED_BOUND, worst
    eng.check_device()


def test_rejections(weights):
    wct = WCT(relu_targets=ALL, weights=weights)
    c, s = _u8(1, 64, 96, 1), _u8(1, 64, 64, 2)
    for kw in (dict(seamless="z"), dict(seamless="xy", swap5=True), dict(seamless="x", swap_targets=["relu3_1"]),
               dict(seamless="x", temporal=wct.temporal_state(0.5))):
        with pytest.raises(ValueError):
            wct.predict_batch(c, s, **kw)
    with pytest.raises(ValueError, match="width 100 is not a multiple of 16"):
        wct.predict_batch(_u8(1, 64, 100, 1), s, seamless="x")
    with pytest.raises(ValueError, match="height 72 is not a multiple of 16"):
        wct.predict_batch(_u8(1, 72, 96, 1), s, seamless="xy", tile_size=32)
    assert wct.predict_batch(_u8(1, 72, 96, 1), s, seamless="x").shape[2] == 96              # y reflects: any height
    eng = wct.engine
    with pytest.raises(ValueError):
        eng.stylize(torch.from_numpy(c).cuda(), torch.from_numpy(s).cuda(), seamless="xy", swap5=True)
