"""Exact feature distribution matching (EFDM, DESIGN.md §3.3.12) on the GPU: the C ABI against the fp64 oracle of
``tests/efdm_ref.py`` over channel counts, style sizes, ties, constant and negative channels; the halo and alpha = 0; byte
identity across workspace sizes, batches and runs; offsets past 2^31; the five-level pipeline; the distribution distance it
is for; and the engine options it works with or rejects.

Tolerance of the C ABI against the oracle (on the device's own SPF16 input, read back as fp32): the run means are fp64
(q interpolated in fp64, prefix sums of at most 2^18 terms: below 2^-30 of max|Q|), rounded once to fp32 (2^-24 of the
value) and stored as SPF16 (hi + lo, lo an fp16 of the rounding error of hi: 2^-22 of the value, or 2^-25 absolute where lo
is subnormal).  So |out - oracle| <= 2^-21 max(|Q|, |x|) + 2^-23.  The inputs are quantised so that adjacent distinct values,
and adjacent style quantiles, lie 2^-8 or more apart: a single wrong rank moves a value by far more than the tolerance."""
import gc
import zlib

import numpy as np
import pytest
import torch

from oracle import nets
from tests import efdm_ref as E
from tests import gpu_util as U
from tests.test_gpu_invariance import assert_bits, planes
from wct_tf_b200 import _capi
from wct_tf_b200.engine import Engine
from wct_tf_b200.wct import WCT
from wct_tf_b200.weights import make_synthetic_weights

pytestmark = pytest.mark.gpu
ALL = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]
FREE_RUN_NOISE_FACTOR = 3          # tests/test_gpu_pipeline.py: the free-running bound, a multiple of the oracle's fp32 noise


def _ws(nbytes):
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device="cuda")


def _tol(q_max, x_max):
    return 2.0 ** -21 * max(q_max, x_max) + 2.0 ** -23


def act_exact(x):
    """SPF16 buffer of fp32 NHWC x (any H, W >= 1: the halo is zero) and the fp32 values it holds (hi + lo)."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    n, h, w, c = x.shape
    hi = x.astype(np.float16)
    lo = (x - hi.astype(np.float32)).astype(np.float16)
    p = np.zeros((2, n, h + 2, w + 2, c), np.float16)
    p[0, :, 1:-1, 1:-1], p[1, :, 1:-1, 1:-1] = hi, lo
    buf = torch.from_numpy(p.view(np.uint8).reshape(-1)).cuda()
    return buf, hi.astype(np.float32) + lo.astype(np.float32)


def prepare(style, ns, hs, ws_, c, max_segments=1 << 30):
    lib = U.lib()
    state = _ws(lib.wctb200_efdm_style_state_bytes(c, ns, hs, ws_))
    ws = _ws(lib.wctb200_efdm_style_workspace_bytes(c, ns, hs, ws_, max_segments))
    _capi.check(lib.wctb200_efdm_style_prepare(style.data_ptr(), ns, hs, ws_, c, state.data_ptr(), ws.data_ptr(), ws.numel(),
                                               U.stream()))
    return state


def apply(content, n, h, w, c, state, ns, hs, ws_, alpha, max_segments=1 << 30, out=None):
    lib = U.lib()
    ws = _ws(lib.wctb200_efdm_workspace_bytes(c, n, h, w, max_segments))
    out = U.act_alloc(n, h, w, c) if out is None else out
    _capi.check(lib.wctb200_efdm_apply(content.data_ptr(), n, h, w, c, state.data_ptr(), ns, hs, ws_, float(alpha), out.data_ptr(),
                                       ws.data_ptr(), ws.numel(), U.stream()))
    return out


def _content(rng, n, h, w, c, kind):
    z = rng.standard_normal((n, h, w, c)) * rng.uniform(0.5, 2.0, c)
    if kind == "ties":            # >= 60 % zeros, the rest on a 2^-8 grid
        x = np.round(np.maximum(z - 0.3, 0) * 256) / 256
    elif kind == "negative":      # both signs on a 2^-8 grid, no zeros forced
        x = np.round(z * 256) / 256
    elif kind == "sparse":        # ~ 80 % zeros: runs of zeros across many sort tiles
        x = np.round(np.maximum(z - 0.85, 0) * 256) / 256
    else:                         # "distinct": continuous, positive, no zeros
        x = np.abs(z) + 0.25
    x[..., 3] = 0.5               # a constant channel
    return x.astype(np.float32)


def _style(rng, ns, hs, ws_, c, zeros):
    """Style values 2^-6 apart (a random permutation of a grid per channel), with a share of exact zeros."""
    m = hs * ws_
    v = np.stack([rng.permutation(m) for _ in range(ns * c)], -1).reshape(m, ns, c).transpose(1, 0, 2)
    v = (v + 1) * 2.0 ** -6 * rng.uniform(0.5, 1.5, c)
    v = np.round(v * 256) / 256
    if zeros:
        v[rng.random(v.shape) < zeros] = 0.0
    v[..., 4] = 1.25              # a constant style channel
    return v.reshape(ns, hs, ws_, c).astype(np.float32)


# (C, N, H, W, Ns, Hs, Ws, content kind, style zero share, alpha).  H*W is no multiple of the 2048-key sort tile.
CASES = {
    "c64_equal_ties": (64, 2, 45, 47, 1, 45, 47, "ties", 0.3, 1.0),
    "c128_style_larger_negative": (128, 2, 37, 61, 2, 50, 70, "negative", 0.0, 0.7),
    "c256_style_smaller_distinct": (256, 1, 65, 67, 1, 23, 29, "distinct", 0.0, 1.0),
    "c512_per_frame_ties": (512, 2, 19, 23, 2, 30, 30, "ties", 0.5, 0.6),
    "c64_long_zero_runs": (64, 1, 160, 160, 1, 96, 96, "sparse", 0.2, 1.0),
    "c64_style_1x1": (64, 2, 5, 7, 1, 1, 1, "negative", 0.0, 1.0),
    "c128_content_2x2": (128, 1, 2, 2, 1, 9, 9, "ties", 0.0, 0.9),
}


def _run_case(name, max_segments=1 << 30):
    c, n, h, w, ns, hs, ws_, kind, zeros, alpha = CASES[name]
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    x32 = _content(rng, n, h, w, c, kind)
    content = U.act_from_numpy(x32)
    x = U.act_to_numpy(content, n, h, w, c)
    style, s = act_exact(_style(rng, ns, hs, ws_, c, zeros))
    state = prepare(style, ns, hs, ws_, c)
    out = apply(content, n, h, w, c, state, ns, hs, ws_, alpha, max_segments)
    return (c, n, h, w, ns, hs, ws_, alpha), x, s, state, out


@pytest.mark.parametrize("name", list(CASES))
def test_apply_vs_fp64(name):
    (c, n, h, w, ns, hs, ws_, alpha), x, s, state, out = _run_case(name)
    U.check_device()
    # the state: every style channel's values, sorted
    got_state = state[:ns * c * hs * ws_ * 4].view(torch.float32).view(ns, c, hs * ws_).cpu().numpy()
    want_state = np.sort(s.reshape(ns, hs * ws_, c), axis=1).transpose(0, 2, 1)
    assert np.array_equal(got_state, want_state)
    ref = E.efdm(x, s, alpha)
    got = U.act_to_numpy(out, n, h, w, c)
    tol = _tol(float(np.abs(s).max()), float(np.abs(x).max()))
    err = float(np.abs(got - ref).max())
    print("%s: max |device - fp64| %.3e (tolerance %.3e)" % (name, err, tol))
    assert err <= tol
    # the reflect halo: every halo cell holds the bytes of its source cell
    p = planes(out, n, h, w, c)
    inner = p[:, :, 1:-1, 1:-1]
    want = np.pad(inner, ((0, 0), (0, 0), (1, 1), (1, 1), (0, 0)), mode="reflect")
    assert_bits(p, want, "%s halo" % name)


def test_alpha_zero_is_the_input_bit_for_bit():
    c, n, h, w = 128, 2, 33, 41
    rng = np.random.default_rng(5)
    content = U.act_from_numpy(_content(rng, n, h, w, c, "ties"))
    style, _ = act_exact(_style(rng, 1, 20, 20, c, 0.2))
    out = apply(content, n, h, w, c, prepare(style, 1, 20, 20, c), 1, 20, 20, 0.0)
    assert_bits(planes(out, n, h, w, c), planes(content, n, h, w, c), "alpha = 0")


@pytest.mark.parametrize("name", ["c64_equal_ties", "c64_long_zero_runs", "c512_per_frame_ties"])
def test_workspace_size_does_not_change_bytes(name):
    c, n, h, w = CASES[name][:4]
    full = planes(_run_case(name)[4], n, h, w, c)
    for segs in (1, 3, 40):
        assert_bits(planes(_run_case(name, max_segments=segs)[4], n, h, w, c), full, "%s, %d segments per chunk" % (name, segs))


def test_style_workspace_size_does_not_change_state():
    c, ns, hs, ws_ = 64, 2, 50, 47
    style, _ = act_exact(_style(np.random.default_rng(8), ns, hs, ws_, c, 0.3))
    full = prepare(style, ns, hs, ws_, c)
    for segs in (1, 5):
        assert torch.equal(prepare(style, ns, hs, ws_, c, max_segments=segs), full)


def _frame(buf, i, n, h, w, c):
    one = U.act_alloc(1, h, w, c, poison=False)
    one.view(torch.int16).view(2, 1, h + 2, w + 2, c).copy_(buf.view(torch.int16).view(2, n, h + 2, w + 2, c)[:, i:i + 1])
    return one


@pytest.mark.parametrize("shared", [True, False], ids=["shared_style", "style_per_frame"])
def test_batch_equals_single_frames(shared):
    c, n, h, w, hs, ws_ = 128, 3, 40, 52, 36, 44
    rng = np.random.default_rng(11)
    content = U.act_from_numpy(_content(rng, n, h, w, c, "ties"))
    ns = 1 if shared else n
    style, _ = act_exact(_style(rng, ns, hs, ws_, c, 0.3))
    state = prepare(style, ns, hs, ws_, c)
    out = apply(content, n, h, w, c, state, ns, hs, ws_, 0.8)
    again = apply(content, n, h, w, c, state, ns, hs, ws_, 0.8)
    assert_bits(planes(again, n, h, w, c), planes(out, n, h, w, c), "two runs")
    p = planes(out, n, h, w, c)
    for i in range(n):
        si = 0 if shared else i
        sty = style.view(torch.int16).view(2, ns, hs + 2, ws_ + 2, c)[:, si:si + 1].contiguous().view(torch.uint8).view(-1)
        one = apply(_frame(content, i, n, h, w, c), 1, h, w, c, prepare(sty, 1, hs, ws_, c), 1, hs, ws_, 0.8)
        assert_bits(planes(one, 1, h, w, c)[:, 0], p[:, i], "frame %d alone" % i)
    if shared:   # a shared style equals the same style repeated per frame
        rep = style.view(torch.int16).view(2, 1, hs + 2, ws_ + 2, c).expand(2, n, hs + 2, ws_ + 2, c).contiguous()
        rep = rep.view(torch.uint8).view(-1)
        per = apply(content, n, h, w, c, prepare(rep, n, hs, ws_, c), n, hs, ws_, 0.8)
        assert_bits(planes(per, n, h, w, c), p, "shared style vs repeated per frame")


def test_rejections():
    lib = U.lib()
    c = 64
    content = U.act_from_numpy(np.ones((2, 4, 4, c), np.float32))
    style, _ = act_exact(np.ones((2, 3, 3, c), np.float32))
    state = prepare(style, 2, 3, 3, c)
    out = U.act_alloc(2, 4, 4, c)
    small = _ws(lib.wctb200_efdm_workspace_bytes(c, 2, 4, 4, 1) - 256)
    ws = _ws(lib.wctb200_efdm_workspace_bytes(c, 2, 4, 4, 1))

    def call(n, ns, buf):
        return lib.wctb200_efdm_apply(content.data_ptr(), n, 4, 4, c, state.data_ptr(), ns, 3, 3, 1.0, out.data_ptr(), buf.data_ptr(),
                                      buf.numel(), U.stream())
    assert call(2, 2, ws) == 0
    assert call(1, 2, ws) == _capi.EINVAL                 # Ns not in {1, N}
    assert call(2, 2, small) == _capi.EWS                 # less than one segment's workspace
    assert lib.wctb200_efdm_workspace_bytes(c, 2, 1, 4, 1) == 0          # the content needs its reflect halo
    assert lib.wctb200_efdm_workspace_bytes(12, 2, 4, 4, 1) == 0         # C a multiple of 8
    assert lib.wctb200_efdm_style_state_bytes(c, 1, 1, 1) > 0
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------- offsets
def test_large_offsets_frame_2_alone():
    """relu1_1 of three 3584^2 frames: frame 2's elements lie past 2^31 in both planes; its bytes equal the frame alone."""
    n, h, w, c = 3, 3584, 3584, 64
    from tests.test_gpu_large_offsets import act_of, pl
    torch.cuda.empty_cache()
    buf = U.act_alloc(n, h, w, c, poison=False)
    dst = pl(buf, n, h, w, c)
    for i in range(n):
        g = torch.Generator(device="cuda").manual_seed(30 + i)
        x = torch.relu(torch.randn(1, h, w, c, generator=g, device="cuda") - 0.3 * (i + 1))
        x = torch.round(x * 256) / 256
        one = act_of(x)
        dst[:, i:i + 1].copy_(pl(one, 1, h, w, c))
        del one, x
    style, _ = act_exact(_style(np.random.default_rng(3), 1, 300, 280, c, 0.4))
    state = prepare(style, 1, 300, 280, c)
    frame = (h + 2) * (w + 2) * c
    # frame 2: its hi plane [2f, 3f) crosses 2^31, its lo plane [5f, 6f) lies past 2^31 and crosses 2^32
    assert 2 * frame < 2 ** 31 < 3 * frame and 2 ** 31 < 5 * frame < 2 ** 32 < 6 * frame
    out = apply(buf, n, h, w, c, state, 1, 300, 280, 1.0, max_segments=16)
    last = pl(out, n, h, w, c)[:, 2:3].clone()
    del out
    one_in = U.act_alloc(1, h, w, c, poison=False)
    pl(one_in, 1, h, w, c).copy_(pl(buf, n, h, w, c)[:, 2:3])
    del buf
    gc.collect()
    torch.cuda.empty_cache()
    one = apply(one_in, 1, h, w, c, state, 1, 300, 280, 1.0, max_segments=64)
    U.check_device()
    assert torch.equal(pl(one, 1, h, w, c), last), "frame 2 of 3 at 3584^2 differs from the frame alone"
    del one, last, one_in
    gc.collect()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------ pipeline
@pytest.fixture(scope="module")
def weights():
    return make_synthetic_weights(42)


def _u8(n, H, W, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, H, W, 3), dtype=np.uint8)


def _style_feats(eng, style_u8):
    """The engine's own style features at every target (the encode its style side runs), as device acts."""
    img = eng_img(eng, style_u8)
    _, feats = eng.encode(img, eng.model.deepest_target, taps=eng.model.style_taps)
    return feats


def eng_img(eng, u8):
    x = torch.empty(u8.shape, dtype=torch.float32, device="cuda")
    t = torch.from_numpy(u8).cuda()
    _capi.check(U.lib().wctb200_image_u8_to_f32(t.data_ptr(), t.numel(), x.data_ptr(), U.stream()))
    return x


def test_teacher_forced_levels(weights):
    """At every level of the five-level 128^2 run, the device's EFDM of its own content feature against its own style
    feature is within the C ABI tolerance of the fp64 oracle, and the level's decode within 1e-3 of fp64."""
    eng = Engine(weights, ALL)
    content, style = _u8(1, 128, 128, 100), _u8(1, 144, 144, 101)
    cap = {}
    eng.stylize(torch.from_numpy(content).cuda(), torch.from_numpy(style).cuda(), alpha=0.8, capture=cap, efdm=True)
    sf = _style_feats(eng, style)
    eng.check_device()
    for i, relu in enumerate(ALL):
        x = eng.act_to_f32(cap["content_feat"][i]).cpu().numpy()
        s = eng.act_to_f32(sf[relu]).cpu().numpy()
        ref = E.efdm(x, s, 0.8)
        got = eng.act_to_f32(cap["transformed"][i]).cpu().numpy()
        e_t, tol = float(np.abs(got - ref).max()), _tol(float(np.abs(s).max()), float(np.abs(x).max()))
        y = nets.decode(got.astype(np.float64), weights, relu, np.float64)
        if i < len(ALL) - 1:
            y = np.clip(y, 0, 1)
        e_out = float(np.abs(cap["level_output"][i].cpu().numpy() - y).max())
        print("%s: transform %.2e (tolerance %.2e)  level output %.2e  zeros %.0f%%" % (relu, e_t, tol, e_out, 100 * (x == 0).mean()))
        assert e_t <= tol and e_out <= 1e-3


def test_free_running_vs_oracle(weights):
    content, style = _u8(1, 128, 128, 1000), _u8(1, 128, 128, 7)
    o64 = E.pipeline_efdm(content[0], style[0], weights, ALL, alpha=0.8, dtype=np.float64)
    o32 = E.pipeline_efdm(content[0], style[0], weights, ALL, alpha=0.8, dtype=np.float32)
    bound = max(1e-3, FREE_RUN_NOISE_FACTOR * float(np.abs(o32 - o64).max()))
    eng = Engine(weights, ALL)
    got = eng.stylize(torch.from_numpy(content).cuda(), torch.from_numpy(style).cuda(), alpha=0.8, efdm=True).cpu().numpy()
    err = float(np.abs(got - o64).max())
    print("free-running EFDM 128^2: vs fp64 oracle %.3e (bound %.3e)" % (err, bound))
    assert err <= bound


def test_distribution_distance_below_wct_and_adain(weights):
    """At alpha = 1 on real encoder features, the per-channel 1-D Wasserstein distance from the style feature: EFDM's is
    below WCT's and AdaIN's at every level, and within the C ABI tolerance of the floor the oracle leaves (ties, and Ms style
    quantiles read at Nc ranks)."""
    eng = Engine(weights, ALL)
    content, style = _u8(1, 128, 128, 3), _u8(1, 160, 112, 4)
    cf_all = _style_feats(eng, content)
    sf = _style_feats(eng, style)
    for relu in ALL:
        cf, s_act = cf_all[relu], sf[relu]
        x = eng.act_to_f32(cf).cpu().numpy()
        s = eng.act_to_f32(s_act).cpu().numpy()
        d = {}
        for name in ("efdm", "wct", "adain"):
            if name == "efdm":
                f, _ = eng.efdm_apply(cf, eng.efdm_prepare(s_act), 1, 1.0)
            else:
                f, _ = eng.transform(cf, s_act, 1.0, adain=name == "adain")
            d[name] = E.w1(eng.act_to_f32(f).cpu().numpy(), s)
        floor = E.floor_w1(x, s)
        tol = _tol(float(np.abs(s).max()), 0.0)
        print("%s: mean W1 efdm %.4g (floor %.4g)  wct %.4g  adain %.4g" % (relu, d["efdm"].mean(), floor.mean(), d["wct"].mean(),
                                                                           d["adain"].mean()))
        assert d["efdm"].mean() < d["wct"].mean() and d["efdm"].mean() < d["adain"].mean()
        assert np.all(d["efdm"] <= floor + tol)
    eng.check_device()


# -------------------------------------------------------------------------------------------------------------- engine
def _f32_bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def test_invariance_batch_groups_styles_and_runs(weights):
    wct = WCT(relu_targets=ALL, weights=weights)
    c, s = _u8(3, 96, 80, 1), _u8(1, 64, 72, 2)
    u8, f = wct.predict_batch(c, s, alpha=0.8, efdm=True, return_float=True)
    u8b, fb = wct.predict_batch(c, s, alpha=0.8, efdm=True, return_float=True)
    assert_bits(_f32_bits(fb), _f32_bits(f), "two runs")
    for i in range(3):
        ui, fi = wct.predict_batch(c[i:i + 1], s, alpha=0.8, efdm=True, return_float=True)
        assert_bits(_f32_bits(fi[0]), _f32_bits(f[i]), "frame %d alone" % i)
    eng = wct.engine
    g0 = eng.groups
    eng.groups = 2
    try:
        ug, fg = wct.predict_batch(c, s, alpha=0.8, efdm=True, return_float=True)
    finally:
        eng.groups = g0
    assert_bits(_f32_bits(fg), _f32_bits(f), "groups = 2")
    ur, fr = wct.predict_batch(c, np.repeat(s, 3, axis=0), alpha=0.8, efdm=True, return_float=True)
    assert_bits(_f32_bits(fr), _f32_bits(f), "the style repeated per frame")
    s3 = _u8(3, 64, 72, 5)                                        # one style per frame, alone and in groups
    per = wct.predict_batch(c, s3, alpha=0.8, efdm=True)
    assert np.array_equal(np.concatenate([wct.predict_batch(c[i:i + 1], s3[i:i + 1], alpha=0.8, efdm=True) for i in range(3)]), per)
    eng.groups = 2
    try:
        assert np.array_equal(wct.predict_batch(c, s3, alpha=0.8, efdm=True), per)
    finally:
        eng.groups = g0
    assert not np.array_equal(u8, wct.predict_batch(c, s, alpha=0.8))          # EFDM is not WCT


def test_passes_outputs_and_predict(weights):
    wct = WCT(relu_targets=ALL, weights=weights, semantics="np")
    c, s = _u8(2, 80, 96, 4), _u8(1, 64, 64, 5)
    one = wct.predict_batch(c, s, alpha=0.7, efdm=True)
    assert np.array_equal(wct.predict_batch(c, s, alpha=0.7, efdm=True, passes=2), wct.predict_batch(one, s, alpha=0.7, efdm=True))
    s2 = _u8(2, 64, 64, 6)
    one2 = wct.predict_batch(c, s2, alpha=0.7, efdm=True)
    assert np.array_equal(wct.predict_batch(c, s2, alpha=0.7, efdm=True, passes=2),
                          wct.predict_batch(one2, s2, alpha=0.7, efdm=True))
    u8, f = wct.predict_batch(c, s, alpha=0.7, efdm=True, return_float=True)
    assert np.array_equal(u8, one) and f.dtype == np.float32
    assert np.array_equal(wct.predict_batch(c, s, alpha=0.7, efdm=True, return_device=True).cpu().numpy(), one)
    out = torch.empty(one.shape, dtype=torch.uint8).pin_memory()
    wct.predict_batch(c, s, alpha=0.7, efdm=True, out=out)
    assert np.array_equal(out.numpy(), one)
    assert np.array_equal(wct.predict(c[0], s[0], alpha=0.7, efdm=True), one[0])


def test_synthesize_and_seamless(weights):
    wct = WCT(relu_targets=ALL, weights=weights)
    style = _u8(1, 128, 144, 2)[0]
    from wct_tf_b200.device_image import noise_u8
    tex = wct.synthesize(style, (128, 192), count=2, seed=5, efdm=True, alpha=0.9)
    noise = noise_u8(2, 128, 192, seed=5, device=wct.engine.device)
    assert np.array_equal(tex, wct.predict_batch(noise, style, efdm=True, alpha=0.9))
    # seamless: a circular shift of the content shifts the wrapped output by the same amount (the check of
    # test_gpu_seamless.py), and the wrapped texture is not the reflect one
    eng = wct.engine
    content = _u8(1, 128, 128, 1000)
    s = torch.from_numpy(style[None]).cuda()
    got = eng.stylize(torch.from_numpy(content).cuda(), s, alpha=0.8, seamless="xy", efdm=True).cpu().numpy()
    rolled = np.roll(content, (32, 48), axis=(1, 2))
    got_r = eng.stylize(torch.from_numpy(rolled).cuda(), s, alpha=0.8, seamless="xy", efdm=True).cpu().numpy()
    e_shift = float(np.abs(got_r - np.roll(got, (32, 48), axis=(1, 2))).max())
    print("seamless xy EFDM: shift equivariance %.3e" % e_shift)
    assert e_shift <= 1e-3
    flat = eng.stylize(torch.from_numpy(content).cuda(), s, alpha=0.8, efdm=True).cpu().numpy()
    assert not np.array_equal(flat, got)
    eng.check_device()


def test_temporal_runs(weights):
    targets = ["relu3_1", "relu1_1"]
    wct = WCT(relu_targets=targets, weights=make_synthetic_weights(1, relu_targets=targets))
    c, s = _u8(3, 64, 64, 1), _u8(1, 64, 64, 2)
    st = wct.temporal_state(0.5)
    out = wct.predict_batch(c, s, efdm=True, temporal=st)
    assert out.shape == (3, 64, 64, 3)
    assert np.array_equal(out[0], wct.predict_batch(c[:1], s, efdm=True)[0])     # the first frame of a clip is unchanged


def test_swap_levels_swap_and_the_others_use_efdm():
    """With swap_targets=["relu1_1"] (the last level) the levels before it are the EFDM-only call's, byte for byte, and the
    swap level is the swap's."""
    targets = ["relu3_1", "relu2_1", "relu1_1"]
    eng = Engine(make_synthetic_weights(3, relu_targets=targets), targets)
    c = torch.from_numpy(_u8(2, 64, 64, 7)).cuda()
    s = torch.from_numpy(_u8(1, 64, 64, 8)).cuda()
    cap_sw, cap_e, cap_w = {}, {}, {}
    eng.stylize(c, s, alpha=0.8, capture=cap_sw, swap_targets=["relu1_1"], efdm=True)
    eng.stylize(c, s, alpha=0.8, capture=cap_e, efdm=True)
    eng.stylize(c, s, alpha=0.8, capture=cap_w, swap_targets=["relu1_1"])
    for i in range(2):
        assert torch.equal(cap_sw["transformed"][i].buf, cap_e["transformed"][i].buf)
        assert not torch.equal(cap_sw["transformed"][i].buf, cap_w["transformed"][i].buf)
    # the swap level: the swap of its own input (the swap-only call's input differs, so compare with a swap of it)
    st, _ = eng.swap_state(eng.prepare_call(s, swap_targets=["relu1_1"]), "relu1_1", 3, 1)
    torch.cuda.synchronize()
    sf = _style_feats(eng, s.cpu().numpy())["relu1_1"]
    f, _ = eng.swap_apply(cap_sw["content_feat"][2], st, (sf.H, sf.W), 0.6)
    assert torch.equal(f.buf, cap_sw["transformed"][2].buf)
    eng.check_device()


_REJECT = [dict(adain=True), dict(ost=True), dict(mst=2), dict(content_mask="mask"), dict(style_weights=[1.0]),
           dict(strength_map="map"), dict(content_weights="weights"), dict(tile_size=64), dict(prepared=True)]


@pytest.mark.parametrize("kw", _REJECT, ids=[next(iter(k)) for k in _REJECT])
def test_rejected_combinations(kw):
    targets = ["relu3_1", "relu1_1"]
    wct = WCT(relu_targets=targets, weights=make_synthetic_weights(1, relu_targets=targets))
    c, s = _u8(1, 64, 64, 1), _u8(1, 64, 64, 2)
    kw = dict(kw)
    styles = s
    if kw.get("content_mask") == "mask":
        kw["content_mask"], styles = np.zeros((8, 8), np.uint8), [s[0]]
    if "style_weights" in kw:
        styles = [s[0]]
    if kw.get("strength_map") == "map":
        kw["strength_map"] = np.ones((8, 8), np.float32)
    if kw.get("content_weights") == "weights":
        kw["content_weights"], styles = np.ones((1, 8, 8), np.float32), [s[0]]
    if kw.pop("prepared", False):
        styles = wct.prepare_style(s[0])
    with pytest.raises(ValueError, match="efdm"):
        wct.predict_batch(c, styles, efdm=True, **kw)
    with pytest.raises(ValueError):
        wct.predict(c[0], styles if not isinstance(styles, np.ndarray) else s[0], efdm=True, **kw)
    eng = wct.engine
    with pytest.raises(ValueError, match="efdm"):
        eng.stylize(torch.from_numpy(c).cuda(), eng.prepare_call(torch.from_numpy(s).cuda()), efdm=True)
