"""Per-frame bit invariance on one GPU: a frame's result does not depend on the batch it runs in, on the stream groups the
batch is cut into, or on the run.  Multi-GPU sharding relies on it (DESIGN.md §3.3 A).

Every comparison is on raw bits -- both SPF16 planes with the halo, fp32 and uint8 outputs -- with no tolerance: a race or a
batch-dependent index that moves a value by one ulp is a failure here, where a 1e-3 parity bound would hide it.  The
single-frame runs read byte copies of the batch's own frames, so any difference comes from the kernels.
"""
import numpy as np
import pytest
import torch

from wct_tf_b200 import _capi
from wct_tf_b200.engine import Engine
from wct_tf_b200.wct import WCT
from wct_tf_b200.weights import make_synthetic_weights
from tests import gpu_util as U

pytestmark = pytest.mark.gpu
ALL = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]
N = 5
SEMS = dict(tf=(1e-8, 0.0, 1e-5, 1), np=(0.0, 1e-5, 1e-5, 0))     # eps_cov, eps_eig, thresh, readd


def planes(buf, n, h, w, c):
    """Raw bits of an SPF16 buffer: int16 [2 planes][n][h+2][w+2][c]."""
    torch.cuda.synchronize()
    return buf.view(torch.int16).view(2, n, h + 2, w + 2, c).cpu().numpy()


def frame_copy(buf, i, n, h, w, c):
    """A new one-frame SPF16 buffer holding the bytes of frame i of `buf` (both planes, halo included)."""
    src = buf.view(torch.int16).view(2, n, h + 2, w + 2, c)
    out = U.act_alloc(1, h, w, c, poison=False)
    out.view(torch.int16).view(2, 1, h + 2, w + 2, c).copy_(src[:, i:i + 1])
    return out


def feats(n, h, w, c, seed, offset=0.3):
    """Relu-like features with channel correlations; each frame has its own content and scale."""
    rng = np.random.default_rng(seed)
    mix = rng.standard_normal((c, c)) / np.sqrt(c)
    x = rng.standard_normal((n, h, w, c)) @ mix
    x *= (1.0 + 0.25 * np.arange(n))[:, None, None, None]
    return np.maximum(x + offset, 0).astype(np.float32)


def assert_bits(a, b, what):
    assert a.shape == b.shape, (what, a.shape, b.shape)
    if not np.array_equal(a, b):
        diff = np.argwhere(a != b)
        raise AssertionError("%s: %d of %d elements differ in their bits, first at %s"
                             % (what, len(diff), a.size, tuple(diff[0])))


def f32_bits(t):
    torch.cuda.synchronize()
    return t.contiguous().view(torch.int32).cpu().numpy()


# ---------------------------------------------------------------------------------------------------------------------
# entry points: frame i of a batch of N == the same frame alone
# ---------------------------------------------------------------------------------------------------------------------
def _conv_weights(cin, cout, seed, up2=False):
    rng = np.random.default_rng(seed)
    k = (rng.normal(0, 1, (3, 3, cin, cout)) * np.sqrt(2.0 / (9 * cin))).astype(np.float32)
    b = rng.normal(0, 0.3, cout).astype(np.float32)
    d_k, d_b = U.dev(k), U.dev(b)
    lib = U.lib()
    if up2:
        wsp = torch.empty(lib.wctb200_conv_weight_bytes(16, cin, cout), dtype=torch.uint8, device="cuda")
        _capi.check(lib.wctb200_prep_conv_weights_up2(d_k.data_ptr(), cin, cout, wsp.data_ptr(), U.stream()))
    else:
        wsp = torch.empty(lib.wctb200_conv_weight_bytes(9, cin, cout), dtype=torch.uint8, device="cuda")
        _capi.check(lib.wctb200_prep_conv_weights(d_k.data_ptr(), 9, cin, cout, wsp.data_ptr(), U.stream()))
    return wsp, d_b


@pytest.mark.parametrize("flags", [_capi.RELU, _capi.RELU | _capi.POOL2, _capi.RELU | _capi.HALO_EDGE, 0],
                         ids=["plain", "pool2", "halo_edge", "linear"])
@pytest.mark.parametrize("shape", [(64, 96, 64, 64), (33, 47, 128, 256), (16, 24, 512, 512)], ids=lambda s: "x".join(map(str, s)))
def test_conv3x3_batch_equals_single(shape, flags):
    h, w, cin, cout = shape
    lib = U.lib()
    xin = U.act_from_numpy(feats(N, h, w, cin, 1))
    wsp, d_b = _conv_weights(cin, cout, 2)
    ho, wo = ((h + 1) // 2, (w + 1) // 2) if flags & _capi.POOL2 else (h, w)
    out = U.act_alloc(N, ho, wo, cout)
    _capi.check(lib.wctb200_conv3x3(xin.data_ptr(), N, h, w, cin, wsp.data_ptr(), d_b.data_ptr(), cout, flags, out.data_ptr(), U.stream()))
    batch = planes(out, N, ho, wo, cout)
    for i in range(N):
        one = U.act_alloc(1, ho, wo, cout)
        _capi.check(lib.wctb200_conv3x3(frame_copy(xin, i, N, h, w, cin).data_ptr(), 1, h, w, cin, wsp.data_ptr(), d_b.data_ptr(),
                                        cout, flags, one.data_ptr(), U.stream()))
        assert_bits(planes(one, 1, ho, wo, cout)[:, 0], batch[:, i], "conv3x3 frame %d" % i)
    U.check_device()


@pytest.mark.parametrize("shape", [(32, 48, 64, 64), (17, 23, 256, 128), (8, 12, 512, 512)], ids=lambda s: "x".join(map(str, s)))
def test_conv3x3_up2_batch_equals_single(shape):
    h, w, cin, cout = shape
    lib = U.lib()
    xin = U.act_from_numpy(feats(N, h, w, cin, 3))
    wup, d_b = _conv_weights(cin, cout, 4, up2=True)
    out = U.act_alloc(N, 2 * h, 2 * w, cout)
    _capi.check(lib.wctb200_conv3x3_up2(xin.data_ptr(), N, h, w, cin, wup.data_ptr(), d_b.data_ptr(), cout, _capi.RELU,
                                        out.data_ptr(), U.stream()))
    batch = planes(out, N, 2 * h, 2 * w, cout)
    for i in range(N):
        one = U.act_alloc(1, 2 * h, 2 * w, cout)
        _capi.check(lib.wctb200_conv3x3_up2(frame_copy(xin, i, N, h, w, cin).data_ptr(), 1, h, w, cin, wup.data_ptr(), d_b.data_ptr(),
                                            cout, _capi.RELU, one.data_ptr(), U.stream()))
        assert_bits(planes(one, 1, 2 * h, 2 * w, cout)[:, 0], batch[:, i], "conv3x3_up2 frame %d" % i)
    U.check_device()


@pytest.mark.parametrize("hw", [(64, 96), (37, 53), (128, 130)], ids=lambda s: "x".join(map(str, s)))
def test_conv_head_batch_equals_single(hw):
    h, w = hw
    rng = np.random.default_rng(5)
    img = U.dev(rng.random((N, h, w, 3)).astype(np.float32))
    wf = U.dev((rng.standard_normal((27, 64)) * 0.3).astype(np.float32))
    bf = U.dev(rng.standard_normal(64).astype(np.float32) * 0.1)
    lib = U.lib()
    out = U.act_alloc(N, h, w, 64)
    _capi.check(lib.wctb200_conv_head(img.data_ptr(), N, h, w, wf.data_ptr(), bf.data_ptr(), out.data_ptr(), U.stream()))
    batch = planes(out, N, h, w, 64)
    for i in range(N):
        one = U.act_alloc(1, h, w, 64)
        x1 = img[i:i + 1].contiguous()
        _capi.check(lib.wctb200_conv_head(x1.data_ptr(), 1, h, w, wf.data_ptr(), bf.data_ptr(), one.data_ptr(), U.stream()))
        assert_bits(planes(one, 1, h, w, 64)[:, 0], batch[:, i], "conv_head frame %d" % i)
    U.check_device()


@pytest.mark.parametrize("clip", [False, True])
@pytest.mark.parametrize("shape", [(64, 96, 64), (37, 45, 64), (70, 300, 64), (40, 33, 128)], ids=lambda s: "x".join(map(str, s)))
def test_conv_tail_batch_equals_single(shape, clip):
    h, w, c = shape
    rng = np.random.default_rng(6)
    xin = U.act_from_numpy(feats(N, h, w, c, 7))
    k = U.dev((rng.normal(0, 1, (9 * c, 3)) * 0.05).astype(np.float32))
    b = U.dev(np.array([0.5, 0.4, 0.6], dtype=np.float32))
    flags = _capi.CLIP01 if clip else 0
    lib = U.lib()
    img = torch.full((N, h, w, 3), float("nan"), dtype=torch.float32, device="cuda")
    _capi.check(lib.wctb200_conv_tail(xin.data_ptr(), N, h, w, c, k.data_ptr(), b.data_ptr(), flags, img.data_ptr(), U.stream()))
    batch = f32_bits(img)
    for i in range(N):
        one = torch.full((1, h, w, 3), float("nan"), dtype=torch.float32, device="cuda")
        _capi.check(lib.wctb200_conv_tail(frame_copy(xin, i, N, h, w, c).data_ptr(), 1, h, w, c, k.data_ptr(), b.data_ptr(), flags,
                                          one.data_ptr(), U.stream()))
        assert_bits(f32_bits(one)[0], batch[i], "conv_tail frame %d" % i)
    U.check_device()


@pytest.mark.parametrize("shape", [(64, 96, 64), (33, 47, 256), (16, 24, 512), (128, 128, 128)], ids=lambda s: "x".join(map(str, s)))
def test_covariance_batch_equals_single(shape):
    h, w, c = shape
    lib = U.lib()
    xin = U.act_from_numpy(feats(N, h, w, c, 8))
    mean = torch.empty((N, c), dtype=torch.float32, device="cuda")
    cov = torch.empty((N, c, c), dtype=torch.float32, device="cuda")
    _capi.check(lib.wctb200_covariance(xin.data_ptr(), N, h, w, c, 1e-8, mean.data_ptr(), cov.data_ptr(), U.stream()))
    bm, bc = f32_bits(mean), f32_bits(cov)
    for i in range(N):
        m1 = torch.empty((1, c), dtype=torch.float32, device="cuda")
        c1 = torch.empty((1, c, c), dtype=torch.float32, device="cuda")
        _capi.check(lib.wctb200_covariance(frame_copy(xin, i, N, h, w, c).data_ptr(), 1, h, w, c, 1e-8, m1.data_ptr(), c1.data_ptr(),
                                           U.stream()))
        assert_bits(f32_bits(m1)[0], bm[i], "covariance mean frame %d" % i)
        assert_bits(f32_bits(c1)[0], bc[i], "covariance frame %d" % i)
    U.check_device()


def _wct_level(cin, nc, hc, wc, sin, ns, hs, ws_, c, sem, alpha=0.7):
    eps_cov, eps_eig, thresh, readd = SEMS[sem]
    out = U.act_alloc(nc, hc, wc, c)
    ws = torch.empty(U.lib().wctb200_wct_workspace_bytes(c, nc, ns), dtype=torch.uint8, device="cuda")
    k = torch.full((2 * (nc + ns),), -7, dtype=torch.int32, device="cuda")
    _capi.check(U.lib().wctb200_wct_level(cin.data_ptr(), nc, hc, wc, sin.data_ptr(), ns, hs, ws_, c, alpha, eps_cov, eps_eig, thresh,
                                          readd, out.data_ptr(), k.data_ptr(), ws.data_ptr(), ws.numel(), U.stream()))
    return planes(out, nc, hc, wc, c), k.cpu().numpy()


def _split_k(k, nc, ns):
    """k_out -> (k_c [nc], k_s [ns], sweeps_c [nc], sweeps_s [ns])"""
    return k[:nc], k[nc:nc + ns], k[nc + ns:2 * nc + ns], k[2 * nc + ns:]


WCT_SHAPES = [(40, 56, 24, 36, 64), (24, 20, 18, 26, 256), (16, 12, 14, 10, 512)]    # hc, wc, hs, ws, C (C = 512: HW < C)


@pytest.mark.parametrize("shared_style", [True, False], ids=["Ns1", "NsNc"])
@pytest.mark.parametrize("sem", ["tf", "np"])
@pytest.mark.parametrize("shape", WCT_SHAPES, ids=lambda s: "C%d" % s[4])
def test_wct_level_batch_equals_single(shape, sem, shared_style):
    hc, wc, hs, ws_, c = shape
    ns = 1 if shared_style else N
    cin = U.act_from_numpy(feats(N, hc, wc, c, 11))
    sin = U.act_from_numpy(feats(ns, hs, ws_, c, 12))
    batch, kb = _wct_level(cin, N, hc, wc, sin, ns, hs, ws_, c, sem)
    kc, ks, swc, sws = _split_k(kb, N, ns)
    for i in range(N):
        si = 0 if shared_style else i
        s1 = sin if shared_style else frame_copy(sin, i, ns, hs, ws_, c)
        one, k1 = _wct_level(frame_copy(cin, i, N, hc, wc, c), 1, hc, wc, s1, 1, hs, ws_, c, sem)
        assert_bits(one[:, 0], batch[:, i], "wct_level %s frame %d" % (sem, i))
        assert k1.tolist() == [kc[i], ks[si], swc[i], sws[si]], (i, k1, kb)
    U.check_device()


@pytest.mark.parametrize("shared_style", [True, False], ids=["Ns1", "NsNc"])
@pytest.mark.parametrize("shape", WCT_SHAPES[:2], ids=lambda s: "C%d" % s[4])
def test_wct_prepare_apply_batch_equals_single(shape, shared_style):
    hc, wc, hs, ws_, c = shape
    ns = 1 if shared_style else N
    lib = U.lib()
    eps_cov, eps_eig, thresh, readd = SEMS["tf"]
    cin = U.act_from_numpy(feats(N, hc, wc, c, 13))
    sin = U.act_from_numpy(feats(ns, hs, ws_, c, 14))

    def run(content, nc, style, n_s):
        ws = torch.empty(lib.wctb200_wct_workspace_bytes(c, nc, n_s), dtype=torch.uint8, device="cuda")
        state = torch.empty(lib.wctb200_wct_style_state_bytes(c, n_s), dtype=torch.uint8, device="cuda")
        _capi.check(lib.wctb200_wct_style_prepare(style.data_ptr(), n_s, hs, ws_, c, eps_cov, eps_eig, thresh, state.data_ptr(),
                                                  ws.data_ptr(), ws.numel(), U.stream()))
        out = U.act_alloc(nc, hc, wc, c)
        k = torch.full((2 * (nc + n_s),), -7, dtype=torch.int32, device="cuda")
        _capi.check(lib.wctb200_wct_apply(content.data_ptr(), nc, hc, wc, c, state.data_ptr(), n_s, 0.7, eps_cov, eps_eig, thresh, readd,
                                          out.data_ptr(), k.data_ptr(), ws.data_ptr(), ws.numel(), U.stream()))
        return planes(out, nc, hc, wc, c), k.cpu().numpy()

    batch, kb = run(cin, N, sin, ns)
    kc, ks, swc, sws = _split_k(kb, N, ns)
    for i in range(N):
        si = 0 if shared_style else i
        s1 = sin if shared_style else frame_copy(sin, i, ns, hs, ws_, c)
        one, k1 = run(frame_copy(cin, i, N, hc, wc, c), 1, s1, 1)
        assert_bits(one[:, 0], batch[:, i], "wct_apply frame %d" % i)
        assert k1.tolist() == [kc[i], ks[si], swc[i], sws[si]], (i, k1, kb)
    U.check_device()


def _adain(cin, nc, hc, wc, sin, ns, hs, ws_, c, alpha=0.8):
    out = U.act_alloc(nc, hc, wc, c)
    ws = torch.empty(U.lib().wctb200_wct_workspace_bytes(c, nc, ns), dtype=torch.uint8, device="cuda")
    _capi.check(U.lib().wctb200_adain_level(cin.data_ptr(), nc, hc, wc, sin.data_ptr(), ns, hs, ws_, c, alpha, 1e-5, out.data_ptr(),
                                            ws.data_ptr(), ws.numel(), U.stream()))
    return planes(out, nc, hc, wc, c)


@pytest.mark.parametrize("shared_style", [True, False], ids=["Ns1", "NsNc"])
@pytest.mark.parametrize("shape", [(64, 96, 48, 40, 64), (32, 48, 30, 20, 128), (16, 24, 12, 20, 512)], ids=lambda s: "C%d" % s[4])
def test_adain_level_batch_equals_single(shape, shared_style):
    """64x96 at C = 64 is a map where the batch size used to change how a frame's pixels were split between CTAs."""
    hc, wc, hs, ws_, c = shape
    ns = 1 if shared_style else N
    cin = U.act_from_numpy(feats(N, hc, wc, c, 15))
    sin = U.act_from_numpy(feats(ns, hs, ws_, c, 16))
    batch = _adain(cin, N, hc, wc, sin, ns, hs, ws_, c)
    for i in range(N):
        s1 = sin if shared_style else frame_copy(sin, i, ns, hs, ws_, c)
        one = _adain(frame_copy(cin, i, N, hc, wc, c), 1, hc, wc, s1, 1, hs, ws_, c)
        assert_bits(one[:, 0], batch[:, i], "adain_level frame %d" % i)
    U.check_device()


# ---------------------------------------------------------------------------------------------------------------------
# repeat runs: the same call twice gives the same bytes
# ---------------------------------------------------------------------------------------------------------------------
def test_adain_level_repeat_runs_equal():
    """1 x 256 x 256 x 64: hundreds of CTAs contribute to every channel's moments."""
    cin = U.act_from_numpy(feats(1, 256, 256, 64, 17, offset=2.0))
    sin = U.act_from_numpy(feats(1, 256, 256, 64, 18))
    first = _adain(cin, 1, 256, 256, sin, 1, 256, 256, 64)
    for r in range(3):
        assert_bits(_adain(cin, 1, 256, 256, sin, 1, 256, 256, 64), first, "adain_level run %d" % (r + 1))
    U.check_device()


def test_wct_level_repeat_runs_equal():
    """relu1_1 of a 512 x 512 frame: 64 covariance CTAs per frame, full split-K."""
    cin = U.act_from_numpy(feats(1, 512, 512, 64, 19))
    sin = U.act_from_numpy(feats(1, 256, 256, 64, 20))
    first, k0 = _wct_level(cin, 1, 512, 512, sin, 1, 256, 256, 64, "tf")
    for r in range(2):
        again, k = _wct_level(cin, 1, 512, 512, sin, 1, 256, 256, 64, "tf")
        assert_bits(again, first, "wct_level run %d" % (r + 1))
        assert k.tolist() == k0.tolist()
    U.check_device()


# ---------------------------------------------------------------------------------------------------------------------
# the engine: batch == single frames, every level, every transform
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def weights():
    return make_synthetic_weights(42)


def _imgs(n, h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, h, w, 3), dtype=np.uint8)


def _act_bits(a, i=None):
    p = planes(a.buf, a.N, a.H, a.W, a.C)
    return p if i is None else p[:, i]


def _stylize(eng, content, style, capture=None, **kw):
    cap = {} if capture else None
    out = eng.stylize(torch.from_numpy(content).cuda(), torch.from_numpy(style).cuda(), alpha=0.7, capture=cap, **kw)
    eng.check_device()
    return f32_bits(out), cap


def _assert_capture_frame(cap_b, i, cap_1, what):
    for key in ("content_feat", "transformed"):
        for lvl, (ab, a1) in enumerate(zip(cap_b[key], cap_1[key])):
            assert_bits(_act_bits(a1, 0), _act_bits(ab, i), "%s: %s level %d frame %d" % (what, key, lvl, i))
    for key in ("level_input", "level_output"):
        for lvl, (tb, t1) in enumerate(zip(cap_b[key], cap_1[key])):
            assert_bits(f32_bits(t1)[0], f32_bits(tb)[i], "%s: %s level %d frame %d" % (what, key, lvl, i))


@pytest.mark.parametrize("mode", ["tf", "np", "adain"])
@pytest.mark.parametrize("shared_style", [False, True], ids=["per_frame_styles", "one_style"])
def test_engine_batch_equals_single_frames(weights, mode, shared_style):
    eng = Engine(weights, ALL, semantics="np" if mode == "np" else "tf")
    adain = mode == "adain"
    contents = _imgs(4, 96, 64, 31)
    styles = _imgs(1 if shared_style else 4, 80, 72, 32)
    out, cap = _stylize(eng, contents, styles, capture=True, adain=adain)
    for i in range(4):
        s = styles if shared_style else styles[i:i + 1]
        one, cap1 = _stylize(eng, contents[i:i + 1], s, capture=True, adain=adain)
        assert_bits(one[0], out[i], "%s output frame %d" % (mode, i))
        _assert_capture_frame(cap, i, cap1, mode)


def test_engine_swap5_independent_of_other_calls(weights):
    """Style swap takes one content/style pair per call: a frame gives the same bits, every level's features included, whatever
    ran before it on the engine."""
    t5 = ["relu5_1", "relu3_1", "relu1_1"]
    w5 = make_synthetic_weights(15, relu_targets=t5)
    eng = Engine(w5, t5, semantics="tf")
    contents, style = _imgs(3, 64, 64, 33), _imgs(1, 72, 64, 34)
    kw = dict(swap5=True, ss_patch_size=3, ss_stride=1)
    first = [_stylize(eng, contents[i:i + 1], style, capture=True, **kw) for i in range(3)]
    _stylize(eng, _imgs(1, 96, 80, 35), _imgs(1, 64, 64, 36), **kw)           # other sizes in between
    for i in (2, 0, 1):
        out, cap = _stylize(eng, contents[i:i + 1], style, capture=True, **kw)
        assert_bits(out, first[i][0], "swap5 output frame %d" % i)
        _assert_capture_frame(first[i][1], 0, cap, "swap5")


@pytest.mark.parametrize("mode", ["tf", "adain"])
def test_engine_groups_equal_bytes(weights, mode):
    """Engine.groups only changes the schedule: sub-batches on independent stream pairs give the same bytes."""
    eng = Engine(weights, ALL, semantics="tf")
    adain = mode == "adain"
    contents = _imgs(4, 64, 80, 41)
    for styles in (_imgs(4, 72, 64, 42), _imgs(1, 72, 64, 43)):
        res = {}
        for g in (1, 2, 4):
            eng.groups = g
            res[g], _ = _stylize(eng, contents, styles, adain=adain)
        eng.groups = 1
        assert_bits(res[2], res[1], "groups 2 vs 1")
        assert_bits(res[4], res[1], "groups 4 vs 1")


def test_predict_batch_adain_equals_per_frame_predict(weights):
    """WCT.predict_batch runs its batch as two stream groups; AdaIN's moments must not depend on that split."""
    targets = ["relu3_1", "relu2_1", "relu1_1"]
    wct = WCT(checkpoints=None, relu_targets=targets, vgg_path=None, weights=weights)
    c, s = _imgs(5, 64, 72, 51), _imgs(1, 56, 48, 52)
    batch = wct.predict_batch(c, s, alpha=0.7, adain=True)
    for i in range(5):
        assert np.array_equal(wct.predict(c[i], s[0], alpha=0.7, adain=True), batch[i]), i
