"""Prepared styles on the GPU: the split entry points and ``WCT.prepare_style`` / ``load_style`` give the bytes of the
one-shot calls.  Every comparison is exact, on raw bits (both SPF16 planes with the halo, ``k_out``) or on uint8 frames."""
import ctypes

import numpy as np
import pytest
import torch

from wct_tf_b200 import _capi
from wct_tf_b200.model import RELU_CHANNELS
from wct_tf_b200.prepared import unpack_adain_state, unpack_wct_state
from wct_tf_b200.wct import WCT
from wct_tf_b200.weights import make_synthetic_weights
from tests import gpu_util as U
from tests.test_gpu_invariance import assert_bits, f32_bits, feats, frame_copy, planes

pytestmark = pytest.mark.gpu
ALL = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]
TF = (1e-8, 1e-5)                 # eps_cov, thresh of the style swap (the TF graph's)


def _imgs(n, h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, h, w, 3), dtype=np.uint8)


def _ws(nbytes):
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device="cuda")


# ------------------------------------------------------------------------------------------------------------------- AdaIN
@pytest.mark.parametrize("c", [64, 128, 256, 512])
@pytest.mark.parametrize("ns", [1, 3], ids=["shared", "per_frame"])
def test_adain_prepare_apply_equals_level(c, ns):
    lib = U.lib()
    nc, hc, wc, hs, ws_ = 3, 19, 23, 17, 29
    content = U.act_from_numpy(feats(nc, hc, wc, c, 1))
    style = U.act_from_numpy(feats(ns, hs, ws_, c, 2, offset=0.5))
    ref = U.act_alloc(nc, hc, wc, c)
    ws = _ws(lib.wctb200_wct_workspace_bytes(c, nc, ns))
    _capi.check(lib.wctb200_adain_level(content.data_ptr(), nc, hc, wc, style.data_ptr(), ns, hs, ws_, c, 0.7, 1e-5, ref.data_ptr(),
                                        ws.data_ptr(), ws.numel(), U.stream()))
    om, ov = ctypes.c_size_t(), ctypes.c_size_t()
    nbytes = lib.wctb200_adain_style_state_layout(c, ns, ctypes.byref(om), ctypes.byref(ov))
    assert nbytes == lib.wctb200_adain_style_state_bytes(c, ns) and om.value == 0 and ov.value >= ns * c * 4
    state = _ws(nbytes)
    _capi.check(lib.wctb200_adain_style_prepare(style.data_ptr(), ns, hs, ws_, c, state.data_ptr(), U.stream()))
    out = U.act_alloc(nc, hc, wc, c)
    ws2 = _ws(lib.wctb200_wct_workspace_bytes(c, nc, 0))
    _capi.check(lib.wctb200_adain_apply(content.data_ptr(), nc, hc, wc, c, state.data_ptr(), ns, 0.7, 1e-5, out.data_ptr(),
                                        ws2.data_ptr(), ws2.numel(), U.stream()))
    assert_bits(planes(out, nc, hc, wc, c), planes(ref, nc, hc, wc, c), "adain_apply")
    assert lib.wctb200_adain_apply(content.data_ptr(), nc, hc, wc, c, None, ns, 0.7, 1e-5, out.data_ptr(), ws2.data_ptr(),
                                   ws2.numel(), U.stream()) == _capi.EINVAL
    U.check_device()


@pytest.mark.parametrize("c", [64, 128, 256, 512])
@pytest.mark.parametrize("nw", [1, 3], ids=["shared_row", "per_frame_rows"])
def test_adain_apply_blend_equals_blend(c, nw):
    lib = U.lib()
    nc, hc, wc, K = 3, 21, 18, 3
    sizes = [(17, 29), (24, 20), (9, 13)]
    content = U.act_from_numpy(feats(nc, hc, wc, c, 3))
    styles = [U.act_from_numpy(feats(1, h, w, c, 10 + k, offset=0.2 * k)) for k, (h, w) in enumerate(sizes)]
    wts = U.dev(np.random.default_rng(4).random((nw, K)).astype(np.float32))
    ref = U.act_alloc(nc, hc, wc, c)
    ws = _ws(lib.wctb200_adain_blend_workspace_bytes(c, nc, K))
    _capi.check(lib.wctb200_adain_blend(content.data_ptr(), nc, hc, wc, c, _capi.pointer_array([s.data_ptr() for s in styles]),
                                        _capi.int_array([h for h, _ in sizes]), _capi.int_array([w for _, w in sizes]), K,
                                        wts.data_ptr(), nw, 0.8, 1e-5, ref.data_ptr(), ws.data_ptr(), ws.numel(), U.stream()))
    states = []
    for s, (h, w) in zip(styles, sizes):
        st = _ws(lib.wctb200_adain_style_state_bytes(c, 1))
        _capi.check(lib.wctb200_adain_style_prepare(s.data_ptr(), 1, h, w, c, st.data_ptr(), U.stream()))
        states.append(st)
    out = U.act_alloc(nc, hc, wc, c)
    ws2 = _ws(lib.wctb200_wct_workspace_bytes(c, nc, 0))
    ptrs = _capi.pointer_array([s.data_ptr() for s in states])
    _capi.check(lib.wctb200_adain_apply_blend(content.data_ptr(), nc, hc, wc, c, ptrs, K, wts.data_ptr(), nw, 0.8, 1e-5,
                                              out.data_ptr(), ws2.data_ptr(), ws2.numel(), U.stream()))
    assert_bits(planes(out, nc, hc, wc, c), planes(ref, nc, hc, wc, c), "adain_apply_blend")
    for bad_k in (0, 9):
        assert lib.wctb200_adain_apply_blend(content.data_ptr(), nc, hc, wc, c, ptrs, bad_k, wts.data_ptr(), nw, 0.8, 1e-5,
                                             out.data_ptr(), ws2.data_ptr(), ws2.numel(), U.stream()) == _capi.EINVAL
    assert lib.wctb200_adain_apply_blend(content.data_ptr(), nc, hc, wc, c, ptrs, K, wts.data_ptr(), 2, 0.8, 1e-5,
                                         out.data_ptr(), ws2.data_ptr(), ws2.numel(), U.stream()) == _capi.EINVAL
    U.check_device()


def test_wct_style_state_layout():
    lib = U.lib()
    for c, ns in [(64, 1), (128, 3), (512, 2)]:
        om, oc, ok = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_size_t()
        total = lib.wctb200_wct_style_state_layout(c, ns, ctypes.byref(om), ctypes.byref(oc), ctypes.byref(ok))
        assert total == lib.wctb200_wct_style_state_bytes(c, ns)
        assert om.value == 0 and oc.value >= ns * c * 4 and ok.value >= oc.value + ns * c * c * 4 and total >= ok.value + 8 * ns
    assert lib.wctb200_wct_style_state_layout(64, 0, None, None, None) == 0


# -------------------------------------------------------------------------------------------------------------- style swap
SWAP_CASES = [  # C, content h x w, style h x w, patch, stride
    (512, (12, 15), (14, 11), 3, 1),
    (256, (17, 21), (19, 16), 5, 2),
    (128, (16, 18), (20, 17), 9, 1),
    (64, (20, 22), (24, 19), 13, 1),
]


@pytest.mark.parametrize("case", SWAP_CASES, ids=lambda k: "c%d_p%d_s%d" % (k[0], k[3], k[4]))
@pytest.mark.parametrize("nc", [1, 3, 5])
def test_style_swap_prepare_apply_equals_level(case, nc):
    """Frame i of one batched apply == style_swap_level on frame i alone, k_out included."""
    lib = U.lib()
    c, (hc, wc), (hs, ws_), p, s = case
    content = U.act_from_numpy(feats(nc, hc, wc, c, 21))
    style = U.act_from_numpy(feats(1, hs, ws_, c, 22, offset=0.4))
    state = _ws(lib.wctb200_style_swap_state_bytes(c, hs, ws_, p, s))
    pws = _ws(lib.wctb200_style_swap_prepare_workspace_bytes(c, hs, ws_, p, s))
    kprep = torch.full((1,), -7, dtype=torch.int32, device="cuda")
    _capi.check(lib.wctb200_style_swap_prepare(style.data_ptr(), hs, ws_, c, p, s, *TF, state.data_ptr(), kprep.data_ptr(),
                                               pws.data_ptr(), pws.numel(), U.stream()))
    before = state.clone()
    out = U.act_alloc(nc, hc, wc, c)
    aws = _ws(lib.wctb200_style_swap_apply_workspace_bytes(c, nc, hc, wc, hs, ws_, p, s))
    kout = torch.full((nc + 1,), -7, dtype=torch.int32, device="cuda")
    _capi.check(lib.wctb200_style_swap_apply(content.data_ptr(), nc, hc, wc, c, state.data_ptr(), hs, ws_, p, s, 0.6, *TF,
                                             out.data_ptr(), kout.data_ptr(), aws.data_ptr(), aws.numel(), U.stream()))
    batch = planes(out, nc, hc, wc, c)
    kb = kout.cpu().numpy()
    assert torch.equal(state, before), "the apply wrote its state"
    for i in range(nc):
        one = U.act_alloc(1, hc, wc, c)
        lws = _ws(lib.wctb200_style_swap_workspace_bytes(c, hc, wc, hs, ws_, p, s))
        k1 = torch.full((2,), -7, dtype=torch.int32, device="cuda")
        _capi.check(lib.wctb200_style_swap_level(frame_copy(content, i, nc, hc, wc, c).data_ptr(), hc, wc, style.data_ptr(), hs, ws_,
                                                 c, p, s, 0.6, *TF, one.data_ptr(), k1.data_ptr(), lws.data_ptr(), lws.numel(),
                                                 U.stream()))
        assert_bits(planes(one, 1, hc, wc, c)[:, 0], batch[:, i], "style_swap_apply frame %d" % i)
        k1 = k1.cpu().numpy()
        assert (kb[i], kb[nc]) == (k1[0], k1[1]) and k1[1] == kprep.cpu().numpy()[0] and k1[0] > 0
    U.check_device()


def test_style_swap_split_rejections():
    lib = U.lib()
    c, hc, wc, hs, ws_ = 64, 12, 12, 10, 10
    content = U.act_from_numpy(feats(2, hc, wc, c, 5))
    style = U.act_from_numpy(feats(1, hs, ws_, c, 6))
    state = _ws(lib.wctb200_style_swap_state_bytes(c, hs, ws_, 3, 1))
    pws = _ws(lib.wctb200_style_swap_prepare_workspace_bytes(c, hs, ws_, 3, 1))
    _capi.check(lib.wctb200_style_swap_prepare(style.data_ptr(), hs, ws_, c, 3, 1, *TF, state.data_ptr(), None, pws.data_ptr(),
                                               pws.numel(), U.stream()))
    out = U.act_alloc(2, hc, wc, c)
    aws = _ws(lib.wctb200_style_swap_apply_workspace_bytes(c, 2, hc, wc, hs, ws_, 3, 1))

    def apply(nc=2, st=state, p=3, s=1):
        return lib.wctb200_style_swap_apply(content.data_ptr(), nc, hc, wc, c, st.data_ptr() if st is not None else None, hs, ws_,
                                            p, s, 0.6, *TF, out.data_ptr(), None, aws.data_ptr(), aws.numel(), U.stream())
    assert apply() == 0
    assert apply(st=None) == _capi.EINVAL
    assert apply(nc=0) == _capi.EINVAL
    assert apply(p=3, s=2) == _capi.EINVAL              # (12 - 3) is odd: stride 2 does not tile 12
    assert apply(p=17) == _capi.EINVAL
    assert lib.wctb200_style_swap_state_bytes(c, 2, 2, 3, 1) == 0
    assert lib.wctb200_style_swap_prepare(style.data_ptr(), hs, ws_, c, 11, 1, *TF, state.data_ptr(), None, pws.data_ptr(),
                                          pws.numel(), U.stream()) == _capi.EINVAL
    U.check_device()


# -------------------------------------------------------------------------------------------------------------- the model
@pytest.fixture(scope="module")
def weights():
    return make_synthetic_weights(42)


@pytest.fixture(scope="module")
def wct_tf(weights):
    return WCT(relu_targets=ALL, weights=weights)


@pytest.mark.parametrize("sem", ["tf", "np"])
@pytest.mark.parametrize("mode", ["wct", "adain", "passes2"])
def test_predict_batch_prepared_equals_image(weights, sem, mode):
    wct = WCT(relu_targets=ALL, weights=weights, semantics=sem)
    c, s = _imgs(3, 64, 80, 1), _imgs(1, 72, 56, 2)
    kw = dict(alpha=0.8, adain=mode == "adain", passes=2 if mode == "passes2" else 1)
    ps = wct.prepare_style(s)
    assert ps.n == 1 and ps.image.shape == s.shape and np.array_equal(ps.image, s)
    assert np.array_equal(wct.predict_batch(c, ps, **kw), wct.predict_batch(c, s, **kw))
    assert np.array_equal(wct.predict(c[0], ps, alpha=0.8), wct.predict(c[0], s[0], alpha=0.8))


@pytest.mark.parametrize("adain", [False, True], ids=["wct", "adain"])
def test_per_frame_prepared_styles(wct_tf, adain):
    c, s = _imgs(4, 48, 64, 3), _imgs(4, 56, 40, 4)
    ps = wct_tf.prepare_style(torch.from_numpy(s).cuda())
    assert ps.n == 4
    assert np.array_equal(wct_tf.predict_batch(c, ps, adain=adain, passes=2), wct_tf.predict_batch(c, s, adain=adain, passes=2))


@pytest.mark.parametrize("adain", [False, True], ids=["wct", "adain"])
@pytest.mark.parametrize("rows", ["shared", "per_frame"])
def test_interpolation_with_prepared_styles(wct_tf, adain, rows):
    c = _imgs(3, 48, 48, 5)
    styles = [_imgs(1, 40 + 8 * k, 48, 6 + k)[0] for k in range(3)]
    w = np.array([0.2, 0.5, 0.3]) if rows == "shared" else np.random.default_rng(7).random((3, 3)) + 0.1
    prepared = [wct_tf.prepare_style(x) for x in styles]
    mixed = [prepared[0], styles[1], prepared[2]]
    ref = wct_tf.predict_batch(c, styles, adain=adain, style_weights=w)
    assert np.array_equal(wct_tf.predict_batch(c, prepared, adain=adain, style_weights=w), ref)
    assert np.array_equal(wct_tf.predict_batch(c, mixed, adain=adain, style_weights=w), ref)


def test_mask_with_prepared_styles(wct_tf):
    c = _imgs(2, 64, 48, 8)
    styles = [_imgs(1, 40, 40, 9)[0], _imgs(1, 56, 32, 10)[0]]
    mask = (np.arange(64)[:, None] + np.arange(48)[None] > 50).astype(np.uint8)
    ref = wct_tf.predict_batch(c, styles, content_mask=mask, passes=2)
    assert np.array_equal(wct_tf.predict_batch(c, [wct_tf.prepare_style(x) for x in styles], content_mask=mask, passes=2), ref)


def test_synthesize_with_prepared_style(wct_tf):
    s = _imgs(1, 64, 64, 11)[0]
    ps = wct_tf.prepare_style(s)
    assert np.array_equal(wct_tf.synthesize(ps, (48, 40), count=3, seed=5), wct_tf.synthesize(s, (48, 40), count=3, seed=5))


@pytest.mark.parametrize("refit", [False, True], ids=["p3s1", "p3s2_refit"])
@pytest.mark.parametrize("adain", [False, True], ids=["wct", "adain"])
def test_swap5_batched_equals_single_frames(weights, refit, adain):
    """One shared style, N = 4 frames: one batched swap per sub-batch == four single-frame calls, and a prepared style
    gives the same bytes; with stride 2 the content is refitted (centre-cropped) first."""
    wct = WCT(relu_targets=ALL, weights=weights, ss_patch_size=3, ss_stride=2 if refit else 1)
    c, s = _imgs(4, 96 if refit else 80, 112, 12), _imgs(1, 96, 80, 13)
    kw = dict(alpha=0.7, adain=adain, swap5=True, ss_alpha=0.5)
    batch = wct.predict_batch(c, s, **kw)
    assert batch.shape[1:3] == ((80, 112) if refit else (80, 112))
    singles = np.stack([wct.predict_batch(c[i], s, **kw)[0] for i in range(4)])
    assert np.array_equal(batch, singles)
    ps = wct.prepare_style(s)
    assert np.array_equal(wct.predict_batch(c, ps, **kw), batch)
    assert np.array_equal(wct.predict_batch(c, ps, passes=2, **kw), wct.predict_batch(c, s, passes=2, **kw))
    # one style per frame: frame by frame, prepared or not
    s4 = _imgs(4, 64, 72, 14)
    assert np.array_equal(wct.predict_batch(c, wct.prepare_style(s4), **kw), wct.predict_batch(c, s4, **kw))


def test_save_load_round_trip(weights, tmp_path):
    wct = WCT(relu_targets=ALL, weights=weights)
    s = _imgs(2, 64, 56, 15)
    ps = wct.prepare_style(s)
    path = str(tmp_path / "two.wctstyle")
    ps.save(path)
    loaded = wct.load_style(path)
    assert loaded.n == 2 and np.array_equal(loaded.image, s)
    lib = U.lib()
    for relu in ALL:                    # every field of the states, bit for bit (the alignment padding is not a field)
        c = RELU_CHANNELS[relu]
        for a, b in zip(unpack_wct_state(lib, loaded.wct[relu], c, 2) + unpack_adain_state(lib, loaded.adain[relu], c, 2),
                        unpack_wct_state(lib, ps.wct[relu], c, 2) + unpack_adain_state(lib, ps.adain[relu], c, 2)):
            assert_bits(a.view(np.int32), b.view(np.int32), relu)
    f = ps.feat5
    n2 = 2 * f.N * (f.H + 2) * (f.W + 2) * f.C * 2
    assert torch.equal(loaded.feat5.buf[:n2], ps.feat5.buf[:n2])
    c = _imgs(2, 64, 64, 16)
    for kw in (dict(), dict(adain=True), dict(swap5=True, ss_alpha=0.5), dict(passes=2)):
        assert np.array_equal(wct.predict_batch(c, loaded, **kw), wct.predict_batch(c, ps, **kw)), kw
    one = wct.prepare_style(s[0])
    one.save(path)
    # other decoders and a subset of the targets: the same encoder serves
    w2 = make_synthetic_weights(43)
    w2["vgg"] = weights["vgg"]
    sub = WCT(relu_targets=["relu4_1", "relu2_1"], weights=w2)
    got = sub.predict_batch(c, sub.load_style(path), alpha=0.9)
    assert np.array_equal(got, sub.predict_batch(c, s[0], alpha=0.9))
    # other encoder weights or other semantics: refused, naming the field
    with pytest.raises(ValueError, match="relu5_1/fingerprint|relu4_1/fingerprint"):
        WCT(relu_targets=ALL, weights=make_synthetic_weights(44)).load_style(path)
    with pytest.raises(ValueError, match="eps_cov"):
        WCT(relu_targets=ALL, weights=weights, semantics="np").load_style(path)
    # a prepared style of another model is refused in memory too
    with pytest.raises(ValueError, match="encoder"):
        WCT(relu_targets=ALL, weights=make_synthetic_weights(44)).predict_batch(c, one)
    with pytest.raises(ValueError, match="eps_cov"):
        WCT(relu_targets=ALL, weights=weights, semantics="np").predict_batch(c, one)


def test_state_read_only_and_independent_of_other_calls(wct_tf):
    """A prepared style's device bytes do not change in three applies, and its outputs do not depend on what ran in
    between (other styles, other sizes, other modes; in the manner of test_engine_swap5_independent_of_other_calls)."""
    s = _imgs(1, 64, 64, 17)
    ps = wct_tf.prepare_style(s)
    c = _imgs(3, 64, 48, 18)
    first = wct_tf.predict_batch(c, ps, swap5=True, ss_alpha=0.5)
    snap = [t.clone() for t in ps.tensors()]
    outs = []
    for k in range(3):
        wct_tf.predict_batch(_imgs(2, 80 + 16 * k, 64, 19 + k), _imgs(1, 48, 96, 30 + k), adain=bool(k % 2), swap5=k == 2)
        outs.append(wct_tf.predict_batch(c, ps, swap5=True, ss_alpha=0.5))
    torch.cuda.synchronize()
    for a, b in zip(snap, ps.tensors()):
        assert torch.equal(a, b)
    for o in outs:
        assert np.array_equal(o, first)
    del ps
    assert np.array_equal(wct_tf.predict_batch(c, s, swap5=True, ss_alpha=0.5), first)
