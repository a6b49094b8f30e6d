"""The softmax style swap (DESIGN.md §3.3.17) on the CPU: the float64 oracle's weights and limits, the option check, and
the API's forwarding of ``ss_temperature`` through a recording stub engine."""
import contextlib

import numpy as np
import pytest
import torch

from oracle import ref_ops
from tests import softmax_swap_ref as SR
from tests import swap_labels_ref as SLR
from wct_tf_b200 import options
from wct_tf_b200 import wct as W
from wct_tf_b200.engine import Engine
from wct_tf_b200.prepared import PreparedStyle


def _feats(seed, hc, hs, c=8):
    rng = np.random.default_rng(seed)
    content = np.maximum(rng.standard_normal((1, hc, hc, c)) + 0.3, 0)
    style = np.maximum(rng.standard_normal((1, hs, hs, c)) + 0.4, 0)
    return content, style


def _whitened(seed, hc, hs, c=8):
    content, style = _feats(seed, hc, hs, c)
    _, inf = ref_ops.wct_style_swap(content, style, 0.6, 3, 1, return_info=True)
    return inf["wc_feat"][0], inf["ws_feat"][0]


def _allowed(hc, hs, p, s, kc, ks):
    """The allowed sets of vertical stripes of kc labels on the content and ks labels on the style (label 2 absent from
    a two-label style)."""
    cl = (np.arange(hc)[None, :].repeat(hc, 0) * kc // hc).astype(np.uint8)
    sl = (np.arange(hs)[None, :].repeat(hs, 0) * ks // hs).astype(np.uint8)
    return SLR.allowed(SLR.anchor_labels(cl, hc, hc, p, s), SLR.patch_labels(sl, hs, hs, p, s))


@pytest.mark.parametrize("ps", [(3, 1), (5, 2)])
@pytest.mark.parametrize("tau", [1e-3, 0.05, 1.0])
def test_weights_sum_to_one_and_vanish_outside_the_allowed_set(ps, tau):
    p, s = ps
    hc, hs = (9, 10) if p == 3 else (11, 15)
    wc, ws = _whitened(3 * p + s, hc, hs)
    allowed = _allowed(hc, hs, p, s, 3, 2)
    assert (~allowed).any() and allowed.any(axis=2).all()
    for mask in (None, allowed):
        _, inf = SR.style_swap_softmax(wc, ws, p, s, tau, mask, return_info=True)
        w = inf["w"]
        assert np.allclose(w.sum(axis=2), 1.0, atol=1e-12)
        assert (w >= 0).all()
        if mask is not None:
            assert (w[~mask] == 0).all()


def test_z_is_scale_free_and_keeps_the_hard_ranking():
    wc, ws = _whitened(11, 9, 10)
    _, a = SR.style_swap_softmax(wc, ws, 3, 1, 0.05, return_info=True)
    _, b = SR.style_swap_softmax(7.5 * wc, ws, 3, 1, 0.05, return_info=True)
    assert np.allclose(a["z"], b["z"], rtol=1e-12, atol=1e-12)
    assert np.array_equal(a["z"].argmax(axis=2), a["scores"].argmax(axis=2))
    # every (tap, channel) column of the filters has unit norm, so |z| <= ||f_n|| / sqrt(K / n_p) and mean ||f_n||^2 <= K / n_p
    assert np.abs(a["z"]).max() <= np.sqrt(a["z"].shape[2]) + 1e-9


def test_a_zero_window_takes_the_uniform_mean():
    wc, ws = _whitened(5, 9, 10)
    wc = wc.copy()
    wc[:3, :3] = 0.0                                     # anchor (0, 0) sees only zeros
    _, inf = SR.style_swap_softmax(wc, ws, 3, 1, 0.01, return_info=True)
    assert inf["norms"][0, 0] == 0
    assert np.allclose(inf["w"][0, 0], 1.0 / inf["w"].shape[2])


def _margin_pixels(z, hc, wc, p, s, tau):
    """Pixels (Y, X) every covering anchor of which has a top-two gap of z above 50 tau."""
    top2 = np.sort(z, axis=2)[..., -2:]
    ok_a = (top2[..., 1] - top2[..., 0]) > 50 * tau
    ok = np.ones((hc, wc), bool)
    ho, wo = ok_a.shape
    for y in range(ho):
        for x in range(wo):
            if not ok_a[y, x]:
                ok[y * s:y * s + p, x * s:x * s + p] = False
    return ok


@pytest.mark.parametrize("ps", [(3, 1), (5, 2)])
def test_small_temperature_is_the_hard_swap(ps):
    p, s = ps
    hc, hs = (11, 12) if p == 3 else (11, 15)
    content, style = _feats(17 + p, hc, hs)
    tau = 1e-4
    got, inf = SR.wct_style_swap_softmax(content, style, 0.6, tau, p, s, return_info=True)
    ref = ref_ops.wct_style_swap(content, style, 0.6, p, s)
    ok = _margin_pixels(inf["z"], hc, hc, p, s, tau)
    assert ok.sum() > 0.5 * ok.size
    assert np.allclose(got[0][ok], ref[0][ok], rtol=1e-9, atol=1e-9)
    hard_sw, _ = ref_ops.style_swap(inf["wc_feat"], inf["ws_feat"], p, s, return_info=True)
    assert np.allclose(inf["swapped"][ok], hard_sw[0][ok], rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("ps", [(3, 1), (5, 2)])
def test_large_temperature_is_the_uniform_mean(ps):
    p, s = ps
    hc, hs = (9, 10) if p == 3 else (11, 15)
    wc, ws = _whitened(23 + p, hc, hs)
    got = SR.style_swap_softmax(wc, ws, p, s, 1e4)
    want = SR.uniform_swap(ws, hc, hc, p, s)
    assert np.abs(got - want).max() <= 1e-3 * np.abs(want).max()
    allowed = _allowed(hc, hs, p, s, 2, 3)
    assert (~allowed).any()
    got = SR.style_swap_softmax(wc, ws, p, s, 1e4, allowed)
    want = SR.uniform_swap(ws, hc, hc, p, s, allowed)
    assert np.abs(got - want).max() <= 1e-3 * np.abs(want).max()


@pytest.mark.parametrize("t", [0.05, 1, 3e-5, 1e-30, np.float32(0.5), np.int64(2)])
def test_check_ss_temperature_accepts(t):
    assert options.check_ss_temperature(t, True) == float(t)
    assert isinstance(options.check_ss_temperature(t, True), float)


def test_check_ss_temperature_none_is_off():
    assert options.check_ss_temperature(None, False) is None
    assert options.check_ss_temperature(None, True) is None


@pytest.mark.parametrize("t", [0, -0.1, float("nan"), float("inf"), -float("inf"), True, False, "0.1", [0.1]])
def test_check_ss_temperature_rejects_values(t):
    with pytest.raises(ValueError, match="ss_temperature must be a finite number > 0"):
        options.check_ss_temperature(t, True)
    with pytest.raises(ValueError, match="--ss-temperature must be"):
        options.check_ss_temperature(t, True, options.CLI)


@pytest.mark.parametrize("t", [1e-300, 1e-40, 1e39])
def test_check_ss_temperature_rejects_what_float32_cannot_divide_by(t):
    """The device takes tau as a float32: values that round to 0, to a subnormal (no finite 1/tau) or to inf."""
    with pytest.raises(ValueError, match="float32's normal range"):
        options.check_ss_temperature(t, True)


def test_check_ss_temperature_needs_the_swap():
    with pytest.raises(ValueError, match="ss_temperature needs swap5 / swap_targets"):
        options.check_ss_temperature(0.1, False)
    with pytest.raises(ValueError, match="--ss-temperature needs --swap5 / --swap-targets"):
        options.check_ss_temperature(0.1, False, options.CLI)
    # a parameter of the swap: no entry of its own in the options table
    assert "ss_temperature" not in options.SPELLINGS and "ss_temperature" not in options.AROUND
    assert all("ss_temperature" not in (a,) + tuple(b) for a, b, _ in options.EXCLUDES)


class _Level(object):
    def __init__(self, relu):
        self.relu_target = relu


class RecordingEngine(object):
    """Records every Engine.stylize call (style argument, keyword arguments); returns zero frames."""
    device = "cpu"

    def __init__(self):
        self.calls = []
        self.model = type("Model", (), dict(levels=[_Level(r) for r in
                                                     ("relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1")]))()

    swap_levels = Engine.swap_levels

    def stylize(self, c, s, **kw):
        self.calls.append((s, kw))
        return torch.zeros(c.shape, dtype=torch.float32)

    def to_u8(self, x):
        return x.to(torch.uint8)

    def check_device(self):
        pass

    def prepare_call(self, a, **kw):
        return a


@pytest.fixture
def api(monkeypatch):
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    empty = torch.empty
    monkeypatch.setattr(torch, "empty", lambda *a, pin_memory=False, **k: empty(*a, **k))
    m = W.WCT.__new__(W.WCT)
    m.ss_patch_size, m.ss_stride, m.verbose = 3, 1, False
    m.engine = RecordingEngine()
    m.model = m.engine.model
    return m


def _imgs(n, h, w, seed=0):
    return np.random.default_rng(seed).integers(0, 256, (n, h, w, 3), dtype=np.uint8)


def test_predict_batch_forwards_the_temperature(api):
    c, s = _imgs(2, 32, 32), _imgs(1, 16, 16, 1)
    api.predict_batch(c, s, swap_targets=["relu3_1"], ss_temperature=0.05, passes=2)
    (_, kw0), (_, kw1) = api.engine.calls
    assert kw0["ss_temperature"] == 0.05 and kw0["swap_targets"] == ["relu3_1"]
    assert kw1["ss_temperature"] is None and kw1["swap_targets"] is None      # the swap acts in the first pass only
    api.engine.calls.clear()
    api.predict(c[0], s[0], swap5=True, ss_temperature=2)
    assert api.engine.calls[0][1]["ss_temperature"] == 2.0 and api.engine.calls[0][1]["swap5"]
    api.engine.calls.clear()
    api.predict_batch(c, PreparedStyle(1, {}, ["relu5_1"]), swap5=True, ss_temperature=0.1)
    assert api.engine.calls[0][1]["ss_temperature"] == 0.1
    api.engine.calls.clear()
    api.predict_batch(c, s, swap5=True)
    assert api.engine.calls[0][1]["ss_temperature"] is None


def test_synthesize_forwards_the_temperature(api, monkeypatch):
    from wct_tf_b200 import device_image
    monkeypatch.setattr(device_image, "noise_u8", lambda n, h, w, seed=0, first_index=0, device=None: torch.zeros(
        (n, h, w, 3), dtype=torch.uint8))
    api.synthesize(_imgs(1, 16, 16), (32, 48), count=2, swap_targets=["relu3_1"], ss_temperature=0.02)
    assert api.engine.calls[0][1]["ss_temperature"] == 0.02


@pytest.mark.parametrize("kw,match", [
    (dict(ss_temperature=0.1), "ss_temperature needs swap5 / swap_targets"),
    (dict(swap5=True, ss_temperature=0.0), "finite number > 0"),
    (dict(swap5=True, ss_temperature=float("nan")), "finite number > 0"),
    (dict(swap5=True, ss_temperature=True), "finite number > 0"),
])
def test_predict_batch_rejects_before_device_work(api, kw, match):
    with pytest.raises(ValueError, match=match):
        api.predict_batch(_imgs(2, 32, 32), _imgs(1, 16, 16), **kw)
    assert api.engine.calls == []
