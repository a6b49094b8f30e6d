"""Coarse-to-fine stylisation (DESIGN.md §3.3.16) on the GPU: the join kernel against ``tests/coarse_ref.py`` byte for
byte (non-integer ratios, h > H, h = g, 1-pixel frames, 4096^2, batch invariance); ``levels=`` against an engine built with
only those targets; the composition identity of ``predict_batch(coarse_to_fine=)`` with every option it combines with,
tiled and untiled; and one 4096^2 frame."""
import gc

import numpy as np
import pytest
import torch

from tests import coarse_ref as R
from tests import test_gpu_luminance as L
from wct_tf_b200 import device_image as D
from wct_tf_b200.temporal import stabilize_
from wct_tf_b200.wct import WCT
from wct_tf_b200.weights import make_synthetic_weights

pytestmark = pytest.mark.gpu
ALL = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]
FINE = ("relu3_1", "relu2_1", "relu1_1")
_smooth, _cuda = L._smooth, L._cuda


def _frames(n, h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, h, w, 3), dtype=np.uint8)


# ------------------------------------------------------------------------------------------------------------- kernel
@pytest.mark.parametrize("hw,coarse", [((1000, 1496), (256, 368)), ((10, 12), (16, 16)), ((16, 16), (16, 16)),
                                       ((40, 50), (16, 16)), ((1, 37), (16, 16)), ((37, 1), (16, 16)), ((1, 1), (16, 32)),
                                       ((97, 61), (48, 32))],
                         ids=["ratio", "h_above_H", "same", "h_is_g", "one_row", "one_column", "one_pixel", "odd"])
def test_join_equals_the_oracle(hw, coarse):
    c, d, s = _frames(3, *hw, 1), _frames(3, *coarse, 2), _frames(3, *coarse, 3)
    want = R.join(c, d, s)
    got = D.coarse_join(_cuda(c), _cuda(d), _cuda(s)).cpu().numpy()
    assert np.array_equal(got, want), int((got != want).sum())
    for i in range(3):                                              # frame n of N = 3 is the N = 1 call
        one = D.coarse_join(_cuda(c[i]), _cuda(d[i]), _cuda(s[i])).cpu().numpy()
        assert np.array_equal(one, want[i])


def test_join_4096_from_1024():
    try:
        c = _smooth(1, 4096, 4096, 4)
        d, s = _smooth(1, 1024, 1024, 5), _smooth(1, 1024, 1024, 6)
        got = D.coarse_join(_cuda(c), _cuda(d), _cuda(s)).cpu().numpy()
        assert np.array_equal(got, R.join(c, d, s))
    finally:
        gc.collect()
        torch.cuda.empty_cache()


def test_join_rejects_mismatched_frames():
    c, d = _cuda(_frames(2, 32, 32, 1)), _cuda(_frames(2, 16, 16, 2))
    with pytest.raises(ValueError, match="coarse_join"):
        D.coarse_join(c, d, d[:, :8])
    with pytest.raises(ValueError, match="coarse_join"):
        D.coarse_join(c, d[:1], d[:1])


# ------------------------------------------------------------------------------------------------------------- levels
@pytest.fixture(scope="module")
def weights():
    return make_synthetic_weights(42)


@pytest.fixture(scope="module")
def wct(weights):
    return WCT(relu_targets=ALL, weights=weights)


@pytest.mark.parametrize("subset", [["relu3_1", "relu2_1", "relu1_1"], ["relu5_1", "relu1_1"], ["relu4_1"]])
def test_levels_equal_an_engine_of_those_targets(wct, weights, subset):
    sub = WCT(relu_targets=subset, weights=weights).engine
    eng = wct.engine
    c = _cuda(_smooth(2, 64, 96, 7))
    s = _cuda(_smooth(1, 48, 56, 8))
    want = sub.stylize(c, s, alpha=0.8).cpu().numpy()
    got = eng.stylize(c, s, alpha=0.8, levels=list(reversed(subset))).cpu().numpy()   # run in the model's order
    assert np.array_equal(got, want)
    ps = wct.prepare_style(s)                                        # a side made for every level serves the subset
    assert np.array_equal(eng.stylize(c, ps, alpha=0.8, levels=subset).cpu().numpy(), want)
    tiled = eng.stylize_tiled(c[:1], s, alpha=0.8, tile_size=32, levels=subset).cpu().numpy()
    assert np.array_equal(tiled, sub.stylize_tiled(c[:1], s, alpha=0.8, tile_size=32).cpu().numpy())


def test_all_levels_are_todays_bytes(wct):
    eng = wct.engine
    c = _cuda(_smooth(2, 64, 64, 9))
    s = _cuda(_smooth(1, 48, 56, 8))
    base = eng.stylize(c, s).cpu().numpy()
    assert np.array_equal(eng.stylize(c, s, levels=None).cpu().numpy(), base)
    assert np.array_equal(eng.stylize(c, s, levels=ALL).cpu().numpy(), base)
    with pytest.raises(ValueError, match="mst"):
        eng.stylize(c, s, mst=2, levels=FINE)
    with pytest.raises(ValueError, match="relu6_1"):
        eng.stylize(c, s, levels=["relu6_1"])


# -------------------------------------------------------------------------------------------------------- composition
def _fine_stage(wct, j, name, styles, opts, tile=None):
    """``Engine.stylize(levels=FINE)`` (or ``stylize_tiled``) of the joined frames with the engine's spelling of ``opts``."""
    eng = wct.engine
    n = j.shape[0]
    if name == "mask":
        return eng.stylize(j, None, labels=_cuda(opts["content_mask"])[None], region_styles=[_cuda(x[None]) for x in styles],
                           region_masks=[None if m is None else _cuda(m) for m in opts["style_masks"]], levels=FINE)
    if name == "interp":
        w = torch.from_numpy(WCT.normalize_weights(opts["style_weights"], n, len(styles))).cuda()
        return eng.stylize(j, None, interp_styles=[_cuda(x[None]) for x in styles], interp_weights=w, levels=FINE)
    s = styles if not isinstance(styles, np.ndarray) else _cuda(styles if styles.ndim == 4 else styles[None])
    kw = {k: v for k, v in opts.items() if k in ("adain", "ost", "efdm", "efdm_slices")}
    if "strength_map" in opts:
        kw["strength_map"] = WCT.check_soft_map(opts["strength_map"], n, "strength_map").cuda()
    if tile is not None:
        return eng.stylize_tiled(j, s, tile_size=tile, levels=FINE, **kw)
    return eng.stylize(j, s, levels=FINE, **kw)


def _compose(wct, c, styles, f, name="plain", tile=None, **opts):
    """uint8 stylize(levels=FINE) of coarse_join(C, D, predict(D)), D = imresize(C, coarse_size), from the public pieces."""
    cd = _cuda(c)
    d = D.imresize(cd, R.coarse_size(c.shape[1], c.shape[2], f, 16))
    tile_kw = {} if tile is None else dict(tile_size=tile)
    s = wct.predict_batch(d, styles, return_device=True, **tile_kw, **opts)
    j = D.coarse_join(cd, d, s)
    return wct.engine.to_u8(_fine_stage(wct, j, name, styles, opts, tile)).cpu().numpy()


def _case(name, n=2):
    """(content, styles, options) of a composition case."""
    c = _smooth(n, 96, 128, 1)
    s = _smooth(1, 48, 56, 2)[0]
    s2 = _smooth(1, 40, 40, 3)[0]
    if name == "plain":
        return c, s, {}
    if name in ("adain", "ost"):
        return c, s, {name: True}
    if name == "efdm_slices":
        return c, s, dict(efdm=True, efdm_slices=2)
    if name == "per_frame":
        return c, _smooth(n, 48, 48, 7), {}
    if name == "mask":
        lab = np.zeros((96, 128), np.uint8)
        lab[:, 64:] = 1
        sm = np.zeros((40, 40), np.uint8)
        sm[:, 20:] = 1
        return c, [s, s2], dict(content_mask=lab, style_masks=[None, sm])
    if name == "interp":
        return c, [s, s2], dict(style_weights=np.array([[3.0, 1.0], [1.0, 1.0]])[:n])
    if name == "strength_map":
        return c, s, dict(strength_map=np.linspace(0, 1, 96 * 128, dtype=np.float32).reshape(96, 128))
    raise KeyError(name)


CASES = ["plain", "adain", "ost", "efdm_slices", "per_frame", "mask", "interp", "strength_map"]


@pytest.mark.parametrize("name", CASES)
def test_composition_identity(wct, name):
    c, styles, opts = _case(name)
    got = wct.predict_batch(c, styles, coarse_to_fine=2, **opts)
    want = _compose(wct, c, styles, 2, name, **opts)
    assert got.shape == want.shape == c.shape
    assert np.array_equal(got, want), (name, int((got != want).sum()))


def test_composition_identity_np_semantics(weights):
    model = WCT(relu_targets=ALL, weights=weights, semantics="np")
    c, s, _ = _case("plain")
    assert np.array_equal(model.predict_batch(c, s, coarse_to_fine=3), _compose(model, c, s, 3))


def test_composition_identity_prepared_and_fine_targets(wct):
    c, s, _ = _case("plain")
    ps = wct.prepare_style(s)
    want = _compose(wct, c, s, 2)
    assert np.array_equal(wct.predict_batch(c, ps, coarse_to_fine=2), want)
    got = wct.predict_batch(c, ps, coarse_to_fine=2, fine_targets=["relu1_1", "relu2_1"])
    cd = _cuda(c)
    d = D.imresize(cd, R.coarse_size(96, 128, 2, 16))
    j = D.coarse_join(cd, d, wct.predict_batch(d, ps, return_device=True))
    assert np.array_equal(got, wct.engine.to_u8(wct.engine.stylize(j, ps, levels=["relu2_1", "relu1_1"])).cpu().numpy())


def test_composition_identity_passes_and_float(wct):
    c, s, _ = _case("plain")
    once = _compose(wct, c, s, 2)
    assert np.array_equal(wct.predict_batch(c, s, coarse_to_fine=2, passes=2), _compose(wct, once, s, 2))
    u8, f32 = wct.predict_batch(c, s, coarse_to_fine=2, return_float=True)
    assert np.array_equal(u8, once) and f32.dtype == np.float32 and f32.shape == c.shape
    assert np.array_equal(wct.engine.to_u8(_cuda(f32)).cpu().numpy(), once)


def test_composition_identity_luminance_only(wct):
    c, s, _ = _case("plain")
    gs = L._grey_host(s)
    got = wct.predict_batch(c, s, luminance_only=True, coarse_to_fine=2)
    assert np.array_equal(got, L._compose(wct, c, _cuda(gs[None]), L._shared(gs), coarse_to_fine=2))


def test_composition_identity_temporal(wct):
    c = _smooth(4, 96, 128, 8)
    c[1:] = np.clip(c[:1].astype(np.int16) + np.arange(1, 4)[:, None, None, None], 0, 255).astype(np.uint8)   # a slow pan
    s = _smooth(1, 48, 56, 2)[0]
    a, b = wct.temporal_state(0.6), wct.temporal_state(0.6)
    got = np.concatenate([wct.predict_batch(c[:2], s, coarse_to_fine=2, temporal=a),
                          wct.predict_batch(c[2:], s, coarse_to_fine=2, temporal=a)])
    want = []
    for part in (c[:2], c[2:]):
        out = _cuda(_compose(wct, part, s, 2))
        stabilize_(b, _cuda(part), out)
        want.append(out.cpu().numpy())
    assert np.array_equal(got, np.concatenate(want))


def test_composition_identity_synthesize(wct):
    s = _smooth(1, 48, 56, 2)[0]
    got = wct.synthesize(s, (96, 128), count=2, seed=5, coarse_to_fine=2)
    noise = D.noise_u8(2, 96, 128, seed=5).cpu().numpy()
    assert np.array_equal(got, _compose(wct, noise, s, 2))


def test_off_means_off(wct):
    c, s, _ = _case("plain")
    assert np.array_equal(wct.predict_batch(c, s, coarse_to_fine=None), wct.predict_batch(c, s))
    assert np.array_equal(wct.predict(c[0], s, coarse_to_fine=2), wct.predict_batch(c[:1], s, coarse_to_fine=2)[0])


def test_rejections(wct):
    c, s, _ = _case("plain")
    for kw, msg in ((dict(swap5=True), "swap"), (dict(seamless="xy"), "seamless"), (dict(mst=2), "mst"),
                    (dict(coarse_to_fine=None, fine_targets=["relu1_1"]), "needs coarse_to_fine"),
                    (dict(coarse_to_fine=20), "2..16"), (dict(fine_targets=["relu1_1", "relu1_1"]), "more than once")):
        with pytest.raises(ValueError, match=msg):
            wct.predict_batch(c, s, **dict(dict(coarse_to_fine=2), **kw))


# -------------------------------------------------------------------------------------------------------------- tiles
def test_a_tile_covering_each_stage_is_untiled(wct):
    c, s, _ = _case("plain")
    for opts in ({}, dict(adain=True), dict(ost=True)):
        assert np.array_equal(wct.predict_batch(c, s, coarse_to_fine=2, tile_size=128, **opts),
                              wct.predict_batch(c, s, coarse_to_fine=2, **opts)), opts


def test_tiled_2048_equals_the_tiled_composition(wct):
    try:
        c = _smooth(1, 2048, 2048, 11)
        s = _smooth(1, 256, 256, 12)[0]
        got = wct.predict_batch(c, s, coarse_to_fine=2, tile_size=512)
        assert np.array_equal(got, _compose(wct, c, s, 2, tile=512))
    finally:
        gc.collect()
        torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------- the size the feature is for
def test_4096_frame(wct):
    try:
        c = _smooth(1, 4096, 4096, 13)
        s = _smooth(1, 512, 512, 14)[0]
        got = wct.predict_batch(c, s, coarse_to_fine=4)
        assert np.array_equal(got, _compose(wct, c, s, 4))
    finally:
        gc.collect()
        torch.cuda.empty_cache()
