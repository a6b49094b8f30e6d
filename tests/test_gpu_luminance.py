"""Luminance-only transfer (DESIGN.md §3.3.15) on the GPU: the moments, match and merge kernels against
``tests/luminance_ref.py`` (odd sizes, N = 1..5, a frame past 2^31 bytes), the composition identity of
``predict_batch(luminance_only=True)`` with every option it combines with, the colour guarantee, batch and run invariance,
and the rejections."""
import gc

import numpy as np
import pytest
import torch

from tests import gpu_util as U
from tests import luminance_ref as R
from wct_tf_b200 import _capi
from wct_tf_b200 import device_image as D
from wct_tf_b200.wct import WCT
from wct_tf_b200.weights import make_synthetic_weights

pytestmark = pytest.mark.gpu
ALL = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]


def _frames(n, h, w, seed, lo=0, hi=256):
    return np.random.default_rng(seed).integers(lo, hi, (n, h, w, 3), dtype=np.uint8)


def _smooth(n, h, w, seed):
    """Frames with structure (gradients and blobs) rather than white noise, so that stylisation has something to keep."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w] / max(h, w)
    out = []
    for _ in range(n):
        a = rng.uniform(0, 2 * np.pi, 3)
        f = [128 + 100 * np.sin(6 * x * np.cos(t) + 5 * y * np.sin(t) + t) for t in a]
        out.append(np.clip(np.stack(f, -1) + rng.normal(0, 8, (h, w, 3)), 0, 255).astype(np.uint8))
    return np.stack(out)


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _assert_rounded(got, pre, what):
    """Within 1 LSB of the clipped, rounded oracle everywhere, and equal where the value before rounding is more than
    1e-3 from a half-integer."""
    want = R.round_clip(pre)
    diff = np.abs(got.astype(np.int32) - want.astype(np.int32))
    assert diff.max() <= 1, (what, int(diff.max()))
    clear = np.abs(np.abs(pre - np.floor(pre)) - 0.5) > 1e-3
    assert np.array_equal(got[clear], want[clear]), (what, int((got != want)[clear].sum()))


# ---------------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("n", [1, 2, 3, 4, 5])
def test_batched_moments_are_exact(n):
    x = _frames(n, 37, 53, n)
    lib = U.lib()
    sums = torch.empty((n, 9), dtype=torch.int64, device="cuda")
    _capi.check(lib.wctb200_rgb_moments_batch_u8(_cuda(x).data_ptr(), n, 37 * 53, sums.data_ptr(), U.stream()))
    got = sums.cpu().numpy()
    v = x.reshape(n, -1, 3).astype(np.int64)
    for i in range(n):
        want = list(v[i].sum(0)) + [int((v[i][:, a] * v[i][:, b]).sum()) for a, b in ((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))]
        assert list(got[i]) == want
        one = torch.empty(9, dtype=torch.int64, device="cuda")
        _capi.check(lib.wctb200_rgb_moments_u8(_cuda(x[i]).data_ptr(), 37 * 53, one.data_ptr(), U.stream()))
        assert list(one.cpu().numpy()) == want                             # the N = 1 entry, as before
    npf, s1, s2 = D.luminance_moments(_cuda(x))
    assert (npf, s1, s2) == R.moments(x)


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("hw", [(1, 1), (7, 13), (61, 45)])
def test_match_and_merge_against_the_oracle(n, hw):
    c, s = _frames(n, *hw, 10 + n), _frames(n, *hw, 20 + n)
    mc, sc = R.stats(c)
    rng = np.random.default_rng(n)
    ms, ss = rng.uniform(20, 230, n), rng.uniform(0, 90, n)
    ss[0] = 0.0 if n > 2 else ss[0]                                         # a degenerate spread
    k = R.params(mc, sc, ms, ss)
    (k_, b), (k_inv, b_m) = D.luminance_params(mc, sc, ms, ss)
    assert np.array_equal(k_, k)
    g = D.luminance_match(_cuda(c), k_, b).cpu().numpy()
    pre = R.match_pre(c, mc, ms, k)
    _assert_rounded(g, np.repeat(pre[..., None], 3, -1), "match")
    assert np.array_equal(D.luminance_grey(_cuda(s)).cpu().numpy(), R.grey(s))           # k = 1, b = 0: exact
    out = D.luminance_merge(_cuda(c), _cuda(s), k_inv, b_m).cpu().numpy()
    _assert_rounded(out, R.merge_pre(c, R.luma_int(s) / 1000.0, mc, ms, k), "merge")
    # frame i's bytes do not depend on the batch
    for i in range(n):
        assert np.array_equal(D.luminance_match(_cuda(c[i]), k_[i], b[i]).cpu().numpy(), g[i])
        assert np.array_equal(D.luminance_merge(_cuda(c[i]), _cuda(s[i]), k_inv[i], b_m[i]).cpu().numpy(), out[i])


def test_one_frame_past_2_31_bytes():
    """A 64000 x 12000 frame (2.3 GB) built from one 64-row band repeated: its moments are 1000 times the band's, and the
    band past byte 2^31 is matched and merged as the band alone."""
    band_c, band_s = _frames(1, 64, 12000, 1), _frames(1, 64, 12000, 2)
    reps = 1000
    assert 3 * 64 * 12000 * reps > 2 ** 31
    try:
        c = _cuda(band_c).repeat(1, reps, 1, 1)
        npf, s1, s2 = D.luminance_moments(c)
        n0, b1, b2 = R.moments(band_c)
        assert npf == n0 * reps and s1 == [b1[0] * reps] and s2 == [b2[0] * reps]
        mc, sc = D.luminance_stats(c)
        (k, b), (k_inv, b_m) = D.luminance_params(mc, sc, 100.0, 40.0)
        g = D.luminance_match(c, k, b)
        tail = g[0, -64:].cpu().numpy()
        del g
        pre = R.match_pre(band_c, mc, np.array([100.0]), k)
        _assert_rounded(tail[None], np.repeat(pre[..., None], 3, -1), "match past 2^31")
        s = _cuda(band_s).repeat(1, reps, 1, 1)
        out = D.luminance_merge(c, s, k_inv, b_m)
        tail = out[0, -64:].cpu().numpy()
        _assert_rounded(tail[None], R.merge_pre(band_c, R.luma_int(band_s) / 1000.0, mc, np.array([100.0]), k),
                        "merge past 2^31")
    finally:
        c = s = out = None
        gc.collect()
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------- API
@pytest.fixture(scope="module")
def weights():
    return make_synthetic_weights(42)


@pytest.fixture(scope="module")
def wct(weights):
    return WCT(relu_targets=ALL, weights=weights)


def _grey_host(x):
    return R.grey(np.asarray(x))


def _compose(model, c, styles, style_stats, crop=False, temporal=None, **opts):
    """luminance_merge(c, predict_batch(luminance_match(c, k, b), grey(styles), **opts), 1/k, b'), with the statistics
    from the oracle: ``style_stats`` = (mean_s, sd_s) per frame or shared.  ``crop``: the content is first fitted to a
    stride swap (``WCT.swap_fit``), and the statistics, the match and the merge use that content."""
    cc = model.swap_fit(_cuda(c), opts.get("swap5"), opts.get("swap_targets"), lambda a: a).cpu().numpy() if crop else c
    mc, sc = R.stats(cc)
    (k, b), (k_inv, b_m) = D.luminance_params(mc, sc, *style_stats)
    g = D.luminance_match(_cuda(cc), k, b)
    s = model.predict_batch(g, styles, return_device=True, **opts)
    cd = _cuda(cc)
    if tuple(s.shape[1:3]) != cc.shape[1:3]:                  # a size the decoders round up: the content resized to it
        cd = D.imresize(cd, s.shape[1:3])
    out = D.luminance_merge(cd, s, k_inv, b_m)
    if temporal is not None:
        from wct_tf_b200.temporal import stabilize_
        stabilize_(temporal, cd, out)
    return out.cpu().numpy()


def _shared(style):
    m, s = R.stats(style[None] if style.ndim == 3 else style)
    return m, s


def _case(name, n=2, size=64):
    """(content, styles for the luminance call, grey styles for the composition, style statistics, options)."""
    c = _smooth(n, size, size, 1)
    s = _smooth(1, 48, 56, 2)[0]
    s2 = _smooth(1, 40, 40, 3)[0]
    gs, gs2 = _grey_host(s), _grey_host(s2)
    one = (s, gs, _shared(gs), {})
    lab = np.zeros((size, size), np.uint8)
    lab[:, size // 2:] = 1
    if name == "plain":
        return (c,) + one
    if name in ("adain", "ost"):
        return (c,) + one[:3] + ({name: True},)
    if name == "efdm_slices":
        return (c,) + one[:3] + (dict(efdm=True, efdm_slices=2),)
    if name == "mst":
        return (c,) + one[:3] + (dict(mst=2),)
    if name == "swap_labels":
        slab = np.zeros(s.shape[:2], np.uint8)
        slab[:, : s.shape[1] // 3] = 1
        return (c,) + one[:3] + (dict(swap_targets=["relu3_1"], swap_labels=(lab, slab)),)
    if name in ("content_mask", "content_weights"):
        pooled = R.pooled([gs, gs2])
        if name == "content_mask":
            opts = dict(content_mask=lab, style_masks=[None, (lab[:40, :40] * 0 + 1).astype(np.uint8)])
        else:
            w = np.stack([np.linspace(0, 1, size)[None].repeat(size, 0)] * 2) * np.array([0.7, 0.3])[:, None, None]
            opts = dict(content_weights=w.astype(np.float32))
        return c, [s, s2], [gs, gs2], pooled, opts
    if name == "style_weights":
        w = np.array([[3.0, 1.0], [1.0, 1.0]])[:n]
        m1, d1 = _shared(gs)
        m2, d2 = _shared(gs2)
        wn = w / w.sum(1, keepdims=True)
        return c, [s, s2], [gs, gs2], R.weighted_mixture([m1[0], m2[0]], [d1[0], d2[0]], wn), dict(style_weights=w)
    if name == "strength_map":
        return (c,) + one[:3] + (dict(strength_map=np.linspace(0, 1, size * size, dtype=np.float32).reshape(size, size)),)
    if name == "tile_size":
        return (c,) + one[:3] + (dict(tile_size=32),)
    if name == "seamless":
        return (c,) + one[:3] + (dict(seamless="xy"),)
    if name == "passes":
        return (c,) + one[:3] + (dict(passes=2),)
    if name == "per_frame":
        ss = _smooth(n, 48, 48, 7)
        gss = R.grey(ss)
        return c, ss, gss, R.stats(gss), {}
    raise KeyError(name)


CASES = ["plain", "adain", "ost", "efdm_slices", "mst", "swap_labels", "content_mask", "content_weights", "style_weights",
         "strength_map", "tile_size", "seamless", "passes", "per_frame"]


@pytest.mark.parametrize("name", CASES)
def test_composition_identity(wct, name):
    c, styles, greys, stats, opts = _case(name)
    got = wct.predict_batch(c, styles, luminance_only=True, **opts)
    grey_dev = [_cuda(g[None]) for g in greys] if isinstance(greys, list) else _cuda(greys if greys.ndim == 4 else greys[None])
    want = _compose(wct, c, grey_dev, stats, **opts)
    assert got.shape == want.shape == c.shape
    assert np.array_equal(got, want), (name, int((got != want).sum()))


def test_composition_identity_stride_swap_crop(weights):
    model = WCT(relu_targets=ALL, weights=weights, ss_patch_size=3, ss_stride=2)
    c = _smooth(2, 72, 88, 4)
    s = _smooth(1, 64, 64, 5)[0]
    gs = _grey_host(s)
    got = model.predict_batch(c, s, luminance_only=True, swap5=True)
    assert got.shape[1:3] != (72, 88)
    want = _compose(model, c, _cuda(gs[None]), _shared(gs), crop=True, swap5=True)
    assert np.array_equal(got, want)
    # swap_targets with a stride and a content label map of the content's size, cropped with it
    c2 = _smooth(2, 70, 90, 14)
    lab = np.zeros((70, 90), np.uint8)
    lab[:, 45:] = 1
    slab = np.zeros((64, 64), np.uint8)
    slab[:, :20] = 1
    opts = dict(swap_targets=["relu5_1"], swap_labels=(lab, slab))
    got = model.predict_batch(c2, s, luminance_only=True, **opts)
    fit = model.swap_fit(_cuda(c2), False, ["relu5_1"], lambda a: a).shape[1:3]
    assert fit == (70, 80)                                   # 90 -> 80; 70 encodes to 5 and stays
    cl = WCT._crop_labels(lab[None], (70, 90), fit)
    want = _compose(model, c2, _cuda(gs[None]), _shared(gs), crop=True, swap_targets=["relu5_1"], swap_labels=(cl, slab))
    assert np.array_equal(got, want)


def test_composition_identity_prepared_and_reloaded(wct, tmp_path):
    c = _smooth(2, 64, 64, 6)
    s = _smooth(1, 48, 56, 2)[0]
    gs = _grey_host(s)
    ps = wct.prepare_style(s, luminance_only=True)
    assert np.array_equal(ps.image[0], gs)
    want = _compose(wct, c, _cuda(gs[None]), _shared(gs))
    assert np.array_equal(wct.predict_batch(c, ps, luminance_only=True), want)
    assert np.array_equal(wct.predict_batch(c, s, luminance_only=True), want)            # same as the image
    path = str(tmp_path / "s.wctstyle")
    ps.save(path)
    assert np.array_equal(wct.predict_batch(c, wct.load_style(path), luminance_only=True), want)


def test_composition_identity_temporal(wct):
    c = _smooth(4, 64, 64, 8)
    c[1:] = np.clip(c[:1].astype(np.int16) + np.arange(1, 4)[:, None, None, None], 0, 255).astype(np.uint8)   # a slow pan
    s = _smooth(1, 48, 56, 2)[0]
    gs = _grey_host(s)
    a, b = wct.temporal_state(0.6), wct.temporal_state(0.6)
    got = np.concatenate([wct.predict_batch(c[:2], s, luminance_only=True, temporal=a),
                          wct.predict_batch(c[2:], s, luminance_only=True, temporal=a)])
    want = np.concatenate([_compose(wct, c[:2], _cuda(gs[None]), _shared(gs), temporal=b),
                           _compose(wct, c[2:], _cuda(gs[None]), _shared(gs), temporal=b)])
    assert np.array_equal(got, want)
    plain = wct.predict_batch(c, s, luminance_only=True)
    assert not np.array_equal(got[1:], plain[1:])                            # stabilisation acted, after the merge


def test_output_keeps_the_contents_colours(wct):
    c = _smooth(1, 256, 256, 9)
    s = _smooth(1, 128, 128, 10)[0]
    gs = _grey_host(s)
    out = wct.predict_batch(c, s, luminance_only=True)
    mc, sc = R.stats(c)
    ms, ss = _shared(gs)
    k = R.params(mc, sc, ms, ss)
    (k_, b), _ = D.luminance_params(mc, sc, ms, ss)
    stylised = wct.predict_batch(D.luminance_match(_cuda(c), k_, b), _cuda(gs[None]), return_device=True).cpu().numpy()
    pre = R.merge_pre(c, R.luma_int(stylised) / 1000.0, mc, ms, k)
    free = ((pre >= 0) & (pre <= 255)).all(-1)
    assert free.mean() > 0.5
    for a, b_, bound in zip(R.iq(out), R.iq(c), R.IQ_BOUND):
        assert np.abs(a - b_)[free].max() <= bound + 1e-4
    assert np.abs(out.astype(np.int32) - c).max() > 20                      # and the luminance did change


def test_batch_and_run_invariance(wct):
    c = _smooth(3, 64, 64, 11)
    s = _smooth(1, 48, 56, 2)[0]
    batch = wct.predict_batch(c, s, luminance_only=True)
    for i in range(3):
        assert np.array_equal(wct.predict_batch(c[i:i + 1], s, luminance_only=True)[0], batch[i])
    assert np.array_equal(wct.predict_batch(c, s, luminance_only=True), batch)


def test_off_means_off(wct):
    c = _smooth(2, 64, 64, 12)
    s = _smooth(1, 48, 56, 2)[0]
    assert np.array_equal(wct.predict_batch(c, s, luminance_only=False), wct.predict_batch(c, s))
    assert np.array_equal(wct.predict(c[0], s, luminance_only=False), wct.predict(c[0], s))


def test_rejections(wct):
    c = _smooth(1, 64, 64, 13)
    s = _smooth(1, 48, 56, 2)[0]
    with pytest.raises(ValueError, match="return_float"):
        wct.predict_batch(c, s, luminance_only=True, return_float=True)
    with pytest.raises(ValueError, match="no colours to keep"):
        wct.synthesize(s, 64, luminance_only=True)
    with pytest.raises(ValueError, match="prepared grey"):
        wct.predict_batch(c, wct.prepare_style(s), luminance_only=True)
    grey_ps = wct.prepare_style(s, luminance_only=True)
    assert np.array_equal(wct.predict_batch(c, grey_ps), wct.predict_batch(c, _grey_host(s)))   # simply a grey style
