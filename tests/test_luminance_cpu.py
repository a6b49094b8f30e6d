"""Luminance-only transfer (DESIGN.md §3.3.15) without a GPU: the oracle's own properties, the options row, the flags of
stylize.py / stylize_video.py / prepare_styles.py and the calls they make (stub models and host image ops), and the API
rejections, which come before any device work."""
import numpy as np
import pytest
import torch
from PIL import Image

import prepare_styles
import stylize
import stylize_video as V
from tests import luminance_ref as R
from tests.test_interp_cli import HostImageOps, _base
from tests.test_options_cpu import stub  # noqa: F401  (fixture)
from wct_tf_b200 import options
from wct_tf_b200 import wct as W
from wct_tf_b200.prepared import PreparedStyle

ALL = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]


def _frames(n, h, w, seed, lo=0, hi=256):
    return np.random.default_rng(seed).integers(lo, hi, (n, h, w, 3), dtype=np.uint8)


# ------------------------------------------------------------------------------------------------------------ oracle
def test_merging_the_unrounded_match_returns_the_content():
    c = _frames(3, 17, 23, 0)
    mc, sc = R.stats(c)
    ms, ss = np.array([90.0, 140.0, 20.0]), np.array([30.0, 5.0, 60.0])
    k = R.params(mc, sc, ms, ss)
    pre = R.merge_pre(c, R.match_pre(c, mc, ms, k), mc, ms, k)
    assert np.allclose(pre, c, atol=1e-9)
    assert np.array_equal(R.round_clip(pre), c)


def test_merging_the_rounded_match_returns_the_content_when_k_is_at_least_one():
    # the grey's rounding error e becomes e / k in the merge: below half an LSB when k >= 1
    c = _frames(2, 31, 19, 1, 60, 200)                   # a narrow content: sd_s > sd_c
    mc, sc = R.stats(c)
    ms, ss = np.array([128.0, 100.0]), 1.5 * sc
    k = R.params(mc, sc, ms, ss)
    assert (k > 1).all()
    g = R.match(c, mc, ms, k)
    pre = R.match_pre(c, mc, ms, k)
    free = ((pre > 0) & (pre < 255))[..., None] & np.ones(3, bool)
    out = R.merge(c, g, mc, ms, k)
    assert free.mean() > 0.9
    assert np.array_equal(out[free], c[free])


def test_iq_of_the_merge_is_the_contents_within_the_rounding_bound():
    c, s = _frames(2, 40, 40, 2), _frames(2, 40, 40, 3)
    mc, sc = R.stats(c)
    k = R.params(mc, sc, 110.0, 50.0)
    pre = R.merge_pre(c, R.luma_int(s) / 1000.0, mc, 110.0, k)
    out = R.round_clip(pre)
    free = ((pre >= 0) & (pre <= 255)).all(axis=-1)
    assert free.mean() > 0.5
    for a, b, bound in zip(R.iq(out), R.iq(c), R.IQ_BOUND):
        assert np.abs(a - b)[free].max() <= bound + 1e-9


def test_mixture_moments_equal_the_moments_of_the_concatenated_pixels():
    imgs = [_frames(1, h, w, 10 + i)[0] for i, (h, w) in enumerate([(7, 9), (16, 5), (11, 11)])]
    means, sds = zip(*[tuple(v[0] for v in R.stats(x[None])) for x in imgs])
    npix = np.array([x.shape[0] * x.shape[1] for x in imgs], np.float64)
    mu, sd = R.weighted_mixture(means, sds, npix / npix.sum())
    mu_p, sd_p = R.pooled(imgs)
    assert abs(mu - mu_p) < 1e-9 and abs(sd - sd_p) < 1e-9


def test_degenerate_spreads_give_k_one():
    assert np.array_equal(R.params([10.0, 10.0, 10.0], [0.0, 3.0, 0.0], [5.0, 5.0, 5.0], [2.0, 0.0, 0.0]), [1.0, 1.0, 1.0])
    flat = np.full((1, 4, 4, 3), 77, np.uint8)
    assert R.stats(flat)[1][0] == 0.0


def test_grey_is_exact_on_grey_images():
    v = np.arange(256, dtype=np.uint8)
    img = np.repeat(v[None, :, None], 3, axis=-1)
    assert np.array_equal(R.grey(img), img)


def test_package_host_arithmetic_matches_the_oracle():
    from wct_tf_b200 import device_image as D
    c = _frames(3, 9, 13, 4)
    n, s1, s2 = R.moments(c)
    assert np.allclose(np.array(D.luminance_stats_from_moments(n, s1, s2)), np.array(R.stats(c)), rtol=0, atol=1e-12)
    (k, b), (k_inv, b_m) = D.luminance_params([100.0, 50.0, 9.0], [20.0, 0.0, 3.0], [120.0, 80.0, 7.0], [10.0, 4.0, 0.0])
    assert np.array_equal(k, R.params([100.0, 50.0, 9.0], [20.0, 0.0, 3.0], [120.0, 80.0, 7.0], [10.0, 4.0, 0.0]))
    assert np.allclose(b, [120.0 - 50.0, 80.0 - 50.0, 7.0 - 9.0]) and np.allclose(k_inv * k, 1.0)
    assert np.allclose(b_m, [100.0 - 240.0, 50.0 - 80.0, 9.0 - 7.0])


# ------------------------------------------------------------------------------------------------------- options row
@pytest.mark.parametrize("other", sorted(options.SPELLINGS))
def test_luminance_only_combines_with_everything_but_return_float(other):
    active = {"luminance_only", other} | ({"content_mask"} if other in ("mask_feather", "style_masks") else set())
    if other == "return_float":
        with pytest.raises(ValueError, match="luminance_only does not combine with return_float"):
            options.check(active, options.API)
    else:
        options.check(active, options.API)
    assert options.API["luminance_only"] == "luminance_only" and options.ENGINE["luminance_only"] is None
    assert options.CLI["luminance_only"] == "--luminance-only"


# ---------------------------------------------------------------------------------------------------------- API stub
def _args(n):
    rng = np.random.default_rng(0)
    return rng.integers(0, 256, (n, 32, 32, 3), dtype=np.uint8), rng.integers(0, 256, (1, 16, 16, 3), dtype=np.uint8)


def test_api_rejects_return_float_before_device_work(stub):  # noqa: F811
    c, s = _args(2)
    with pytest.raises(ValueError, match="return_float"):
        stub.predict_batch(c, s, luminance_only=True, return_float=True)
    assert stub.engine.calls == []


def test_api_rejects_a_colour_prepared_style_before_device_work(stub, monkeypatch):  # noqa: F811
    def no_device(*a, **k):
        raise AssertionError("device work before the check")
    monkeypatch.setattr(W, "_to_dev", no_device)
    c, _ = _args(1)
    ps = PreparedStyle(1, {}, ALL)
    ps.image = _frames(1, 8, 8, 5)
    with pytest.raises(ValueError, match="prepare_style\\(style, luminance_only=True\\)"):
        stub.predict_batch(c, ps, luminance_only=True)
    ps.image = None
    with pytest.raises(ValueError, match="prepared grey"):
        stub.predict_batch(c, ps, luminance_only=True)
    with pytest.raises(ValueError, match="prepared grey"):
        stub.predict_batch(c, [ps, ps], luminance_only=True, style_weights=[1, 1])
    assert stub.engine.calls == []


def test_synthesize_rejects_luminance_only_before_device_work(stub, monkeypatch):  # noqa: F811
    import wct_tf_b200.device_image as D

    def no_noise(*a, **k):
        raise AssertionError("noise made before the check")
    monkeypatch.setattr(D, "noise_u8", no_noise)
    with pytest.raises(ValueError, match="no colours to keep"):
        stub.synthesize(_args(1)[1], 32, luminance_only=True)


# --------------------------------------------------------------------------------------------------------- stylize.py
def test_stylize_flag_parses_and_defaults_off(tmp_path):
    assert not stylize.parse_args(_base(tmp_path) + ["--style-path", "s.png"]).luminance_only
    a = stylize.parse_args(_base(tmp_path) + ["--style-path", "s.png", "--luminance-only", "--adain", "--passes", "2"])
    assert a.luminance_only
    for extra in (["--interp-styles", "a.png", "b.png", "--interp-weights", "1", "1"],
                  ["--mask-styles", "a.png", "b.png", "--content-mask", "m.png"], ["--style-path", "s.wctstyle"],
                  ["--style-path", "s.png", "--swap5", "--ost"], ["--style-path", "s.png", "--mst", "2", "--tile-size", "0"]):
        assert stylize.parse_args(_base(tmp_path) + extra + ["--luminance-only"]).luminance_only


@pytest.mark.parametrize("extra, words", [(["--keep-colors"], "--keep-colors"), (["--noise"], "--noise")])
def test_stylize_flag_rejections(tmp_path, extra, words, capsys):
    argv = ["--relu-targets", "relu1_1", "--style-path", "s.png", "--out-path", str(tmp_path), "--luminance-only"] + extra
    if "--noise" not in extra:
        argv += ["--content-path", "c.png"]
    with pytest.raises(SystemExit):
        stylize.parse_args(argv)
    err = capsys.readouterr().err
    assert "--luminance-only" in err and words in err


class _FakeWCT(object):
    class engine(object):
        device = None

    def __init__(self):
        self.calls = []

    def predict_batch(self, contents, styles, **kw):
        self.calls.append(kw)
        c = np.asarray(contents)
        return (c[None] if c.ndim == 3 else c) + 1


def test_stylize_runs_every_pass_in_one_luminance_call(tmp_path):
    Image.fromarray(np.full((8, 12, 3), 10, np.uint8)).save(str(tmp_path / "c.png"))
    Image.fromarray(np.full((6, 6, 3), 50, np.uint8)).save(str(tmp_path / "s.png"))
    fake = _FakeWCT()
    argv = _base(tmp_path) + ["--style-path", str(tmp_path / "s.png"), "--passes", "3", "--luminance-only", "--adain"]
    assert stylize.main(argv, model_factory=lambda a: fake, image_ops=HostImageOps) == 1
    assert len(fake.calls) == 1
    assert fake.calls[0]["luminance_only"] is True and fake.calls[0]["passes"] == 3 and fake.calls[0]["adain"]
    assert (tmp_path / "out" / "c_s.png").exists()                            # output name unchanged


# --------------------------------------------------------------------------------------------------- stylize_video.py
def _clip(tmp_path, sizes):
    frames = tmp_path / "clip"
    frames.mkdir()
    for i, hw in enumerate(sizes):
        Image.fromarray(np.full(hw + (3,), i + 1, dtype=np.uint8)).save(str(frames / ("frame_%d.png" % (i + 1))))
    Image.fromarray(np.full((6, 6, 3), 50, np.uint8)).save(str(tmp_path / "s.png"))
    return ["--relu-targets", "relu1_1", "--in-path", str(frames), "--out-path", str(tmp_path / "out"), "--style-path",
            str(tmp_path / "s.png")]


def test_video_flag_parses_and_rejects_keep_colors(tmp_path, capsys):
    argv = ["--relu-targets", "relu1_1", "--in-path", "x", "--out-path", "y", "--style-path", "s.png"]
    assert not V.parse_args(argv).luminance_only
    assert V.parse_args(argv + ["--luminance-only", "--temporal", "0.5"]).luminance_only
    with pytest.raises(SystemExit):
        V.parse_args(argv + ["--luminance-only", "--keep-colors"])
    assert "--keep-colors" in capsys.readouterr().err


def test_video_keeps_batches_with_luminance_only(tmp_path):
    argv = _clip(tmp_path, [(8, 12)] * 5 + [(16, 12)])                      # frame 6 is ragged: one call on its own
    calls = []

    class Fake(_FakeWCT):
        def predict_batch(self, contents, styles, **kw):
            c = np.asarray(contents)
            c = c[None] if c.ndim == 3 else c
            calls.append(([int(x[0, 0, 0]) for x in c], kw))
            return c + 1

    n = V.main(argv + ["--luminance-only", "--batch", "2", "--passes", "2"], wct_factory=lambda a: Fake(),
               image_ops=HostImageOps)
    assert n == 6
    assert [c[0] for c in calls] == [[1, 2], [3, 4], [5], [6]]
    for _, kw in calls:
        assert kw["luminance_only"] is True and kw["passes"] == 2              # merged once, after the last pass
    assert (tmp_path / "out" / "clip_s_frames" / "frame_6.png").exists()


# -------------------------------------------------------------------------------------------------- prepare_styles.py
def test_prepare_styles_prepares_the_grey_under_the_same_name(tmp_path):
    Image.fromarray(np.full((6, 6, 3), 50, np.uint8)).save(str(tmp_path / "starry.png"))
    made = []

    class Prepared(object):
        def save(self, path):
            made.append(path)

    class Model(object):
        class engine(object):
            device = None

        def prepare_style(self, img, **kw):
            made.append(kw)
            return Prepared()

    argv = ["--relu-targets", "relu1_1", "--style-path", str(tmp_path / "starry.png"), "--out-path", str(tmp_path / "p")]
    for extra, want in (([], {}), (["--luminance-only"], {"luminance_only": True})):
        del made[:]
        assert prepare_styles.main(argv + extra, model_factory=lambda a: Model(), image_ops=HostImageOps) == 1
        assert made == [want, str(tmp_path / "p" / "starry.wctstyle")]
