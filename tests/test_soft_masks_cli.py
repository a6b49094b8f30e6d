"""CLI soft spatial control (stylize.py --strength-map / --mask-feather / --mask-weights, stylize_video.py
--strength-map): flag errors, the options passed to predict_batch and the output names; no GPU needed (fake WCT)."""
import numpy as np
import pytest
from PIL import Image

import stylize
import stylize_video


def _base(tmp_path):
    return ["--relu-targets", "relu1_1", "--synthetic-weights", "1", "--content-path", str(tmp_path / "c.png"),
            "--out-path", str(tmp_path / "out")]


@pytest.mark.parametrize("extra", [
    ["--style-path", "s.png", "--mask-feather", "4"],                                      # feather without a mask
    ["--content-mask", "m.png", "--mask-styles", "a.png", "--mask-feather", "0"],
    ["--content-mask", "m.png", "--mask-styles", "a.png", "--mask-feather", "nan"],
    ["--content-mask", "m.png", "--mask-styles", "a.png", "--mask-weights", "w.png"],       # weights with a mask
    ["--mask-styles", "a.png", "b.png", "--mask-weights", "w.png"],                        # one map per style
    ["--mask-styles", "a.png", "--mask-weights", "w.png", "--adain"],
    ["--style-path", "s.png", "--strength-map", "p.png", "--swap5"],
    ["--style-path", "s.png", "--strength-map", "p.png", "--mst", "2"],
    ["--style-path", "s.png", "--strength-map", "p.png", "--tile-size", "64"],
    ["--interp-styles", "a.png", "b.png", "--interp-weights", "1", "1", "--strength-map", "p.png"],
])
def test_soft_flag_errors(tmp_path, extra):
    with pytest.raises(SystemExit):
        stylize.parse_args(_base(tmp_path) + extra)


def test_soft_flags_default_off():
    a = stylize.parse_args(["--relu-targets", "relu1_1"])
    assert a.strength_map is None and a.mask_feather is None and a.mask_weights is None
    assert stylize.soft_kw(a) == {}


def test_video_strength_map_rejections():
    base = ["--relu-targets", "relu1_1", "--in-path", "v.mp4", "--out-path", "o.mp4", "--style-path", "s.png"]
    assert stylize_video.parse_args(base + ["--strength-map", "p.png"]).strength_map == "p.png"
    with pytest.raises(SystemExit):
        stylize_video.parse_args(base + ["--strength-map", "p.png", "--swap5"])


class _Fake(object):
    def __init__(self):
        self.calls = []

    class engine(object):
        device = None

    def predict_batch(self, contents, styles, return_device=False, **kw):
        self.calls.append(kw)
        c = np.asarray(contents)
        return (c[None] if c.ndim == 3 else c) + 1


class _HostImageOps(object):
    to_device = staticmethod(lambda img, device=None: np.asarray(img))
    to_host = staticmethod(lambda img: np.asarray(img))
    resize_to = staticmethod(lambda img, size: img)


def _images(tmp_path):
    Image.fromarray(np.full((8, 12, 3), 10, np.uint8)).save(str(tmp_path / "c.png"))
    for name, v in (("sky", 50), ("sea", 90)):
        Image.fromarray(np.full((6, 6, 3), v, np.uint8)).save(str(tmp_path / (name + ".png")))
    ramp = np.tile(np.linspace(0, 255, 12).astype(np.uint8), (8, 1))
    Image.fromarray(ramp, mode="L").save(str(tmp_path / "p.png"))
    Image.fromarray(255 - ramp, mode="L").save(str(tmp_path / "q.png"))
    m = np.zeros((8, 12), np.uint8)
    m[:, 6:] = 255
    Image.fromarray(m, mode="L").save(str(tmp_path / "m.png"))
    return ramp


def test_strength_map_run(tmp_path):
    ramp = _images(tmp_path)
    fake = _Fake()
    argv = _base(tmp_path) + ["--style-path", str(tmp_path / "sky.png"), "--strength-map", str(tmp_path / "p.png")]
    assert stylize.main(argv, model_factory=lambda a: fake, image_ops=_HostImageOps) == 1
    assert (tmp_path / "out" / "c_sky.png").exists()
    assert np.array_equal(fake.calls[0]["strength_map"], ramp)


def test_feathered_mask_run(tmp_path):
    _images(tmp_path)
    fake = _Fake()
    argv = _base(tmp_path) + ["--content-mask", str(tmp_path / "m.png"), "--mask-styles", str(tmp_path / "sky.png"),
                              str(tmp_path / "sea.png"), "--mask-feather", "3"]
    assert stylize.main(argv, model_factory=lambda a: fake, image_ops=_HostImageOps) == 1
    assert (tmp_path / "out" / "c_sky+sea.png").exists()
    kw = fake.calls[0]
    assert kw["mask_feather"] == 3.0 and kw["content_mask"].max() == 1


def test_mask_weights_run(tmp_path):
    ramp = _images(tmp_path)
    fake = _Fake()
    argv = _base(tmp_path) + ["--mask-styles", str(tmp_path / "sky.png"), str(tmp_path / "sea.png"), "--mask-weights",
                              str(tmp_path / "p.png"), str(tmp_path / "q.png")]
    assert stylize.main(argv, model_factory=lambda a: fake, image_ops=_HostImageOps) == 1
    assert (tmp_path / "out" / "c_sky+sea.png").exists()
    kw = fake.calls[0]
    assert "content_mask" not in kw
    assert np.array_equal(kw["content_weights"], np.stack([ramp, 255 - ramp]))


def test_api_rejections():
    from wct_tf_b200.wct import WCT
    ok = WCT.check_soft_map(np.full((4, 5), 255, np.uint8), 1, "strength_map")
    assert ok.dtype.is_floating_point and float(ok.max()) == 1.0
    for bad in (np.full((4, 5), 1.5), np.full((4, 5), np.nan), np.zeros((2, 2, 4, 5)), np.zeros((4, 5), np.int32)):
        with pytest.raises(ValueError):
            WCT.check_soft_map(bad, 1, "strength_map")
    w = WCT.check_soft_map(np.full((2, 3, 3), 0.8), 1, "content_weights", planes=2)     # sum 1.6 -> divided by it
    assert np.allclose(w.numpy().sum(1), 1.0)
    with pytest.raises(ValueError):
        WCT.check_soft_map(np.full((3, 3, 3), 0.2), 1, "content_weights", planes=2)
