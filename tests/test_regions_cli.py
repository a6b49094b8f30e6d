"""CLI spatial control (stylize.py --content-mask / --mask-styles): flag errors, mask quantisation, output naming and
the call the driver makes; no GPU needed (fake WCT)."""
import numpy as np
import pytest
from PIL import Image

import stylize
from tests.regions_ref import mask_regions


def _base(tmp_path):
    return ["--relu-targets", "relu1_1", "--synthetic-weights", "1", "--content-path", str(tmp_path / "c.png"),
            "--out-path", str(tmp_path / "out")]


@pytest.mark.parametrize("extra", [["--style-path", "s.png"], ["--adain"], ["--swap5"], ["--concat"], ["-r", "2"], []])
def test_mask_flag_errors(tmp_path, extra):
    argv = _base(tmp_path) + ["--content-mask", "m.png"] + ([] if extra == [] else ["--mask-styles", "a.png"]) + extra
    with pytest.raises(SystemExit):
        stylize.parse_args(argv)


def test_mask_styles_without_mask_is_an_error(tmp_path):
    with pytest.raises(SystemExit):
        stylize.parse_args(_base(tmp_path) + ["--mask-styles", "a.png"])


def test_mask_flags_default_off():
    a = stylize.parse_args(["--relu-targets", "relu1_1"])
    assert a.content_mask is None and a.mask_styles is None


def test_mask_file_quantisation(tmp_path):
    gray = np.tile(np.arange(256, dtype=np.uint8), (3, 1))
    Image.fromarray(gray, mode="L").save(str(tmp_path / "m.png"))
    Image.fromarray(np.stack([gray] * 3, -1)).save(str(tmp_path / "rgb.png"))       # read as 8-bit grayscale
    for R in (1, 2, 3, 5):
        assert np.array_equal(stylize.read_mask(str(tmp_path / "m.png"), R), mask_regions(gray, R))
        assert np.array_equal(stylize.read_mask(str(tmp_path / "rgb.png"), R), mask_regions(gray, R))
    bw = np.zeros((4, 4), np.uint8)
    bw[:, 2:] = 255
    Image.fromarray(bw, mode="L").save(str(tmp_path / "bw.png"))
    assert np.array_equal(stylize.read_mask(str(tmp_path / "bw.png"), 2), bw // 255)   # black/white -> background/foreground


def test_masked_run_calls_predict_batch_and_names_output(tmp_path):
    Image.fromarray(np.full((8, 12, 3), 10, np.uint8)).save(str(tmp_path / "c.png"))
    for name, v in (("sky", 50), ("sea", 90)):
        Image.fromarray(np.full((6, 6, 3), v, np.uint8)).save(str(tmp_path / (name + ".png")))
    mask = np.zeros((8, 12), np.uint8)
    mask[4:] = 200
    Image.fromarray(mask, mode="L").save(str(tmp_path / "m.png"))
    calls = []

    class FakeWCT(object):
        class engine(object):
            device = None

        def predict_batch(self, contents, styles, alpha=1, content_mask=None, return_device=False, **kw):
            calls.append(([int(np.asarray(s)[0, 0, 0]) for s in styles], np.asarray(content_mask).copy(), alpha, kw))
            c = np.asarray(contents)
            return (c[None] if c.ndim == 3 else c) + 1

    class HostImageOps(object):
        to_device = staticmethod(lambda img, device=None: np.asarray(img))
        to_host = staticmethod(lambda img: np.asarray(img))
        resize_to = staticmethod(lambda img, size: img)

    argv = _base(tmp_path) + ["--content-mask", str(tmp_path / "m.png"), "--mask-styles", str(tmp_path / "sky.png"),
                              str(tmp_path / "sea.png"), "--alpha", "0.7", "--passes", "2"]
    n = stylize.main(argv, model_factory=lambda a: FakeWCT(), image_ops=HostImageOps)
    assert n == 1
    out = tmp_path / "out" / "c_sky+sea.png"
    assert out.exists()
    assert np.array_equal(np.asarray(Image.open(str(out))), np.full((8, 12, 3), 12, np.uint8))   # two passes
    assert len(calls) == 2
    for styles, m, alpha, kw in calls:
        assert styles == [50, 90] and alpha == 0.7 and not kw
        assert np.array_equal(m, (mask.astype(int) * 2 // 256).astype(np.uint8))
