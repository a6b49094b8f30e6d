"""CLI texture synthesis (stylize.py --noise, --noise-size, --noise-count, --noise-seed): flag defaults and errors, output
naming and the predict_batch calls the driver makes for a style file or folder, a blend and a mask; no GPU needed (fake WCT,
host image ops with the NumPy noise of tests/texture_ref.py)."""
import numpy as np
import pytest
from PIL import Image

import stylize
from tests.texture_ref import noise_u8


def _base(tmp_path):
    return ["--relu-targets", "relu1_1", "--synthetic-weights", "1", "--out-path", str(tmp_path / "out")]


def test_noise_flags_default_off():
    a = stylize.parse_args(["--relu-targets", "relu1_1"])
    assert not a.noise and a.noise_size is None and a.noise_count is None and a.noise_seed is None


def test_noise_flag_defaults_and_values(tmp_path):
    a = stylize.parse_args(_base(tmp_path) + ["--noise", "--style-path", "s.png"])
    assert a.noise and a.noise_size == [512, 512] and a.noise_count == 1 and a.noise_seed == 0
    b = stylize.parse_args(_base(tmp_path) + ["--noise", "--noise-size", "768", "512", "--noise-count", "4", "--noise-seed",
                                              str(2**64 - 1), "--style-path", "s.png", "--passes", "2", "--adain", "--concat"])
    assert b.noise_size == [768, 512] and b.noise_count == 4 and b.noise_seed == 2**64 - 1


@pytest.mark.parametrize("extra", [["--content-path", "c.png"], ["--content-size", "256"], ["--keep-colors"],
                                   ["--noise-count", "0"], ["--noise-count", "-2"], ["--noise-size", "0", "512"],
                                   ["--noise-size", "512", "-1"], ["--noise-seed", "-1"], ["--noise-seed", str(2**64)]])
def test_noise_flag_errors(tmp_path, extra):
    with pytest.raises(SystemExit):
        stylize.parse_args(_base(tmp_path) + ["--noise", "--style-path", "s.png"] + extra)


@pytest.mark.parametrize("extra", [["--noise-size", "64", "64"], ["--noise-count", "2"], ["--noise-seed", "3"]])
def test_noise_options_need_noise(tmp_path, extra):
    with pytest.raises(SystemExit):
        stylize.parse_args(_base(tmp_path) + ["--content-path", "c.png", "--style-path", "s.png"] + extra)


def test_noise_names():
    assert stylize.noise_names(0, 4) == ["noise0-0.png", "noise0-1.png", "noise0-2.png", "noise0-3.png"]
    assert stylize.interp_output_name(stylize.noise_names(0, 1)[0], ["a.jpg", "b.jpg"], [3, 1]) == "noise0-0_a-0.75+b-0.25.png"
    assert stylize.mask_output_name(stylize.noise_names(7, 1)[0], ["sky.jpg", "sea.jpg"]) == "noise7-0_sky+sea.png"


class HostImageOps(object):
    to_device = staticmethod(lambda img, device=None: np.asarray(img))
    to_host = staticmethod(lambda img: np.asarray(img))
    resize_to = staticmethod(lambda img, size: img)
    center_crop = staticmethod(lambda img, size: img)
    concat_with_style = staticmethod(lambda style, result: np.concatenate([np.zeros_like(result), result], axis=1))

    @staticmethod
    def noise_u8(count, height, width, seed=0, first_index=0, device=None):
        return noise_u8(count, height, width, 3, seed=seed, first_index=first_index)


class FakeWCT(object):
    class engine(object):
        device = None

    def __init__(self):
        self.calls = []

    def predict_batch(self, contents, styles, **kw):
        c = np.asarray(contents)
        self.calls.append((c.copy(), styles, kw))
        return (c[None] if c.ndim == 3 else c) + 1


def _styles(tmp_path, names_values, folder=None):
    d = tmp_path if folder is None else tmp_path / folder
    d.mkdir(exist_ok=True)
    for name, v in names_values:
        Image.fromarray(np.full((6, 6, 3), v, np.uint8)).save(str(d / (name + ".png")))
    return d


def _read(path):
    return np.asarray(Image.open(str(path)))


def test_style_file_one_batched_call_per_pass_and_names(tmp_path):
    _styles(tmp_path, [("starry", 40)])
    wct = FakeWCT()
    argv = _base(tmp_path) + ["--noise", "--noise-count", "4", "--noise-size", "8", "12", "--noise-seed", "5", "--style-path",
                              str(tmp_path / "starry.png"), "--alpha", "0.7", "--adain", "--passes", "2"]
    n = stylize.main(argv, model_factory=lambda a: wct, image_ops=HostImageOps)
    assert n == 4
    ref = noise_u8(4, 8, 12, 3, seed=5)
    assert len(wct.calls) == 2                                        # one call per pass, all four frames in each
    first, second = wct.calls
    assert first[0].dtype == np.uint8 and first[0].shape == (4, 8, 12, 3) and np.array_equal(first[0], ref)
    assert np.array_equal(second[0], ref + 1)
    assert int(np.asarray(first[1])[0, 0, 0]) == 40
    assert first[2]["alpha"] == 0.7 and first[2]["adain"] and first[2]["return_device"]
    for i in range(4):
        assert np.array_equal(_read(tmp_path / "out" / ("noise5-%d_starry.png" % i)), ref[i] + 2)
    assert sorted(p.name for p in (tmp_path / "out").iterdir()) == ["noise5-%d_starry.png" % i for i in range(4)]


def test_style_folder_one_call_per_style_with_concat(tmp_path):
    sdir = _styles(tmp_path, [("a", 10), ("b", 20)], folder="styles")
    wct = FakeWCT()
    argv = _base(tmp_path) + ["--noise", "--noise-count", "3", "--noise-size", "6", "5", "--style-path", str(sdir), "--concat",
                              "--swap5"]
    assert stylize.main(argv, model_factory=lambda a: wct, image_ops=HostImageOps) == 6
    assert len(wct.calls) == 2
    assert sorted(int(np.asarray(c[1])[0, 0, 0]) for c in wct.calls) == [10, 20]
    ref = noise_u8(3, 6, 5, 3, seed=0)
    for c in wct.calls:
        assert np.array_equal(c[0], ref) and c[2]["swap5"]
    for s in ("a", "b"):
        for i in range(3):
            out = _read(tmp_path / "out" / ("noise0-%d_%s.png" % (i, s)))
            assert out.shape == (6, 10, 3) and np.array_equal(out[:, 5:], ref[i] + 1)


def test_blend_one_call_and_names(tmp_path):
    _styles(tmp_path, [("a", 50), ("b", 90)])
    wct = FakeWCT()
    argv = _base(tmp_path) + ["--noise", "--noise-count", "2", "--noise-size", "4", "4", "--interp-styles", str(tmp_path / "a.png"),
                              str(tmp_path / "b.png"), "--interp-weights", "3", "1"]
    assert stylize.main(argv, model_factory=lambda a: wct, image_ops=HostImageOps) == 2
    assert len(wct.calls) == 1
    contents, styles, kw = wct.calls[0]
    assert np.array_equal(contents, noise_u8(2, 4, 4, 3)) and [int(np.asarray(s)[0, 0, 0]) for s in styles] == [50, 90]
    assert np.array_equal(kw["style_weights"], [3.0, 1.0])
    for i in range(2):
        assert (tmp_path / "out" / ("noise0-%d_a-0.75+b-0.25.png" % i)).exists()


def test_mask_one_call_and_names(tmp_path):
    _styles(tmp_path, [("sky", 50), ("sea", 90)])
    mask = np.zeros((4, 6), np.uint8)
    mask[2:] = 255
    Image.fromarray(mask, mode="L").save(str(tmp_path / "m.png"))
    wct = FakeWCT()
    argv = _base(tmp_path) + ["--noise", "--noise-count", "3", "--noise-size", "4", "6", "--noise-seed", "9", "--content-mask",
                              str(tmp_path / "m.png"), "--mask-styles", str(tmp_path / "sky.png"), str(tmp_path / "sea.png")]
    assert stylize.main(argv, model_factory=lambda a: wct, image_ops=HostImageOps) == 3
    assert len(wct.calls) == 1
    contents, styles, kw = wct.calls[0]
    assert np.array_equal(contents, noise_u8(3, 4, 6, 3, seed=9)) and np.array_equal(kw["content_mask"], mask // 255)
    for i in range(3):
        assert (tmp_path / "out" / ("noise9-%d_sky+sea.png" % i)).exists()
