"""stylize.py --swap-labels: parsing, the joint colour -> label mapping of the two maps, every parser error, and what reaches
predict_batch; no GPU needed (fake WCT and host image ops)."""
import numpy as np
import pytest
from PIL import Image

import stylize
from tests.test_interp_cli import HostImageOps
from tests.test_swap_levels_cli import FakeWCT

TARGETS = ["--relu-targets", "relu5_1", "relu4_1", "relu3_1", "--synthetic-weights", "1"]


def _maps(tmp_path):
    c = np.zeros((8, 12, 3), np.uint8)
    c[:, 6:] = (0, 0, 255)
    c[6:, :] = (255, 0, 0)
    s = np.zeros((6, 6, 3), np.uint8)
    s[3:] = (0, 0, 255)
    s[:, :2] = (0, 255, 0)
    Image.fromarray(c).save(str(tmp_path / "cm.png"))
    Image.fromarray(s).save(str(tmp_path / "sm.png"))
    Image.fromarray(np.full((8, 12, 3), 10, np.uint8)).save(str(tmp_path / "c.png"))
    Image.fromarray(np.full((6, 6, 3), 50, np.uint8)).save(str(tmp_path / "s.png"))
    return c, s


def _argv(tmp_path, *extra):
    return TARGETS + ["--content-path", str(tmp_path / "c.png"), "--style-path", str(tmp_path / "s.png"), "--out-path",
                      str(tmp_path / "out"), "--swap-targets", "relu3_1", "--swap-labels", str(tmp_path / "cm.png"),
                      str(tmp_path / "sm.png")] + list(extra)


def test_joint_colour_labels(tmp_path):
    c, s = _maps(tmp_path)
    a = stylize.parse_args(_argv(tmp_path))
    cl, sl = a.swap_label_maps
    # colours sorted by packed 24-bit value: black 0x000000, blue 0x0000ff, green 0x00ff00, red 0xff0000
    packed = {(0, 0, 0): 0, (0, 0, 255): 1, (0, 255, 0): 2, (255, 0, 0): 3}
    assert cl.dtype == np.uint8 and cl.shape == (8, 12) and sl.shape == (6, 6)
    assert np.array_equal(cl, np.vectorize(lambda *p: packed[p])(c[..., 0], c[..., 1], c[..., 2]))
    assert np.array_equal(sl, np.vectorize(lambda *p: packed[p])(s[..., 0], s[..., 1], s[..., 2]))


def test_grey_maps(tmp_path):
    _maps(tmp_path)
    Image.fromarray(np.array([[0, 200], [90, 90]], np.uint8)).save(str(tmp_path / "cm.png"))
    Image.fromarray(np.array([[90, 0]], np.uint8)).save(str(tmp_path / "sm.png"))
    cl, sl = stylize.parse_args(_argv(tmp_path)).swap_label_maps
    assert cl.tolist() == [[0, 2], [1, 1]] and sl.tolist() == [[1, 0]]


def test_too_many_colours(tmp_path, capsys):
    _maps(tmp_path)
    noisy = np.random.default_rng(0).integers(0, 256, (20, 20, 3), dtype=np.uint8)
    Image.fromarray(noisy).save(str(tmp_path / "cm.png"))
    with pytest.raises(SystemExit):
        stylize.parse_args(_argv(tmp_path))
    err = capsys.readouterr().err
    assert "at most 256" in err and "flat colours (PNG, not JPEG)" in err


@pytest.mark.parametrize("case,match", [
    ("no_swap", "needs --swap5 or --swap-targets"),
    ("style_folder", "one --style-path file"),
    ("random", "one --style-path file"),
    ("content_folder", "one --content-path file or --noise"),
    ("crop", "takes no --crop-size"),
    ("missing_map", "--swap-labels"),
    ("one_map", "--swap-labels"),
    ("content_mask", "--content-mask"),
])
def test_parser_errors(tmp_path, capsys, case, match):
    _maps(tmp_path)
    argv = _argv(tmp_path)
    if case == "no_swap":
        i = argv.index("--swap-targets")
        del argv[i:i + 2]
    elif case == "style_folder":
        argv[argv.index("--style-path") + 1] = str(tmp_path)
    elif case == "random":
        argv += ["-r", "2"]
    elif case == "content_folder":
        argv[argv.index("--content-path") + 1] = str(tmp_path)
    elif case == "crop":
        argv += ["--crop-size", "4"]
    elif case == "missing_map":
        argv[argv.index("--swap-labels") + 2] = str(tmp_path / "nope.png")
    elif case == "one_map":
        i = argv.index("--swap-labels")
        argv = argv[:i + 2]
    elif case == "content_mask":
        argv += ["--content-mask", str(tmp_path / "cm.png"), "--mask-styles", str(tmp_path / "s.png")]
        i = argv.index("--style-path")
        del argv[i:i + 2]
    with pytest.raises(SystemExit):
        stylize.parse_args(argv)
    assert match in capsys.readouterr().err


def test_swap5_noise_and_prepared_parse(tmp_path):
    _maps(tmp_path)
    argv = _argv(tmp_path)
    i = argv.index("--swap-targets")
    argv[i:i + 2] = ["--swap5"]
    assert stylize.parse_args(argv).swap_label_maps[0].shape == (8, 12)
    j = argv.index("--content-path")
    del argv[j:j + 2]
    assert stylize.parse_args(argv + ["--noise", "--noise-count", "3"]).noise
    argv[argv.index("--style-path") + 1] = str(tmp_path / "s.wctstyle")
    assert stylize.parse_args(argv + ["--noise"]).swap_labels is not None


def test_labels_reach_predict_batch(tmp_path):
    _maps(tmp_path)
    calls = []
    assert stylize.main(_argv(tmp_path, "--ss-alpha", "0.5"), model_factory=lambda a: FakeWCT(calls),
                        image_ops=HostImageOps) == 1
    cl, sl = calls[0]["swap_labels"]
    assert cl.shape == (8, 12) and sl.shape == (6, 6) and calls[0]["swap_targets"] == ["relu3_1"]
    assert (tmp_path / "out" / "c_s.png").exists()              # output names are unchanged
    calls.clear()
    argv = _argv(tmp_path)
    i = argv.index("--swap-labels")
    stylize.main(argv[:i], model_factory=lambda a: FakeWCT(calls), image_ops=HostImageOps)
    assert "swap_labels" not in calls[0]
