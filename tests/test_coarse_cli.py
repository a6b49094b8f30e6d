"""stylize.py / stylize_video.py --coarse-to-fine and --fine-targets: the flags parse, are checked by the shared options
table and value check, and reach every stylising call (none without them), in stylize.py's one-style, mask and
interpolation modes and on both paths of stylize_video.py.  No GPU needed (fake models and host image ops)."""
import numpy as np
import pytest
from PIL import Image

import stylize
import stylize_video as V
from tests.test_interp_cli import HostImageOps
from tests.test_temporal_cli import FakeTemporalWCT, _argv, _clip
from tests.test_tiles_cpu import FakeWCT, _base


def test_flags_parse(tmp_path):
    a = stylize.parse_args(_base(tmp_path) + ["--style-path", "s.png"])
    assert a.coarse_to_fine == 0 and a.fine_targets is None
    a = stylize.parse_args(_base(tmp_path) + ["--style-path", "s.png", "--coarse-to-fine", "4", "--fine-targets", "relu3_1",
                                              "relu4_1"])
    assert a.coarse_to_fine == 4 and a.fine_targets == ["relu3_1", "relu4_1"]
    a = V.parse_args(_argv(tmp_path, "x", "s.png", ["--coarse-to-fine", "16"]))
    assert a.coarse_to_fine == 16 and a.fine_targets is None
    # combines with the options the table allows
    stylize.parse_args(_base(tmp_path) + ["--style-path", "s.png", "--coarse-to-fine", "2", "--tile-size", "512", "--adain",
                                          "--luminance-only", "--passes", "2"])


@pytest.mark.parametrize("extra,msg", [
    (["--coarse-to-fine", "1"], "--coarse-to-fine must be an integer factor in 2..16"),
    (["--coarse-to-fine", "17"], "--coarse-to-fine must be an integer factor in 2..16"),
    (["--coarse-to-fine", "-2"], "--coarse-to-fine must be an integer factor in 2..16"),
    (["--fine-targets", "relu1_1"], "--fine-targets needs --coarse-to-fine"),
    (["--coarse-to-fine", "0", "--fine-targets", "relu1_1"], "--fine-targets needs --coarse-to-fine"),
    (["--coarse-to-fine", "2", "--fine-targets", "relu2_1"], "--fine-targets: relu2_1 is not a relu target"),
    (["--coarse-to-fine", "2", "--fine-targets", "relu1_1", "relu1_1"], "--fine-targets names a relu target more than once"),
    (["--coarse-to-fine", "2", "--swap5"], "--coarse-to-fine does not combine with --swap5 / --swap-targets"),
    (["--coarse-to-fine", "2", "--seamless", "xy"], "--coarse-to-fine does not combine with --seamless"),
    (["--coarse-to-fine", "2", "--mst", "2"], "--coarse-to-fine does not combine with --mst"),
], ids=["one", "above_16", "negative", "fine_alone", "fine_with_zero", "foreign", "repeated", "swap", "seamless", "mst"])
def test_parser_errors(tmp_path, extra, msg, capsys):
    targets = ["--relu-targets", "relu5_1", "relu4_1", "relu1_1"]
    with pytest.raises(SystemExit):
        stylize.parse_args(targets + _base(tmp_path)[4:] + ["--style-path", "s.png"] + extra)
    assert msg in capsys.readouterr().err
    with pytest.raises(SystemExit):
        V.parse_args(targets + _argv(tmp_path, "x", "s.png", extra)[2:])
    assert msg in capsys.readouterr().err


def test_default_fine_targets_need_a_fine_level(tmp_path, capsys):
    with pytest.raises(SystemExit):
        stylize.parse_args(["--relu-targets", "relu5_1", "relu4_1"] + _base(tmp_path)[4:] + ["--style-path", "s.png",
                                                                                              "--coarse-to-fine", "2"])
    assert "none of the default fine targets" in capsys.readouterr().err


def _images(tmp_path):
    Image.fromarray(np.full((8, 12, 3), 10, np.uint8)).save(str(tmp_path / "c.png"))
    for name in ("s", "t"):
        Image.fromarray(np.full((6, 6, 3), 50, np.uint8)).save(str(tmp_path / (name + ".png")))
    Image.fromarray(np.zeros((8, 12), np.uint8)).save(str(tmp_path / "m.png"))


@pytest.mark.parametrize("mode", ["one", "mask", "interp"])
def test_stylize_passes_the_options(tmp_path, mode):
    _images(tmp_path)
    s, t = str(tmp_path / "s.png"), str(tmp_path / "t.png")
    extra = {"one": ["--style-path", s], "mask": ["--content-mask", str(tmp_path / "m.png"), "--mask-styles", s, t],
             "interp": ["--interp-styles", s, t, "--interp-weights", "1", "2"]}[mode]
    calls = []
    argv = _base(tmp_path) + extra + ["--coarse-to-fine", "3", "--fine-targets", "relu4_1", "--passes", "2"]
    assert stylize.main(argv, model_factory=lambda a: FakeWCT(calls), image_ops=HostImageOps) == 1
    assert len(calls) == 2 and all(kw["coarse_to_fine"] == 3 and kw["fine_targets"] == ["relu4_1"] for kw in calls)
    calls.clear()
    stylize.main(_base(tmp_path) + extra, model_factory=lambda a: FakeWCT(calls), image_ops=HostImageOps)
    assert all("coarse_to_fine" not in kw and "fine_targets" not in kw for kw in calls)


@pytest.mark.parametrize("temporal", [[], ["--temporal", "0.5"]], ids=["plain", "temporal"])
def test_video_every_call_carries_the_options(tmp_path, temporal):
    frames, styles = _clip(tmp_path, [(8, 12)] * 3 + [(16, 12)])
    calls, states = [], []
    n = V.main(_argv(tmp_path, frames, styles / "a.png", ["--batch", "2", "--passes", "2", "--coarse-to-fine", "2"] + temporal),
               wct_factory=lambda a: FakeTemporalWCT(calls, states), image_ops=HostImageOps)
    assert n == 4
    frames_in = [c[0] for c in calls]
    assert [4] in frames_in and [1, 2] in frames_in            # the batched and the frame-by-frame path both ran
    assert all(kw.get("coarse_to_fine") == 2 and kw.get("fine_targets") is None for _, _, kw in calls)
    calls.clear()
    V.main(_argv(tmp_path, frames, styles / "a.png", ["--batch", "2"]), wct_factory=lambda a: FakeTemporalWCT(calls, states),
           image_ops=HostImageOps)
    assert all("coarse_to_fine" not in kw for _, _, kw in calls)
