"""stylize.py / stylize_video.py --ost: the flag parses, every stylising call carries ost=True (and none without the flag),
on the batched and the frame-by-frame path, and it is a parser error with --adain, --content-mask and --interp-styles.
No GPU needed (fake models and host image ops)."""
import numpy as np
import pytest
from PIL import Image

import stylize
import stylize_video as V
from tests.test_interp_cli import HostImageOps
from tests.test_temporal_cli import FakeTemporalWCT, _argv, _clip
from tests.test_tiles_cpu import FakeWCT, _base


def test_flag_parses(tmp_path):
    assert not stylize.parse_args(_base(tmp_path) + ["--style-path", "s.png"]).ost
    a = stylize.parse_args(_base(tmp_path) + ["--style-path", "s.png", "--ost", "--tile-size", "64"])
    assert a.ost and a.tile_size == 64
    assert V.parse_args(_argv(tmp_path, "x", "s.png", ["--ost", "--temporal", "0.5"])).ost


@pytest.mark.parametrize("extra", [["--style-path", "s.png", "--adain"],
                                   ["--content-mask", "m.png", "--mask-styles", "x.png"],
                                   ["--interp-styles", "a.png", "b.png", "--interp-weights", "1", "1"]],
                         ids=["adain", "content_mask", "interp"])
def test_parser_errors(tmp_path, extra, capsys):
    with pytest.raises(SystemExit):
        stylize.parse_args(_base(tmp_path) + extra + ["--ost"])
    assert "--ost" in capsys.readouterr().err


@pytest.mark.parametrize("extra", [["--adain"], ["--interp-styles", "a.png", "--interp-weights", "1"]], ids=["adain", "interp"])
def test_video_parser_errors(tmp_path, extra, capsys):
    argv = _argv(tmp_path, "x", "s.png", extra + ["--ost"])
    if "--interp-styles" in extra:
        argv.remove("--style-path")
        argv.remove("s.png")
    with pytest.raises(SystemExit):
        V.parse_args(argv)
    assert "--ost" in capsys.readouterr().err


def test_stylize_passes_ost(tmp_path):
    Image.fromarray(np.full((8, 12, 3), 10, np.uint8)).save(str(tmp_path / "c.png"))
    Image.fromarray(np.full((6, 6, 3), 50, np.uint8)).save(str(tmp_path / "s.png"))
    calls = []
    argv = _base(tmp_path) + ["--style-path", str(tmp_path / "s.png"), "--ost", "--passes", "2"]
    assert stylize.main(argv, model_factory=lambda a: FakeWCT(calls), image_ops=HostImageOps) == 1
    assert len(calls) == 2 and all(kw["ost"] is True for kw in calls)
    assert (tmp_path / "out" / "c_s.png").exists()
    calls.clear()
    stylize.main(_base(tmp_path) + ["--style-path", str(tmp_path / "s.png")], model_factory=lambda a: FakeWCT(calls),
                 image_ops=HostImageOps)
    assert "ost" not in calls[0]


@pytest.mark.parametrize("temporal", [[], ["--temporal", "0.5"]], ids=["plain", "temporal"])
def test_video_every_call_carries_ost(tmp_path, temporal):
    frames, styles = _clip(tmp_path, [(8, 12)] * 3 + [(16, 12)])
    calls, states = [], []
    n = V.main(_argv(tmp_path, frames, styles / "a.png", ["--batch", "2", "--passes", "2", "--ost"] + temporal),
               wct_factory=lambda a: FakeTemporalWCT(calls, states), image_ops=HostImageOps)
    assert n == 4
    frames_in = [c[0] for c in calls]
    assert [4] in frames_in and [1, 2] in frames_in            # the batched and the frame-by-frame path both ran
    assert all(kw.get("ost") is True for _, _, kw in calls)
    calls.clear()
    V.main(_argv(tmp_path, frames, styles / "a.png", ["--batch", "2"]), wct_factory=lambda a: FakeTemporalWCT(calls, states),
           image_ops=HostImageOps)
    assert all("ost" not in kw for _, _, kw in calls)
