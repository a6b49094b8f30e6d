"""stylize.py / stylize_video.py --efdm-slices: the flag parses, needs --efdm, is range-checked, and reaches every
stylising call (none without it), on the batched and the frame-by-frame path.  No GPU needed (fake models and host image
ops)."""
import numpy as np
import pytest
from PIL import Image

import stylize
import stylize_video as V
from tests.test_interp_cli import HostImageOps
from tests.test_temporal_cli import FakeTemporalWCT, _argv, _clip
from tests.test_tiles_cpu import FakeWCT, _base


def test_flag_parses(tmp_path):
    assert stylize.parse_args(_base(tmp_path) + ["--style-path", "s.png", "--efdm"]).efdm_slices == 0
    a = stylize.parse_args(_base(tmp_path) + ["--style-path", "s.png", "--efdm", "--efdm-slices", "8"])
    assert a.efdm and a.efdm_slices == 8
    assert V.parse_args(_argv(tmp_path, "x", "s.png", ["--efdm", "--efdm-slices", "32"])).efdm_slices == 32


@pytest.mark.parametrize("extra,msg", [(["--efdm-slices", "4"], "--efdm-slices needs --efdm"),
                                       (["--efdm", "--efdm-slices", "33"], "--efdm-slices must be an integer in 0..32"),
                                       (["--efdm", "--efdm-slices", "-1"], "--efdm-slices must be an integer in 0..32"),
                                       (["--efdm", "--efdm-slices", "2.5"], "--efdm-slices"),
                                       (["--efdm", "--efdm-slices", "4", "--adain"], "--adain")],
                         ids=["needs_efdm", "above_32", "negative", "not_integer", "adain"])
def test_parser_errors(tmp_path, extra, msg, capsys):
    with pytest.raises(SystemExit):
        stylize.parse_args(_base(tmp_path) + ["--style-path", "s.png"] + extra)
    assert msg in capsys.readouterr().err
    with pytest.raises(SystemExit):
        V.parse_args(_argv(tmp_path, "x", "s.png", extra))
    assert msg in capsys.readouterr().err


def test_stylize_passes_slices(tmp_path):
    Image.fromarray(np.full((8, 12, 3), 10, np.uint8)).save(str(tmp_path / "c.png"))
    Image.fromarray(np.full((6, 6, 3), 50, np.uint8)).save(str(tmp_path / "s.png"))
    calls = []
    argv = _base(tmp_path) + ["--style-path", str(tmp_path / "s.png"), "--efdm", "--efdm-slices", "4", "--passes", "2"]
    assert stylize.main(argv, model_factory=lambda a: FakeWCT(calls), image_ops=HostImageOps) == 1
    assert len(calls) == 2 and all(kw["efdm"] is True and kw["efdm_slices"] == 4 for kw in calls)
    calls.clear()
    stylize.main(_base(tmp_path) + ["--style-path", str(tmp_path / "s.png"), "--efdm"], model_factory=lambda a: FakeWCT(calls),
                 image_ops=HostImageOps)
    assert "efdm_slices" not in calls[0]


@pytest.mark.parametrize("temporal", [[], ["--temporal", "0.5"]], ids=["plain", "temporal"])
def test_video_every_call_carries_slices(tmp_path, temporal):
    frames, styles = _clip(tmp_path, [(8, 12)] * 3 + [(16, 12)])
    calls, states = [], []
    n = V.main(_argv(tmp_path, frames, styles / "a.png", ["--batch", "2", "--passes", "2", "--efdm", "--efdm-slices", "3"]
                     + temporal), wct_factory=lambda a: FakeTemporalWCT(calls, states), image_ops=HostImageOps)
    assert n == 4
    frames_in = [c[0] for c in calls]
    assert [4] in frames_in and [1, 2] in frames_in            # the batched and the frame-by-frame path both ran
    assert all(kw.get("efdm") is True and kw.get("efdm_slices") == 3 for _, _, kw in calls)
    calls.clear()
    V.main(_argv(tmp_path, frames, styles / "a.png", ["--batch", "2", "--efdm"]), wct_factory=lambda a: FakeTemporalWCT(calls, states),
           image_ops=HostImageOps)
    assert all("efdm_slices" not in kw for _, _, kw in calls)
