"""stylize.py / stylize_video.py --efdm: the flag parses, every stylising call carries efdm=True (and none without the
flag), on the batched and the frame-by-frame path, and every combination the engine rejects is a parser error.  No GPU
needed (fake models and host image ops)."""
import numpy as np
import pytest
from PIL import Image

import stylize
import stylize_video as V
from tests.test_interp_cli import HostImageOps
from tests.test_temporal_cli import FakeTemporalWCT, _argv, _clip
from tests.test_tiles_cpu import FakeWCT, _base


def test_flag_parses(tmp_path):
    assert not stylize.parse_args(_base(tmp_path) + ["--style-path", "s.png"]).efdm
    a = stylize.parse_args(_base(tmp_path) + ["--style-path", "s.png", "--efdm", "--passes", "2"])
    assert a.efdm and a.passes == 2
    assert V.parse_args(_argv(tmp_path, "x", "s.png", ["--efdm", "--temporal", "0.5"])).efdm


_ERRORS = [(["--style-path", "s.png", "--efdm", "--adain"], "--adain"),
           (["--style-path", "s.png", "--efdm", "--ost"], "--ost"),
           (["--style-path", "s.png", "--efdm", "--mst", "3"], "--mst"),
           (["--content-mask", "m.png", "--mask-styles", "x.png", "--efdm"], "--content-mask"),
           (["--mask-styles", "x.png", "--mask-weights", "w.png", "--efdm"], "--mask-weights"),
           (["--content-mask", "m.png", "--mask-styles", "x.png", "--mask-feather", "2", "--efdm"], "--content-mask"),
           (["--style-path", "s.png", "--strength-map", "m.png", "--efdm"], "--strength-map"),
           (["--interp-styles", "a.png", "b.png", "--interp-weights", "1", "1", "--efdm"], "--interp-styles"),
           (["--style-path", "s.png", "--efdm", "--tile-size", "64"], "--tile-size"),
           (["--style-path", "s.wctstyle", "--efdm"], ".wctstyle")]


@pytest.mark.parametrize("extra,msg", _ERRORS, ids=[m for _, m in _ERRORS])
def test_parser_errors(tmp_path, extra, msg, capsys):
    with pytest.raises(SystemExit):
        stylize.parse_args(_base(tmp_path) + extra)
    assert msg in capsys.readouterr().err


@pytest.mark.parametrize("extra,msg", [(["--adain"], "--adain"), (["--ost"], "--ost"), (["--mst", "2"], "--mst"),
                                       (["--strength-map", "m.png"], "--strength-map")], ids=["adain", "ost", "mst", "strength"])
def test_video_parser_errors(tmp_path, extra, msg, capsys):
    with pytest.raises(SystemExit):
        V.parse_args(_argv(tmp_path, "x", "s.png", extra + ["--efdm"]))
    assert msg in capsys.readouterr().err


def test_stylize_passes_efdm(tmp_path):
    Image.fromarray(np.full((8, 12, 3), 10, np.uint8)).save(str(tmp_path / "c.png"))
    Image.fromarray(np.full((6, 6, 3), 50, np.uint8)).save(str(tmp_path / "s.png"))
    calls = []
    argv = _base(tmp_path) + ["--style-path", str(tmp_path / "s.png"), "--efdm", "--passes", "2"]
    assert stylize.main(argv, model_factory=lambda a: FakeWCT(calls), image_ops=HostImageOps) == 1
    assert len(calls) == 2 and all(kw["efdm"] is True for kw in calls)
    assert (tmp_path / "out" / "c_s.png").exists()
    calls.clear()
    stylize.main(_base(tmp_path) + ["--style-path", str(tmp_path / "s.png")], model_factory=lambda a: FakeWCT(calls),
                 image_ops=HostImageOps)
    assert "efdm" not in calls[0]


@pytest.mark.parametrize("temporal", [[], ["--temporal", "0.5"]], ids=["plain", "temporal"])
def test_video_every_call_carries_efdm(tmp_path, temporal):
    frames, styles = _clip(tmp_path, [(8, 12)] * 3 + [(16, 12)])
    calls, states = [], []
    n = V.main(_argv(tmp_path, frames, styles / "a.png", ["--batch", "2", "--passes", "2", "--efdm"] + temporal),
               wct_factory=lambda a: FakeTemporalWCT(calls, states), image_ops=HostImageOps)
    assert n == 4
    frames_in = [c[0] for c in calls]
    assert [4] in frames_in and [1, 2] in frames_in            # the batched and the frame-by-frame path both ran
    assert all(kw.get("efdm") is True for _, _, kw in calls)
    calls.clear()
    V.main(_argv(tmp_path, frames, styles / "a.png", ["--batch", "2"]), wct_factory=lambda a: FakeTemporalWCT(calls, states),
           image_ops=HostImageOps)
    assert all("efdm" not in kw for _, _, kw in calls)
