"""stylize.py / stylize_video.py --mst K [--mst-smooth LAMBDA]: the flags parse with their defaults, every stylising call
carries mst and mst_smooth (and none without the flag), on the batched and the frame-by-frame path, and every combination
the engine rejects is a parser error.  No GPU needed (fake models and host image ops)."""
import numpy as np
import pytest
from PIL import Image

import stylize
import stylize_video as V
from tests.test_interp_cli import HostImageOps
from tests.test_temporal_cli import FakeTemporalWCT, _argv, _clip
from tests.test_tiles_cpu import FakeWCT, _base


def test_flags_and_defaults(tmp_path):
    a = stylize.parse_args(_base(tmp_path) + ["--style-path", "s.png"])
    assert a.mst is None and a.mst_smooth is None
    a = stylize.parse_args(_base(tmp_path) + ["--style-path", "s.png", "--mst", "3"])
    assert a.mst == 3 and a.mst_smooth == 0.05
    a = stylize.parse_args(_base(tmp_path) + ["--style-path", "s.png", "--mst", "8", "--mst-smooth", "0", "--passes", "2"])
    assert a.mst == 8 and a.mst_smooth == 0.0
    v = V.parse_args(_argv(tmp_path, "x", "s.png", ["--mst", "2", "--mst-smooth", "0.2", "--temporal", "0.5"]))
    assert v.mst == 2 and v.mst_smooth == 0.2


_ERRORS = [(["--style-path", "s.png", "--mst", "0"], "--mst"),
           (["--style-path", "s.png", "--mst", "9"], "--mst"),
           (["--style-path", "s.png", "--mst", "3", "--mst-smooth", "-0.1"], "--mst-smooth"),
           (["--style-path", "s.png", "--mst", "3", "--mst-smooth", "nan"], "--mst-smooth"),
           (["--style-path", "s.png", "--mst", "3", "--mst-smooth", "inf"], "--mst-smooth"),
           (["--style-path", "s.png", "--mst-smooth", "0.1"], "--mst-smooth needs --mst"),
           (["--style-path", "s.png", "--mst", "3", "--adain"], "--adain"),
           (["--style-path", "s.png", "--mst", "3", "--ost"], "--ost"),
           (["--content-mask", "m.png", "--mask-styles", "x.png", "--mst", "3"], "--content-mask"),
           (["--interp-styles", "a.png", "b.png", "--interp-weights", "1", "1", "--mst", "3"], "--interp-styles"),
           (["--style-path", "s.png", "--mst", "3", "--swap5"], "--swap5"),
           (["--style-path", "s.png", "--mst", "3", "--swap-targets", "relu1_1"], "--swap-targets"),
           (["--style-path", "s.png", "--mst", "3", "--tile-size", "64"], "--tile-size"),
           (["--style-path", "s.png", "--mst", "3", "--seamless", "x"], "--seamless"),
           (["--style-path", "s.wctstyle", "--mst", "3"], ".wctstyle")]


@pytest.mark.parametrize("extra,msg", _ERRORS, ids=["k0", "k9", "lam_neg", "lam_nan", "lam_inf", "smooth_alone", "adain", "ost",
                                                    "content_mask", "interp", "swap5", "swap_targets", "tiles", "seamless",
                                                    "prepared"])
def test_parser_errors(tmp_path, extra, msg, capsys):
    with pytest.raises(SystemExit):
        stylize.parse_args(_base(tmp_path) + extra)
    assert msg in capsys.readouterr().err


def test_prepared_styles_in_a_folder_are_a_parser_error(tmp_path, capsys):
    d = tmp_path / "styles"
    d.mkdir()
    (d / "a.wctstyle").write_bytes(b"")
    with pytest.raises(SystemExit):
        stylize.parse_args(_base(tmp_path) + ["--style-path", str(d), "--mst", "2"])
    assert ".wctstyle" in capsys.readouterr().err


@pytest.mark.parametrize("extra", [["--adain"], ["--ost"], ["--seamless", "x"], ["--swap5"], ["--mst-smooth", "-1"]],
                         ids=["adain", "ost", "seamless", "swap5", "lam_neg"])
def test_video_parser_errors(tmp_path, extra, capsys):
    with pytest.raises(SystemExit):
        V.parse_args(_argv(tmp_path, "x", "s.png", extra + ["--mst", "3"]))
    assert "--mst" in capsys.readouterr().err


def test_video_smooth_needs_mst(tmp_path, capsys):
    with pytest.raises(SystemExit):
        V.parse_args(_argv(tmp_path, "x", "s.png", ["--mst-smooth", "0.1"]))
    assert "--mst-smooth needs --mst" in capsys.readouterr().err


def test_stylize_passes_mst(tmp_path):
    Image.fromarray(np.full((8, 12, 3), 10, np.uint8)).save(str(tmp_path / "c.png"))
    Image.fromarray(np.full((6, 6, 3), 50, np.uint8)).save(str(tmp_path / "s.png"))
    calls = []
    argv = _base(tmp_path) + ["--style-path", str(tmp_path / "s.png"), "--mst", "4", "--mst-smooth", "0.2", "--passes", "2"]
    assert stylize.main(argv, model_factory=lambda a: FakeWCT(calls), image_ops=HostImageOps) == 1
    assert len(calls) == 2 and all(kw["mst"] == 4 and kw["mst_smooth"] == 0.2 for kw in calls)
    assert (tmp_path / "out" / "c_s.png").exists()
    calls.clear()
    stylize.main(_base(tmp_path) + ["--style-path", str(tmp_path / "s.png")], model_factory=lambda a: FakeWCT(calls),
                 image_ops=HostImageOps)
    assert "mst" not in calls[0] and "mst_smooth" not in calls[0]


@pytest.mark.parametrize("temporal", [[], ["--temporal", "0.5"]], ids=["plain", "temporal"])
def test_video_every_call_carries_mst(tmp_path, temporal):
    frames, styles = _clip(tmp_path, [(8, 12)] * 3 + [(16, 12)])
    calls, states = [], []
    n = V.main(_argv(tmp_path, frames, styles / "a.png", ["--batch", "2", "--passes", "2", "--mst", "3"] + temporal),
               wct_factory=lambda a: FakeTemporalWCT(calls, states), image_ops=HostImageOps)
    assert n == 4
    frames_in = [c[0] for c in calls]
    assert [4] in frames_in and [1, 2] in frames_in            # the batched and the frame-by-frame path both ran
    assert all(kw.get("mst") == 3 and kw.get("mst_smooth") == 0.05 for _, _, kw in calls)
    calls.clear()
    V.main(_argv(tmp_path, frames, styles / "a.png", ["--batch", "2"]), wct_factory=lambda a: FakeTemporalWCT(calls, states),
           image_ops=HostImageOps)
    assert all("mst" not in kw for _, _, kw in calls)
