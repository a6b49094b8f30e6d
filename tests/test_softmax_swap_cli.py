"""--ss-temperature (the softmax swap, DESIGN.md §3.3.17) in stylize.py and stylize_video.py: parsing, the parser errors,
and what reaches predict_batch; no GPU needed (fake WCT and host image ops)."""
import numpy as np
import pytest
from PIL import Image

import stylize
import stylize_video as V
from tests.test_interp_cli import HostImageOps
from tests.test_swap_levels_cli import FakeWCT

TARGETS = ["--relu-targets", "relu5_1", "relu4_1", "relu3_1", "--synthetic-weights", "1"]


def _base(tmp_path):
    return TARGETS + ["--content-path", str(tmp_path / "c.png"), "--style-path", str(tmp_path / "s.png"), "--out-path",
                      str(tmp_path / "out")]


def _video(tmp_path):
    return TARGETS + ["--in-path", str(tmp_path / "in.mp4"), "--out-path", str(tmp_path / "out.mp4"), "--style-path",
                      str(tmp_path / "s.png")]


@pytest.mark.parametrize("argv", [_base, _video])
def test_flag_parses_with_a_swap(tmp_path, argv):
    parse = stylize.parse_args if argv is _base else V.parse_args
    a = parse(argv(tmp_path))
    assert a.ss_temperature is None
    a = parse(argv(tmp_path) + ["--swap5", "--ss-temperature", "0.05"])
    assert a.ss_temperature == 0.05
    a = parse(argv(tmp_path) + ["--swap-targets", "relu3_1", "--ss-temperature", "2"])
    assert a.ss_temperature == 2.0


@pytest.mark.parametrize("argv", [_base, _video])
@pytest.mark.parametrize("extra,match", [
    (["--ss-temperature", "0.1"], "--ss-temperature needs --swap5 / --swap-targets"),
    (["--swap5", "--ss-temperature", "0"], "--ss-temperature must be a finite number > 0"),
    (["--swap5", "--ss-temperature", "-1"], "--ss-temperature must be a finite number > 0"),
    (["--swap5", "--ss-temperature", "nan"], "--ss-temperature must be a finite number > 0"),
    (["--swap5", "--ss-temperature", "inf"], "--ss-temperature must be a finite number > 0"),
    (["--swap5", "--ss-temperature", "warm"], "invalid float value"),
])
def test_parser_errors(tmp_path, capsys, argv, extra, match):
    parse = stylize.parse_args if argv is _base else V.parse_args
    with pytest.raises(SystemExit):
        parse(argv(tmp_path) + extra)
    assert match in capsys.readouterr().err


def test_stylize_passes_the_temperature(tmp_path):
    Image.fromarray(np.full((8, 12, 3), 10, np.uint8)).save(str(tmp_path / "c.png"))
    Image.fromarray(np.full((6, 6, 3), 50, np.uint8)).save(str(tmp_path / "s.png"))
    calls = []
    argv = _base(tmp_path) + ["--swap-targets", "relu3_1", "--ss-temperature", "0.03", "--passes", "2"]
    assert stylize.main(argv, model_factory=lambda a: FakeWCT(calls), image_ops=HostImageOps) == 1
    assert len(calls) == 2
    for kw in calls:
        assert kw["ss_temperature"] == 0.03 and kw["swap_targets"] == ["relu3_1"]
    calls.clear()
    stylize.main(_base(tmp_path) + ["--swap5"], model_factory=lambda a: FakeWCT(calls), image_ops=HostImageOps)
    assert "ss_temperature" not in calls[0]
    assert sorted(p.name for p in (tmp_path / "out").iterdir()) == ["c_s.png"]
