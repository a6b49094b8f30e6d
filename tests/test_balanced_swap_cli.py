"""--ss-balance (the balanced swap, DESIGN.md §3.3.18) in stylize.py and stylize_video.py: parsing, the parser errors,
and what reaches predict_batch; no GPU needed (fake WCT and host image ops)."""
import numpy as np
import pytest
from PIL import Image

import stylize
import stylize_video as V
from tests.test_interp_cli import HostImageOps
from tests.test_softmax_swap_cli import _base, _video
from tests.test_swap_levels_cli import FakeWCT


@pytest.mark.parametrize("argv", [_base, _video])
def test_flag_parses_with_a_temperature(tmp_path, argv):
    parse = stylize.parse_args if argv is _base else V.parse_args
    a = parse(argv(tmp_path))
    assert a.ss_balance is None
    a = parse(argv(tmp_path) + ["--swap5", "--ss-temperature", "0.05", "--ss-balance", "4"])
    assert a.ss_balance == 4
    a = parse(argv(tmp_path) + ["--swap-targets", "relu3_1", "--ss-temperature", "2", "--ss-balance", "0"])
    assert a.ss_balance == 0
    a = parse(argv(tmp_path) + ["--swap5", "--ss-balance", "0"])      # 0 is the softmax swap: no temperature needed
    assert a.ss_balance == 0


@pytest.mark.parametrize("argv", [_base, _video])
@pytest.mark.parametrize("extra,match", [
    (["--swap5", "--ss-balance", "4"], "--ss-balance needs --ss-temperature"),
    (["--ss-balance", "4"], "--ss-balance needs --ss-temperature"),
    (["--swap5", "--ss-temperature", "0.1", "--ss-balance", "-1"], "--ss-balance must be an integer in 0..256"),
    (["--swap5", "--ss-temperature", "0.1", "--ss-balance", "257"], "--ss-balance must be an integer in 0..256"),
    (["--swap5", "--ss-temperature", "0.1", "--ss-balance", "1.5"], "invalid int value"),
    (["--swap5", "--ss-temperature", "0.1", "--ss-balance", "many"], "invalid int value"),
])
def test_parser_errors(tmp_path, capsys, argv, extra, match):
    parse = stylize.parse_args if argv is _base else V.parse_args
    with pytest.raises(SystemExit):
        parse(argv(tmp_path) + extra)
    assert match in capsys.readouterr().err


def test_stylize_passes_the_iterations(tmp_path):
    Image.fromarray(np.full((8, 12, 3), 10, np.uint8)).save(str(tmp_path / "c.png"))
    Image.fromarray(np.full((6, 6, 3), 50, np.uint8)).save(str(tmp_path / "s.png"))
    calls = []
    argv = _base(tmp_path) + ["--swap-targets", "relu3_1", "--ss-temperature", "0.03", "--ss-balance", "8", "--passes", "2"]
    assert stylize.main(argv, model_factory=lambda a: FakeWCT(calls), image_ops=HostImageOps) == 1
    assert len(calls) == 2
    for kw in calls:
        assert kw["ss_balance"] == 8 and kw["ss_temperature"] == 0.03 and kw["swap_targets"] == ["relu3_1"]
    calls.clear()
    stylize.main(_base(tmp_path) + ["--swap5", "--ss-temperature", "0.03"], model_factory=lambda a: FakeWCT(calls),
                 image_ops=HostImageOps)
    assert "ss_balance" not in calls[0]
    assert sorted(p.name for p in (tmp_path / "out").iterdir()) == ["c_s.png"]
