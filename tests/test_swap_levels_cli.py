"""CLI style swap at any level (stylize.py / stylize_video.py / prepare_styles.py --swap-targets): parsing, every parser
error and the calls each driver makes; no GPU needed (fake WCT and host image ops)."""
import numpy as np
import pytest
from PIL import Image

import prepare_styles
import stylize
import stylize_video as V
from tests.test_interp_cli import HostImageOps

TARGETS = ["--relu-targets", "relu5_1", "relu4_1", "relu3_1"]


def _base(tmp_path):
    return TARGETS + ["--synthetic-weights", "1", "--content-path", str(tmp_path / "c.png"), "--out-path", str(tmp_path / "out")]


def test_swap_targets_parse(tmp_path):
    a = stylize.parse_args(_base(tmp_path) + ["--style-path", "s.png"])
    assert a.swap_targets is None
    b = stylize.parse_args(_base(tmp_path) + ["--style-path", "s.png", "--swap-targets", "relu4_1", "relu3_1", "--ss-stride", "2"])
    assert b.swap_targets == ["relu4_1", "relu3_1"] and b.ss_stride == 2


@pytest.mark.parametrize("extra", [["--style-path", "s.png", "--swap5"],
                                   ["--style-path", "s.png", "--swap-targets", "relu2_1"],
                                   ["--content-mask", "m.png", "--mask-styles", "x.png"],
                                   ["--interp-styles", "a.png", "b.png", "--interp-weights", "1", "1"]],
                         ids=["swap5", "not_a_target", "content_mask", "interp"])
def test_swap_targets_parser_errors(tmp_path, extra, capsys):
    argv = _base(tmp_path) + extra
    if "--swap-targets" not in extra:
        argv += ["--swap-targets", "relu3_1"]
    with pytest.raises(SystemExit):
        stylize.parse_args(argv)
    assert "--swap-targets" in capsys.readouterr().err


class FakeWCT(object):
    class engine(object):
        device = None

    def __init__(self, calls):
        self.calls = calls

    def predict_batch(self, contents, styles, **kw):
        self.calls.append(kw)
        c = np.asarray(contents)
        return (c[None] if c.ndim == 3 else c) + 1


def _images(tmp_path):
    Image.fromarray(np.full((8, 12, 3), 10, np.uint8)).save(str(tmp_path / "c.png"))
    Image.fromarray(np.full((6, 6, 3), 50, np.uint8)).save(str(tmp_path / "s.png"))


def test_stylize_passes_swap_targets(tmp_path):
    _images(tmp_path)
    calls = []
    argv = _base(tmp_path) + ["--style-path", str(tmp_path / "s.png"), "--swap-targets", "relu3_1", "--passes", "2",
                              "--ss-alpha", "0.5"]
    assert stylize.main(argv, model_factory=lambda a: FakeWCT(calls), image_ops=HostImageOps) == 1
    assert len(calls) == 2                      # stylize.py repeats its call per pass, as with --swap5
    for kw in calls:
        assert kw["swap_targets"] == ["relu3_1"] and kw["swap5"] is False and kw["ss_alpha"] == 0.5
    calls.clear()
    stylize.main(_base(tmp_path) + ["--style-path", str(tmp_path / "s.png")], model_factory=lambda a: FakeWCT(calls),
                 image_ops=HostImageOps)
    assert "swap_targets" not in calls[0]


def _video(tmp_path, sizes):
    frames = tmp_path / "clip"
    frames.mkdir()
    for i, hw in enumerate(sizes):
        Image.fromarray(np.full(hw + (3,), i + 1, dtype=np.uint8)).save(str(frames / ("frame_%d.png" % (i + 1))))
    Image.fromarray(np.full((6, 6, 3), 50, np.uint8)).save(str(tmp_path / "s.png"))
    return TARGETS + ["--in-path", str(frames), "--out-path", str(tmp_path / "out"), "--style-path", str(tmp_path / "s.png")]


@pytest.mark.parametrize("extra", [["--swap5"], ["--swap-targets", "relu1_1"], ["--interp-styles", "a.png", "b.png", "--morph"]],
                         ids=["swap5", "not_a_target", "morph"])
def test_video_swap_targets_parser_errors(tmp_path, extra):
    argv = TARGETS + ["--in-path", "x", "--out-path", "y"] + extra
    if "--interp-styles" not in extra:
        argv += ["--style-path", "s.png"]
    if "--swap-targets" not in extra:
        argv += ["--swap-targets", "relu3_1"]
    with pytest.raises(SystemExit):
        V.parse_args(argv)


def test_video_batches_swap_targets(tmp_path):
    argv = _video(tmp_path, [(8, 12)] * 3 + [(16, 12)]) + ["--swap-targets", "relu3_1", "--batch", "3", "--passes", "2"]
    calls = []
    assert V.main(argv, wct_factory=lambda a: FakeWCT(calls), image_ops=HostImageOps) == 4
    batched, single = calls[0], calls[1:]
    assert batched["swap_targets"] == ["relu3_1"] and batched["passes"] == 2 and "swap5" not in batched
    # the ragged frame: one call per pass, the swap in the first only
    assert single[0]["swap_targets"] == ["relu3_1"] and "swap_targets" not in single[1] and not single[1]["swap5"]


class FakePrepModel(object):
    class engine(object):
        device = None

    def __init__(self, calls):
        self.calls = calls

    def prepare_style(self, img, **kw):
        self.calls.append(kw)
        return self

    def save(self, path):
        open(path, "w").close()


def test_prepare_styles_swap_targets(tmp_path):
    _images(tmp_path)
    calls = []
    argv = TARGETS + ["--synthetic-weights", "1", "--style-path", str(tmp_path / "s.png"), "--out-path", str(tmp_path / "p")]
    prepare_styles.main(argv + ["--swap-targets", "relu3_1"], model_factory=lambda a: FakePrepModel(calls),
                        image_ops=HostImageOps)
    prepare_styles.main(argv, model_factory=lambda a: FakePrepModel(calls), image_ops=HostImageOps)
    assert calls == [dict(swap_targets=["relu3_1"]), {}]
    with pytest.raises(SystemExit):
        prepare_styles.main(argv + ["--swap-targets", "relu2_1"], model_factory=lambda a: FakePrepModel(calls),
                            image_ops=HostImageOps)
