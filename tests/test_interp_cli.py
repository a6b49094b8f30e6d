"""CLI style interpolation (stylize.py / stylize_video.py --interp-styles, --interp-weights, --morph): flag errors and defaults,
output naming and the predict_batch calls both drivers make; no GPU needed (fake WCT and host image ops)."""
import numpy as np
import pytest
from PIL import Image

import stylize
import stylize_video as V


def _base(tmp_path):
    return ["--relu-targets", "relu1_1", "--synthetic-weights", "1", "--content-path", str(tmp_path / "c.png"),
            "--out-path", str(tmp_path / "out")]


@pytest.mark.parametrize("extra", [["--style-path", "s.png"], ["-r", "2"], ["--swap5"], ["--concat"],
                                   ["--content-mask", "m.png", "--mask-styles", "x.png"],
                                   ["--interp-weights", "1", "2", "3"],                      # lengths differ
                                   ["--interp-weights", "1", "-1"], ["--interp-weights", "0", "0"],
                                   ["--interp-weights", "nan", "1"]])
def test_interp_flag_errors(tmp_path, extra):
    argv = _base(tmp_path) + ["--interp-styles", "a.png", "b.png"] + extra
    if "--interp-weights" not in extra:
        argv += ["--interp-weights", "1", "1"]
    with pytest.raises(SystemExit):
        stylize.parse_args(argv)


def test_interp_flags_need_each_other_and_at_most_8(tmp_path):
    for extra in (["--interp-styles", "a.png"], ["--interp-weights", "1"],
                  ["--interp-styles"] + ["s%d.png" % i for i in range(9)] + ["--interp-weights"] + ["1"] * 9):
        with pytest.raises(SystemExit):
            stylize.parse_args(_base(tmp_path) + extra)


def test_interp_flags_default_off_and_allowed_combinations(tmp_path):
    a = stylize.parse_args(["--relu-targets", "relu1_1"])
    assert a.interp_styles is None and a.interp_weights is None
    b = stylize.parse_args(_base(tmp_path) + ["--interp-styles", "a.png", "b.png", "--interp-weights", "1", "3", "--adain",
                                              "--alpha", "0.5", "--passes", "2", "--keep-colors", "--style-size", "64",
                                              "--crop-size", "32"])
    assert b.interp_styles == ["a.png", "b.png"] and b.interp_weights == [1.0, 3.0] and b.adain and b.keep_colors


def test_interp_output_names():
    assert stylize.interp_output_name("/x/c.jpg", ["/s/a.png", "b.jpg"], [1, 3]) == "c_a-0.25+b-0.75.jpg"
    assert stylize.interp_output_name("c.png", ["a.png", "b.png", "d.png"], [1, 1, 1]) == "c_a-0.333333+b-0.333333+d-0.333333.png"
    assert stylize.interp_output_name("c.png", ["a.png"], [2.5]) == "c_a-1.png"
    assert stylize.interp_output_name("c.png", ["a.png", "b.png"], [0, 5]) == "c_a-0+b-1.png"


class HostImageOps(object):
    to_device = staticmethod(lambda img, device=None: np.asarray(img))
    to_host = staticmethod(lambda img: np.asarray(img))
    resize_to = staticmethod(lambda img, size: img)
    center_crop = staticmethod(lambda img, size: img)
    preserve_colors_np = staticmethod(lambda style, content: np.asarray(style) + 1)


def test_interp_run_calls_predict_batch_and_names_output(tmp_path):
    Image.fromarray(np.full((8, 12, 3), 10, np.uint8)).save(str(tmp_path / "c.png"))
    for name, v in (("sky", 50), ("sea", 90)):
        Image.fromarray(np.full((6, 6, 3), v, np.uint8)).save(str(tmp_path / (name + ".png")))
    calls = []

    class FakeWCT(object):
        class engine(object):
            device = None

        def predict_batch(self, contents, styles, alpha=1, adain=False, style_weights=None, return_device=False, **kw):
            calls.append(([int(np.asarray(s)[0, 0, 0]) for s in styles], np.asarray(style_weights).copy(), alpha, adain, kw))
            c = np.asarray(contents)
            return (c[None] if c.ndim == 3 else c) + 1

    argv = _base(tmp_path) + ["--interp-styles", str(tmp_path / "sky.png"), str(tmp_path / "sea.png"), "--interp-weights", "3",
                              "1", "--alpha", "0.7", "--passes", "2", "--adain", "--keep-colors"]
    n = stylize.main(argv, model_factory=lambda a: FakeWCT(), image_ops=HostImageOps)
    assert n == 1
    out = tmp_path / "out" / "c_sky-0.75+sea-0.25.png"
    assert out.exists()
    assert np.array_equal(np.asarray(Image.open(str(out))), np.full((8, 12, 3), 12, np.uint8))   # two passes
    assert len(calls) == 2
    for styles, w, alpha, adain, kw in calls:
        assert styles == [51, 91] and alpha == 0.7 and adain and not kw                          # CORAL on each style
        assert np.array_equal(w, [3.0, 1.0])                                                     # normalised by predict_batch


def _video_frames(tmp_path, sizes):
    frames = tmp_path / "clip"
    frames.mkdir()
    for i, hw in enumerate(sizes):
        Image.fromarray(np.full(hw + (3,), i + 1, dtype=np.uint8)).save(str(frames / ("frame_%d.png" % (i + 1))))
    for name, v in (("a", 50), ("b", 90), ("d", 130)):
        Image.fromarray(np.full((6, 6, 3), v, np.uint8)).save(str(tmp_path / (name + ".png")))
    return frames


def _video_argv(tmp_path, frames, extra):
    return (["--relu-targets", "relu1_1", "--in-path", str(frames), "--out-path", str(tmp_path / "out"), "--interp-styles"]
            + [str(tmp_path / (n + ".png")) for n in ("a", "b", "d")] + extra)


@pytest.mark.parametrize("extra", [[], ["--morph", "--interp-weights", "1", "1", "1"], ["--style-path", "s.png", "--morph"],
                                   ["--morph", "--swap5"], ["--morph", "--concat"], ["--interp-weights", "1", "1"]])
def test_video_interp_flag_errors(tmp_path, extra):
    with pytest.raises(SystemExit):
        V.parse_args(_video_argv(tmp_path, tmp_path, extra))


def test_video_flags_default_off_and_style_required(tmp_path):
    a = V.parse_args(["--relu-targets", "relu1_1", "--in-path", "x", "--out-path", "y", "--style-path", "s.png"])
    assert a.interp_styles is None and a.interp_weights is None and not a.morph
    with pytest.raises(SystemExit):
        V.parse_args(["--relu-targets", "relu1_1", "--in-path", "x", "--out-path", "y"])
    with pytest.raises(SystemExit):                                         # --morph needs K >= 2
        V.parse_args(["--relu-targets", "relu1_1", "--in-path", "x", "--out-path", "y", "--interp-styles", "a.png", "--morph"])


class FakeVideoWCT(object):
    def __init__(self, calls):
        self.calls = calls

    def predict_batch(self, contents, styles, alpha=1, adain=False, passes=None, swap5=False, style_weights=None, **kw):
        c = np.asarray(contents)
        c = c[None] if c.ndim == 3 else c
        self.calls.append(([int(x[0, 0, 0]) for x in c], [int(np.asarray(s)[0, 0, 0]) for s in styles],
                           np.asarray(style_weights).copy(), passes))
        return c + 1


def test_video_morph_rows_follow_the_clip_index(tmp_path):
    frames = _video_frames(tmp_path, [(8, 12)] * 4 + [(16, 12)])                # frame 5 is ragged: per-frame fallback
    calls = []
    n = V.main(_video_argv(tmp_path, frames, ["--morph", "--batch", "2"]), wct_factory=lambda a: FakeVideoWCT(calls),
               image_ops=HostImageOps)
    assert n == 5
    w = V.morph_weights(5, 3)
    assert [c[0] for c in calls] == [[1, 2], [3, 4], [5]]
    for c, rows in zip(calls, (w[0:2], w[2:4], w[4:5])):
        assert c[1] == [50, 90, 130] and np.array_equal(c[2], rows)
    assert calls[0][3] == 1 and calls[2][3] is None                            # batched passes / one call per frame
    assert (tmp_path / "out" / "clip_morph_a+b+d_frames" / "frame_5.png").exists()


def test_video_fixed_blend_and_keep_colors(tmp_path):
    frames = _video_frames(tmp_path, [(8, 12)] * 3)
    calls = []
    n = V.main(_video_argv(tmp_path, frames, ["--interp-weights", "2", "1", "1", "--batch", "2", "--keep-colors"]),
               wct_factory=lambda a: FakeVideoWCT(calls), image_ops=HostImageOps)
    assert n == 3
    assert [c[0] for c in calls] == [[1], [2], [3]]                             # --keep-colors: one call per frame
    for c in calls:
        assert c[1] == [51, 91, 131] and np.array_equal(c[2], [2.0, 1.0, 1.0])
    assert (tmp_path / "out" / "clip_a-0.5+b-0.25+d-0.25_frames" / "frame_3.png").exists()
