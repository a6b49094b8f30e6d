"""stylize_video.py --temporal: flag errors, the default (off: predict_batch called exactly as without the flag) and one
temporal state per (clip, style) run, carried across batches and through the frame-by-frame path.  No GPU needed (a fake
WCT and host image ops)."""
import numpy as np
import pytest
from PIL import Image

import stylize_video as V
from tests.test_interp_cli import HostImageOps


def _clip(tmp_path, sizes):
    frames = tmp_path / "clip"
    frames.mkdir()
    for i, hw in enumerate(sizes):
        Image.fromarray(np.full(hw + (3,), i + 1, dtype=np.uint8)).save(str(frames / ("frame_%d.png" % (i + 1))))
    styles = tmp_path / "styles"
    styles.mkdir()
    for name, v in (("a", 50), ("b", 90)):
        Image.fromarray(np.full((6, 6, 3), v, np.uint8)).save(str(styles / (name + ".png")))
    return frames, styles


def _argv(tmp_path, frames, style, extra):
    return ["--relu-targets", "relu1_1", "--in-path", str(frames), "--out-path", str(tmp_path / "out"), "--style-path",
            str(style)] + extra


@pytest.mark.parametrize("value", ["-0.1", "1", "1.5", "nan"])
def test_temporal_flag_errors(tmp_path, value):
    with pytest.raises(SystemExit):
        V.parse_args(_argv(tmp_path, "x", "s.png", ["--temporal", value]))


def test_temporal_flag_default_off():
    a = V.parse_args(["--relu-targets", "relu1_1", "--in-path", "x", "--out-path", "y", "--style-path", "s.png"])
    assert a.temporal == 0.0
    b = V.parse_args(["--relu-targets", "relu1_1", "--in-path", "x", "--out-path", "y", "--style-path", "s.png",
                      "--temporal", "0.8"])
    assert b.temporal == 0.8


class FakeState(object):
    def __init__(self, strength):
        self.strength = strength


class FakeTemporalWCT(object):
    def __init__(self, calls, states):
        self.calls, self.states = calls, states

    def temporal_state(self, strength):
        s = FakeState(strength)
        self.states.append(s)
        return s

    def predict_batch(self, contents, styles, **kw):
        c = np.asarray(contents)
        c = c[None] if c.ndim == 3 else c
        self.calls.append(([int(x[0, 0, 0]) for x in c], int(np.asarray(styles).reshape(-1)[0]), dict(kw)))
        return c + 1


def test_default_calls_predict_batch_without_temporal(tmp_path):
    frames, styles = _clip(tmp_path, [(8, 12)] * 3 + [(16, 12)])
    calls, states = [], []
    n = V.main(_argv(tmp_path, frames, styles / "a.png", ["--batch", "2", "--passes", "2"]),
               wct_factory=lambda a: FakeTemporalWCT(calls, states), image_ops=HostImageOps)
    assert n == 4 and not states
    assert all("temporal" not in kw for _, _, kw in calls)
    # batched frames 1-2 (one call, two passes), then frame 3 alone and ragged frame 4: one call per pass each
    assert [c[0] for c in calls] == [[1, 2], [3], [4], [4], [5]]


def test_one_state_per_clip_and_style_across_batches_and_frame_path(tmp_path):
    frames, styles = _clip(tmp_path, [(8, 12)] * 3 + [(16, 12)] + [(8, 12)])
    calls, states = [], []
    n = V.main(_argv(tmp_path, frames, styles, ["--batch", "2", "--temporal", "0.8", "--passes", "2"]),
               wct_factory=lambda a: FakeTemporalWCT(calls, states), image_ops=HostImageOps)
    assert n == 10                                               # 5 frames x 2 styles
    assert len(states) == 2 and all(s.strength == 0.8 for s in states)
    per_style = {}
    for frames_in, style, kw in calls:
        assert kw["passes"] == 2                                 # every pass in one call, stabilised after the last
        per_style.setdefault(style, []).append((frames_in, kw["temporal"]))
    assert sorted(per_style) == [50, 90]
    for (style, seq), state in zip(sorted(per_style.items()), states):
        assert [f for f, _ in seq] == [[1, 2], [3], [4], [5]]    # batch of 2, then the ragged batch frame by frame
        assert all(t is state for _, t in seq)
    assert (tmp_path / "out" / "clip_a_frames" / "frame_5.png").exists()
