"""Seamless stylisation on the CPU: the wrap oracle (tests/seamless_ref.py), the mode and size checks of model.py and the
command-line flags (DESIGN.md §3.3.9)."""
import numpy as np
import pytest

from oracle import nets
from tests import seamless_ref as S
from wct_tf_b200.model import check_seamless, seamless_axes
from wct_tf_b200.weights import make_synthetic_weights

ALL = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]


@pytest.fixture(scope="module")
def weights():
    return make_synthetic_weights(42)


def _img(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def test_unwrapped_oracle_is_nets(weights):
    """wrap="" pads by reflection on both axes, one after the other: the same values as oracle/nets.py."""
    x = _img(40, 56, 3)[None] / 255.0
    for relu in ("relu1_1", "relu3_1"):
        a = S.encode(x, weights, [relu], np.float64)[relu]
        b = nets.encode(x, weights, [relu], np.float64)[relu]
        assert np.array_equal(a, b)
        assert np.array_equal(S.decode(a, weights, relu, np.float64), nets.decode(a, weights, relu, np.float64))


def test_wrap_pad_is_circular_on_wrapped_axes_only():
    import torch
    x = torch.arange(12, dtype=torch.float64).reshape(1, 1, 3, 4)
    p = S.pad(x, "x")[0, 0].numpy()
    assert np.array_equal(p[1:-1, 0], x[0, 0, :, -1].numpy()) and np.array_equal(p[1:-1, -1], x[0, 0, :, 0].numpy())
    assert np.array_equal(p[0], p[2]) and np.array_equal(p[-1], p[-3])                    # y reflects
    q = S.pad(x, "xy")[0, 0].numpy()
    assert np.array_equal(q, np.pad(x[0, 0].numpy(), 1, mode="wrap"))


@pytest.mark.parametrize("wrap,size,shifts", [
    ("x", (48, 64), [(0, 16), (0, 48)]),
    ("xy", (64, 64), [(16, 32), (48, 16)]),
])
def test_wrap_oracle_is_shift_equivariant(weights, wrap, size, shifts):
    """A circular shift of the content by multiples of 16 pixels along the wrapped axes shifts the five-level output by the
    same amount: every conv is circular there and every pool keeps its pairs.  Only the order of the statistics' sums
    differs, so float64 agrees to about 1e-8."""
    content, style = _img(*size, 1000), _img(48, 48, 7)
    base = S.pipeline(content, style, weights, ALL, alpha=0.8, dtype=np.float64, wrap=wrap)
    for dy, dx in shifts:
        got = S.pipeline(np.roll(content, (dy, dx), axis=(0, 1)), style, weights, ALL, alpha=0.8, dtype=np.float64, wrap=wrap)
        err = np.abs(got - np.roll(base, (dy, dx), axis=(1, 2))).max()
        print("%s shift (%d, %d): %.2e" % (wrap, dy, dx, err))
        assert err <= 1e-8


def test_reflect_oracle_is_not_shift_equivariant(weights):
    """The control: with reflect padding the same shift moves the seam into the image."""
    content, style = _img(48, 64, 1000), _img(48, 48, 7)
    base = S.pipeline(content, style, weights, ["relu2_1", "relu1_1"], alpha=0.8, dtype=np.float64)
    got = S.pipeline(np.roll(content, 32, axis=1), style, weights, ["relu2_1", "relu1_1"], alpha=0.8, dtype=np.float64)
    assert np.abs(got - np.roll(base, 32, axis=2)).max() > 1e-3


def test_seamless_axes_values():
    assert seamless_axes(None) == (False, False)
    assert seamless_axes("x") == (True, False)
    assert seamless_axes("y") == (False, True)
    assert seamless_axes("xy") == (True, True)
    for bad in ("yx", "X", "", "z", True, 1, ["x"]):
        with pytest.raises(ValueError, match="seamless must be"):
            seamless_axes(bad)


def test_check_seamless_divisibility():
    assert check_seamless("xy", 512, 1024, ALL) == (True, True)
    assert check_seamless("x", 100, 2048, ALL) == (True, False)          # the reflected axis may have any size
    assert check_seamless("y", 96, 33, ALL) == (False, True)
    assert check_seamless(None, 7, 9, ALL) == (False, False)
    with pytest.raises(ValueError, match="width 1000 is not a multiple of 16"):
        check_seamless("x", 512, 1000, ALL)
    with pytest.raises(ValueError, match="height 100 is not a multiple of 16"):
        check_seamless("xy", 100, 512, ALL)
    # the multiple follows the deepest target: relu3_1 pools twice
    assert check_seamless("xy", 20, 36, ["relu3_1", "relu1_1"]) == (True, True)
    with pytest.raises(ValueError, match="width 18 is not a multiple of 4"):
        check_seamless("xy", 20, 18, ["relu1_1", "relu3_1"])
    assert check_seamless("xy", 3, 5, ["relu1_1"]) == (True, True)


BASE = ["--relu-targets", "relu5_1", "relu1_1", "--style-path", "s.png", "--out-path", "out"]


@pytest.mark.parametrize("mode", ["x", "y", "xy"])
def test_cli_parses_seamless(mode):
    import stylize
    import stylize_video
    assert stylize.parse_args(BASE + ["--content-path", "c.png", "--seamless", mode]).seamless == mode
    assert stylize.parse_args(BASE + ["--noise", "--seamless", mode]).seamless == mode
    assert stylize.parse_args(BASE + ["--content-path", "c.png"]).seamless is None
    v = stylize_video.parse_args(["--relu-targets", "relu1_1", "--in-path", "v.mp4", "--out-path", "o", "--style-path", "s.png",
                                  "--seamless", mode])
    assert v.seamless == mode


@pytest.mark.parametrize("extra", [["--swap5"], ["--swap-targets", "relu1_1"], ["--seamless", "yx"]])
def test_cli_rejects_seamless_combinations(extra):
    import stylize
    args = BASE + ["--content-path", "c.png"] + (["--seamless", "x"] if extra[0] != "--seamless" else []) + extra
    with pytest.raises(SystemExit):
        stylize.parse_args(args)


def test_video_cli_rejects_seamless_with_temporal():
    import stylize_video
    base = ["--relu-targets", "relu1_1", "--in-path", "v.mp4", "--out-path", "o", "--style-path", "s.png", "--seamless", "x"]
    with pytest.raises(SystemExit):
        stylize_video.parse_args(base + ["--temporal", "0.5"])
    with pytest.raises(SystemExit):
        stylize_video.parse_args(base + ["--swap5"])
    assert stylize_video.parse_args(base + ["--temporal", "0"]).seamless == "x"


def test_header_and_bindings_declare_the_seamless_entries():
    import os
    from wct_tf_b200 import _capi
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "wctb200.h")).read()
    assert "#define WCTB200_HALO_WRAP_X 16" in header and "#define WCTB200_HALO_WRAP_Y 32" in header
    assert (_capi.HALO_WRAP_X, _capi.HALO_WRAP_Y) == (16, 32)
    for name in ("wctb200_act_halo", "wctb200_conv_head_flags"):
        assert name in _capi.SIGNATURES and name in header
