"""Tiled stylisation on the host (no GPU): the halos walked from the plans, the tile grid, the record oracle against the
float64 statistics of a union of rectangles, the argument checks, and the stylize.py flag."""
import numpy as np
import pytest
from PIL import Image

import stylize
from tests import tiles_ref as R
from tests.test_interp_cli import HostImageOps
from wct_tf_b200.engine import Engine
from wct_tf_b200.model import RELU_LEVEL, tile_grid, tile_halos

# DESIGN.md §3.3.7, derived by hand from encoder_plan / decoder_plan
HALOS = {"relu5_1": (80, 160), "relu4_1": (32, 64), "relu3_1": (12, 24), "relu2_1": (4, 8), "relu1_1": (1, 3)}


@pytest.mark.parametrize("relu", sorted(HALOS))
def test_tile_halos_table(relu):
    h_a, h_b = tile_halos(relu)
    assert (h_a, h_b) == HALOS[relu]
    g = 2 ** (RELU_LEVEL[relu] - 1)
    assert h_a % g == 0 and h_b % g == 0


@pytest.mark.parametrize("hw,T", [((1000, 1496), 512), ((64, 64), 64), ((17, 300), 16), ((2048, 2048), 1024),
                                  ((33, 49), 1024), ((1040, 1040), 512)])
def test_tile_grid_partitions(hw, T):
    H, W = hw
    tiles = tile_grid(H, W, T)
    cover = np.zeros((H, W), np.int32)
    for y0, y1, x0, x1 in tiles:
        assert y0 % 16 == 0 and x0 % 16 == 0 and y0 < y1 <= H and x0 < x1 <= W
        assert (y1 == H or y1 % 16 == 0) and (x1 == W or x1 % 16 == 0)
        assert y1 - y0 <= T and x1 - x0 <= T
        cover[y0:y1, x0:x1] += 1
    assert (cover == 1).all()
    assert max(t[1] for t in tiles) == H and max(t[3] for t in tiles) == W
    assert tiles == sorted(tiles)                       # row-major: the fold order is fixed


@pytest.mark.parametrize("hw,T", [((1000, 1496), 512), ((1040, 1008), 512), ((100, 100), 48)])
@pytest.mark.parametrize("relu", sorted(HALOS))
def test_interior_feature_rectangles_partition(hw, T, relu):
    """The interior feature rectangles [y0/g, ceil(y1/g)) x ... partition the ceil(H/g) x ceil(W/g) feature map, and lie
    inside the feature map of their crop (widened by h_A, clipped to the image)."""
    H, W = hw
    g = 2 ** (RELU_LEVEL[relu] - 1)
    h_a, _ = tile_halos(relu)
    cover = np.zeros((-(-H // g), -(-W // g)), np.int32)
    for y0, y1, x0, x1 in tile_grid(H, W, T):
        cover[y0 // g:-(-y1 // g), x0 // g:-(-x1 // g)] += 1
        cy0, cy1 = max(0, y0 - h_a), min(H, y1 + h_a)
        assert cy0 % g == 0 and -(-y1 // g) - cy0 // g <= -(-(cy1 - cy0) // g)
    assert (cover == 1).all()


def _union_case(seed, C, diag):
    """An image with a strong gradient cut into rectangles of very different means, each recorded on its own shift."""
    rng = np.random.default_rng(seed)
    H, W = 60, 90
    yy, xx = np.mgrid[0:H, 0:W]
    img = rng.standard_normal((H, W, C)) * 0.3 + (yy[..., None] * 4.0 + xx[..., None] * 2.5) * rng.uniform(0.5, 2, C)
    ys, xs = [0, 7, 31, 60], [0, 16, 17, 70, 90]
    rec = R.empty(C, diag)
    for i in range(3):
        for j in range(4):
            px = img[ys[i]:ys[i + 1], xs[j]:xs[j + 1]].reshape(-1, C)
            t = px[::max(1, len(px) // 7)].mean(axis=0)          # a sampled shift, as k_sample_shift takes
            rec = R.accumulate(rec, R.record(px, t, diag))
    return img.reshape(-1, C), rec


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_record_oracle_covariance_of_union(seed):
    x, rec = _union_case(seed, 8, False)
    mean, cov = R.covariance(rec)
    assert rec["n"] == len(x)
    np.testing.assert_allclose(mean, x.mean(axis=0), rtol=1e-12, atol=1e-9)
    np.testing.assert_allclose(cov, np.cov(x, rowvar=False), rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("seed", [0, 1])
def test_record_oracle_moments_of_union(seed):
    x, rec = _union_case(seed, 8, True)
    mean, var = R.moments(rec)
    np.testing.assert_allclose(mean, x.mean(axis=0), rtol=1e-12, atol=1e-9)
    np.testing.assert_allclose(var, x.var(axis=0), rtol=1e-9, atol=1e-9)


def test_record_oracle_identity_and_order():
    rng = np.random.default_rng(5)
    x = rng.standard_normal((50, 4)) + 100
    r = R.record(x, x[0])
    one = R.accumulate(R.empty(4), r)
    for k in ("n", "t", "s", "S"):
        assert np.array_equal(one[k], r[k])
    a, b = R.record(x[:20], x[3]), R.record(x[20:], x[40] - 7)
    ab, ba = R.accumulate(R.accumulate(R.empty(4), a), b), R.accumulate(R.accumulate(R.empty(4), b), a)
    np.testing.assert_allclose(R.covariance(ab)[1], R.covariance(ba)[1], rtol=1e-10)


@pytest.mark.parametrize("bad", [0, -16, 8, 24, 1000, 16.0, "64", True])
def test_check_tile_size_rejects(bad):
    with pytest.raises(ValueError):
        Engine.check_tile_size(bad)


@pytest.mark.parametrize("good", [16, 512, 1024, np.int64(2048)])
def test_check_tile_size_accepts(good):
    assert Engine.check_tile_size(good) == int(good)


# ------------------------------------------------------------------------------------------------------------ stylize.py
TARGETS = ["--relu-targets", "relu5_1", "relu4_1", "relu3_1"]


def _base(tmp_path):
    return TARGETS + ["--synthetic-weights", "1", "--content-path", str(tmp_path / "c.png"), "--out-path", str(tmp_path / "out")]


def test_tile_size_parse(tmp_path):
    assert stylize.parse_args(_base(tmp_path) + ["--style-path", "s.png"]).tile_size == 0
    assert stylize.parse_args(_base(tmp_path) + ["--style-path", "s.png", "--tile-size", "1024"]).tile_size == 1024
    a = stylize.parse_args(_base(tmp_path) + ["--style-path", "s.png", "--tile-size", "512", "--keep-colors", "--concat",
                                              "--content-size", "900", "--passes", "2", "--adain"])
    assert a.tile_size == 512 and a.keep_colors and a.concat and a.passes == 2


@pytest.mark.parametrize("extra", [["--style-path", "s.png", "--tile-size", "100"],
                                   ["--style-path", "s.png", "--tile-size", "-16"],
                                   ["--style-path", "s.png", "--tile-size", "64", "--swap5"],
                                   ["--style-path", "s.png", "--tile-size", "64", "--swap-targets", "relu3_1"],
                                   ["--content-mask", "m.png", "--mask-styles", "x.png", "--tile-size", "64"],
                                   ["--interp-styles", "a.png", "b.png", "--interp-weights", "1", "1", "--tile-size", "64"]],
                         ids=["not_multiple", "negative", "swap5", "swap_targets", "content_mask", "interp"])
def test_tile_size_parser_errors(tmp_path, extra, capsys):
    with pytest.raises(SystemExit):
        stylize.parse_args(_base(tmp_path) + extra)
    assert "--tile-size" in capsys.readouterr().err


class FakeWCT(object):
    class engine(object):
        device = None

    def __init__(self, calls):
        self.calls = calls

    def predict_batch(self, contents, styles, **kw):
        self.calls.append(kw)
        c = np.asarray(contents)
        return (c[None] if c.ndim == 3 else c) + 1


def test_stylize_passes_tile_size(tmp_path):
    Image.fromarray(np.full((8, 12, 3), 10, np.uint8)).save(str(tmp_path / "c.png"))
    Image.fromarray(np.full((6, 6, 3), 50, np.uint8)).save(str(tmp_path / "s.png"))
    calls = []
    argv = _base(tmp_path) + ["--style-path", str(tmp_path / "s.png"), "--tile-size", "256", "--passes", "2"]
    assert stylize.main(argv, model_factory=lambda a: FakeWCT(calls), image_ops=HostImageOps) == 1
    assert len(calls) == 2 and all(kw["tile_size"] == 256 for kw in calls)
    calls.clear()
    stylize.main(_base(tmp_path) + ["--style-path", str(tmp_path / "s.png")], model_factory=lambda a: FakeWCT(calls),
                 image_ops=HostImageOps)
    assert "tile_size" not in calls[0]
