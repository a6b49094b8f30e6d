"""The float32 oracle of the temporal stabilisation (tests/temporal_ref.py, DESIGN.md §3.3.6) on seeded synthetic clips:
flow accuracy, zero motion, occlusion, cuts and the blend's fixed points.  No GPU needed."""
import numpy as np
import pytest

from tests import temporal_ref as R

H, W = 96, 128


@pytest.mark.parametrize("d", [(1.0, 0.0), (-2.0, 1.0), (0.75, 0.5), (0.3, -1.6)])
def test_flow_recovers_translations(d):
    Y = R.luminance(R.translating_clip(2, H, W, d=d, seed=3))
    fl = R.flow_pairs(Y)
    m = 8                                                        # away from the border
    for k, sign in ((0, -1.0), (1, 1.0)):                        # backward t+1 -> t is -d, forward t -> t+1 is +d
        epe = np.hypot(fl[k, 0, m:-m, m:-m] - sign * d[0], fl[k, 1, m:-m, m:-m] - sign * d[1])
        assert np.median(epe) < 0.1, (d, k, np.median(epe))


def test_flow_recovers_a_translation_over_several_levels():
    Y = R.luminance(R.translating_clip(2, 160, 200, d=(2.5, -1.5), seed=5))
    assert len(R.level_sizes(160, 200)) == 3
    fl = R.flow(Y[1], Y[0])
    epe = np.hypot(fl[0, 8:-8, 8:-8] + 2.5, fl[1, 8:-8, 8:-8] - 1.5)
    assert np.median(epe) < 0.1


def test_zero_motion_is_zero_flow_and_full_confidence():
    Y = R.luminance(R.translating_clip(3, H, W, d=(0.0, 0.0), seed=1))
    fl = R.flow_pairs(Y)
    assert fl.dtype == np.float32 and not fl.any()
    masks, counts = R.confidence(Y, fl)
    assert masks.all() and counts == [H * W, H * W]


def test_uncovered_band_is_not_confident():
    # a textured 24 px square moves by (3, 2) px per frame over a background moving by (0.75, 0.5)
    clip = R.translating_clip(2, H, W, d=(0.75, 0.5), seed=3, square=(24, 30, 30, 3, 2))
    Y = R.luminance(clip)
    masks, counts = R.confidence(Y, R.flow_pairs(Y))
    band = np.zeros((H, W), bool)
    band[30:54, 30:54] = True                                    # under the square in frame 0 ...
    band[32:56, 33:57] = False                                   # ... and not in frame 1
    assert band.sum() == 24 * 24 - 22 * 21
    assert masks[0][band].mean() < 0.25
    assert counts[0] > 0.9 * H * W                               # the rest of the frame is confident


def test_cut_frame_gets_no_confidence():
    clip = R.translating_clip(4, H, W, d=(0.75, 0.5), seed=3, cut=3)
    Y = R.luminance(clip)
    masks, counts = R.confidence(Y, R.flow_pairs(Y))
    assert masks[0].mean() > 0.9 and masks[1].mean() > 0.9
    assert counts[2] > 0 and not masks[2].any()                  # some pixels pass by chance; the cut rule zeroes them


def test_blend_fixed_points():
    rng = np.random.default_rng(0)
    clip = R.translating_clip(3, H, W, d=(0.75, 0.5), seed=2)
    sty = rng.integers(0, 256, (3, H, W, 3), dtype=np.uint8)
    out, _ = R.stabilize(clip, sty, 0.0)
    assert np.array_equal(out, sty)                              # beta = 0
    same = np.repeat(clip[:1], 3, axis=0)
    sty_same = np.repeat(sty[:1], 3, axis=0)
    out, _ = R.stabilize(same, sty_same, 0.8)
    assert np.array_equal(out, sty_same)                         # identical frames: zero flow, O_{t-1} = P_t
    out, _ = R.stabilize(clip, sty, 0.8)
    assert np.array_equal(out[0], sty[0]) and not np.array_equal(out[1:], sty[1:])


def test_stabilize_is_independent_of_the_split():
    rng = np.random.default_rng(1)
    clip = R.translating_clip(5, 48, 64, d=(0.5, 0.25), seed=4)
    sty = rng.integers(0, 256, (5, 48, 64, 3), dtype=np.uint8)
    whole, _ = R.stabilize(clip, sty, 0.6)
    a, st = R.stabilize(clip[:2], sty[:2], 0.6)
    b, _ = R.stabilize(clip[2:], sty[2:], 0.6, prev=st)
    assert np.array_equal(whole, np.concatenate([a, b]))
