"""Temporal stabilisation on the GPU: luminance, flows, confidence and the blend against the float32 oracle
(tests/temporal_ref.py) bit for bit, at odd sizes, a 16-rounded relu5_1 output size, 512^2 and 1920x1080; batched flow
problems against the same pairs one at a time; predict_batch(temporal=) independent of the batch split and of the engine's
stream groups, its fixed points, every option it combines with, its rejections, and the warping error it lowers."""
import json
import os

import numpy as np
import pytest
import torch

import tests.gpu_util as U
from tests import temporal_ref as R
from tests.test_gpu_pipeline import ALL
from wct_tf_b200 import temporal as T
from wct_tf_b200.device_image import imresize
from wct_tf_b200.weights import make_synthetic_weights
from wct_tf_b200.wct import WCT

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def wct():
    return WCT(checkpoints=None, relu_targets=ALL, vgg_path=None, weights=make_synthetic_weights(42))


def _device_all(clip, sty, beta, prev=None):
    """luminance, flows, masks, counts and the blended frames from the device for one stack."""
    Y = T.luminance(U.dev(clip))
    Ys = Y if prev is None else torch.cat([U.dev(prev[0])[None], Y])
    flows = T.flow_pairs(Ys)
    masks, counts = T.confidence(Ys, flows)
    out = U.dev(sty)
    T.blend_(out, None if prev is None else U.dev(prev[1]), flows, masks, beta)
    torch.cuda.synchronize()
    return Y.cpu().numpy(), flows.cpu().numpy(), masks.cpu().numpy(), counts.cpu().numpy(), out.cpu().numpy()


@pytest.mark.parametrize("M,H,W", [(3, 37, 53), (2, 5, 9), (3, 112, 144), (2, 512, 512), (2, 1080, 1920)])
def test_device_matches_oracle_bit_for_bit(M, H, W):
    rng = np.random.default_rng(H * W)
    square = (min(H, W) // 4, W // 3, H // 3, 2, 1) if min(H, W) >= 32 else None
    clip = R.translating_clip(M, H, W, d=(1.25, -0.5), seed=M + H, square=square)
    sty = rng.integers(0, 256, (M, H, W, 3), dtype=np.uint8)
    Y, flows, masks, counts, out = _device_all(clip, sty, 0.8)
    Yr = R.luminance(clip)
    assert np.array_equal(Y.view(np.uint32), Yr.view(np.uint32))
    fr = R.flow_pairs(Yr)
    assert np.array_equal(flows.view(np.uint32), fr.view(np.uint32))
    mr, cr = R.confidence(Yr, fr)
    assert np.array_equal(masks, mr) and list(counts) == cr
    assert np.array_equal(out, R.blend(sty, None, fr, mr, 0.8))


def test_blend_with_a_predecessor_matches_oracle():
    rng = np.random.default_rng(7)
    clip = R.translating_clip(3, 64, 80, d=(0.5, 0.75), seed=9)
    sty = rng.integers(0, 256, (3, 64, 80, 3), dtype=np.uint8)
    prev = (R.luminance(clip[0]), sty[0])
    *_, out = _device_all(clip[1:], sty[1:], 0.6, prev=prev)
    ref, _ = R.stabilize(clip[1:], sty[1:], 0.6, prev=prev)
    assert np.array_equal(out, ref)


def test_batched_flow_problems_equal_single_pairs():
    Y = T.luminance(U.dev(R.translating_clip(5, 72, 96, d=(0.8, 0.3), seed=11, cut=3)))
    batched = T.flow_pairs(Y)
    for t in range(4):
        one = T.flow_pairs(Y[t:t + 2].contiguous())
        assert torch.equal(batched[2 * t:2 * t + 2], one)


def test_argument_checks():
    Y = T.luminance(U.dev(R.translating_clip(2, 32, 32, seed=1)))
    with pytest.raises(Exception):
        T.flow_pairs(Y[:1].contiguous())                        # one frame has no pair
    flows = T.flow_pairs(Y)
    masks, _ = T.confidence(Y, flows)
    frames = torch.zeros((2, 32, 32, 3), dtype=torch.uint8, device="cuda")
    with pytest.raises(Exception):
        T.blend_(frames, None, flows, masks, 1.0)


def _content(n, H=60, W=90, seed=0, cut=None):
    return R.translating_clip(n, H, W, d=(0.75, 0.5), seed=seed, cut=cut)


def _style():
    return R.texture(64, 64, 77)


def test_split_and_groups_do_not_change_a_frame(wct):
    clip, style = _content(12), _style()
    runs = []
    for groups in (1, 2):
        wct.engine.groups = groups
        for split in (1, 5, 12):
            st = wct.temporal_state(0.8)
            outs = [wct.predict_batch(clip[i:i + split], style, alpha=0.8, temporal=st) for i in range(0, 12, split)]
            runs.append(np.concatenate(outs))
    wct.engine.groups = 2
    for r in runs[1:]:
        assert np.array_equal(r, runs[0])
    plain = wct.predict_batch(clip, style, alpha=0.8)
    assert plain.shape == (12, 64, 96, 3)                       # relu5_1 rounds 60 x 90 up to multiples of 16
    assert np.array_equal(runs[0][0], plain[0]) and not np.array_equal(runs[0], plain)


def test_strength_zero_identical_frames_and_cut(wct):
    clip, style = _content(6, cut=4), _style()
    plain = wct.predict_batch(clip, style, alpha=0.8)
    assert np.array_equal(wct.predict_batch(clip, style, alpha=0.8, temporal=wct.temporal_state(0.0)), plain)
    same = np.repeat(clip[:1], 4, axis=0)
    assert np.array_equal(wct.predict_batch(same, style, alpha=0.8, temporal=wct.temporal_state(0.9)),
                          wct.predict_batch(same, style, alpha=0.8))
    out = wct.predict_batch(clip, style, alpha=0.8, temporal=wct.temporal_state(0.8))
    assert np.array_equal(out[4], plain[4]) and not np.array_equal(out[5], plain[5])


def test_size_change_restarts_the_clip(wct):
    style = _style()
    st = wct.temporal_state(0.8)
    wct.predict_batch(_content(2), style, temporal=st)
    other = _content(2, H=48, W=48, seed=3)
    assert np.array_equal(wct.predict_batch(other[:1], style, temporal=st), wct.predict_batch(other[:1], style))


def _combos(style):
    other = R.texture(48, 40, 78)
    mask = np.zeros((60, 90), np.uint8)
    mask[:, 45:] = 1
    smask = np.zeros((48, 40), np.uint8)
    smask[24:] = 1
    return {
        "passes": dict(styles=style, passes=2),
        "swap5": dict(styles=style, swap5=True, ss_alpha=0.7),
        "swap_targets": dict(styles=style, swap_targets=["relu4_1"]),
        "style_weights": dict(styles=[style, other], style_weights=[1, 3]),
        "content_mask": dict(styles=[style, other], content_mask=mask),
        "style_masks": dict(styles=[style, other], content_mask=mask, style_masks=[None, smask]),
        "adain": dict(styles=style, adain=True),
    }


@pytest.mark.parametrize("name", ["passes", "swap5", "swap_targets", "style_weights", "content_mask", "style_masks", "adain",
                                  "prepared", "out", "return_device"])
def test_combinations_equal_the_oracle_on_the_plain_output(wct, name):
    clip, style = _content(3), _style()
    kw = _combos(style).get(name, dict(styles=style))
    if name == "prepared":
        kw = dict(styles=wct.prepare_style(style))
    styles = kw.pop("styles")
    plain = wct.predict_batch(clip, styles, alpha=0.8, **kw)
    extra = {}
    if name == "out":
        extra["out"] = torch.empty(plain.shape, dtype=torch.uint8).pin_memory()
    if name == "return_device":
        extra["return_device"] = True
    got = wct.predict_batch(clip, styles, alpha=0.8, temporal=wct.temporal_state(0.7), **dict(kw, **extra))
    got = got.cpu().numpy() if isinstance(got, torch.Tensor) else got
    with torch.cuda.device(wct.engine.device):
        c = imresize(U.dev(clip), plain.shape[1:3]).cpu().numpy()
    ref, _ = R.stabilize(c, plain, 0.7)
    assert np.array_equal(got, ref)


def test_rejections(wct):
    clip, style = _content(2), _style()
    with pytest.raises(ValueError, match="return_float"):
        wct.predict_batch(clip, style, return_float=True, temporal=wct.temporal_state(0.5))
    for bad in (-0.1, 1.0, 2.0, float("nan")):
        with pytest.raises(ValueError):
            wct.temporal_state(bad)


def test_stabilisation_lowers_the_warping_error(wct):
    # integer motion (2, 1) px per frame, so O_{t-1}(x - d) is an exact pixel
    n, H, W, d = 10, 128, 160, (2, 1)
    clip, style = R.translating_clip(n, H, W, d=d, seed=21), _style()
    plain = wct.predict_batch(clip, style, alpha=0.8)
    stab = wct.predict_batch(clip, style, alpha=0.8, temporal=wct.temporal_state(0.8))
    Y = T.luminance(U.dev(clip))
    masks, _ = T.confidence(Y, T.flow_pairs(Y))
    masks = masks.cpu().numpy().astype(bool)
    m = 8

    def warp_error(o):
        errs = []
        for t in range(1, n):
            cur = o[t, m:H - m, m:W - m].astype(np.float64)
            prev = o[t - 1, m - d[1]:H - m - d[1], m - d[0]:W - m - d[0]].astype(np.float64)
            conf = masks[t - 1, m:H - m, m:W - m]
            errs.append(np.abs(cur - prev).mean(axis=-1)[conf])
        return float(np.concatenate(errs).mean())
    e_plain, e_stab = warp_error(plain), warp_error(stab)
    os.makedirs(U.OUT_DIR, exist_ok=True)
    with open(os.path.join(U.OUT_DIR, "temporal_warp_error.json"), "w") as f:
        json.dump(dict(clip=[n, H, W], motion=d, strength=0.8, plain=e_plain, stabilised=e_stab,
                       gpu=torch.cuda.get_device_name()), f)
    assert e_stab < e_plain, (e_stab, e_plain)
