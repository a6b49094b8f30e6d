"""Texture synthesis on the GPU: the device noise (wctb200_noise_u8) against the NumPy Philox4x32-10 oracle
(tests/texture_ref.py) byte for byte, its argument checks, WCT.synthesize against predict_batch on the oracle noise for every
option it forwards, its independence of the batch split, the free-running five-level texture against the fp64 oracle, and the
command line."""
import numpy as np
import pytest
import torch
from PIL import Image

import tests.gpu_util as U
from oracle import nets, ref_ops
from tests.test_gpu_pipeline import ALL, FREE_RUN_NOISE_FACTOR
from tests.texture_ref import noise_u8 as oracle_noise
from wct_tf_b200 import _capi
from wct_tf_b200.device_image import noise_u8
from wct_tf_b200.weights import make_synthetic_weights
from wct_tf_b200.wct import WCT

pytestmark = pytest.mark.gpu
SENTINEL = 0xA5


@pytest.fixture(scope="module")
def weights():
    return make_synthetic_weights(42)


@pytest.fixture(scope="module")
def wct_tf(weights):
    return WCT(checkpoints=None, relu_targets=ALL, vgg_path=None, weights=weights, semantics="tf")


def _capi_noise(N, H, W, C, seed, first, offset=0):
    """wctb200_noise_u8 into a sentinel-filled buffer at byte ``offset``; checks that nothing outside the frames is written."""
    nbytes = N * H * W * C
    buf = torch.full((offset + nbytes + 32,), SENTINEL, dtype=torch.uint8, device="cuda")
    _capi.check(U.lib().wctb200_noise_u8(buf.data_ptr() + offset, N, H, W, C, seed, first, U.stream()))
    U.check_device()
    host = buf.cpu().numpy()
    assert (host[:offset] == SENTINEL).all() and (host[offset + nbytes:] == SENTINEL).all()
    return host[offset:offset + nbytes].reshape(N, H, W, C)


# H*W*C % 16 != 0 for 37x53x3, 9x7x1, 19x23x4 and 1x5x1; seeds and frame indices past 2^32 use the counter's high words
SHAPES = [(1, 1, 1, 3), (3, 37, 53, 3), (4, 9, 7, 1), (3, 19, 23, 4), (5, 1, 5, 1)]
KEYS = [(0, 0), (12345, 7), (2**32 + 11, 2**32 + 3), (2**64 - 1, 2**63 - 6)]
NOISE_CASES = [(s, k) for s in SHAPES for k in KEYS] + [((2, 512, 512, 3), KEYS[0]), ((2, 512, 512, 3), KEYS[3])]


@pytest.mark.parametrize("shape,key", NOISE_CASES, ids=["x".join(map(str, s)) + "-%d" % KEYS.index(k) for s, k in NOISE_CASES])
def test_device_noise_equals_oracle(shape, key):
    seed, first = key
    got = _capi_noise(*shape, seed, first)
    assert np.array_equal(got, oracle_noise(*shape, seed=seed, first_index=first))


@pytest.mark.parametrize("offset", [1, 2, 4, 8, 12])
@pytest.mark.parametrize("shape", [(3, 16, 16, 3), (3, 37, 53, 3)], ids=["aligned_frames", "ragged_frames"])
def test_device_noise_at_any_alignment(shape, offset):
    """16-byte, 4-byte and byte stores: the destination's alignment changes the store width, never the bytes."""
    got = _capi_noise(*shape, 99, 4, offset=offset)
    assert np.array_equal(got, oracle_noise(*shape, seed=99, first_index=4))


def test_python_noise_u8_equals_oracle():
    got = noise_u8(3, 37, 53, seed=2**40 + 1, first_index=2**33)
    assert got.is_cuda and got.dtype == torch.uint8 and tuple(got.shape) == (3, 37, 53, 3)
    assert np.array_equal(got.cpu().numpy(), oracle_noise(3, 37, 53, 3, seed=2**40 + 1, first_index=2**33))
    for bad in (dict(count=0, height=4, width=4), dict(count=1, height=0, width=4), dict(count=1, height=4, width=4, seed=-1),
                dict(count=1, height=4, width=4, seed=2**64), dict(count=1, height=4, width=4, first_index=-1)):
        with pytest.raises(ValueError):
            noise_u8(**bad)


def test_bad_arguments_return_einval_without_a_launch():
    lib = U.lib()
    buf = torch.full((4096,), SENTINEL, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()
    for args in [(None, 1, 4, 4, 3, 0, 0), (p, 0, 4, 4, 3, 0, 0), (p, 1, 0, 4, 3, 0, 0), (p, 1, 4, 0, 3, 0, 0),
                 (p, 1, 4, 4, 0, 0, 0), (p, 1, 4, 4, 5, 0, 0), (p, 1, 4, 4, 3, 0, -1), (p, 2, 4, 4, 3, 0, 2**63 - 2),
                 (p, 2**31 - 1, 2**31 - 1, 2**31 - 1, 4, 0, 0)]:
        assert lib.wctb200_noise_u8(*args, U.stream()) == _capi.EINVAL, args
    U.check_device()
    assert (buf.cpu().numpy() == SENTINEL).all()


# ---------------------------------------------------------------------------------------------------------- WCT.synthesize
def _styles(n, seed=11):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (s, s + 8, 3), dtype=np.uint8) for s in (72, 56, 64)[:n]]


def _halves(h, w):
    m = np.zeros((h, w), np.uint8)
    m[:, w // 2:] = 1
    return m


CASES = {
    "wct_tf": ("tf", 1, dict(alpha=0.8)),
    "wct_np": ("np", 1, dict(alpha=0.8)),
    "adain": ("tf", 1, dict(alpha=0.7, adain=True)),
    "passes2": ("tf", 1, dict(alpha=0.8, passes=2)),
    "swap5": ("tf", 1, dict(alpha=0.8, swap5=True, ss_alpha=0.6)),
    "blend_one_row": ("tf", 2, dict(alpha=0.8, style_weights=[0.3, 0.7])),
    "blend_rows": ("tf", 3, dict(alpha=0.8, style_weights=[[1, 0, 0], [0.2, 0.5, 0.3], [0, 0.25, 0.75]])),
    "adain_blend_rows": ("tf", 2, dict(alpha=0.8, adain=True, style_weights=[[1, 1], [0, 1], [3, 1]])),
    "mask": ("tf", 2, dict(alpha=0.8, content_mask=_halves(48, 40))),
}


@pytest.mark.parametrize("case", list(CASES))
def test_synthesize_equals_predict_batch_on_oracle_noise(weights, wct_tf, case):
    sem, nstyles, kw = CASES[case]
    wct = wct_tf if sem == "tf" else WCT(checkpoints=None, relu_targets=ALL, vgg_path=None, weights=weights, semantics=sem)
    assert wct.engine.groups == 2                              # three frames: the two stream groups take 1 and 2
    styles = _styles(nstyles)
    styles = styles[0] if nstyles == 1 else styles
    got = wct.synthesize(styles, (64, 96), count=3, seed=2**35 + 9, first_index=41, **kw)
    ref = wct.predict_batch(oracle_noise(3, 64, 96, 3, seed=2**35 + 9, first_index=41), styles, **kw)
    assert got.dtype == np.uint8 and got.shape == (3, 64, 96, 3)
    assert np.array_equal(got, ref)
    assert len({got[i].tobytes() for i in range(3)}) == 3     # different noise, different textures


def test_synthesize_square_size_and_device_result(wct_tf):
    style = _styles(1)[0]
    dev = wct_tf.synthesize(style, 64, count=2, seed=3, alpha=0.8, return_device=True)
    assert dev.is_cuda and tuple(dev.shape) == (2, 64, 64, 3)
    assert np.array_equal(dev.cpu().numpy(), wct_tf.predict_batch(oracle_noise(2, 64, 64, 3, seed=3), style, alpha=0.8))


@pytest.mark.parametrize("adain", [False, True])
def test_textures_do_not_depend_on_the_batch_split(wct_tf, adain):
    style = _styles(1)[0]
    kw = dict(alpha=0.8, adain=adain, seed=77)
    whole = wct_tf.synthesize(style, (80, 64), count=5, **kw)
    parts = np.concatenate([wct_tf.synthesize(style, (80, 64), count=2, **kw),
                            wct_tf.synthesize(style, (80, 64), count=3, first_index=2, **kw)])
    assert np.array_equal(whole, parts)
    one = wct_tf.synthesize(style, (80, 64), count=1, first_index=4, **kw)
    assert np.array_equal(one[0], whole[4])
    assert np.array_equal(wct_tf.synthesize(style, (80, 64), count=5, **kw), whole)      # a repeated call is byte-identical


def test_free_running_texture_vs_oracle(weights):
    size = 128
    noise = oracle_noise(1, size, size, 3, seed=1000)
    style = np.random.default_rng(7).integers(0, 256, (size, size, 3), dtype=np.uint8)
    o64, info = nets.pipeline(noise[0], style, weights, ALL, alpha=0.8, semantics="np", dtype=np.float64, return_info=True)
    o32 = nets.pipeline(noise[0], style, weights, ALL, alpha=0.8, semantics="np", dtype=np.float32)
    for inf in info:
        assert ref_ops.spectral_gap_ok(inf["wc"]) and ref_ops.spectral_gap_ok(inf["ws"])
    wct = WCT(checkpoints=None, relu_targets=ALL, vgg_path=None, weights=weights, semantics="np")
    _, got = wct.synthesize(style, size, count=1, seed=1000, alpha=0.8, return_float=True)
    noise_floor = np.abs(o32 - o64).max()
    err = np.abs(got - o64).max()
    print("free-running 5-level texture: engine-vs-fp64 oracle %.3e ; oracle fp32-vs-fp64 %.3e" % (err, noise_floor))
    assert err <= max(1e-3, FREE_RUN_NOISE_FACTOR * noise_floor)


def test_cli_end_to_end(tmp_path):
    import stylize
    from wct_tf_b200 import imageio as io
    targets = ["relu3_1", "relu2_1", "relu1_1"]
    style = np.random.default_rng(5).integers(0, 256, (48, 64, 3), dtype=np.uint8)
    Image.fromarray(style).save(str(tmp_path / "st.png"))
    argv = ["--synthetic-weights", "42", "--relu-targets"] + targets + ["--noise", "--noise-count", "3", "--noise-size", "40",
                                                                       "56", "--noise-seed", "4", "--style-path",
                                                                       str(tmp_path / "st.png"), "--alpha", "0.7"]
    assert stylize.main(argv + ["--out-path", str(tmp_path / "o")]) == 3
    wct = WCT(checkpoints=None, relu_targets=targets, vgg_path=None, weights=make_synthetic_weights(42, relu_targets=targets))
    ref = wct.predict_batch(oracle_noise(3, 40, 56, 3, seed=4), io.get_img(str(tmp_path / "st.png")), alpha=0.7)
    assert sorted(p.name for p in (tmp_path / "o").iterdir()) == ["noise4-%d_st.png" % i for i in range(3)]
    for i in range(3):
        got = np.asarray(Image.open(str(tmp_path / "o" / ("noise4-%d_st.png" % i))))
        assert got.shape == (40, 56, 3) and np.array_equal(got, ref[i])
    stylize.main(argv + ["--out-path", str(tmp_path / "o2")])                            # the same bytes on a rerun
    for i in range(3):
        name = "noise4-%d_st.png" % i
        assert np.array_equal(np.asarray(Image.open(str(tmp_path / "o" / name))), np.asarray(Image.open(str(tmp_path / "o2" / name))))
