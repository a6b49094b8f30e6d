"""Texture-synthesis noise on the CPU: the NumPy Philox4x32-10 oracle (tests/texture_ref.py) against the Random123 known
answers, its (seed, frame index) addressing and its byte statistics, and the C-ABI's argument checks (which return before
any CUDA call, so they run without a GPU)."""
import ctypes

import numpy as np
import pytest

from tests.texture_ref import noise_u8, philox4x32_10

KNOWN_ANSWERS = [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
]


@pytest.mark.parametrize("ctr,key,want", KNOWN_ANSWERS)
def test_philox_known_answers(ctr, key, want):
    assert tuple(int(v) for v in philox4x32_10(np.array([ctr]), key)[0]) == want


def test_byte_layout_is_little_endian_words_of_the_block():
    x = philox4x32_10(np.array([[0, 0, 7, 0]]), (5, 0))[0]
    frame = noise_u8(1, 1, 6, 3, seed=5, first_index=7)[0].reshape(-1)       # 18 bytes: one full block + 2 bytes
    assert frame.shape == (18,)
    assert [int(v) for v in frame[:16]] == [(int(x[j // 4]) >> (8 * (j % 4))) & 255 for j in range(16)]
    y = philox4x32_10(np.array([[1, 0, 7, 0]]), (5, 0))[0]
    assert [int(v) for v in frame[16:]] == [int(y[0]) & 255, (int(y[0]) >> 8) & 255]


@pytest.mark.parametrize("seed,first", [(0, 0), (3, 11), (2**40 + 5, 2**33 + 1)])
def test_frame_n_equals_a_one_frame_call_at_first_index_plus_n(seed, first):
    batch = noise_u8(4, 5, 7, 3, seed=seed, first_index=first)
    for n in range(4):
        assert np.array_equal(batch[n], noise_u8(1, 5, 7, 3, seed=seed, first_index=first + n)[0])


def test_counter_halves_are_all_used():
    """64-bit seeds and frame indices: the high words change the bytes."""
    base = noise_u8(1, 4, 4, 3, seed=1, first_index=1)
    assert not np.array_equal(base, noise_u8(1, 4, 4, 3, seed=1 + 2**32, first_index=1))
    assert not np.array_equal(base, noise_u8(1, 4, 4, 3, seed=1, first_index=1 + 2**32))


def test_different_seeds_or_indices_give_different_frames():
    frames = [noise_u8(1, 16, 16, 3, seed=s, first_index=i)[0] for s in (0, 1, 2) for i in (0, 1, 2)]
    for a in range(len(frames)):
        for b in range(a + 1, len(frames)):
            assert np.mean(frames[a] == frames[b]) < 0.02, (a, b)       # ~1/256 of the bytes agree by chance


def test_byte_histogram_is_uniform():
    """2^24 seeded bytes, 256 bins: chi-square with 255 degrees of freedom (mean 255, sd 22.6).  Deterministic, so it cannot
    flake: the bounds sit about 6 sd from the mean, and also reject a suspiciously flat histogram."""
    x = noise_u8(16, 512, 512, 4, seed=12345, first_index=0).reshape(-1)
    assert x.size == 2**24
    counts = np.bincount(x, minlength=256).astype(np.float64)
    expected = x.size / 256.0
    chi2 = float(((counts - expected) ** 2 / expected).sum())
    print("chi-square over 2^24 bytes: %.1f (255 degrees of freedom)" % chi2)
    assert 120.0 < chi2 < 390.0
    # each of the 16 byte positions of a block on its own, 2^20 bytes each
    for j in range(16):
        cj = np.bincount(x[j::16], minlength=256).astype(np.float64)
        e = x.size / 16 / 256.0
        assert 120.0 < float(((cj - e) ** 2 / e).sum()) < 390.0, j


def test_capi_noise_rejects_bad_arguments_before_any_cuda_call():
    """Every rejection returns WCTB200_EINVAL before the buffer is touched: the fake pointer below is never dereferenced, and
    without a GPU a launch would fail with WCTB200_ECUDA instead."""
    from wct_tf_b200 import _capi
    lib = _capi.load()
    fake = ctypes.c_void_p(0x1000)
    i64max = 2**63 - 1
    for args in [(None, 1, 4, 4, 3, 0, 0), (fake, 0, 4, 4, 3, 0, 0), (fake, 1, 0, 4, 3, 0, 0), (fake, 1, 4, 0, 3, 0, 0),
                 (fake, 1, 4, 4, 0, 0, 0), (fake, 1, 4, 4, 5, 0, 0), (fake, -1, 4, 4, 3, 0, 0), (fake, 1, 4, 4, 3, 0, -1),
                 (fake, 2, 4, 4, 3, 0, i64max - 1), (fake, 1, 4, 4, 3, 0, i64max),
                 (fake, 2**31 - 1, 2**31 - 1, 2**31 - 1, 4, 0, 0)]:
        assert lib.wctb200_noise_u8(*args, None) == _capi.EINVAL, args
        assert lib.wctb200_last_error().startswith(b"noise_u8:")
