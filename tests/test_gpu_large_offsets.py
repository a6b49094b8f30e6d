"""Kernels at activation offsets past 2^31 and 2^32 elements (DESIGN.md §4, "Offsets past 2^31").

An SPF16 buffer is a hi plane and a lo plane of N (H+2)(W+2) C elements each, so at relu1_1 (C = 64) a batch of 2048^2
frames puts the lo plane past 2^31 from the second frame on, and a 4096^2 frame puts its last rows there.  The kernels mix
64-bit offsets with 32-bit shortcuts that rest on guards; a shortcut taken past its guard reads or writes the wrong
element.  A wrong lo-plane address moves a value by about 2^-11 of itself, inside every 1e-3 parity bound, so the checks
here are on raw bits:

  - batch invariance: frame i of an N-frame batch has the bytes of that frame run alone (test_gpu_invariance.py pins it
    small), and the one-frame runs stay far below 2^31;
  - locality: a band of a local op, or of a transform applied pixel by pixel, has the bytes of the same op on a crop.

Each case also compares a window of its last frame (or band) with float64 at the tolerance of the kernel's own parity test.

Geometries (C = 64, a 2048^2 frame's plane is 268.96e6 elements):
  A = 9 x 2048^2   (9.7 GB a buffer): the lo plane is past 2^31 throughout and past 2^32 from frame 7; hi past 2^31 in frames 7, 8.
  B = 17 x 2048^2  (18.3 GB): the lo plane is past 2^32 throughout; hi past 2^32 in frames 15, 16.
  F = 1 x 4096^2   : the lo plane passes 2^31 at padded row 4090.
Same-size ops run at A, ops with one large side at B; every test stays below about 25 GB of device memory.
"""
import ctypes
import gc
import math
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import gpu_util as U
from tests import ost_ref
from tests.test_gpu_layers import conv_ref64
from wct_tf_b200 import _capi
from wct_tf_b200.engine import Engine
from wct_tf_b200.weights import make_synthetic_weights

pytestmark = pytest.mark.gpu
C = 64
A = (9, 2048, 2048)
B = (17, 2048, 2048)
FH = 4096
SEMS = dict(tf=(1e-8, 0.0, 1e-5, 1), np=(0.0, 1e-5, 1e-5, 0))     # eps_cov, eps_eig, thresh, readd
K = 12                                                             # side of the float64 anchor window


@pytest.fixture(autouse=True)
def _release():
    """Every test frees its buffers and reports its peak."""
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    yield
    torch.cuda.synchronize()
    print("peak device memory %.1f GB" % (torch.cuda.max_memory_allocated() / 1e9))
    # pytest keeps a failed test's traceback for post-mortem debugging, and with it that test's 20 GB of buffers
    sys.last_type = sys.last_value = sys.last_traceback = sys.last_exc = None
    gc.collect()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------- buffers
def pl(buf, n, h, w, c):
    """Raw bits of an SPF16 buffer, on the device: int16 [2 planes][n][h+2][w+2][c]."""
    return buf.view(torch.int16).view(2, n, h + 2, w + 2, c)


def feats_dev(h, w, c, seed, scale, offset=0.3):
    """fp32 [1,h,w,c] relu-like features with channel correlations, made on the device."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    mix = torch.randn(c, c, generator=g, device="cuda") / math.sqrt(c)
    x = torch.randn(h * w, c, generator=g, device="cuda") @ mix
    return torch.relu(x * scale + offset).view(1, h, w, c)


def act_of(x):
    """SPF16 of the fp32 NHWC device tensor x."""
    n, h, w, c = x.shape
    buf = U.act_alloc(n, h, w, c, poison=False)
    _capi.check(U.lib().wctb200_act_from_f32(x.data_ptr(), n, h, w, c, buf.data_ptr(), U.stream()))
    return buf


def batch_act(n, h, w, c, seed):
    """An n-frame SPF16 batch, frame i converted alone with its own seed and scale and copied into its slots."""
    buf = U.act_alloc(n, h, w, c, poison=False)
    dst = pl(buf, n, h, w, c)
    for i in range(n):
        one = act_of(feats_dev(h, w, c, seed + i, 1.0 + 0.25 * i))
        dst[:, i:i + 1].copy_(pl(one, 1, h, w, c))
        del one
    return buf


def frame_copy(buf, i, n, h, w, c):
    """A one-frame SPF16 buffer holding the bytes of frame i of `buf` (both planes, halo included)."""
    out = U.act_alloc(1, h, w, c, poison=False)
    pl(out, 1, h, w, c).copy_(pl(buf, n, h, w, c)[:, i:i + 1])
    return out


def crop_rows(buf, n, h, w, c, i, p0, p1):
    """A one-frame SPF16 map of padded rows [p0, p1) of frame i: interior rows p0 .. p1 - 3 of the map, each cell with the
    bytes it has in `buf` (its top and bottom halo rows are the frame's own neighbouring rows)."""
    out = U.act_alloc(1, p1 - p0 - 2, w, c, poison=False)
    pl(out, 1, p1 - p0 - 2, w, c).copy_(pl(buf, n, h, w, c)[:, i:i + 1, p0:p1])
    return out


def window(buf, n, h, w, c, i, py0, py1, px0, px1):
    """float64 values (hi + lo) of padded rows [py0, py1) x columns [px0, px1) of frame i, on the host."""
    p = buf.view(torch.float16).view(2, n, h + 2, w + 2, c)[:, i, py0:py1, px0:px1].double()
    return (p[0] + p[1]).cpu().numpy()


def assert_same(got, want, what):
    """Bitwise equality of two device tensors; the message gives the first differing index."""
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if torch.equal(got, want):
        return
    d = (got != want).reshape(-1)
    first = int(d.to(torch.uint8).argmax())
    idx = np.unravel_index(first, tuple(got.shape))
    raise AssertionError("%s: %d of %d elements differ in their bits, first at %s" % (what, int(d.sum()), d.numel(), idx))


def assert_rel(got, ref, tol, what):
    """|got - ref| <= tol (1 + |ref|), the bound of test_gpu_layers.assert_close."""
    err = np.abs(got - ref) / (1.0 + np.abs(ref))
    assert np.isfinite(got).all() and err.max() <= tol, (what, float(np.nanmax(err)))


def f32_bits(t):
    return t.view(torch.int32)


def conv_weights(cin, cout, seed, up2=False):
    """Host fp32 weights k [3][3][cin][cout], b [cout] and the prepared device operand."""
    rng = np.random.default_rng(seed)
    k = (rng.normal(0, 1, (3, 3, cin, cout)) * np.sqrt(2.0 / (9 * cin))).astype(np.float32)
    b = rng.normal(0, 0.3, cout).astype(np.float32)
    d_k, d_b = U.dev(k), U.dev(b)
    lib = U.lib()
    taps = 16 if up2 else 9
    wsp = torch.empty(lib.wctb200_conv_weight_bytes(taps, cin, cout), dtype=torch.uint8, device="cuda")
    if up2:
        _capi.check(lib.wctb200_prep_conv_weights_up2(d_k.data_ptr(), cin, cout, wsp.data_ptr(), U.stream()))
    else:
        _capi.check(lib.wctb200_prep_conv_weights(d_k.data_ptr(), 9, cin, cout, wsp.data_ptr(), U.stream()))
    torch.cuda.synchronize()
    return k, b, wsp, d_b


def check_frames(out, n, h, w, c, one_of, what, frames=None):
    """Frame i of the batch output `out` equals the one-frame output one_of(i), both planes with the halo."""
    bp = pl(out, n, h, w, c)
    for i in (range(n) if frames is None else frames):
        one = one_of(i)
        assert_same(pl(one, 1, h, w, c)[:, 0], bp[:, i], "%s frame %d" % (what, i))
        del one


# ---------------------------------------------------------------------------------------------------------- conversions
def test_act_from_and_to_f32_at_A():
    n, h, w = A
    lib = U.lib()
    x = torch.empty((n, h, w, C), dtype=torch.float32, device="cuda")
    for i in range(n):
        x[i:i + 1] = feats_dev(h, w, C, 100 + i, 1.0 + 0.25 * i)
    act = U.act_alloc(n, h, w, C)
    _capi.check(lib.wctb200_act_from_f32(x.data_ptr(), n, h, w, C, act.data_ptr(), U.stream()))
    check_frames(act, n, h, w, C, lambda i: act_of(x[i:i + 1]), "act_from_f32")
    # float64: the last frame's bottom-right corner, halo included, is the split of its fp32 values mirrored by REFLECT
    xs = U.split_repr(x[n - 1, h - K:, w - K:].cpu().numpy())
    ref = np.pad(xs, ((0, 1), (0, 1), (0, 0)), mode="reflect")             # + the bottom halo row and right halo column
    assert np.array_equal(window(act, n, h, w, C, n - 1, h - K + 1, h + 2, w - K + 1, w + 2), ref)
    last = x[n - 1, h - K:, w - K:].clone()
    _capi.check(lib.wctb200_act_to_f32(act.data_ptr(), n, h, w, C, x.data_ptr(), U.stream()))    # back into x
    for i in range(n):
        one = torch.empty((1, h, w, C), dtype=torch.float32, device="cuda")
        _capi.check(lib.wctb200_act_to_f32(frame_copy(act, i, n, h, w, C).data_ptr(), 1, h, w, C, one.data_ptr(), U.stream()))
        assert_same(f32_bits(one[0]), f32_bits(x[i]), "act_to_f32 frame %d" % i)
    back = x[n - 1, h - K:, w - K:].cpu().numpy()
    assert np.abs(back - last.cpu().numpy()).max() <= 1e-6 * (1 + float(last.abs().max()))     # test_act_roundtrip bound
    U.check_device()


# ---------------------------------------------------------------------------------------------------------------- convs
@pytest.mark.parametrize("fuse", [-1, 0, 1], ids=["fuse_auto", "fuse_off", "fuse_on"])
@pytest.mark.parametrize("flags", [_capi.RELU, _capi.RELU | _capi.HALO_EDGE, 0], ids=["relu", "halo_edge", "linear"])
def test_conv3x3_at_A(flags, fuse):
    """64 -> 64 at A: the input's lo plane is read through the TMA map past 2^32, the output stored past it.  At Cout = 64 the
    default N tile is 64 (the only one that divides it)."""
    n, h, w = A
    lib = U.lib()
    xin = batch_act(n, h, w, C, 200)
    k, b, wsp, d_b = conv_weights(C, C, 201)
    out = U.act_alloc(n, h, w, C)

    def conv(src, nn, dst):
        _capi.check(lib.wctb200_conv3x3(src.data_ptr(), nn, h, w, C, wsp.data_ptr(), d_b.data_ptr(), C, flags, dst.data_ptr(),
                                        U.stream()))
        return dst

    lib.wctb200_debug_set_conv_fuse(fuse)
    try:
        conv(xin, n, out)
        check_frames(out, n, h, w, C, lambda i: conv(frame_copy(xin, i, n, h, w, C), 1, U.act_alloc(1, h, w, C)), "conv3x3")
    finally:
        lib.wctb200_debug_set_conv_fuse(-1)
    # float64: the bottom-right K x K input corner gives the last K - 1 rows / columns (its first row sees no true neighbour)
    crop = window(xin, n, h, w, C, n - 1, h - K + 1, h + 1, w - K + 1, w + 1)
    ref = conv_ref64(crop[None], k, b, bool(flags & _capi.RELU))[0, 1:, 1:]
    got = window(out, n, h, w, C, n - 1, h - K + 2, h + 1, w - K + 2, w + 1)
    assert_rel(got, ref, 1e-5, "conv3x3 vs float64")                      # test_conv3x3_tensor_core
    U.check_device()


def test_conv3x3_pool2_with_input_B():
    n, h, w = B
    ho, wo = h // 2, w // 2
    lib = U.lib()
    xin = batch_act(n, h, w, C, 300)
    k, b, wsp, d_b = conv_weights(C, C, 301)
    fl = _capi.RELU | _capi.POOL2

    def conv(src, nn):
        dst = U.act_alloc(nn, ho, wo, C)
        _capi.check(lib.wctb200_conv3x3(src.data_ptr(), nn, h, w, C, wsp.data_ptr(), d_b.data_ptr(), C, fl, dst.data_ptr(), U.stream()))
        return dst

    out = conv(xin, n)
    check_frames(out, n, ho, wo, C, lambda i: conv(frame_copy(xin, i, n, h, w, C), 1), "conv3x3 POOL2")
    crop = window(xin, n, h, w, C, n - 1, h - K + 1, h + 1, w - K + 1, w + 1)
    y = torch.from_numpy(conv_ref64(crop[None], k, b, True)).permute(0, 3, 1, 2)
    ref = F.max_pool2d(y, 2, 2).permute(0, 2, 3, 1).numpy()[0, 1:, 1:]         # the first pooled row / column saw the crop edge
    got = window(out, n, ho, wo, C, n - 1, ho - K // 2 + 2, ho + 1, wo - K // 2 + 2, wo + 1)
    assert_rel(got, ref, 1e-5, "conv3x3 POOL2 vs float64")                # test_conv3x3_pool2_equals_conv_then_maxpool
    U.check_device()


def test_maxpool2_with_input_B():
    n, h, w = B
    ho, wo = h // 2, w // 2
    lib = U.lib()
    xin = batch_act(n, h, w, C, 310)

    def pool(src, nn):
        dst = U.act_alloc(nn, ho, wo, C)
        _capi.check(lib.wctb200_maxpool2(src.data_ptr(), nn, h, w, C, dst.data_ptr(), U.stream()))
        return dst

    out = pool(xin, n)
    check_frames(out, n, ho, wo, C, lambda i: pool(frame_copy(xin, i, n, h, w, C), 1), "maxpool2")
    crop = window(xin, n, h, w, C, n - 1, h - K + 1, h + 1, w - K + 1, w + 1)
    ref = crop.reshape(K // 2, 2, K // 2, 2, C).max(axis=(1, 3))
    assert np.array_equal(window(out, n, ho, wo, C, n - 1, ho - K // 2 + 1, ho + 1, wo - K // 2 + 1, wo + 1), ref)
    U.check_device()


def _edge_halo(buf, n, h, w, c):
    """Rewrite the halo of an SPF16 map as EDGE-replicated (the input format of conv3x3_up2)."""
    p = pl(buf, n, h, w, c)
    p[:, :, 0].copy_(p[:, :, 1])
    p[:, :, h + 1].copy_(p[:, :, h])
    p[:, :, :, 0].copy_(p[:, :, :, 1])
    p[:, :, :, w + 1].copy_(p[:, :, :, w])


def test_conv3x3_up2_with_output_B():
    n, h2, w2 = B
    h, w = h2 // 2, w2 // 2
    lib = U.lib()
    xin = batch_act(n, h, w, C, 400)
    _edge_halo(xin, n, h, w, C)
    k, b, wup, d_b = conv_weights(C, C, 401, up2=True)

    def conv(src, nn):
        dst = U.act_alloc(nn, h2, w2, C)
        _capi.check(lib.wctb200_conv3x3_up2(src.data_ptr(), nn, h, w, C, wup.data_ptr(), d_b.data_ptr(), C, _capi.RELU,
                                            dst.data_ptr(), U.stream()))
        return dst

    out = conv(xin, n)
    check_frames(out, n, h2, w2, C, lambda i: conv(frame_copy(xin, i, n, h, w, C), 1), "conv3x3_up2")
    # float64: upsample the bottom-right corner of the input, conv with REFLECT padding (which at the bottom / right edge
    # equals the edge halo of the low-resolution map); the first output row / column saw the crop edge
    k2 = K // 2
    crop = window(xin, n, h, w, C, n - 1, h - k2 + 1, h + 1, w - k2 + 1, w + 1).repeat(2, axis=0).repeat(2, axis=1)
    ref = conv_ref64(crop[None], k, b, True)[0, 1:, 1:]
    got = window(out, n, h2, w2, C, n - 1, h2 - K + 2, h2 + 1, w2 - K + 2, w2 + 1)
    assert_rel(got, ref, 1e-5, "conv3x3_up2 vs float64")                   # test_conv3x3_up2_equals_upsample_then_conv
    U.check_device()


def test_upsample2_with_output_B():
    n, h2, w2 = B
    h, w = h2 // 2, w2 // 2
    lib = U.lib()
    xin = batch_act(n, h, w, C, 410)

    def up(src, nn):
        dst = U.act_alloc(nn, h2, w2, C)
        _capi.check(lib.wctb200_upsample2(src.data_ptr(), nn, h, w, C, dst.data_ptr(), U.stream()))
        return dst

    out = up(xin, n)
    check_frames(out, n, h2, w2, C, lambda i: up(frame_copy(xin, i, n, h, w, C), 1), "upsample2")
    k2 = K // 2
    crop = window(xin, n, h, w, C, n - 1, h - k2 + 1, h + 1, w - k2 + 1, w + 1).repeat(2, axis=0).repeat(2, axis=1)
    ref = np.pad(crop, ((0, 1), (0, 1), (0, 0)), mode="reflect")
    assert np.array_equal(window(out, n, h2, w2, C, n - 1, h2 - K + 1, h2 + 2, w2 - K + 1, w2 + 2), ref)
    U.check_device()


def _head_weights():
    rng = np.random.default_rng(5)
    wf = (rng.standard_normal((27, 64)) * 0.3).astype(np.float32)
    bf = (rng.standard_normal(64) * 0.1).astype(np.float32)
    return wf, bf, U.dev(wf), U.dev(bf)


def _head_ref(img_crop, wf, bf):
    """conv_head in float64 on an image crop: the folded 3x3x3 -> 64 conv with REFLECT padding, + bias, ReLU."""
    return conv_ref64(img_crop[None].astype(np.float64), wf.reshape(3, 3, 3, 64), bf, True)[0]


def _images(n, h, w, seed):
    img = torch.empty((n, h, w, 3), dtype=torch.float32, device="cuda")
    for i in range(n):
        g = torch.Generator(device="cuda").manual_seed(seed + i)
        img[i] = torch.rand((h, w, 3), generator=g, device="cuda")
    return img


@pytest.mark.parametrize("impl", ["tensor-core", "simt"])
def test_conv_head_with_output_B(impl):
    n, h, w = B
    lib = U.lib()
    img = _images(n, h, w, 500)
    wf, bf, d_wf, d_bf = _head_weights()

    def head(src, nn):
        dst = U.act_alloc(nn, h, w, C)
        _capi.check(lib.wctb200_conv_head(src.data_ptr(), nn, h, w, d_wf.data_ptr(), d_bf.data_ptr(), dst.data_ptr(), U.stream()))
        return dst

    if impl == "simt":
        lib.wctb200_debug_set_conv_head_tc(0)
    try:
        out = head(img, n)
        check_frames(out, n, h, w, C, lambda i: head(img[i:i + 1].contiguous(), 1), "conv_head " + impl)
    finally:
        lib.wctb200_debug_set_conv_head_tc(1)
    ref = _head_ref(img[n - 1, h - K:, w - K:].cpu().numpy(), wf, bf)[1:, 1:]
    assert_rel(window(out, n, h, w, C, n - 1, h - K + 2, h + 1, w - K + 2, w + 1), ref, 2e-5, "conv_head vs float64")
    U.check_device()


def _tail_weights():
    rng = np.random.default_rng(6)
    k = (rng.normal(0, 1, (3, 3, C, 3)) * 0.05).astype(np.float32)
    b = np.array([0.5, 0.4, 0.6], dtype=np.float32)
    return k, b, U.dev(k.reshape(9 * C, 3)), U.dev(b)


def _tail(src, nn, h, w, d_k, d_b):
    dst = torch.full((nn, h, w, 3), float("nan"), dtype=torch.float32, device="cuda")
    _capi.check(U.lib().wctb200_conv_tail(src.data_ptr(), nn, h, w, C, d_k.data_ptr(), d_b.data_ptr(), 0, dst.data_ptr(), U.stream()))
    return dst


@pytest.mark.parametrize("impl", ["tensor-core", "simt"])
def test_conv_tail_with_input_B(impl):
    n, h, w = B
    lib = U.lib()
    xin = batch_act(n, h, w, C, 600)
    k, b, d_k, d_b = _tail_weights()
    if impl == "simt":
        lib.wctb200_debug_set_conv_tail_tc(0)
    try:
        out = _tail(xin, n, h, w, d_k, d_b)
        for i in range(n):
            one = _tail(frame_copy(xin, i, n, h, w, C), 1, h, w, d_k, d_b)
            assert_same(f32_bits(one[0]), f32_bits(out[i]), "conv_tail %s frame %d" % (impl, i))
    finally:
        lib.wctb200_debug_set_conv_tail_tc(1)
    crop = window(xin, n, h, w, C, n - 1, h - K + 1, h + 1, w - K + 1, w + 1)
    ref = conv_ref64(crop[None], k, b, False)[0, 1:, 1:]
    assert_rel(out[n - 1, h - K + 1:, w - K + 1:].cpu().numpy(), ref, 2e-5, "conv_tail vs float64")     # test_conv_tail
    U.check_device()


# ------------------------------------------------------------------------------------------------- statistics, transforms
def stats64(buf, n, h, w, c, i, mask=None, rows=256):
    """float64 pixel count, mean [c], unbiased covariance [c][c] and max |x| of frame i (the pixels where mask [h][w] is
    true), summed on the device in bands of `rows` rows."""
    p = buf.view(torch.float16).view(2, n, h + 2, w + 2, c)
    cnt, s, xmax = 0, torch.zeros(c, dtype=torch.float64, device="cuda"), 0.0
    for pass_ in (0, 1):
        S = torch.zeros((c, c), dtype=torch.float64, device="cuda")
        for y in range(0, h, rows):
            x = (p[0, i, 1 + y:1 + min(y + rows, h), 1:w + 1].double() + p[1, i, 1 + y:1 + min(y + rows, h), 1:w + 1].double())
            x = x.reshape(-1, c)
            if mask is not None:
                x = x[mask[y:y + rows].reshape(-1)]
            if pass_ == 0:
                cnt += x.shape[0]
                s += x.sum(0)
                xmax = max(xmax, float(x.abs().max()))
            else:
                d = x - mean
                S += d.T @ d
        if pass_ == 0:
            mean = s / cnt
    return cnt, mean.cpu().numpy(), (S / (cnt - 1)).cpu().numpy(), xmax


def affine_ref(xw, mc, cov_c, ms, cov_s, sem, alpha, ost=False):
    """WCT (T = C_s W_c) or OST (M) of the window pixels xw [.., C] in float64, from float64 statistics."""
    eps_cov, eps_eig, thresh, readd = SEMS[sem]
    eye = np.eye(len(mc))
    M, info = ost_ref.ost_map(cov_c + eps_cov * eye, cov_s + eps_cov * eye, eps_eig, thresh, return_info=True)
    T = M if ost else info["T"]
    d = xw - mc
    base = xw if readd else d
    return alpha * (d @ T.T + ms) + (1 - alpha) * base


def test_covariance_at_B():
    n, h, w = B
    lib = U.lib()
    xin = batch_act(n, h, w, C, 700)

    def cov(src, nn):
        m = torch.full((nn, C), float("nan"), dtype=torch.float32, device="cuda")
        cv = torch.full((nn, C, C), float("nan"), dtype=torch.float32, device="cuda")
        _capi.check(lib.wctb200_covariance(src.data_ptr(), nn, h, w, C, 1e-8, m.data_ptr(), cv.data_ptr(), U.stream()))
        return m, cv

    bm, bc = cov(xin, n)
    for i in range(n):
        m1, c1 = cov(frame_copy(xin, i, n, h, w, C), 1)
        assert_same(f32_bits(m1[0]), f32_bits(bm[i]), "covariance mean frame %d" % i)
        assert_same(f32_bits(c1[0]), f32_bits(bc[i]), "covariance frame %d" % i)
    _, mean, ref, xmax = stats64(xin, n, h, w, C, n - 1)
    # the fp32-summation bound of test_rect_statistics_vs_fp64, per pixel: 1e-6 max|x| on the mean, 1e-6 max|x|^2 on the covariance
    assert np.abs(bm[n - 1].cpu().numpy() - mean).max() <= 1e-6 * xmax
    assert np.abs(bc[n - 1].cpu().numpy() - (ref + 1e-8 * np.eye(C))).max() <= 1e-6 * xmax ** 2
    U.check_device()


def _ws(nbytes):
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device="cuda")


def _style(seed, hs=512, ws_=512):
    return act_of(feats_dev(hs, ws_, C, seed, 0.8, offset=0.2)), hs, ws_


def test_adain_level_at_A():
    n, h, w = A
    lib = U.lib()
    xin = batch_act(n, h, w, C, 800)
    sty, hs, ws_ = _style(801)
    alpha = 0.8

    def run(src, nn):
        dst = U.act_alloc(nn, h, w, C)
        ws = _ws(lib.wctb200_wct_workspace_bytes(C, nn, 1))
        _capi.check(lib.wctb200_adain_level(src.data_ptr(), nn, h, w, sty.data_ptr(), 1, hs, ws_, C, alpha, 1e-5, dst.data_ptr(),
                                            ws.data_ptr(), ws.numel(), U.stream()))
        return dst

    out = run(xin, n)
    check_frames(out, n, h, w, C, lambda i: run(frame_copy(xin, i, n, h, w, C), 1), "adain_level")
    cnt, mc, cc, _ = stats64(xin, n, h, w, C, n - 1)
    cnt_s, ms, cs, _ = stats64(sty, 1, hs, ws_, C, 0)
    vc, vs = np.diag(cc) * (cnt - 1) / cnt, np.diag(cs) * (cnt_s - 1) / cnt_s        # biased moments
    xw = window(xin, n, h, w, C, n - 1, h - K + 1, h + 1, w - K + 1, w + 1)
    ref = alpha * ((xw - mc) / np.sqrt(vc + 1e-5) * np.sqrt(vs) + ms) + (1 - alpha) * xw
    got = window(out, n, h, w, C, n - 1, h - K + 1, h + 1, w - K + 1, w + 1)
    tol = 1e-5 * np.abs(ref).max(axis=(0, 1)) + 1e-4 * alpha * np.sqrt(vs)                # test_adain_vs_fp64 bound
    assert (np.abs(got - ref) <= tol).all(), float((np.abs(got - ref) / tol).max())
    U.check_device()


@pytest.mark.parametrize("sem", ["tf", "np"])
def test_wct_level_at_A(sem):
    n, h, w = A
    lib = U.lib()
    eps_cov, eps_eig, thresh, readd = SEMS[sem]
    xin = batch_act(n, h, w, C, 900)
    sty, hs, ws_ = _style(901)
    alpha = 0.7

    def run(src, nn):
        dst = U.act_alloc(nn, h, w, C)
        ws = _ws(lib.wctb200_wct_workspace_bytes(C, nn, 1))
        k = torch.full((2 * (nn + 1),), -7, dtype=torch.int32, device="cuda")
        _capi.check(lib.wctb200_wct_level(src.data_ptr(), nn, h, w, sty.data_ptr(), 1, hs, ws_, C, alpha, eps_cov, eps_eig, thresh,
                                          readd, dst.data_ptr(), k.data_ptr(), ws.data_ptr(), ws.numel(), U.stream()))
        return dst, k.cpu().tolist()

    out, kb = run(xin, n)
    bp = pl(out, n, h, w, C)
    for i in range(n):
        one, k1 = run(frame_copy(xin, i, n, h, w, C), 1)
        assert_same(pl(one, 1, h, w, C)[:, 0], bp[:, i], "wct_level %s frame %d" % (sem, i))
        assert k1 == [kb[i], kb[n], kb[n + 1 + i], kb[2 * n + 1]], (i, k1, kb)     # k_c, k_s, sweeps_c, sweeps_s
        del one
    _, mc, cc, _ = stats64(xin, n, h, w, C, n - 1)
    _, ms, cs, _ = stats64(sty, 1, hs, ws_, C, 0)
    xw = window(xin, n, h, w, C, n - 1, h - K + 1, h + 1, w - K + 1, w + 1)
    got = window(out, n, h, w, C, n - 1, h - K + 1, h + 1, w - K + 1, w + 1)
    assert np.abs(got - affine_ref(xw, mc, cc, ms, cs, sem, alpha)).max() <= 1e-3           # test_gpu_transform bound
    U.check_device()


def _prepare(sty, hs, ws_, sem="tf"):
    eps_cov, eps_eig, thresh, _ = SEMS[sem]
    lib = U.lib()
    state = torch.empty(lib.wctb200_wct_style_state_bytes(C, 1), dtype=torch.uint8, device="cuda")
    ws = _ws(lib.wctb200_wct_workspace_bytes(C, 1, 1))
    _capi.check(lib.wctb200_wct_style_prepare(sty.data_ptr(), 1, hs, ws_, C, eps_cov, eps_eig, thresh, state.data_ptr(), ws.data_ptr(),
                                              ws.numel(), U.stream()))
    return state


def test_ost_apply_at_A():
    n, h, w = A
    lib = U.lib()
    eps_cov, eps_eig, thresh, readd = SEMS["tf"]
    xin = batch_act(n, h, w, C, 1000)
    sty, hs, ws_ = _style(1001)
    state = _prepare(sty, hs, ws_)
    alpha = 0.8

    def run(src, nn):
        dst = U.act_alloc(nn, h, w, C)
        ws = _ws(lib.wctb200_ost_workspace_bytes(C, nn))
        k = torch.full((5 * nn,), -7, dtype=torch.int32, device="cuda")
        _capi.check(lib.wctb200_ost_apply(src.data_ptr(), nn, h, w, C, state.data_ptr(), 1, alpha, eps_cov, eps_eig, thresh, readd,
                                          dst.data_ptr(), k.data_ptr(), ws.data_ptr(), ws.numel(), U.stream()))
        return dst, k.cpu().tolist()

    out, kb = run(xin, n)
    bp = pl(out, n, h, w, C)
    for i in range(n):
        one, k1 = run(frame_copy(xin, i, n, h, w, C), 1)
        assert_same(pl(one, 1, h, w, C)[:, 0], bp[:, i], "ost_apply frame %d" % i)
        assert k1 == kb[i::n], (i, k1, kb)
        del one
    _, mc, cc, _ = stats64(xin, n, h, w, C, n - 1)
    _, ms, cs, _ = stats64(sty, 1, hs, ws_, C, 0)
    xw = window(xin, n, h, w, C, n - 1, h - K + 1, h + 1, w - K + 1, w + 1)
    got = window(out, n, h, w, C, n - 1, h - K + 1, h + 1, w - K + 1, w + 1)
    assert np.abs(got - affine_ref(xw, mc, cc, ms, cs, "tf", alpha, ost=True)).max() <= 1e-3     # test_ost_apply_vs_fp64
    U.check_device()


def test_wct_apply_regions_at_A():
    """Two labels: frame i is split at column 1024 + 64 i, region 0 on the left takes style 0, region 1 style 1."""
    n, h, w = A
    lib = U.lib()
    eps_cov, eps_eig, thresh, readd = SEMS["tf"]
    xin = batch_act(n, h, w, C, 1100)
    styles = [_style(1101), _style(1102, 384, 640)]
    states = [_prepare(*s) for s in styles]
    cols = torch.arange(w, device="cuda")
    split = [1024 + 64 * i for i in range(n)]
    labels = torch.stack([(cols >= s).to(torch.uint8).expand(h, w) for s in split]).contiguous()
    ptrs = _capi.pointer_array([s.data_ptr() for s in states])
    alpha = 0.7

    def run(src, lab, nn):
        dst = U.act_alloc(nn, h, w, C)
        ws = _ws(lib.wctb200_wct_regions_workspace_bytes(C, nn, 2, h, w))
        k = torch.full((2 * (2 * nn + 2),), -7, dtype=torch.int32, device="cuda")
        _capi.check(lib.wctb200_wct_apply_regions(src.data_ptr(), nn, h, w, C, lab.data_ptr(), 2, ptrs, alpha, eps_cov, eps_eig,
                                                  thresh, readd, dst.data_ptr(), k.data_ptr(), ws.data_ptr(), ws.numel(), U.stream()))
        return dst, k.cpu().tolist()

    out, kb = run(xin, labels, n)
    bp = pl(out, n, h, w, C)
    for i in range(n):
        one, k1 = run(frame_copy(xin, i, n, h, w, C), labels[i:i + 1].contiguous(), 1)
        assert_same(pl(one, 1, h, w, C)[:, 0], bp[:, i], "wct_apply_regions frame %d" % i)
        # [k_c x 2N | k_s x 2 | sweeps_c x 2N | sweeps_s x 2]
        assert k1 == kb[2 * i:2 * i + 2] + kb[2 * n:2 * n + 2] + kb[2 * n + 2 + 2 * i:2 * n + 4 + 2 * i] + kb[4 * n + 2:], (i, k1, kb)
        del one
    # float64: a window of the last frame across its region boundary
    i, s = n - 1, split[n - 1]
    xw = window(xin, n, h, w, C, i, h - K + 1, h + 1, s - K // 2 + 1, s + K // 2 + 1)
    got = window(out, n, h, w, C, i, h - K + 1, h + 1, s - K // 2 + 1, s + K // 2 + 1)
    for r, (sty, hs, ws_) in enumerate(styles):
        _, mc, cc, _ = stats64(xin, n, h, w, C, i, mask=labels[i].bool() if r else ~labels[i].bool())
        _, ms, cs, _ = stats64(sty, 1, hs, ws_, C, 0)
        side = slice(0, K // 2) if r == 0 else slice(K // 2, K)
        ref = affine_ref(xw[:, side], mc, cc, ms, cs, "tf", alpha)
        assert np.abs(got[:, side] - ref).max() <= 1e-3, r
    U.check_device()


def _record(n):
    offs = [ctypes.c_size_t() for _ in range(4)]
    nbytes = U.lib().wctb200_stats_record_layout(C, n, 0, *[ctypes.byref(o) for o in offs])
    return torch.zeros(nbytes, dtype=torch.uint8, device="cuda"), [o.value for o in offs]


def _read_record(buf, offs, n):
    raw = buf.cpu().numpy()

    def arr(o, count):
        return raw[o:o + 8 * count].view(np.float64)
    return (arr(offs[0], n), arr(offs[1], n * C).reshape(n, C), arr(offs[2], n * C).reshape(n, C),
            arr(offs[3], n * C * C).reshape(n, C, C))


def test_wct_stats_rect_in_frame_16_of_B():
    n, h, w = B
    lib = U.lib()
    xin = batch_act(n, h, w, C, 1200)
    y0, x0, rh, rw = h - 300, w - 700, 300, 700
    rb, offs = _record(n)
    _capi.check(lib.wctb200_wct_stats_rect(xin.data_ptr(), n, h, w, C, y0, x0, rh, rw, rb.data_ptr(), U.stream()))
    r1, offs1 = _record(1)
    one = frame_copy(xin, n - 1, n, h, w, C)
    _capi.check(lib.wctb200_wct_stats_rect(one.data_ptr(), 1, h, w, C, y0, x0, rh, rw, r1.data_ptr(), U.stream()))
    got = [a[n - 1] for a in _read_record(rb, offs, n)]
    want = [a[0] for a in _read_record(r1, offs1, 1)]
    for name, g, wv in zip("ntsS", got, want):
        assert np.array_equal(np.asarray(g).view(np.uint64), np.asarray(wv).view(np.uint64)), name
    U.check_device()


# ----------------------------------------------------------------------------------------------- one 4096 x 4096 frame
def test_frame_4096_conv_head_and_tail_bands():
    """Locality at F: the bottom rows of conv_head and conv_tail, whose lo plane lies past 2^31, equal the same op on a crop."""
    h = w = FH
    lib = U.lib()
    wf, bf, d_wf, d_bf = _head_weights()
    img = _images(1, h, w, 1300)
    out = U.act_alloc(1, h, w, C)
    _capi.check(lib.wctb200_conv_head(img.data_ptr(), 1, h, w, d_wf.data_ptr(), d_bf.data_ptr(), out.data_ptr(), U.stream()))
    hc = 18
    crop_img = img[:, h - hc:].contiguous()
    band = U.act_alloc(1, hc, w, C)
    _capi.check(lib.wctb200_conv_head(crop_img.data_ptr(), 1, hc, w, d_wf.data_ptr(), d_bf.data_ptr(), band.data_ptr(), U.stream()))
    # the crop's first row sees a mirrored neighbour; its rows 1.. and its bottom halo are the frame's last 17 rows and halo
    assert_same(pl(band, 1, hc, w, C)[:, 0, 2:], pl(out, 1, h, w, C)[:, 0, h - hc + 2:], "conv_head band")
    ref = _head_ref(img[0, h - K:, w - K:].cpu().numpy(), wf, bf)[1:, 1:]
    assert_rel(window(out, 1, h, w, C, 0, h - K + 2, h + 1, w - K + 2, w + 1), ref, 2e-5, "conv_head vs float64")
    del band, crop_img, img

    # conv_tail reads the head's output; the crop's top halo row is the frame's row above the band, so every row matches
    k, b, d_k, d_b = _tail_weights()
    full = _tail(out, 1, h, w, d_k, d_b)
    crop = crop_rows(out, 1, h, w, C, 0, h - hc, h + 2)
    part = _tail(crop, 1, hc, w, d_k, d_b)
    assert_same(f32_bits(part[0]), f32_bits(full[0, h - hc:]), "conv_tail band")
    xw = window(out, 1, h, w, C, 0, h - K + 1, h + 1, w - K + 1, w + 1)
    assert_rel(full[0, h - K + 1:, w - K + 1:].cpu().numpy(), conv_ref64(xw[None], k, b, False)[0, 1:, 1:], 2e-5,
               "conv_tail vs float64")
    U.check_device()


def test_frame_4096_transform_band():
    """The whole-frame record at F against float64 statistics, and the bottom band of wct_style_prepare + wct_apply at F
    against wct_transform_apply of that record's transform on a crop of the band."""
    h = w = FH
    lib = U.lib()
    eps_cov, eps_eig, thresh, readd = SEMS["tf"]
    xin = act_of(feats_dev(h, w, C, 1400, 1.3))
    rec, offs = _record(1)
    _capi.check(lib.wctb200_wct_stats_rect(xin.data_ptr(), 1, h, w, C, 0, 0, h, w, rec.data_ptr(), U.stream()))
    n_, t, s, S = [a[0] for a in _read_record(rec, offs, 1)]
    assert n_ == h * w
    # float64 sums centred on the record's shift (test_rect_statistics_vs_fp64 bound: fp32 products, fp64 above)
    p = xin.view(torch.float16).view(2, 1, h + 2, w + 2, C)
    td = torch.from_numpy(t).cuda()
    s64 = torch.zeros(C, dtype=torch.float64, device="cuda")
    S64 = torch.zeros((C, C), dtype=torch.float64, device="cuda")
    xmax = 0.0
    for y in range(0, h, 256):
        x = (p[0, 0, 1 + y:1 + y + 256, 1:w + 1].double() + p[1, 0, 1 + y:1 + y + 256, 1:w + 1].double()).reshape(-1, C)
        xmax = max(xmax, float(x.abs().max()))
        d = x - td
        s64 += d.sum(0)
        S64 += d.T @ d
    scale = xmax ** 2 * h * w
    Su = np.triu(S) + np.triu(S, 1).T
    assert np.abs(t + s / n_ - (td + s64 / n_).cpu().numpy()).max() <= 1e-6 * xmax
    assert np.abs(Su - S64.cpu().numpy()).max() <= 1e-6 * scale

    sty, hs, ws_ = _style(1401)
    state = _prepare(sty, hs, ws_)
    alpha = 0.7
    ws = _ws(lib.wctb200_wct_workspace_bytes(C, 1, 1))
    out = U.act_alloc(1, h, w, C)
    _capi.check(lib.wctb200_wct_apply(xin.data_ptr(), 1, h, w, C, state.data_ptr(), 1, alpha, eps_cov, eps_eig, thresh, readd,
                                      out.data_ptr(), None, ws.data_ptr(), ws.numel(), U.stream()))
    tr = torch.empty(lib.wctb200_wct_transform_layout(C, 1, None, None, None), dtype=torch.uint8, device="cuda")
    _capi.check(lib.wctb200_wct_transform_from_stats(rec.data_ptr(), 1, C, state.data_ptr(), 1, alpha, eps_cov, eps_eig, thresh,
                                                     readd, tr.data_ptr(), ws.data_ptr(), ws.numel(), U.stream()))
    hb = 16
    crop = crop_rows(xin, 1, h, w, C, 0, h - hb, h + 2)
    band = U.act_alloc(1, hb, w, C)
    _capi.check(lib.wctb200_wct_transform_apply(crop.data_ptr(), 1, hb, w, C, tr.data_ptr(), band.data_ptr(), U.stream()))
    # the apply writes each halo cell as the mirror of its interior pixel, so the crop's top halo row is not the frame's
    assert_same(pl(band, 1, hb, w, C)[:, 0, 1:], pl(out, 1, h, w, C)[:, 0, h - hb + 1:], "wct_apply band")
    _, mc, cc, _ = stats64(xin, 1, h, w, C, 0)
    _, ms, cs, _ = stats64(sty, 1, hs, ws_, C, 0)
    xw = window(xin, 1, h, w, C, 0, h - K + 1, h + 1, w - K + 1, w + 1)
    got = window(out, 1, h, w, C, 0, h - K + 1, h + 1, w - K + 1, w + 1)
    assert np.abs(got - affine_ref(xw, mc, cc, ms, cs, "tf", alpha)).max() <= 1e-3
    U.check_device()


# -------------------------------------------------------------------------------------------------------------- engine
def test_engine_one_group_17_frames_1080p():
    """relu1_1 of 17 frames at 1920 x 1080 in one group: the hi plane passes 2^31 and the lo plane 2^32."""
    targets = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]
    eng = Engine(make_synthetic_weights(42), targets, semantics="tf")
    eng.groups = 1
    g = torch.Generator(device="cuda").manual_seed(1500)
    content = torch.randint(0, 256, (17, 1080, 1920, 3), generator=g, device="cuda", dtype=torch.uint8)
    style = torch.randint(0, 256, (1, 512, 512, 3), generator=g, device="cuda", dtype=torch.uint8)
    out = eng.to_u8(eng.stylize(content, style, alpha=0.7))
    eng.check_device()
    for i in [0] + list(range(8, 17)):
        one = eng.to_u8(eng.stylize(content[i:i + 1], style, alpha=0.7))
        assert_same(one[0], out[i], "engine frame %d" % i)
    eng.check_device()
