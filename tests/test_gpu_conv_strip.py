"""The conv mainloop stages one activation strip per (filter row, 64-channel slice) and feeds every column tap of that row
from it: column tap kx is a wgmma operand that starts kx rows into the 128B-swizzled strip, not at a swizzle atom.

These cases run each mode on a one-CTA-per-SM grid (every CTA walks many strips back to back through the rings) and on the
default grid, require the same bytes from both, and compare with the float64 references:
- strips whose first row lies above the tensor (top tiles) or whose last rows lie past it (the final tile);
- many channel slices (Cin = 512, K = 4608), where the k-order (filter row, slice, column tap) decides the chunk sums;
- the style swap's kw x kw correlation with kw = 9 .. 16, whose column taps start at every row residue of a swizzle atom
  and run into the next atom."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import tests.gpu_util as U
from oracle import ref_ops
from tests.test_gpu_conv_handoff import _both_grids, _raw, _weights
from tests.test_gpu_layers import _conv_inputs, assert_close, conv_ref64, weight_repr
from wct_tf_b200 import _capi

pytestmark = pytest.mark.gpu


def _with_tile(bn, fuse, run):
    lib = U.lib()
    lib.wctb200_debug_set_conv_bn(bn)
    lib.wctb200_debug_set_conv_fuse(fuse)
    try:
        return _both_grids(run)
    finally:
        lib.wctb200_debug_set_conv_bn(0)
        lib.wctb200_debug_set_conv_fuse(-1)


def _reflected(padded):
    return np.array_equal(padded, np.pad(padded[:, 1:-1, 1:-1], ((0, 0), (1, 1), (1, 1), (0, 0)), mode="reflect"))


CASES_3X3 = [
    # N, H, W, Cin, Cout, BN, fuse
    (3, 9, 5, 64, 128, 128, -1),       # Wp = 7: a tile spans many image rows and images
    (3, 9, 5, 64, 64, 64, 1),
    (1, 20, 126, 128, 128, 128, -1),   # Wp = 128: a tile is one padded row
    (1, 20, 126, 128, 64, 64, 0),
    (1, 20, 126, 128, 64, 64, 1),
    (2, 12, 30, 512, 128, 128, -1),    # K = 4608
]


@pytest.mark.parametrize("case", CASES_3X3, ids=lambda c: "x".join(map(str, c)))
def test_conv3x3_strip(case):
    n, h, w, cin, cout, bn, fuse = case
    x, k, b = _conv_inputs((n, h, w, cin, cout, True), 61)
    lib = U.lib()
    xin, ws, d_b = U.act_from_numpy(x), _weights(k, 9, cin, cout), U.dev(b)

    def run():
        out = U.act_alloc(n, h, w, cout)
        _capi.check(lib.wctb200_conv3x3(xin.data_ptr(), n, h, w, cin, ws.data_ptr(), d_b.data_ptr(), cout, _capi.RELU,
                                        out.data_ptr(), U.stream()))
        return out

    one, dflt = _with_tile(bn, fuse, run)
    assert np.array_equal(_raw(one), _raw(dflt))
    padded = U.act_raw_padded(dflt, n, h, w, cout)
    assert np.isfinite(padded).all(), "cells left unwritten"
    assert _reflected(padded)
    assert_close(padded[:, 1:-1, 1:-1], conv_ref64(U.split_repr(x), weight_repr(k), b, True), tol=1e-5,
                 name="strip_3x3_%d_%d_bn%d" % (cin, cout, bn))


@pytest.mark.parametrize("bn", [64, 128])
def test_conv3x3_pool2_strip(bn):
    n, h, w, cin, cout = 2, 33, 141, 128, 128      # odd sizes: ragged right column and bottom row; three column segments
    x, k, b = _conv_inputs((n, h, w, cin, cout, True), 62)
    lib = U.lib()
    xin, ws, d_b = U.act_from_numpy(x), _weights(k, 9, cin, cout), U.dev(b)
    ho, wo = (h + 1) // 2, (w + 1) // 2

    def run():
        out = U.act_alloc(n, ho, wo, cout)
        _capi.check(lib.wctb200_conv3x3(xin.data_ptr(), n, h, w, cin, ws.data_ptr(), d_b.data_ptr(), cout,
                                        _capi.RELU | _capi.POOL2, out.data_ptr(), U.stream()))
        return out

    one, dflt = _with_tile(bn, -1, run)
    assert np.array_equal(_raw(one), _raw(dflt))
    padded = U.act_raw_padded(dflt, n, ho, wo, cout)
    assert np.isfinite(padded).all(), "pooled cells left unwritten"
    assert _reflected(padded)
    ref = conv_ref64(U.split_repr(x), weight_repr(k), b, True)
    ref = F.max_pool2d(torch.from_numpy(ref).permute(0, 3, 1, 2), 2, 2, ceil_mode=True).permute(0, 2, 3, 1).numpy()
    assert_close(padded[:, 1:-1, 1:-1], ref, tol=1e-5, name="strip_pool2_bn%d" % bn)


CASES_UP2 = [
    # N, H, W (low resolution), Cin, Cout, BN, fuse
    (2, 20, 33, 64, 128, 128, -1),
    (2, 20, 33, 128, 64, 64, 0),
    (2, 20, 33, 128, 64, 64, 1),
    (1, 12, 14, 512, 128, 128, -1),
]


@pytest.mark.parametrize("case", CASES_UP2, ids=lambda c: "x".join(map(str, c)))
def test_conv3x3_up2_strip(case):
    n, h, w, cin, cout, bn, fuse = case
    x, k, b = _conv_inputs((n, h, w, cin, cout, True), 63)
    lib = U.lib()
    xin, ws, d_b = U.act_from_numpy(x), _weights(k, 9, cin, cout, up2=True), U.dev(b)
    lowp = U.act_raw_padded(xin, n, h, w, cin)

    def run():
        out = U.act_alloc(n, 2 * h, 2 * w, cout)
        _capi.check(lib.wctb200_conv3x3_up2(xin.data_ptr(), n, h, w, cin, ws.data_ptr(), d_b.data_ptr(), cout, _capi.RELU,
                                            out.data_ptr(), U.stream()))
        return out

    one, dflt = _with_tile(bn, fuse, run)
    assert np.array_equal(_raw(one), _raw(dflt))
    padded = U.act_raw_padded(dflt, n, 2 * h, 2 * w, cout)
    assert np.isfinite(padded).all(), "cells left unwritten"
    # the input carries a reflect halo, not the edge halo the engine gives an UP2 input: compare where no output reads it
    up = np.repeat(np.repeat(lowp[:, 1:-1, 1:-1], 2, axis=1), 2, axis=2)
    ref = conv_ref64(up, k, b, True)
    assert_close(padded[:, 3:-3, 3:-3], ref[:, 2:-2, 2:-2], tol=1e-5, name="strip_up2_%d_%d_bn%d" % (cin, cout, bn))


@pytest.mark.parametrize("patch, hwc, hws", [(9, (12, 21), (12, 12)), (13, (15, 24), (14, 15)), (16, (18, 29), (18, 18))])
def test_style_swap_wide_patch_strip(patch, hwc, hws):
    """The style swap's patch correlation is a kw x kw conv (kw = patch) fed from strips of 127 + kw rows."""
    C, alpha = 64, 0.6
    rng = np.random.default_rng(20)

    def feat(hw):
        m = rng.standard_normal((C, C)) / np.sqrt(C)
        return np.maximum(rng.standard_normal((hw[0] * hw[1], C)) @ m + 0.3, 0.0).reshape(1, hw[0], hw[1], C).astype(np.float32)

    content, style = feat(hwc), feat(hws)
    ref, info = ref_ops.wct_style_swap(U.split_repr(content).astype(np.float64), U.split_repr(style).astype(np.float64), alpha,
                                       patch_size=patch, stride=1, return_info=True)
    assert ref_ops.spectral_gap_ok(info["wc"]) and ref_ops.spectral_gap_ok(info["ws"]), "ill-posed vector (eigenvalue near the cut)"
    assert info["margin"].min() > 2e-3, "ill-posed vector (arg-max decided by %.1e)" % info["margin"].min()
    lib = U.lib()
    cin, sin = U.act_from_numpy(content), U.act_from_numpy(style)
    nbytes = lib.wctb200_style_swap_workspace_bytes(C, hwc[0], hwc[1], hws[0], hws[1], patch, 1)
    assert nbytes > 0
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")

    def run():
        out = U.act_alloc(1, hwc[0], hwc[1], C)
        kbuf = torch.zeros(2, dtype=torch.int32, device="cuda")
        _capi.check(lib.wctb200_style_swap_level(cin.data_ptr(), hwc[0], hwc[1], sin.data_ptr(), hws[0], hws[1], C, patch, 1,
                                                 alpha, 1e-8, 1e-5, out.data_ptr(), kbuf.data_ptr(), ws.data_ptr(), ws.numel(),
                                                 U.stream()))
        assert tuple(kbuf.cpu().tolist()) == (info["k_c"], info["k_s"])
        return out

    one, dflt = _both_grids(run)
    assert np.array_equal(_raw(one), _raw(dflt))
    got = U.act_to_numpy(dflt, 1, hwc[0], hwc[1], C)
    err = np.abs(got - ref).max()
    print("style swap patch %d: max-abs vs fp64 oracle %.2e" % (patch, err))
    assert err <= 1e-3
    assert _reflected(U.act_raw_padded(dflt, 1, hwc[0], hwc[1], C))
