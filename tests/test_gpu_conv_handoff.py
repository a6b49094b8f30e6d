"""The conv epilogue runs on its own warps and takes each finished tile over from the MMA warps through one shared-memory
buffer.  Its output must not depend on how the tiles are spread over the CTAs: one CTA per SM (every CTA walks many tiles,
hand-offs back to back) gives the same bytes as the default over-subscribed grid, halo cells included, and both agree
with the float64 references."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import tests.gpu_util as U
from tests.test_gpu_layers import _conv_inputs, assert_close, conv_ref64, weight_repr
from tests.test_gpu_regions import _apply_regions, _feats, _prepare, blobs
from wct_tf_b200 import _capi

pytestmark = pytest.mark.gpu

DEFAULT_OVERSUB = 4          # the library's conv grid: 4 CTAs per SM


def _both_grids(run):
    """run() on a grid of one CTA per SM, then on the default grid; returns the two results."""
    lib = U.lib()
    lib.wctb200_debug_set_conv_oversub(1)
    try:
        one = run()
        U.check_device()
    finally:
        lib.wctb200_debug_set_conv_oversub(DEFAULT_OVERSUB)
    dflt = run()
    U.check_device()
    return one, dflt


def _raw(buf):
    return buf.view(torch.int16).cpu().numpy()


def _weights(k, taps, cin, cout, up2=False):
    lib = U.lib()
    ws = torch.empty(lib.wctb200_conv_weight_bytes(16 if up2 else taps, cin, cout), dtype=torch.uint8, device="cuda")
    d_k = U.dev(k)
    if up2:
        _capi.check(lib.wctb200_prep_conv_weights_up2(d_k.data_ptr(), cin, cout, ws.data_ptr(), U.stream()))
    else:
        _capi.check(lib.wctb200_prep_conv_weights(d_k.data_ptr(), taps, cin, cout, ws.data_ptr(), U.stream()))
    return ws


@pytest.mark.parametrize("bn", [64, 0])          # 0: the default tile, 128 for Cout = 128
def test_conv3x3_handoff_grid_independent(bn):
    n, h, w, cin, cout = 2, 100, 130, 64, 128      # 400 tiles at BN = 64: ~3 per CTA on a one-CTA-per-SM grid
    x, k, b = _conv_inputs((n, h, w, cin, cout, True), 41)
    lib = U.lib()
    xin, ws, d_b = U.act_from_numpy(x), _weights(k, 9, cin, cout), U.dev(b)

    def run():
        out = U.act_alloc(n, h, w, cout)
        _capi.check(lib.wctb200_conv3x3(xin.data_ptr(), n, h, w, cin, ws.data_ptr(), d_b.data_ptr(), cout, _capi.RELU,
                                        out.data_ptr(), U.stream()))
        return out

    lib.wctb200_debug_set_conv_bn(bn)
    try:
        one, dflt = _both_grids(run)
    finally:
        lib.wctb200_debug_set_conv_bn(0)
    assert np.array_equal(_raw(one), _raw(dflt))
    padded = U.act_raw_padded(dflt, n, h, w, cout)
    assert np.isfinite(padded).all(), "cells left unwritten"
    assert np.array_equal(padded, np.pad(padded[:, 1:-1, 1:-1], ((0, 0), (1, 1), (1, 1), (0, 0)), mode="reflect"))
    assert_close(padded[:, 1:-1, 1:-1], conv_ref64(U.split_repr(x), weight_repr(k), b, True), tol=1e-5, name="handoff_3x3")


def test_conv3x3_up2_handoff_grid_independent():
    n, h, w, cin, cout = 2, 48, 64, 64, 64         # 4 parity classes x 52 tiles
    x, k, b = _conv_inputs((n, h, w, cin, cout, True), 42)
    lib = U.lib()
    xin, ws, d_b = U.act_from_numpy(x), _weights(k, 9, cin, cout, up2=True), U.dev(b)
    lowp = U.act_raw_padded(xin, n, h, w, cin)

    def run():
        out = U.act_alloc(n, 2 * h, 2 * w, cout)
        _capi.check(lib.wctb200_conv3x3_up2(xin.data_ptr(), n, h, w, cin, ws.data_ptr(), d_b.data_ptr(), cout, _capi.RELU,
                                            out.data_ptr(), U.stream()))
        return out

    one, dflt = _both_grids(run)
    assert np.array_equal(_raw(one), _raw(dflt))
    padded = U.act_raw_padded(dflt, n, 2 * h, 2 * w, cout)
    assert np.isfinite(padded).all(), "cells left unwritten"
    # the input carries a reflect halo, not the edge halo the engine gives an UP2 input: compare the interior with the
    # conv of the upsampled interior only where no output reads the halo
    up = np.repeat(np.repeat(lowp[:, 1:-1, 1:-1], 2, axis=1), 2, axis=2)
    ref = conv_ref64(up, k, b, True)
    assert_close(padded[:, 3:-3, 3:-3], ref[:, 2:-2, 2:-2], tol=1e-5, name="handoff_up2")


def test_conv3x3_pool2_handoff_grid_independent():
    n, h, w, cin, cout = 2, 95, 131, 64, 64        # odd sizes: ragged right column and bottom row of the 'same' pooling
    x, k, b = _conv_inputs((n, h, w, cin, cout, True), 43)
    lib = U.lib()
    xin, ws, d_b = U.act_from_numpy(x), _weights(k, 9, cin, cout), U.dev(b)
    ho, wo = (h + 1) // 2, (w + 1) // 2

    def run():
        out = U.act_alloc(n, ho, wo, cout)
        _capi.check(lib.wctb200_conv3x3(xin.data_ptr(), n, h, w, cin, ws.data_ptr(), d_b.data_ptr(), cout,
                                        _capi.RELU | _capi.POOL2, out.data_ptr(), U.stream()))
        return out

    one, dflt = _both_grids(run)
    assert np.array_equal(_raw(one), _raw(dflt))
    padded = U.act_raw_padded(dflt, n, ho, wo, cout)
    assert np.isfinite(padded).all(), "pooled cells left unwritten"
    assert np.array_equal(padded, np.pad(padded[:, 1:-1, 1:-1], ((0, 0), (1, 1), (1, 1), (0, 0)), mode="reflect"))
    ref = conv_ref64(U.split_repr(x), weight_repr(k), b, True)
    ref = F.max_pool2d(torch.from_numpy(ref).permute(0, 3, 1, 2), 2, 2, ceil_mode=True).permute(0, 2, 3, 1).numpy()
    assert_close(padded[:, 1:-1, 1:-1], ref, tol=1e-5, name="handoff_pool2")


def test_apply_per_image_handoff_grid_independent():
    """wctb200_wct_apply with one style per frame: the 1x1 apply conv runs per-image tiles with per-image weight sets."""
    nc, hc, wc, c = 3, 64, 128, 128
    content, style = _feats((nc, hc, wc, c), 44), _feats((nc, 24, 32, c), 45)
    state = _prepare(style)
    lib = U.lib()
    cin = U.act_from_numpy(content)
    ws = torch.empty(lib.wctb200_wct_workspace_bytes(c, nc, 0), dtype=torch.uint8, device="cuda")

    def run():
        out = torch.zeros(lib.wctb200_act_bytes(nc, hc, wc, c), dtype=torch.uint8, device="cuda")
        _capi.check(lib.wctb200_wct_apply(cin.data_ptr(), nc, hc, wc, c, state.data_ptr(), nc, 0.7, 1e-8, 0.0, 1e-5, 1,
                                          out.data_ptr(), None, ws.data_ptr(), ws.numel(), U.stream()))
        return out

    one, dflt = _both_grids(run)
    assert np.array_equal(_raw(one), _raw(dflt))
    padded = U.act_raw_padded(dflt, nc, hc, wc, c)
    assert np.isfinite(padded).all()
    assert np.array_equal(padded, np.pad(padded[:, 1:-1, 1:-1], ((0, 0), (1, 1), (1, 1), (0, 0)), mode="reflect"))
    # frame i alone against style i alone: the per-image weight set of the batched apply is that frame's own transform
    for i in range(nc):
        si = _prepare(style[i:i + 1])
        ci = U.act_from_numpy(content[i:i + 1])
        wsi = torch.empty(lib.wctb200_wct_workspace_bytes(c, 1, 0), dtype=torch.uint8, device="cuda")
        oi = torch.zeros(lib.wctb200_act_bytes(1, hc, wc, c), dtype=torch.uint8, device="cuda")
        _capi.check(lib.wctb200_wct_apply(ci.data_ptr(), 1, hc, wc, c, si.data_ptr(), 1, 0.7, 1e-8, 0.0, 1e-5, 1,
                                          oi.data_ptr(), None, wsi.data_ptr(), wsi.numel(), U.stream()))
        U.check_device()
        assert_close(padded[i], U.act_raw_padded(oi, 1, hc, wc, c)[0], tol=1e-4, name="handoff_apply_%d" % i)


def test_apply_regions_handoff_grid_independent():
    """Regions apply: one hand-off per region present in a tile, then the copy of the pixels that keep their input."""
    nc, hc, wc, c = 2, 64, 128, 128
    content = _feats((nc, hc, wc, c), 46)
    states = [_prepare(_feats((1, 16, 16, c), 47 + r)) for r in range(2)]
    lab = np.stack([blobs(hc, wc, 2, 50 + i) for i in range(nc)])      # label 2 = unstyled strip
    (cin, one, _), (_, dflt, _) = _both_grids(lambda: _apply_regions(content, lab, states, 1.0))
    assert np.array_equal(_raw(one), _raw(dflt))
    padded = U.act_raw_padded(dflt, nc, hc, wc, c)
    assert np.isfinite(padded).all()
    keep = np.pad(lab >= 2, ((0, 0), (1, 1), (1, 1)), mode="reflect")
    planes_in = _raw(cin).reshape(2, nc, hc + 2, wc + 2, c)
    planes_out = _raw(dflt).reshape(2, nc, hc + 2, wc + 2, c)
    assert np.array_equal(planes_out[:, keep], planes_in[:, keep])
