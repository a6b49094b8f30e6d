"""GPU: the conv's split-fp16 accumulation (conv_tc.cu, DESIGN.md §3.1).

The large a_hi*b_hi products accumulate in chunks of two k-iterations, each added into the running sum with round-to-nearest
FADDs; the small cross products a_hi*b_lo + a_lo*b_hi accumulate in one tensor-core accumulator over the whole K and are added
once at the end.  These tests pin that scheme where it is weakest, on heavy cancellation at the longest K, and pin that the
cross-product accumulator adds exactly nothing when every cross term is zero."""
import numpy as np
import pytest
import torch

from wct_tf_b200 import _capi
from tests import gpu_util as U
from tests.test_gpu_layers import conv_ref64, weight_repr

pytestmark = pytest.mark.gpu


def _run_conv(x, k, up2=False, fuse=-1, products=3):
    """3x3 conv (up2: the UP2 conv) without bias or ReLU; returns (output buffer, fp32 output)."""
    n, h, w, cin = x.shape
    cout = k.shape[3]
    lib = U.lib()
    xin = U.act_from_numpy(x)
    d_k = U.dev(k)
    bias = torch.zeros(cout, dtype=torch.float32, device="cuda")
    ws = torch.empty(lib.wctb200_conv_weight_bytes(16 if up2 else 9, cin, cout), dtype=torch.uint8, device="cuda")
    if up2:
        _capi.check(lib.wctb200_prep_conv_weights_up2(d_k.data_ptr(), cin, cout, ws.data_ptr(), U.stream()))
    else:
        _capi.check(lib.wctb200_prep_conv_weights(d_k.data_ptr(), 9, cin, cout, ws.data_ptr(), U.stream()))
    ho, wo = (2 * h, 2 * w) if up2 else (h, w)
    out = U.act_alloc(n, ho, wo, cout)
    fn = lib.wctb200_conv3x3_up2 if up2 else lib.wctb200_conv3x3
    lib.wctb200_debug_set_conv_fuse(fuse)
    assert lib.wctb200_debug_set_conv_products(products) == products
    try:
        _capi.check(fn(xin.data_ptr(), n, h, w, cin, ws.data_ptr(), bias.data_ptr(), cout, 0, out.data_ptr(), U.stream()))
        U.check_device()
    finally:
        lib.wctb200_debug_set_conv_fuse(-1)
        lib.wctb200_debug_set_conv_products(3)
    return out, U.act_to_numpy(out, n, ho, wo, cout)


CANCEL_CASES = [
    # N, H, W, Cin, Cout, fuse
    (1, 12, 12, 512, 512, -1),         # K = 4608, BN = 128: 36 chunks of a_hi b_hi, one cross-product accumulator
    (2, 20, 24, 64, 64, -1),           # BN = 64, fused a_hi [b_hi | b_lo]; 9 k-iterations, the last chunk a short one
    (2, 20, 24, 64, 64, 0),            # BN = 64 without the fused product
]


@pytest.mark.parametrize("case", CANCEL_CASES, ids=lambda c: "x".join(map(str, c)))
def test_conv_heavy_cancellation_against_fp64(case):
    """Mixed-sign activations in channel pairs that differ by ~1e-3, weights of opposite sign on the two channels of a
    pair: every output is a sum whose terms cancel to ~1e-5 of sum |a||b|.  Against float64 of the stored split operands
    the error stays within 2^-21 sum |a||b|: eight fp32 unit roundoffs of the magnitude the conv adds up, where a
    cross-product accumulator that kept a stale value or dropped a product would be off by ~2^-18 or more."""
    n, h, w, cin, cout, fuse = case
    rng = np.random.default_rng(11)
    base = rng.normal(0.0, 1.0, (n, h, w, cin // 2))
    x = np.empty((n, h, w, cin), dtype=np.float32)
    x[..., 0::2] = base
    x[..., 1::2] = base + rng.normal(0.0, 1e-3, base.shape)
    kb = rng.normal(0.0, np.sqrt(2.0 / (9 * cin)), (3, 3, cin // 2, cout))
    k = np.empty((3, 3, cin, cout), dtype=np.float32)
    k[:, :, 0::2] = kb
    k[:, :, 1::2] = -kb
    _, got = _run_conv(x, k, fuse=fuse)
    xs, ks = U.split_repr(x), weight_repr(k)
    ref = conv_ref64(xs, ks, np.zeros(cout), False)
    mag = conv_ref64(np.abs(xs), np.abs(ks), np.zeros(cout), False)          # sum |a||b| per output
    assert np.isfinite(got).all()
    err = np.abs(got - ref) / mag
    print("K=%d: max |err| / sum|a||b| = %.3g (2^%.1f), median |ref| / sum|a||b| = %.2g" % (
        9 * cin, err.max(), np.log2(err.max()), np.median(np.abs(ref) / mag)))
    assert np.median(np.abs(ref) / mag) < 1e-3, "the inputs do not cancel"
    if err.max() > 2.0 ** -21:
        U.dump("fail_conv_cancel_%d_%d" % (cin, cout), got=got, ref=ref, mag=mag)
    assert err.max() <= 2.0 ** -21


ZERO_CROSS_CASES = [
    # N, H, W, Cin, Cout, up2, fuse
    (1, 12, 12, 512, 512, False, -1),  # 72 k-iterations: whole chunks only
    (2, 20, 24, 64, 64, False, -1),    # 9 k-iterations: a short last chunk, fused product
    (2, 20, 24, 64, 64, False, 0),
    (1, 16, 16, 128, 64, False, -1),   # two channel slices per filter row
    (2, 9, 11, 64, 64, True, -1),      # UP2: 4 k-iterations per parity class
]


@pytest.mark.parametrize("case", ZERO_CROSS_CASES, ids=lambda c: "x".join(map(str, c)))
def test_conv_zero_cross_terms_equal_one_product(case):
    """Activations and weights that fp16 holds exactly (the weights also after their power-of-two scaling) have a_lo = b_lo
    = 0, so every cross product is zero.  The three-product conv must then give the bits of the one-product conv: the
    cross-product accumulator starts every pass at zero and adds exactly nothing, in every tile and every pass."""
    n, h, w, cin, cout, up2, fuse = case
    rng = np.random.default_rng(12)
    x = (rng.integers(-64, 65, (n, h, w, cin)) / 64.0).astype(np.float32)
    # |m| <= 255: the UP2 weights are sums of up to four taps, which must stay within fp16's 11 significant bits
    k = (rng.integers(-255, 256, (3, 3, cin, cout)) / 256.0).astype(np.float32)
    assert np.array_equal(U.split_repr(x), x.astype(np.float64))
    assert np.array_equal(weight_repr(k), k.astype(np.float64))
    buf3, got3 = _run_conv(x, k, up2=up2, fuse=fuse, products=3)
    buf1, got1 = _run_conv(x, k, up2=up2, fuse=fuse, products=1)
    assert np.isfinite(got3).all()
    assert torch.equal(buf3, buf1), "max |3 products - 1 product| = %.3g" % np.abs(got3 - got1).max()
    if not up2:
        ref = conv_ref64(x, k, np.zeros(cout), False)
        assert np.abs(got3 - ref).max() <= 1e-5 * (1 + np.abs(ref).max())
