"""Spatial control on the GPU: label resize, per-region covariance, the regions apply and the masked pipeline
against the fp64 region oracle (tests/regions_ref.py)."""
import numpy as np
import pytest
import torch

import tests.gpu_util as U
from oracle import nets, ref_ops
from tests.regions_ref import pipeline_regions, resize_labels, wct_regions
from tests.test_gpu_pipeline import ALL, FREE_RUN_NOISE_FACTOR
from wct_tf_b200 import _capi
from wct_tf_b200.engine import Engine, SEMANTICS
from wct_tf_b200.weights import make_synthetic_weights
from wct_tf_b200.wct import WCT

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def weights():
    return make_synthetic_weights(42)


def halves(h, w):
    m = np.zeros((h, w), np.uint8)
    m[:, w // 2:] = 1
    return m


def blobs(h, w, R, seed, strip=True):
    """R random disc-shaped regions over region 0, plus (strip) an unlabelled band of label R at the bottom."""
    rng = np.random.default_rng(seed)
    m = np.zeros((h, w), np.uint8)
    yy, xx = np.mgrid[:h, :w]
    for r in range(1, R):
        cy, cx, rad = rng.integers(0, h), rng.integers(0, w), rng.integers(h // 6, h // 3)
        m[(yy - cy) ** 2 + (xx - cx) ** 2 < rad * rad] = r
    if strip:
        m[h - max(1, h // 8):, :] = R
    return m


@pytest.mark.parametrize("n,hm,wm,hf,wf", [(1, 512, 512, 64, 64), (2, 37, 101, 9, 13), (3, 5, 7, 33, 65), (1, 1, 1, 4, 3)])
def test_labels_resize_matches_rule(n, hm, wm, hf, wf):
    mask = np.random.default_rng(hm + wf).integers(0, 256, (n, hm, wm), dtype=np.uint8)
    src = U.dev(mask)
    dst = torch.empty((n, hf, wf), dtype=torch.uint8, device="cuda")
    _capi.check(U.lib().wctb200_labels_resize_nearest(src.data_ptr(), n, hm, wm, hf, wf, dst.data_ptr(), U.stream()))
    U.check_device()
    assert np.array_equal(dst.cpu().numpy(), resize_labels(mask, hf, wf))


@pytest.mark.parametrize("shape", [(1, 16, 33, 64), (2, 9, 40, 128), (1, 12, 21, 256), (2, 8, 9, 512), (1, 70, 130, 64)])
def test_covariance_regions_match_float64(shape):
    """Means and covariances over each region's pixel set (tolerance of test_covariance_kernels).  Region 1 has no pixel,
    region 2 one pixel, region 3 a mean far from the frame mean."""
    rng = np.random.default_rng(sum(shape))
    n, h, w, c = shape
    R = 4
    x = np.maximum(rng.standard_normal(shape) @ (rng.standard_normal((c, c)) / np.sqrt(c)) + 0.3, 0).astype(np.float32)
    lab = np.zeros((n, h, w), np.uint8)
    lab[:, :, w // 2:] = 3
    lab[:, 0, 0] = 2
    lab[:, h // 2:, : w // 3] = 7                       # label >= R: in no region
    x[lab == 3] += 40.0                                 # region 3 sits far from the frame mean
    buf = U.act_from_numpy(x)
    mean = torch.empty((n * R, c), dtype=torch.float32, device="cuda")
    cov = torch.empty((n * R, c, c), dtype=torch.float32, device="cuda")
    counts = torch.empty(n * R, dtype=torch.int32, device="cuda")
    _capi.check(U.lib().wctb200_covariance_regions(buf.data_ptr(), n, h, w, c, U.dev(lab).data_ptr(), R, 1e-8, mean.data_ptr(),
                                                   cov.data_ptr(), counts.data_ptr(), U.stream()))
    U.check_device()
    xs = U.split_repr(x)
    for i in range(n):
        for r in range(R):
            z = i * R + r
            px = xs[i][lab[i] == r]
            assert counts[z].item() == len(px)
            got = cov[z].cpu().numpy()
            if len(px) < 2:
                assert np.array_equal(got, np.eye(c, dtype=np.float32))
                continue
            ref = np.cov(px.T) + 1e-8 * np.eye(c)
            assert np.abs(mean[z].cpu().numpy() - px.mean(0)).max() <= 1e-6 * max(1.0, np.abs(px.mean(0)).max())
            assert np.abs(got - ref).max() <= 1.5e-6 * max(1.0, np.abs(ref).max()), (z, np.abs(got - ref).max())
            assert np.array_equal(got, got.T)


def _prepare(style, sem="tf"):
    lib = U.lib()
    ns, hs, ws_, c = style.shape
    sp = SEMANTICS[sem]
    sin = U.act_from_numpy(style)
    ws = torch.empty(lib.wctb200_wct_workspace_bytes(c, 0, ns), dtype=torch.uint8, device="cuda")
    state = torch.empty(lib.wctb200_wct_style_state_bytes(c, ns), dtype=torch.uint8, device="cuda")
    _capi.check(lib.wctb200_wct_style_prepare(sin.data_ptr(), ns, hs, ws_, c, sp["eps_cov"], sp["eps_eig"], sp["thresh"],
                                              state.data_ptr(), ws.data_ptr(), ws.numel(), U.stream()))
    return state


def _apply_regions(content, lab, states, alpha, sem="tf"):
    lib = U.lib()
    nc, hc, wc, c = content.shape
    R = len(states)
    sp = SEMANTICS[sem]
    cin = U.act_from_numpy(content)
    out = torch.zeros(lib.wctb200_act_bytes(nc, hc, wc, c), dtype=torch.uint8, device="cuda")
    ws = torch.empty(lib.wctb200_wct_regions_workspace_bytes(c, nc, R, hc, wc), dtype=torch.uint8, device="cuda")
    kbuf = torch.zeros(2 * (nc * R + R), dtype=torch.int32, device="cuda")
    _capi.check(lib.wctb200_wct_apply_regions(cin.data_ptr(), nc, hc, wc, c, U.dev(lab).data_ptr(), R,
                                              _capi.pointer_array([s.data_ptr() for s in states]), alpha, sp["eps_cov"],
                                              sp["eps_eig"], sp["thresh"], sp["readd"], out.data_ptr(), kbuf.data_ptr(),
                                              ws.data_ptr(), ws.numel(), U.stream()))
    U.check_device()
    return cin, out, kbuf.cpu().numpy()


def _feats(shape, seed):
    rng = np.random.default_rng(seed)
    c = shape[-1]
    return np.maximum(rng.standard_normal(shape) @ (rng.standard_normal((c, c)) / np.sqrt(c)) + 0.3, 0).astype(np.float32)


@pytest.mark.parametrize("shape", [(2, 24, 40, 128), (1, 33, 17, 64), (3, 8, 8, 512)])
def test_one_region_is_byte_identical_to_wct_apply(shape):
    nc, hc, wc, c = shape
    content, style = _feats(shape, 1), _feats((1, 20, 30, c), 2)
    state = _prepare(style)
    lib = U.lib()
    cin = U.act_from_numpy(content)
    ref = torch.zeros(lib.wctb200_act_bytes(nc, hc, wc, c), dtype=torch.uint8, device="cuda")
    ws = torch.empty(lib.wctb200_wct_workspace_bytes(c, nc, 0), dtype=torch.uint8, device="cuda")
    _capi.check(lib.wctb200_wct_apply(cin.data_ptr(), nc, hc, wc, c, state.data_ptr(), 1, 0.7, 1e-8, 0.0, 1e-5, 1, ref.data_ptr(),
                                      None, ws.data_ptr(), ws.numel(), U.stream()))
    _, out, k = _apply_regions(content, np.zeros((nc, hc, wc), np.uint8), [state], 0.7)
    assert torch.equal(out, ref)
    assert (k[:nc] > 0).all()


def test_unstyled_pixels_keep_their_bytes_interior_and_halo():
    nc, hc, wc, c = 2, 19, 45, 128
    content = _feats((nc, hc, wc, c), 3)
    states = [_prepare(_feats((1, 16, 16, c), 4 + r)) for r in range(2)]
    lab = np.stack([blobs(hc, wc, 2, 10 + i) for i in range(nc)])      # label 2 = unstyled strip
    lab[:, 0, 3] = 1                                                    # and region 1 ...
    lab[1, :, :] = np.where(lab[1] == 1, 0, lab[1])
    lab[1, 5, 5] = 1                                                    # ... a single pixel in frame 1: skipped
    cin, out, k = _apply_regions(content, lab, states, 1.0)
    assert k[1 * 2 + 1] == -1
    planes_in = cin.view(torch.int16).view(2, nc, hc + 2, wc + 2, c).cpu().numpy()
    planes_out = out.view(torch.int16).view(2, nc, hc + 2, wc + 2, c).cpu().numpy()
    # padded cell -> the interior pixel it holds (reflect halo)
    ry = np.abs(np.arange(hc + 2) - 1)
    ry = np.where(ry > hc - 1, 2 * (hc - 1) - ry, ry)
    rx = np.abs(np.arange(wc + 2) - 1)
    rx = np.where(rx > wc - 1, 2 * (wc - 1) - rx, rx)
    keep = lab >= 2
    keep[1] |= lab[1] == 1
    kp = keep[:, ry[:, None], rx[None, :]]                              # [n, hc+2, wc+2]
    assert np.array_equal(planes_out[:, kp], planes_in[:, kp])
    assert not np.array_equal(planes_out[:, ~kp], planes_in[:, ~kp])


def test_bad_region_count_is_rejected():
    c = 64
    state = _prepare(_feats((1, 8, 8, c), 1))
    with pytest.raises(_capi.WctB200Error):
        _apply_regions(_feats((1, 8, 8, c), 2), np.zeros((1, 8, 8), np.uint8), [state] * 9, 1.0)


def _teacher_forced_regions(weights, sem, mask, csize, ssizes, alpha=0.8, seed=100):
    targets = ALL
    R = len(ssizes)
    eng = Engine(weights, targets, semantics=sem)
    rng = np.random.default_rng(seed)
    content = rng.integers(0, 256, (1, csize, csize, 3), dtype=np.uint8)
    styles = [rng.integers(0, 256, (1, s, s, 3), dtype=np.uint8) for s in ssizes]
    cap = {}
    out = eng.stylize(torch.from_numpy(content).cuda(), None, alpha=alpha, want_info=True, capture=cap,
                      labels=torch.from_numpy(mask).cuda(), region_styles=[torch.from_numpy(s).cuda() for s in styles])
    eng.check_device()
    sfe = [nets.encode(nets.preprocess(s).astype(np.float64), weights, targets, np.float64) for s in styles]
    worst = 0.0
    for i, relu in enumerate(targets):
        x = cap["level_input"][i].cpu().numpy().astype(np.float64)
        cf = nets.encode(x, weights, [relu], np.float64)[relu]
        got_cf = eng.act_to_f32(cap["content_feat"][i]).cpu().numpy()
        e_enc = np.abs(got_cf - cf).max()
        lab = resize_labels(mask, cf.shape[1], cf.shape[2])
        f, info = wct_regions(cf, [s[relu] for s in sfe], lab, alpha, sem, return_info=True)
        k = eng.last_info[i].cpu().numpy()
        for r, inf in enumerate(info):
            if inf["k_c"] >= 0:
                assert ref_ops.spectral_gap_ok(inf["wc"]), "ill-posed vector (%s, region %d)" % (relu, r)
            assert ref_ops.spectral_gap_ok(inf["ws"])
            assert (k[r], k[R + r]) == (inf["k_c"], inf["k_s"]), (relu, r, k, inf["k_c"], inf["k_s"])
        got_f = eng.act_to_f32(cap["transformed"][i]).cpu().numpy()
        e_wct = np.abs(got_f - f).max()
        y = nets.decode(np.asarray(f, dtype=np.float64), weights, relu, np.float64)
        if i < len(targets) - 1:
            y = np.clip(y, 0, 1)
        e_out = np.abs(cap["level_output"][i].cpu().numpy() - y).max()
        print("%s %dx%d R=%d: encoder %.2e  transform %.2e  level output %.2e" % (relu, csize, csize, R, e_enc, e_wct, e_out))
        worst = max(worst, e_enc, e_wct, e_out)
    assert out.shape == (1, csize, csize, 3)
    return worst


@pytest.mark.parametrize("sem", ["tf", "np"])
@pytest.mark.parametrize("R", [2, 3])
def test_teacher_forced_regions_128(weights, sem, R):
    mask = halves(128, 128) if R == 2 else blobs(128, 128, R, 5)
    ssizes = [144, 96, 112][:R]
    assert _teacher_forced_regions(weights, sem, mask, 128, ssizes) <= 1e-3


def test_teacher_forced_regions_512_tf(weights):
    # top 3/4 vs bottom 1/4: at relu5_1 (32 x 32, C = 512) the regions hold 768 and 256 pixels.  Halves would give 512 pixels
    # for 512 channels, whose covariance has eigenvalues around the 1e-5 cut (an ill-posed vector for any fp32 engine).
    mask = np.zeros((512, 512), np.uint8)
    mask[384:] = 1
    assert _teacher_forced_regions(weights, "tf", mask, 512, [512, 256], seed=1000) <= 1e-3


def test_free_running_regions_vs_oracle(weights):
    size = 128
    rng = np.random.default_rng(1000)
    content = rng.integers(0, 256, (1, size, size, 3), dtype=np.uint8)
    styles = [rng.integers(0, 256, (1, s, s, 3), dtype=np.uint8) for s in (128, 96)]
    mask = blobs(97, 131, 2, 8)                                         # any resolution: sampled per level
    o64 = pipeline_regions(content[0], [s[0] for s in styles], mask, weights, ALL, alpha=0.8, semantics="np", dtype=np.float64)
    o32 = pipeline_regions(content[0], [s[0] for s in styles], mask, weights, ALL, alpha=0.8, semantics="np", dtype=np.float32)
    eng = Engine(weights, ALL, semantics="np")
    out = eng.stylize(torch.from_numpy(content).cuda(), None, alpha=0.8, labels=torch.from_numpy(mask).cuda(),
                      region_styles=[torch.from_numpy(s).cuda() for s in styles])
    eng.check_device()
    noise = np.abs(o32 - o64).max()
    err = np.abs(out.cpu().numpy() - o64).max()
    print("free-running masked 5-level: engine-vs-fp64 oracle %.3e ; oracle fp32-vs-fp64 %.3e" % (err, noise))
    assert err <= max(1e-3, FREE_RUN_NOISE_FACTOR * noise)


def test_predict_batch_mask_all_zero_equals_unmasked(weights):
    wct = WCT(checkpoints=None, relu_targets=ALL, vgg_path=None, weights=weights)
    rng = np.random.default_rng(3)
    c = rng.integers(0, 256, (3, 96, 80, 3), dtype=np.uint8)
    s = rng.integers(0, 256, (70, 90, 3), dtype=np.uint8)
    plain = wct.predict_batch(c, s, alpha=0.8)
    masked = wct.predict_batch(c, [s], alpha=0.8, content_mask=np.zeros((50, 40), np.uint8))
    assert np.array_equal(masked, plain)


def test_batch_with_different_masks_equals_single_frames(weights):
    wct = WCT(checkpoints=None, relu_targets=ALL, vgg_path=None, weights=weights)
    assert wct.engine.groups == 2
    rng = np.random.default_rng(4)
    c = rng.integers(0, 256, (3, 64, 96, 3), dtype=np.uint8)
    styles = [rng.integers(0, 256, (s, s, 3), dtype=np.uint8) for s in (64, 80, 48)]
    masks = np.stack([halves(64, 96), blobs(64, 96, 3, 1), blobs(64, 96, 3, 2)])
    batch = wct.predict_batch(c, styles, alpha=0.8, content_mask=masks)
    for i in range(3):
        one = wct.predict_batch(c[i:i + 1], styles, alpha=0.8, content_mask=masks[i])
        assert np.array_equal(one[0], batch[i])


def test_mask_with_adain_or_swap5_is_rejected(weights):
    wct = WCT(checkpoints=None, relu_targets=ALL, vgg_path=None, weights=weights)
    c = np.zeros((32, 32, 3), np.uint8)
    with pytest.raises(ValueError):
        wct.predict(c, [c], adain=True, content_mask=np.zeros((32, 32), np.uint8))
    with pytest.raises(ValueError):
        wct.predict(c, [c], swap5=True, content_mask=np.zeros((32, 32), np.uint8))
