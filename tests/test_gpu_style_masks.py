"""Style masks on the GPU: the masked style prepare against wct_style_prepare and the fp64 oracle, the empty-region
sentinel in the regions apply, the masked pipeline against tests/style_masks_ref.py, byte identity with today's
content-mask calls, invariance, sharing of one (style, mask) side, and the rejections."""
import numpy as np
import pytest
import torch

import tests.gpu_util as U
from oracle import nets, ref_ops
from tests.regions_ref import resize_labels
from tests.style_masks_ref import pipeline_style_masks, wct_style_masks
from tests.test_gpu_pipeline import ALL, FREE_RUN_NOISE_FACTOR
from tests.test_gpu_regions import _apply_regions, _feats, _prepare, blobs, halves
from tests.texture_ref import noise_u8 as oracle_noise
from wct_tf_b200 import _capi
from wct_tf_b200.engine import Engine, SEMANTICS
from wct_tf_b200.prepared import slice_wct_state, unpack_wct_state
from wct_tf_b200.weights import make_synthetic_weights
from wct_tf_b200.wct import WCT

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def weights():
    return make_synthetic_weights(42)


@pytest.fixture(scope="module")
def wct(weights):
    return WCT(checkpoints=None, relu_targets=ALL, vgg_path=None, weights=weights)


def _prepare_regions(style, lab, R, sem="tf"):
    """wctb200_wct_style_prepare_regions of one style feature map (float32 [1,Hs,Ws,C]) -> (state, k_out)."""
    lib = U.lib()
    _, hs, ws_, c = style.shape
    sp = SEMANTICS[sem]
    sin = U.act_from_numpy(style)
    ws = torch.empty(lib.wctb200_wct_style_prepare_regions_workspace_bytes(c, R, hs, ws_), dtype=torch.uint8, device="cuda")
    state = torch.empty(lib.wctb200_wct_style_state_bytes(c, R), dtype=torch.uint8, device="cuda")
    k = torch.zeros(2 * R, dtype=torch.int32, device="cuda")
    _capi.check(lib.wctb200_wct_style_prepare_regions(sin.data_ptr(), hs, ws_, c, U.dev(lab).data_ptr(), R, sp["eps_cov"],
                                                      sp["eps_eig"], sp["thresh"], state.data_ptr(), k.data_ptr(), ws.data_ptr(),
                                                      ws.numel(), U.stream()))
    U.check_device()
    return state, k.cpu().numpy()


# ---------------------------------------------------------------------------------------------------------- C-ABI
@pytest.mark.parametrize("c", [64, 128, 256, 512])
def test_uniform_mask_entry_is_byte_identical_to_wct_style_prepare(c):
    style = _feats((1, 21, 34, c), c)
    ref = unpack_wct_state(U.lib(), _prepare(style), c, 1)
    for R in (1, 2, 4):
        for r in range(R):
            state, k = _prepare_regions(style, np.full((21, 34), r, np.uint8), R)
            mean, cs, kk = unpack_wct_state(U.lib(), state, c, R)
            assert np.array_equal(mean[r].view(np.int32), ref[0][0].view(np.int32)), (R, r)
            assert np.array_equal(cs[r].view(np.int32), ref[1][0].view(np.int32)), (R, r)
            assert tuple(kk[r]) == tuple(ref[2][0]) and k[r] == ref[2][0][0]
            for o in range(R):
                if o != r:
                    assert tuple(kk[o]) == (-1, 0) and not mean[o].any() and not cs[o].any()


def _oracle_side(px, sem, dtype):
    """mean, C_s^2 (kept part, + eps_eig) and k_s of a pixel set [m, C] in ``dtype`` (wct_generic's style side)."""
    sp = SEMANTICS[sem]
    x = px.astype(dtype)
    ms = x.mean(0)
    cov = np.cov(x.T).astype(dtype) + np.eye(x.shape[1], dtype=dtype) * dtype(sp["eps_cov"])
    E, w, _ = np.linalg.svd(cov)
    k = int((w > sp["thresh"]).sum())
    return ms, (E[:, :k] * (w[:k] + sp["eps_eig"])) @ E[:, :k].T, k


@pytest.mark.parametrize("sem", ["tf", "np"])
@pytest.mark.parametrize("case", ["halves", "blobs", "ragged"])
def test_masked_prepare_matches_float64(sem, case):
    shapes = {"halves": (24, 40, 128), "blobs": (37, 45, 64), "ragged": (19, 27, 256)}
    hs, ws_, c = shapes[case]
    R = 3
    style = _feats((1, hs, ws_, c), hs + ws_)
    lab = {"halves": halves(hs, ws_), "blobs": blobs(hs, ws_, R, 7), "ragged": blobs(hs, ws_, R, 9)}[case]
    state, _ = _prepare_regions(style, lab, R, sem)
    mean, cs, k = unpack_wct_state(U.lib(), state, c, R)
    px_all = U.split_repr(style)[0]
    for r in range(R):
        px = px_all[lab == r]
        if len(px) < 2:
            assert tuple(k[r]) == (-1, 0)
            continue
        m64, s64, k64 = _oracle_side(px, sem, np.float64)
        _, _, k32 = _oracle_side(px, sem, np.float32)
        assert np.abs(mean[r] - m64).max() <= 1e-6 * max(1.0, np.abs(m64).max()), (r, np.abs(mean[r] - m64).max())
        got = cs[r].astype(np.float64) @ cs[r].T.astype(np.float64)
        err = np.abs(got - s64).max() / np.abs(s64).max()
        print("%s %s region %d (%d px, C %d): k_s %d / %d, C_s C_s^T rel err %.2e" % (case, sem, r, len(px), c, k[r][0], k64, err))
        assert err <= 2e-4
        if k32 == k64:
            assert k[r][0] == k64


def test_empty_style_region_keeps_the_content_interior_and_halo():
    nc, hc, wc, c = 2, 19, 45, 128
    content = _feats((nc, hc, wc, c), 3)
    style = _feats((1, 16, 16, c), 4)
    state, k = _prepare_regions(style, np.zeros((16, 16), np.uint8), 2)        # entry 1: no pixel
    assert tuple(k) == (k[0], -1, k[2], 0) and k[0] > 0
    states = [slice_wct_state(U.lib(), state, c, 2, r, r + 1) for r in range(2)]
    lab = np.stack([halves(hc, wc), blobs(hc, wc, 2, 11, strip=False)])
    cin, out, kout = _apply_regions(content, lab, states, 1.0)
    R = 2
    assert kout[0 * R + 1] == -1 and kout[1 * R + 1] == -1 and kout[0] > 0 and kout[nc * R + 1] == -1
    planes_in = cin.view(torch.int16).view(2, nc, hc + 2, wc + 2, c).cpu().numpy()
    planes_out = out.view(torch.int16).view(2, nc, hc + 2, wc + 2, c).cpu().numpy()
    ry = np.abs(np.arange(hc + 2) - 1)
    ry = np.where(ry > hc - 1, 2 * (hc - 1) - ry, ry)
    rx = np.abs(np.arange(wc + 2) - 1)
    rx = np.where(rx > wc - 1, 2 * (wc - 1) - rx, rx)
    kp = (lab == 1)[:, ry[:, None], rx[None, :]]
    assert np.array_equal(planes_out[:, kp], planes_in[:, kp])
    assert not np.array_equal(planes_out[:, ~kp], planes_in[:, ~kp])


# ---------------------------------------------------------------------------------------------------------- pipeline
def _teacher_forced(weights, sem, mask, smasks, csize, ssizes, alpha=0.8, seed=200):
    targets = ALL
    R = len(ssizes)
    eng = Engine(weights, targets, semantics=sem)
    rng = np.random.default_rng(seed)
    content = rng.integers(0, 256, (1, csize, csize, 3), dtype=np.uint8)
    styles = [rng.integers(0, 256, (1, s, s, 3), dtype=np.uint8) for s in ssizes]
    cap = {}
    eng.stylize(torch.from_numpy(content).cuda(), None, alpha=alpha, want_info=True, capture=cap, labels=torch.from_numpy(mask).cuda(),
                region_styles=[torch.from_numpy(s).cuda() for s in styles],
                region_masks=[None if m is None else torch.from_numpy(m).cuda() for m in smasks])
    eng.check_device()
    sfe = [nets.encode(nets.preprocess(s).astype(np.float64), weights, targets, np.float64) for s in styles]
    worst, empty = 0.0, 0
    for i, relu in enumerate(targets):
        x = cap["level_input"][i].cpu().numpy().astype(np.float64)
        cf = nets.encode(x, weights, [relu], np.float64)[relu]
        lab = resize_labels(mask, cf.shape[1], cf.shape[2])
        sfs = [s[relu] for s in sfe]
        slabs = [None if m is None else resize_labels(m, sf.shape[1], sf.shape[2]) for m, sf in zip(smasks, sfs)]
        f, info = wct_style_masks(cf, sfs, lab, slabs, alpha, sem, return_info=True)
        k = eng.last_info[i].cpu().numpy()
        for r, inf in enumerate(info):
            empty += inf["k_s"] == -1
            if inf["k_c"] >= 0:
                assert ref_ops.spectral_gap_ok(inf["wc"]) and ref_ops.spectral_gap_ok(inf["ws"]), (relu, r)
            assert (k[r], k[R + r]) == (inf["k_c"], inf["k_s"]), (relu, r, k, inf["k_c"], inf["k_s"])
        e = np.abs(eng.act_to_f32(cap["transformed"][i]).cpu().numpy() - f).max()
        print("%s %s: transform %.2e" % (sem, relu, e))
        worst = max(worst, e)
    return worst, empty


def test_teacher_forced_style_masks_tf(weights):
    # sky / sea: region r of the content takes region r of ONE painting
    smask = np.zeros((144, 144), np.uint8)
    smask[:60] = 1
    worst, _ = _teacher_forced(weights, "tf", halves(128, 128), [smask, smask], 128, [144, 144])
    assert worst <= 1e-3


def test_teacher_forced_style_masks_np_with_a_vanishing_style_region(weights):
    # style 1's region is a 6-row strip: no relu5_1 sample falls in it (the sentinel), the finer levels see it
    smask = np.zeros((144, 144), np.uint8)
    smask[:6] = 1
    worst, empty = _teacher_forced(weights, "np", blobs(128, 128, 2, 5), [None, smask], 128, [112, 144])
    assert empty >= 1
    assert worst <= 1e-3


def test_free_running_style_masks_vs_oracle(weights):
    rng = np.random.default_rng(1001)
    content = rng.integers(0, 256, (1, 128, 128, 3), dtype=np.uint8)
    style = rng.integers(0, 256, (1, 128, 160, 3), dtype=np.uint8)
    mask, smask = blobs(97, 131, 2, 8), blobs(61, 77, 2, 3)            # any resolutions
    args = (content[0], [style[0], style[0]], mask, [smask, smask], weights, ALL)
    o64 = pipeline_style_masks(*args, alpha=0.8, semantics="np", dtype=np.float64)
    o32 = pipeline_style_masks(*args, alpha=0.8, semantics="np", dtype=np.float32)
    eng = Engine(weights, ALL, semantics="np")
    s, m = torch.from_numpy(style).cuda(), torch.from_numpy(smask).cuda()
    out = eng.stylize(torch.from_numpy(content).cuda(), None, alpha=0.8, labels=torch.from_numpy(mask).cuda(), region_styles=[s, s],
                      region_masks=[m, m])
    eng.check_device()
    noise = np.abs(o32 - o64).max()
    err = np.abs(out.cpu().numpy() - o64).max()
    print("free-running style-masked 5-level: engine-vs-fp64 %.3e ; oracle fp32-vs-fp64 %.3e" % (err, noise))
    assert err <= max(1e-3, FREE_RUN_NOISE_FACTOR * noise)


# ---------------------------------------------------------------------------------------------------------- WCT API
def _inputs(seed, n=3):
    rng = np.random.default_rng(seed)
    c = rng.integers(0, 256, (n, 64, 96, 3), dtype=np.uint8)
    styles = [rng.integers(0, 256, (s, s + 8, 3), dtype=np.uint8) for s in (56, 72)]
    return c, styles, blobs(64, 96, 2, seed, strip=True)


def test_none_and_uniform_style_masks_are_byte_identical_to_the_content_mask_call(wct):
    c, styles, mask = _inputs(3)
    plain = wct.predict_batch(c, styles, alpha=0.8, content_mask=mask)
    assert np.array_equal(wct.predict_batch(c, styles, alpha=0.8, content_mask=mask, style_masks=[None, None]), plain)
    uniform = [np.full((5, 7), r, np.uint8) for r in range(2)]
    assert np.array_equal(wct.predict_batch(c, styles, alpha=0.8, content_mask=mask, style_masks=uniform), plain)


def test_batch_groups_passes_and_synthesize_are_invariant(wct):
    c, styles, mask = _inputs(4)
    painting = styles[1]
    sm = blobs(72, 80, 2, 6, strip=False)
    kw = dict(alpha=0.8, content_mask=mask, style_masks=[sm, sm])
    batch = wct.predict_batch(c, [painting, painting], **kw)
    for i in range(3):
        assert np.array_equal(wct.predict_batch(c[i:i + 1], [painting, painting], **kw)[0], batch[i])
    wct.engine.groups = 1
    try:
        assert np.array_equal(wct.predict_batch(c, [painting, painting], **kw), batch)
    finally:
        wct.engine.groups = 2
    two = wct.predict_batch(c, [painting, painting], passes=2, **kw)
    assert np.array_equal(two, wct.predict_batch(batch, [painting, painting], **kw))
    tex = wct.synthesize([painting, painting], (64, 96), count=3, seed=17, **kw)
    assert np.array_equal(tex, wct.predict_batch(oracle_noise(3, 64, 96, seed=17), [painting, painting], **kw))


def test_shared_style_and_mask_launch_one_encode(wct):
    c, styles, _ = _inputs(5, n=1)
    R = 3
    mask = np.repeat(np.arange(R, dtype=np.uint8), 32)[None].repeat(64, 0)
    sm = blobs(72, 80, R, 2, strip=False)
    copies = [styles[1].copy() for _ in range(R)]
    eng = wct.engine

    def launches(ss):
        n0 = eng.launches
        wct.predict_batch(c, ss, alpha=0.8, content_mask=mask, style_masks=[sm] * R)
        return eng.launches - n0

    shared, distinct = launches([styles[1]] * R), launches(copies)
    # one masked style side: the u8 -> f32 conversion, one encoder pass, and a labels resize and a masked prepare per level
    sdev, mdev = torch.from_numpy(styles[1][None]).cuda(), torch.from_numpy(sm).cuda()
    n0 = eng.launches
    eng.prepare_regions_call([sdev], eng.check_region_masks([mdev], [sdev]))
    eng.check_device()
    per_side = eng.launches - n0
    assert per_side > 0 and distinct - shared == (R - 1) * per_side, (shared, distinct, per_side)
    # the shared call's output is the distinct call's
    a = wct.predict_batch(c, [styles[1]] * R, alpha=0.8, content_mask=mask, style_masks=[sm] * R)
    b = wct.predict_batch(c, copies, alpha=0.8, content_mask=mask, style_masks=[sm] * R)
    assert np.array_equal(a, b)


def test_style_mask_rejections(wct):
    c = np.zeros((32, 32, 3), np.uint8)
    s = np.full((32, 32, 3), 7, np.uint8)
    m = np.zeros((32, 32), np.uint8)
    ps = wct.prepare_style(s)
    bad = [dict(style=[s, s], content_mask=m, style_masks=[m]),                       # not one entry per style
           dict(style=[s], content_mask=m, style_masks=[m.astype(np.int32)]),         # not uint8
           dict(style=[s], content_mask=m, style_masks=[m[None]]),                    # not 2-D
           dict(style=[s], style_masks=[m]),                                          # no content mask
           dict(style=[ps], content_mask=m, style_masks=[m]),                         # a prepared style has no features
           dict(style=[s], content_mask=m, style_masks=[m], adain=True),
           dict(style=[s], content_mask=m, style_masks=[m], swap5=True),
           dict(style=[s], content_mask=m, style_masks=[m], style_weights=[1.0])]
    for kw in bad:
        style = kw.pop("style")
        with pytest.raises(ValueError):
            wct.predict(c, style, **kw)
        with pytest.raises(ValueError):
            wct.predict_batch(c[None], style, **kw)
    # a prepared style without a mask is fine next to a masked image
    out = wct.predict(c, [ps, s], content_mask=halves(32, 32), style_masks=[None, m])
    assert out.shape == (32, 32, 3)
