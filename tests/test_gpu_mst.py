"""Multimodal style transfer on the GPU: the ICM kernel bit for bit against tests/mst_ref.py, the data term against float64,
the k-means++ draws and the Lloyd fixed point against the oracle, the engine against ``pipeline_mst`` teacher-forced on the
device's labels, byte identity of K = 1 with plain WCT, a semantic check on flat colours, invariance, and the rejections."""
import numpy as np
import pytest
import torch

import tests.gpu_util as U
from oracle import nets
from tests import mst_ref as M
from tests.regions_ref import resize_labels
from tests.style_masks_ref import wct_style_masks
from tests.test_gpu_pipeline import ALL
from tests.texture_ref import noise_u8 as oracle_noise
from wct_tf_b200 import _capi
from wct_tf_b200.engine import Engine
from wct_tf_b200.weights import make_synthetic_weights
from wct_tf_b200.wct import WCT

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def weights():
    return make_synthetic_weights(42)


@pytest.fixture(scope="module")
def wct(weights):
    return WCT(checkpoints=None, relu_targets=ALL, vgg_path=None, weights=weights)


# ---------------------------------------------------------------------------------------------------------- C-ABI
def _smooth(D, lam, sweeps=M.SWEEPS):
    N, H, W, K = D.shape
    d = U.dev(np.ascontiguousarray(D, np.float32))
    lab = torch.full((N, H, W), 77, dtype=torch.uint8, device="cuda")
    _capi.check(U.lib().wctb200_mst_smooth(d.data_ptr(), N, H, W, K, float(lam), sweeps, lab.data_ptr(), U.stream()))
    U.check_device()
    return lab.cpu().numpy()


def _data_term(feat, centres, counts):
    N, H, W, C = feat.shape
    K = centres.shape[0]
    buf = U.act_from_numpy(feat)
    D = torch.empty((N, H, W, K), dtype=torch.float32, device="cuda")
    cen, cnt = U.dev(centres.astype(np.float32)), U.dev(np.asarray(counts, np.int32))     # alive until the kernel has run
    _capi.check(U.lib().wctb200_mst_data_term(buf.data_ptr(), N, H, W, C, cen.data_ptr(), cnt.data_ptr(), K, D.data_ptr(),
                                              U.stream()))
    U.check_device()
    return D.cpu().numpy()


def _clusters(feat, K, level):
    """wctb200_mst_style_clusters of feat float32 [Hs,Ws,C] -> (labels [Hs,Ws], centres [K,C], info, oracle unit directions)."""
    lib = U.lib()
    Hs, Ws, C = feat.shape
    buf = U.act_from_numpy(feat[None])
    lab = torch.full((Hs * Ws,), 77, dtype=torch.uint8, device="cuda")
    cen = torch.empty((K, C), dtype=torch.float32, device="cuda")
    info = torch.empty(2 * K + 1, dtype=torch.int32, device="cuda")
    ws = torch.empty(lib.wctb200_mst_style_clusters_workspace_bytes(Hs, Ws, C, K), dtype=torch.uint8, device="cuda")
    _capi.check(lib.wctb200_mst_style_clusters(buf.data_ptr(), Hs, Ws, C, K, level, lab.data_ptr(), cen.data_ptr(), info.data_ptr(),
                                               ws.data_ptr(), ws.numel(), U.stream()))
    U.check_device()
    return (lab.cpu().numpy().reshape(Hs, Ws), cen.cpu().numpy().astype(np.float64), info.cpu().numpy(),
            M.unit(U.split_repr(feat).reshape(-1, C)))


def _blobs(shape, K, seed, noise=0.3):
    H, W, C = shape
    rng = np.random.default_rng(seed)
    dirs = rng.standard_normal((K, C))
    truth = rng.integers(0, K, H * W)
    f = dirs[truth] + noise * rng.standard_normal((H * W, C))
    return f.reshape(H, W, C).astype(np.float32), truth


@pytest.mark.parametrize("lam", [0.0, 0.05, 1.0])
@pytest.mark.parametrize("K", [2, 3, 4, 5, 6, 7, 8])
def test_smooth_is_bit_identical_to_the_oracle(K, lam):
    for i, (N, H, W) in enumerate([(3, 13, 17), (2, 1, 9), (2, 8, 1), (1, 31, 29), (2, 64, 48)]):
        rng = np.random.default_rng(100 * K + i)
        D = (np.floor(rng.random((N, H, W, K)) * 24) / 64).astype(np.float32)     # coarse values: many exact ties
        if K >= 3:
            D[..., 1] = np.inf
        if K >= 5:
            D[0, 0, 0, :] = np.inf                                             # a pixel with no finite cost
        assert np.array_equal(_smooth(D, lam), M.icm(D, lam)), (N, H, W)
    if lam == 0.0:
        assert np.array_equal(_smooth(D, lam, sweeps=0), np.argmin(D, -1))


@pytest.mark.parametrize("C", [64, 128, 256, 512])
def test_data_term_against_float64(C):
    rng = np.random.default_rng(C)
    feat = (rng.standard_normal((2, 9, 11, C)) * rng.random((2, 9, 11, 1)) * 3).astype(np.float32)
    feat[1, 4, 5] = 0
    centres = M.unit(rng.standard_normal((5, C)))
    counts = [5, 1, 9, 0, 3]
    got = _data_term(feat, centres.astype(np.float32), counts)
    ref = M.data_term(U.split_repr(feat), centres.astype(np.float32).astype(np.float64), counts)
    assert np.array_equal(np.isinf(got), np.isinf(ref)) and np.isinf(got[..., [1, 3]]).all()
    fin = np.isfinite(ref)
    err = np.abs(got[fin] - ref[fin]).max()
    print("C=%d data term max err %.2e" % (C, err))
    assert err <= 1e-6


@pytest.mark.parametrize("C,K,blobs", [(64, 4, True), (512, 3, True), (128, 5, False), (256, 8, False)])
def test_kmeanspp_draws_are_valid(C, K, blobs):
    feat = _blobs((37, 41, C), K, C + K)[0] if blobs else np.random.default_rng(C).standard_normal((37, 41, C)).astype(np.float32)
    _, _, info, u = _clusters(feat, K, level=3)
    M.check_draws(u, list(info[:K]), level=3, tol=1e-5)
    # the same feature, level and K give the same draws; another level others
    assert np.array_equal(_clusters(feat, K, level=3)[2], info)
    assert not np.array_equal(_clusters(feat, K, level=1)[2][:K], info[:K])


@pytest.mark.parametrize("C,K,level", [(64, 3, 0), (256, 6, 2), (512, 8, 4)])
def test_lloyd_step_teacher_forced_on_the_device_state(C, K, level):
    feat, _ = _blobs((29, 33, C), K, 7 * C + K, noise=0.8)
    lab, cen, info, u = _clusters(feat, K, level)
    lab = lab.reshape(-1)
    it = int(info[K])
    assert 1 <= it < M.LLOYD_MAX, info
    assert np.array_equal(info[K + 1:], np.bincount(lab, minlength=K))
    # the centres are the update of the device's labels, and the labels the assign of the centres (the loop converged)
    assert np.abs(M.update(u, lab, cen) - cen).max() <= 1e-6
    again, margin = M.assign(u, cen)
    bad = (again != lab) & (margin >= 1e-5)
    assert not bad.any(), np.flatnonzero(bad)[:10]


@pytest.mark.parametrize("C,K", [(64, 3), (512, 4)])
def test_blobs_partition_equals_the_oracle(C, K):
    feat, truth = _blobs((40, 40, C), K, 3 * C + K, noise=0.2)
    lab, cen, info, u = _clusters(feat, K, level=1)
    olab, oc, oit, ocnt = M.lloyd(u, list(info[:K]))
    assert np.array_equal(lab.reshape(-1), olab)
    assert np.abs(cen - oc).max() <= 1e-6 and int(info[K]) == oit
    perm = {int(t): int(l) for t, l in zip(truth, olab)}
    assert np.array_equal(np.vectorize(perm.get)(truth), olab)


def test_k1_labels_are_zero():
    feat = np.random.default_rng(0).standard_normal((12, 10, 128)).astype(np.float32)
    lab, cen, info, u = _clusters(feat, 1, level=0)
    assert not lab.any() and info[2] == 120
    assert np.abs(cen[0] - M.unit(u.sum(0))).max() <= 1e-6


# ---------------------------------------------------------------------------------------------------------- engine
def _imgs(seed, n, hw, shw):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (n,) + hw + (3,), dtype=np.uint8), rng.integers(0, 256, shw + (3,), dtype=np.uint8)


@pytest.mark.parametrize("sem", ["tf", "np"])
def test_mst_1_is_byte_identical_to_plain_wct(weights, sem):
    m = WCT(checkpoints=None, relu_targets=ALL, vgg_path=None, weights=weights, semantics=sem)
    c, s = _imgs(1, 3, (64, 80), (72, 64))
    u8, f = m.predict_batch(c, s, alpha=0.8, return_float=True)
    u8m, fm = m.predict_batch(c, s, alpha=0.8, return_float=True, mst=1, mst_smooth=0.3)
    assert np.array_equal(u8, u8m) and np.array_equal(f.view(np.int32), fm.view(np.int32))


@pytest.mark.parametrize("sem", ["tf", "np"])
def test_teacher_forced_levels_against_pipeline_mst(weights, sem):
    K, lam, alpha = 3, 0.05, 0.8
    eng = Engine(weights, ALL, semantics=sem)
    c, s = _imgs(11, 1, (128, 128), (144, 144))
    cap = {}
    eng.stylize(torch.from_numpy(c).cuda(), torch.from_numpy(s[None]).cuda(), alpha=alpha, capture=cap, mst=K, mst_smooth=lam)
    eng.check_device()
    sfe = nets.encode(nets.preprocess(s[None]).astype(np.float64), weights, ALL, np.float64)
    worst, agree = 0.0, []
    for i, relu in enumerate(ALL):
        slab = cap["mst_style_labels"][i].cpu().numpy()[0]
        clab = cap["mst_content_labels"][i].cpu().numpy()[0]
        cen = cap["mst_centres"][i].cpu().numpy().astype(np.float64)
        info = cap["mst_info"][i].cpu().numpy()
        assert np.array_equal(info[K + 1:], np.bincount(slab.reshape(-1), minlength=K)), relu
        x = cap["level_input"][i].cpu().numpy().astype(np.float64)
        cf = nets.encode(x, weights, [relu], np.float64)[relu]
        f = wct_style_masks(cf, [sfe[relu]] * K, clab, [slab] * K, alpha, sem)
        e = np.abs(eng.act_to_f32(cap["transformed"][i]).cpu().numpy() - f).max()
        # the device's content labels against the oracle's ICM on the device's own content feature and centres
        cdev = eng.act_to_f32(cap["content_feat"][i]).cpu().numpy().astype(np.float64)
        olab = M.content_labels(cdev, cen, info[K + 1:], lam)[0]
        agree.append(float((olab == clab).mean()))
        print("%s %s: transform %.2e, label agreement %.4f, iterations %d" % (sem, relu, e, agree[-1], info[K]))
        worst = max(worst, e)
    assert worst <= 1e-3
    assert min(agree) >= 0.99, agree


@pytest.mark.parametrize("relu", ["relu3_1", "relu2_1", "relu1_1"])
def test_semantic_flat_colours(relu):
    # one level per model, so that the level's content is the flat image itself (a later level of a chain would see the
    # decoded output of the level before it)
    m = WCT(checkpoints=None, relu_targets=[relu], vgg_path=None, weights=make_synthetic_weights(42, relu_targets=[relu]))
    # 256^2: the feature column at the colour edge sees both colours (one column of 64 at relu2_1 of a 128^2 image)
    H = 256
    content = np.zeros((H, H, 3), np.uint8)
    content[:, :H // 2] = (220, 30, 30)
    content[:, H // 2:] = (30, 40, 220)
    style = np.zeros((H, H, 3), np.uint8)
    style[:H // 2] = (230, 20, 20)
    style[H // 2:] = (20, 30, 230)
    cmask = np.zeros((H, H), np.uint8)
    cmask[:, H // 2:] = 1
    smask = np.zeros((H, H), np.uint8)
    smask[H // 2:] = 1
    cap = {}
    out_mst = m.engine.stylize(torch.from_numpy(content[None]).cuda(), torch.from_numpy(style[None]).cuda(), alpha=1.0, capture=cap,
                               mst=2, mst_smooth=0.05).cpu().numpy()
    lab = cap["mst_content_labels"][0].cpu().numpy()[0]
    hand = resize_labels(cmask, lab.shape[0], lab.shape[1])
    a = max((lab == hand).mean(), (lab == 1 - hand).mean())
    _, out_masks = m.predict_batch(content, [style, style], alpha=1.0, content_mask=cmask, style_masks=[smask, smask],
                                   return_float=True)
    _, out_plain = m.predict_batch(content, style, alpha=1.0, return_float=True)
    d_masks, d_plain = np.abs(out_mst - out_masks).mean(), np.abs(out_mst - out_plain).mean()
    print("%s: agreement with the hand mask %.4f; mean |mst - masks| %.4f, |mst - plain| %.4f" % (relu, a, d_masks, d_plain))
    assert a >= 0.99
    assert d_masks < d_plain


def test_frames_do_not_depend_on_batch_groups_passes(wct):
    c, s = _imgs(5, 30, (64, 64), (64, 80))
    kw = dict(alpha=0.9, mst=3, mst_smooth=0.05)
    wct.engine.groups = 2
    out30 = wct.predict_batch(c, s, **kw)
    assert np.array_equal(wct.predict_batch(c[:7], s, **kw), out30[:7])
    assert np.array_equal(wct.predict_batch(c[12:13], s, **kw), out30[12:13])
    wct.engine.groups = 1
    try:
        assert np.array_equal(wct.predict_batch(c, s, **kw), out30)
    finally:
        wct.engine.groups = 2
    two = wct.predict_batch(c[:4], s, passes=2, **kw)
    assert np.array_equal(two, wct.predict_batch(out30[:4], s, **kw))
    syn = wct.synthesize(s, 64, count=3, seed=9, first_index=2, **kw)
    assert np.array_equal(syn, wct.predict_batch(oracle_noise(3, 64, 64, seed=9, first_index=2), s, **kw))


def test_temporal_acts_after_the_pipeline(wct):
    c, s = _imgs(6, 3, (64, 64), (64, 64))
    plain = wct.predict_batch(c, s, mst=2)
    st = wct.temporal_state(0.5)
    out = wct.predict_batch(c, s, mst=2, temporal=st)
    assert np.array_equal(out[0], plain[0]) and out.shape == plain.shape


@pytest.mark.parametrize("kw", [dict(mst=0), dict(mst=9), dict(mst=2.0), dict(mst=2, mst_smooth=-1.0),
                                dict(mst=2, mst_smooth=float("nan")), dict(mst=2, adain=True), dict(mst=2, ost=True),
                                dict(mst=2, swap5=True), dict(mst=2, swap_targets=["relu3_1"]), dict(mst=2, tile_size=64),
                                dict(mst=2, seamless="x")],
                         ids=["k0", "k9", "kfloat", "lam_neg", "lam_nan", "adain", "ost", "swap5", "swap_targets", "tiles",
                              "seamless"])
def test_rejections(wct, kw):
    c, s = _imgs(7, 2, (64, 64), (64, 64))
    with pytest.raises(ValueError):
        wct.predict_batch(c, s, **kw)


def test_rejections_of_styles_and_modes(wct):
    c, s = _imgs(8, 2, (64, 64), (64, 64))
    with pytest.raises(ValueError):
        wct.predict_batch(c, np.stack([s, s]), mst=2)                       # one style per frame
    with pytest.raises(ValueError):
        wct.predict_batch(c, wct.prepare_style(s), mst=2)                   # a prepared style
    with pytest.raises(ValueError):
        wct.predict_batch(c, [s, s], mst=2, content_mask=np.zeros((64, 64), np.uint8))
    with pytest.raises(ValueError):
        wct.predict_batch(c, [s, s], mst=2, style_weights=[1, 1])
    with pytest.raises(ValueError):
        wct.engine.stylize(torch.from_numpy(c).cuda(), wct.prepare_style(s), mst=2)
    with pytest.raises(ValueError):
        wct.predict(c[0], s, mst=2, content_mask=np.zeros((64, 64), np.uint8))
    assert wct.predict(c[0], s, mst=2).shape == (64, 64, 3)
