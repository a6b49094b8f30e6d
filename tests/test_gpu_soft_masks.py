"""Soft spatial control on the GPU (DESIGN.md §3.3.11): feathering and the area resample against float64, the weighted
record against the reliability-weighted covariance, byte identities with the hard-mask and plain paths, and the
visible behaviour of feathered masks and strength ramps."""
import numpy as np
import pytest
import torch

import tests.gpu_util as U
from oracle import nets, ref_ops
from tests.soft_masks_ref import apply_soft, feather, pipeline_soft, record_stats, resize_area, weighted_stats, wct_soft
from tests.test_gpu_pipeline import ALL, FREE_RUN_NOISE_FACTOR
from wct_tf_b200.engine import Engine
from wct_tf_b200 import _capi
from wct_tf_b200.weights import make_synthetic_weights
from wct_tf_b200.wct import WCT

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def wct():
    return WCT(checkpoints=None, relu_targets=ALL, vgg_path=None, weights=make_synthetic_weights(42))


@pytest.mark.parametrize("n,hm,wm,R,sigma", [(1, 64, 48, 2, 4.0), (2, 37, 101, 3, 1.5), (1, 9, 7, 1, 6.0)])
def test_feather_matches_fp64(n, hm, wm, R, sigma):
    lab = np.random.default_rng(hm).integers(0, R + 1, (n, hm, wm)).astype(np.uint8)
    out = torch.empty((n, R, hm, wm), dtype=torch.float32, device="cuda")
    _capi.check(U.lib().wctb200_mask_feather(U.dev(lab).data_ptr(), n, hm, wm, R, sigma, out.data_ptr(), U.stream()))
    U.check_device()
    assert np.abs(out.cpu().numpy() - feather(lab, R, sigma)).max() <= 1e-6


@pytest.mark.parametrize("hm,wm,hf,wf", [(64, 64, 64, 64), (512, 384, 32, 24), (37, 101, 9, 13), (5, 7, 33, 65)])
def test_area_resize_matches_fp64(hm, wm, hf, wf):
    m = np.random.default_rng(wm).random((2, 3, hm, wm)).astype(np.float32)
    out = torch.empty((2, 3, hf, wf), dtype=torch.float32, device="cuda")
    _capi.check(U.lib().wctb200_weights_resize_area(U.dev(m).data_ptr(), 2, 3, hm, wm, hf, wf, out.data_ptr(), U.stream()))
    U.check_device()
    got = out.cpu().numpy()
    if (hm, wm) == (hf, wf):
        assert np.array_equal(got, m)
    assert np.abs(got - resize_area(m, hf, wf)).max() <= 1e-6


def _record(buf, C, P):
    import ctypes
    o = [ctypes.c_size_t() for _ in range(4)]
    U.lib().wctb200_stats_record_layout(C, P, 0, *[ctypes.byref(x) for x in o])
    b = buf.cpu().numpy()
    f = lambda i, cnt: b[o[i].value:o[i].value + 8 * cnt].view(np.float64)
    return f(0, P), f(1, P * C).reshape(P, C), f(2, P * C).reshape(P, C), f(3, P * C * C).reshape(P, C, C)


@pytest.mark.parametrize("C", [64, 128, 256, 512])
def test_weighted_record_matches_fp64(C):
    rng = np.random.default_rng(C)
    N, H, W, K = 2, 21, 67, 4
    x = rng.standard_normal((N, H, W, C)).astype(np.float32)
    x[:, :, W // 2:, :] += 40.0                           # region 1 sits far from the frame mean
    yy, xx = np.mgrid[:H, :W]
    w = np.zeros((N, K, H, W), np.float32)
    w[:, 0] = np.clip(1.0 - xx / (W / 2.0), 0, 1)
    w[:, 1] = (xx >= W // 2) * rng.random((H, W))
    w[1, 2, 3, 5] = 0.7                                   # a problem with n_eff < 2
    # plane 3 carries no weight at all
    rec = torch.zeros(U.lib().wctb200_stats_record_layout(C, N * K, 0, None, None, None, None), dtype=torch.uint8, device="cuda")
    act = U.act_from_numpy(x)
    _capi.check(U.lib().wctb200_wct_stats_weighted(act.data_ptr(), N, H, W, C, U.dev(w).data_ptr(), K, rec.data_ptr(), U.stream()))
    U.check_device()
    rn, rt, rs, rS = _record(rec, C, N * K)
    xs = U.act_to_numpy(act, N, H, W, C).astype(np.float64)
    for n in range(N):
        for k in range(K):
            m, cov, ne = weighted_stats(xs[n], w[n, k])
            z = n * K + k
            if m is None:
                assert rn[z] == 0
                continue
            assert abs(rn[z] - ne) <= 1e-9 * ne
            if ne < 2:
                continue
            m2, c2 = record_stats(rn[z], rt[z], rs[z], rS[z])
            scale = max(1.0, np.abs(cov).max())
            assert np.abs(m2 - m).max() <= 1e-4 * max(1.0, np.abs(m).max())
            assert np.abs(c2 - cov).max() <= 2e-4 * scale, (n, k)


def _pair(rng, h=64, w=64):
    return rng.integers(0, 256, (1, h, w, 3), dtype=np.uint8), rng.integers(0, 256, (1, 48, 56, 3), dtype=np.uint8)


@pytest.mark.parametrize("mode", ["wct", "wct_np", "ost", "adain"])
def test_unit_strength_is_the_plain_call(wct, mode):
    if mode == "wct_np":
        wct = WCT(checkpoints=None, relu_targets=ALL, vgg_path=None, weights=make_synthetic_weights(42), semantics="np")
    c, s = _pair(np.random.default_rng(1))
    c = np.concatenate([c, c[:, ::-1]])
    kw = dict(alpha=0.8, ost=mode == "ost", adain=mode == "adain")
    plain = wct.predict_batch(c, s, **kw)
    soft = wct.predict_batch(c, s, strength_map=np.ones((64, 64), np.float32), **kw)
    assert np.array_equal(plain, soft)


@pytest.mark.parametrize("semantics", ["tf", "np"])
def test_one_hot_weights_are_the_hard_mask(semantics):
    w = WCT(checkpoints=None, relu_targets=ALL, vgg_path=None, weights=make_synthetic_weights(42), semantics=semantics)
    rng = np.random.default_rng(2)
    c, s0 = _pair(rng, 80, 96)
    s1 = rng.integers(0, 256, (40, 40, 3), dtype=np.uint8)
    mask = np.zeros((80, 96), np.uint8)
    mask[:, 40:] = 1
    mask[70:, :] = 3                                       # labels >= R keep the content
    mask[0, 0] = 2                                         # a region that vanishes at every coarse level
    styles = [s0[0], s1, s1]
    hard = w.predict_batch(c, styles, alpha=0.9, content_mask=mask)
    soft = w.predict_batch(c, styles, alpha=0.9, content_mask=mask, strength_map=np.ones((80, 96), np.float32))
    assert np.array_equal(hard, soft)


def test_feathered_boundary_is_smoother(wct):
    c = np.full((1, 128, 128, 3), 128, np.uint8)
    s0 = np.zeros((64, 64, 3), np.uint8)
    s0[..., 0] = 220
    s1 = np.zeros((64, 64, 3), np.uint8)
    s1[..., 2] = 220
    s0[::2] += 20
    s1[::3] += 30
    mask = np.zeros((128, 128), np.uint8)
    mask[:, 64:] = 1
    hard = wct.predict_batch(c, [s0, s1], content_mask=mask).astype(np.float64)
    soft = wct.predict_batch(c, [s0, s1], content_mask=mask, mask_feather=16).astype(np.float64)
    jump = lambda o: np.abs(np.diff(o[0].mean(0), axis=0)).max()
    assert jump(soft) < jump(hard)


def test_strength_ramp_is_monotone(wct):
    """With a left-to-right strength ramp the change against the strength-0 output (every level keeps its feature: the
    decoders' reconstruction) grows from left to right, column means within 1 grey level."""
    rng = np.random.default_rng(3)
    c, s = _pair(rng, 64, 128)
    ramp = np.tile(np.linspace(0, 1, 128, dtype=np.float32), (64, 1))
    out = wct.predict_batch(c, s, alpha=1, strength_map=ramp).astype(np.float64)
    base = wct.predict_batch(c, s, alpha=1, strength_map=np.zeros_like(ramp)).astype(np.float64)
    d = np.abs(out[0] - base[0]).mean(axis=(0, 2))
    smooth = np.convolve(d, np.ones(16) / 16, mode="valid")
    assert (np.diff(smooth) >= -1.0).all()
    assert smooth[-1] > smooth[0] + 5.0


@pytest.mark.parametrize("case", ["strength", "feathered"])
def test_batch_groups_and_passes_invariance(wct, case):
    """A frame's bytes do not depend on the batch (N in 1, 7, 30), the sub-batch groups or the passes."""
    rng = np.random.default_rng(4)
    c = rng.integers(0, 256, (30, 64, 64, 3), dtype=np.uint8)
    s = rng.integers(0, 256, (48, 48, 3), dtype=np.uint8)
    s2 = rng.integers(0, 256, (40, 56, 3), dtype=np.uint8)
    mask = np.zeros((64, 64), np.uint8)
    mask[:, 30:] = 1
    ramp = np.tile(np.linspace(0.2, 1, 64, dtype=np.float32), (64, 1))
    st, kw = (s, {}) if case == "strength" else ([s, s2], dict(content_mask=mask, mask_feather=5.0))
    eng = wct.engine
    g0 = eng.groups
    try:
        for passes in (1, 2):
            runs = {}
            for groups in (1, 3):
                eng.groups = groups
                runs[(30, groups)] = wct.predict_batch(c, st, strength_map=ramp, passes=passes, **kw)
                runs[(7, groups)] = wct.predict_batch(c[:7], st, strength_map=ramp, passes=passes, **kw)
            eng.groups = 1
            for i in (0, 3, 6):
                one = wct.predict_batch(c[i:i + 1], st, strength_map=ramp, passes=passes, **kw)
                for key, out in runs.items():
                    assert np.array_equal(out[i:i + 1], one), (passes, key, i)
            assert np.array_equal(runs[(30, 1)], runs[(30, 3)]), passes
    finally:
        eng.groups = g0


def test_seamless_with_strength():
    """seamless="x" with a strength map constant along x: a circular shift of the content along x shifts the output by
    the same amount (one level, float output, within 1e-3 as the seamless tests allow), so opposite edges still join."""
    from wct_tf_b200.engine import Engine
    eng = Engine(make_synthetic_weights(42), ["relu3_1"])
    rng = np.random.default_rng(5)
    c = rng.integers(0, 256, (1, 64, 96, 3), dtype=np.uint8)
    s = torch.from_numpy(rng.integers(0, 256, (1, 48, 48, 3), dtype=np.uint8)).cuda()
    ramp = torch.linspace(0, 1, 64, device="cuda").view(1, 64, 1).expand(1, 64, 96).contiguous()
    a = eng.stylize(torch.from_numpy(c).cuda(), s, alpha=0.8, seamless="x", strength_map=ramp).cpu().numpy()
    b = eng.stylize(torch.from_numpy(np.roll(c, 24, axis=2)).cuda(), s, alpha=0.8, seamless="x", strength_map=ramp).cpu().numpy()
    eng.check_device()
    assert np.abs(b - np.roll(a, 24, axis=2)).max() <= 1e-3


def test_rejections(wct):
    c, s = _pair(np.random.default_rng(6))
    with pytest.raises(ValueError):
        wct.predict_batch(c, s, mask_feather=3.0)
    with pytest.raises(ValueError):
        wct.predict_batch(c, s, strength_map=np.full((8, 8), 2.0))
    with pytest.raises(ValueError):
        wct.predict_batch(c, s, strength_map=np.ones((8, 8)), tile_size=64)
    with pytest.raises(ValueError):
        wct.predict_batch(c, [s[0]], content_mask=np.zeros((8, 8), np.uint8), content_weights=np.ones((1, 8, 8)))
    with pytest.raises(ValueError):
        wct.predict_batch(c, [s[0]], content_weights=np.ones((1, 8, 8)), adain=True)


# --------------------------------------------------------------------------------------------- the weighted apply
def _transform(C, P, seed, dead=()):
    """A WCT transform buffer of P problems: M = I + a small random matrix (split fp16), a random bias, k_c = -1 for the
    problems in ``dead``.  Returns (device buffer, M as float64 [P,C,C] of its two planes, bias [P,C])."""
    import ctypes
    rng = np.random.default_rng(seed)
    o = [ctypes.c_size_t() for _ in range(3)]
    nbytes = U.lib().wctb200_wct_transform_layout(C, P, *[ctypes.byref(x) for x in o])
    om, ob, ok = [x.value for x in o]
    M = np.eye(C)[None] + rng.standard_normal((P, C, C)) * (0.3 / np.sqrt(C))
    hi = M.astype(np.float16)
    lo = (M - hi.astype(np.float64)).astype(np.float16)
    bias = rng.standard_normal((P, C)).astype(np.float32)
    kk = np.zeros(2 * P, np.int32)
    kk[:P] = C
    for z in dead:
        kk[z] = -1
    buf = np.zeros(nbytes, np.uint8)
    buf[om:om + P * 2 * C * C * 2] = np.stack([hi, lo], 1).reshape(-1).view(np.uint8)
    buf[ob:ob + P * C * 4] = bias.reshape(-1).view(np.uint8)
    buf[ok:ok + 2 * P * 4] = kk.view(np.uint8)
    Mq = hi.astype(np.float64) + lo.astype(np.float64)
    return U.dev(buf), Mq, bias.astype(np.float64)


def _soft_maps(N, K, H, W, seed):
    """Fractional weights summing to <= 1, a band where every weight is 0 (it keeps its input), and a strength ramp."""
    rng = np.random.default_rng(seed)
    w = rng.random((N, K + 1, H, W))
    w = (w / w.sum(1, keepdims=True))[:, :K].astype(np.float32)
    w[:, :, :, -3:] = 0.0
    s = np.tile(np.linspace(0.1, 1.0, W, dtype=np.float32), (N, H, 1))
    return w, s


@pytest.mark.parametrize("C", [64, 128, 256, 512])
def test_weighted_apply_matches_fp64(C):
    """wctb200_wct_transform_apply_weighted against float64 ``apply_soft``: fractional weights, a strength map, a k_c = -1
    problem (its weight counts as 0), and pixels whose weights are all 0 (their bytes, halo included, are the input's)."""
    N, K, H, W = 2, 3, 19, 45
    rng = np.random.default_rng(C)
    x = rng.standard_normal((N, H, W, C)).astype(np.float32)
    w, s = _soft_maps(N, K, H, W, C + 1)
    tr, M, b = _transform(C, N * K, C + 2, dead=(1 * K + 2,))
    act = U.act_from_numpy(x)
    out = U.act_alloc(N, H, W, C)
    d_w, d_s = U.dev(w), U.dev(s)                         # held until the kernel has read them
    _capi.check(U.lib().wctb200_wct_transform_apply_weighted(act.data_ptr(), N, H, W, C, tr.data_ptr(), K, d_w.data_ptr(),
                                                              d_s.data_ptr(), out.data_ptr(), U.stream()))
    U.check_device()
    xin = U.act_raw_padded(act, N, H, W, C)
    got = U.act_raw_padded(out, N, H, W, C)
    worst = 0.0
    for n in range(N):
        v = s[n][None].astype(np.float64) * w[n].astype(np.float64)
        if n == 1:
            v[2] = 0.0
        ref = apply_soft(xin[n, 1:-1, 1:-1], M[n * K:(n + 1) * K], b[n * K:(n + 1) * K], v)
        err = np.abs(got[n, 1:-1, 1:-1] - ref).max() / max(1.0, np.abs(ref).max())
        worst = max(worst, err)
    print("weighted apply C=%d: max rel error %.2e" % (C, worst))
    assert worst <= 1e-5
    raw_in = act.view(torch.float16).view(2, N, H + 2, W + 2, C).cpu().numpy()
    raw_out = out.view(torch.float16).view(2, N, H + 2, W + 2, C).cpu().numpy()
    assert np.array_equal(raw_out[:, :, :, -4:].view(np.uint16), raw_in[:, :, :, -4:].view(np.uint16))   # kept band + halo


# --------------------------------------------------------------------------------------------- teacher-forced levels
def _teacher_forced_soft(weights, sem, mask, R, sigma, ssizes, size=128, alpha=0.8, seed=100):
    eng = Engine(weights, ALL, semantics=sem)
    rng = np.random.default_rng(seed)
    content = rng.integers(0, 256, (1, size, size, 3), dtype=np.uint8)
    styles = [rng.integers(0, 256, (1, q, q, 3), dtype=np.uint8) for q in ssizes]
    ramp = np.tile(np.linspace(0.0, 1.0, size, dtype=np.float32), (size, 1))
    cap = {}
    eng.stylize(torch.from_numpy(content).cuda(), None, alpha=alpha, capture=cap, labels=torch.from_numpy(mask).cuda(),
                region_styles=[torch.from_numpy(q).cuda() for q in styles], mask_feather=sigma,
                strength_map=torch.from_numpy(ramp[None]).cuda())
    eng.check_device()
    planes = feather(mask[None], R, sigma)[0]
    sfe = [nets.encode(nets.preprocess(q).astype(np.float64), weights, ALL, np.float64) for q in styles]
    worst = 0.0
    for i, relu in enumerate(ALL):
        x = cap["level_input"][i].cpu().numpy().astype(np.float64)
        cf = nets.encode(x, weights, [relu], np.float64)[relu]
        h, w = cf.shape[1:3]
        f, info = wct_soft(cf, [q[relu] for q in sfe], resize_area(planes, h, w), resize_area(ramp, h, w), alpha, sem,
                           return_info=True)
        for r, inf in enumerate(info):       # an eigenvalue at the 1e-5 cut would make the kept set a coin toss
            assert inf["k_c"] < 0 or ref_ops.spectral_gap_ok(inf["wc"]), "ill-posed vector (%s, region %d)" % (relu, r)
        got_f = eng.act_to_f32(cap["transformed"][i]).cpu().numpy()
        e_f = np.abs(got_f - f).max()
        y = nets.decode(np.asarray(f, dtype=np.float64), weights, relu, np.float64)
        if i < len(ALL) - 1:
            y = np.clip(y, 0, 1)
        e_out = np.abs(cap["level_output"][i].cpu().numpy() - y).max()
        print("%s %s R=%d: transform %.2e  level output %.2e" % (sem, relu, R, e_f, e_out))
        worst = max(worst, e_f, e_out)
    return worst


@pytest.mark.parametrize("sem", ["tf", "np"])
@pytest.mark.parametrize("R", [2, 3])
def test_teacher_forced_soft_128(sem, R):
    # feathering spreads small weights over a region's neighbourhood, so a small region's weighted covariance can have
    # eigenvalues all the way down through the 1e-5 cut (a kept set decided by rounding); the oracle's spectral-gap check
    # above guards against that.  Two halves, or three vertical bands, feathered by sigma = 6.
    mask = np.zeros((128, 128), np.uint8)
    if R == 2:
        mask[:, 64:] = 1
    else:
        mask[:, 40:] = 1
        mask[:, 88:] = 2
    sigma = 6.0
    worst = _teacher_forced_soft(make_synthetic_weights(42), sem, mask, R, sigma, [144, 96, 112][:R])
    print("teacher-forced soft %s R=%d: max %.2e" % (sem, R, worst))
    assert worst <= 1e-3


def test_free_running_soft_vs_oracle():
    weights = make_synthetic_weights(42)
    size = 128
    rng = np.random.default_rng(1000)
    content = rng.integers(0, 256, (1, size, size, 3), dtype=np.uint8)
    styles = [rng.integers(0, 256, (1, q, q, 3), dtype=np.uint8) for q in (128, 96)]
    mask = np.zeros((97, 131), np.uint8)                                # any resolution: area-averaged per level
    mask[:, 61:] = 1
    planes = feather(mask[None], 2, 2.0)[0]
    ramp = np.tile(np.linspace(0.3, 1.0, 131), (97, 1))
    o64 = pipeline_soft(content[0], [q[0] for q in styles], planes, ramp, weights, ALL, alpha=0.8, semantics="np", dtype=np.float64)
    o32 = pipeline_soft(content[0], [q[0] for q in styles], planes, ramp, weights, ALL, alpha=0.8, semantics="np", dtype=np.float32)
    noise = np.abs(o32 - o64).max()
    eng = Engine(weights, ALL, semantics="np")
    got = eng.stylize(torch.from_numpy(content).cuda(), None, alpha=0.8, labels=torch.from_numpy(mask).cuda(),
                      region_styles=[torch.from_numpy(q).cuda() for q in styles], mask_feather=2.0,
                      strength_map=torch.from_numpy(ramp.astype(np.float32)[None]).cuda()).cpu().numpy()
    eng.check_device()
    err = np.abs(got - o64).max()
    print("free-running soft: %.3e (oracle fp32 noise %.3e)" % (err, noise))
    assert err <= max(1e-3, FREE_RUN_NOISE_FACTOR * noise)


# --------------------------------------------------------------------------------------------- style masks
def test_soft_paths_with_style_masks(wct):
    """Hard mask + unit strength, and one-hot content_weights aligned to every level's grid, equal the hard mask with style
    masks byte for byte; the style mask leaves region 2 empty (k_s = -1: region 2 keeps the content)."""
    rng = np.random.default_rng(9)
    c = rng.integers(0, 256, (2, 128, 128, 3), dtype=np.uint8)
    st = [rng.integers(0, 256, (96, 96, 3), dtype=np.uint8) for _ in range(2)]
    styles = [st[0], st[1], st[1]]
    mask = np.zeros((128, 128), np.uint8)
    mask[:, 48:96] = 1
    mask[:, 96:] = 2
    smask = np.zeros((96, 96), np.uint8)
    smask[48:] = 1                                         # no style pixel is labelled 2
    sms = [smask, smask, smask]
    hard = wct.predict_batch(c, styles, alpha=0.9, content_mask=mask, style_masks=sms)
    unit = wct.predict_batch(c, styles, alpha=0.9, content_mask=mask, style_masks=sms, strength_map=np.ones((128, 128), np.float32))
    onehot = np.stack([(mask == k).astype(np.float32) for k in range(3)])
    soft = wct.predict_batch(c, styles, alpha=0.9, content_weights=onehot, style_masks=sms)
    assert np.array_equal(hard, unit)
    assert np.array_equal(hard, soft)
    assert not np.array_equal(hard[:, :, :40], c[:, :, :40])


# --------------------------------------------------------------------------------------------- offsets past 2^31
def test_weighted_stats_and_apply_past_2_31():
    """At 9 x 2048^2 x 64 the lo plane lies past 2^31 (past 2^32 from frame 7): each frame's weighted record and weighted
    apply have the bytes of that frame run alone."""
    import gc
    from tests.test_gpu_large_offsets import A, C as C64, batch_act, frame_copy
    n, h, w = A
    K = 2
    lib = U.lib()
    xin = batch_act(n, h, w, C64, 1300)
    wts = torch.rand((n, K, h, w), generator=torch.Generator(device="cuda").manual_seed(7), device="cuda")
    wts = wts / (wts.sum(1, keepdim=True) + 0.25)
    stren = torch.linspace(0.2, 1.0, w, device="cuda").expand(n, h, w).contiguous()
    nb = lib.wctb200_stats_record_layout(C64, n * K, 0, None, None, None, None)
    rec = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    _capi.check(lib.wctb200_wct_stats_weighted(xin.data_ptr(), n, h, w, C64, wts.data_ptr(), K, rec.data_ptr(), U.stream()))
    got_rec = _record(rec, C64, n * K)
    tr, _, _ = _transform(C64, n * K, 31)
    out = U.act_alloc(n, h, w, C64, poison=False)
    _capi.check(lib.wctb200_wct_transform_apply_weighted(xin.data_ptr(), n, h, w, C64, tr.data_ptr(), K, wts.data_ptr(),
                                                          stren.data_ptr(), out.data_ptr(), U.stream()))
    U.check_device()
    planes = out.view(torch.float16).view(2, n, h + 2, w + 2, C64)
    for i in (0, 4, 7, n - 1):
        one = frame_copy(xin, i, n, h, w, C64)
        r1 = torch.zeros(lib.wctb200_stats_record_layout(C64, K, 0, None, None, None, None), dtype=torch.uint8, device="cuda")
        wi = wts[i:i + 1].contiguous()
        _capi.check(lib.wctb200_wct_stats_weighted(one.data_ptr(), 1, h, w, C64, wi.data_ptr(), K, r1.data_ptr(), U.stream()))
        want = _record(r1, C64, K)
        for name, g, wv in zip("ntsS", got_rec, want):
            assert np.array_equal(np.asarray(g[i * K:(i + 1) * K]).view(np.uint64), np.asarray(wv).view(np.uint64)), (i, name)
        t1, _, _ = _transform_slice(tr, C64, n * K, i * K, K)
        o1 = U.act_alloc(1, h, w, C64, poison=False)
        _capi.check(lib.wctb200_wct_transform_apply_weighted(one.data_ptr(), 1, h, w, C64, t1.data_ptr(), K, wi.data_ptr(),
                                                              stren[i:i + 1].contiguous().data_ptr(), o1.data_ptr(), U.stream()))
        U.check_device()
        p1 = o1.view(torch.float16).view(2, 1, h + 2, w + 2, C64)
        assert torch.equal(p1[:, 0].view(torch.int16), planes[:, i].view(torch.int16)), i
        del one, o1
    del xin, out
    gc.collect()
    torch.cuda.empty_cache()


def _transform_slice(tr, C, P, z0, cnt):
    """Problems [z0, z0 + cnt) of a transform buffer of P problems, as a buffer of cnt problems."""
    import ctypes
    o = [ctypes.c_size_t() for _ in range(3)]
    U.lib().wctb200_wct_transform_layout(C, P, *[ctypes.byref(x) for x in o])
    q = [ctypes.c_size_t() for _ in range(3)]
    nb = U.lib().wctb200_wct_transform_layout(C, cnt, *[ctypes.byref(x) for x in q])
    out = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    (om, ob, ok), (qm, qb, qk) = [x.value for x in o], [x.value for x in q]
    mb = 2 * C * C * 2
    out[qm:qm + cnt * mb] = tr[om + z0 * mb:om + (z0 + cnt) * mb]
    out[qb:qb + cnt * C * 4] = tr[ob + z0 * C * 4:ob + (z0 + cnt) * C * 4]
    out[qk:qk + cnt * 4] = tr[ok + z0 * 4:ok + (z0 + cnt) * 4]
    out[qk + cnt * 4:qk + 2 * cnt * 4] = tr[ok + (P + z0) * 4:ok + (P + z0 + cnt) * 4]
    return out, None, None
