"""The optimal-transport transform (OST, DESIGN.md §3.3.8) on the GPU: the C ABI against the fp64 oracle of
``tests/ost_ref.py`` on both B^1/2 paths, its defining properties, batch and record invariance, the five-level pipeline,
and the engine options it works with or rejects."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import nets, ref_ops
from tests import gpu_util as U
from tests import ost_ref as O
from tests.test_gpu_invariance import assert_bits, frame_copy, planes
from wct_tf_b200 import _capi
from wct_tf_b200.engine import SEMANTICS, Engine
from wct_tf_b200.wct import WCT
from wct_tf_b200.weights import make_synthetic_weights

pytestmark = pytest.mark.gpu
ALL = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]
FREE_RUN_NOISE_FACTOR = 3          # tests/test_gpu_pipeline.py: the free-running bound, a multiple of the oracle's fp32 noise
TF_TILED_BOUND = 1e-4              # tests/test_gpu_tiles.py: tiled vs untiled teacher-forced level


def _ws(nbytes):
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device="cuda")


def _gauss(n, h, w, c, seed, rank=None, lo=0.5, hi=2.0, offset=0.3):
    """Features whose covariance has eigenvalues in [lo, hi] (times the sampling spread) on `rank` of the C directions."""
    rng = np.random.default_rng(seed)
    q, _ = np.linalg.qr(rng.standard_normal((c, c)))
    k = c if rank is None else rank
    mix = (q[:, :k] * np.sqrt(rng.uniform(lo, hi, k))) @ q[:, :k].T
    x = rng.standard_normal((n, h, w, c)) @ mix + offset * rng.uniform(0.5, 1.5, c)
    return x.astype(np.float32)


CASES = {   # (content rank, style rank) as a fraction of C; 64 x 64 pixels: the sample covariances stay well-conditioned
    "full": (None, None),
    "content_rank_deficient": (0.5, None),
    "style_rank_deficient": (None, 0.5),
}


def _prepare(lib, style, ns, hs, ws_, c, s):
    state = _ws(lib.wctb200_wct_style_state_bytes(c, ns))
    ws = _ws(lib.wctb200_wct_workspace_bytes(c, 0, ns))
    _capi.check(lib.wctb200_wct_style_prepare(style.data_ptr(), ns, hs, ws_, c, s["eps_cov"], s["eps_eig"], s["thresh"],
                                              state.data_ptr(), ws.data_ptr(), ws.numel(), U.stream()))
    return state


def _ost(lib, content, nc, h, w, c, state, ns, alpha, s, ws=None):
    ws = _ws(lib.wctb200_ost_workspace_bytes(c, nc)) if ws is None else ws
    out = U.act_alloc(nc, h, w, c)
    k = torch.zeros(5 * nc, dtype=torch.int32, device="cuda")
    _capi.check(lib.wctb200_ost_apply(content.data_ptr(), nc, h, w, c, state.data_ptr(), ns, float(alpha), s["eps_cov"],
                                      s["eps_eig"], s["thresh"], s["readd"], out.data_ptr(), k.data_ptr(), ws.data_ptr(),
                                      ws.numel(), U.stream()))
    return out, k.cpu().numpy()


def _wct(lib, content, nc, h, w, c, state, ns, alpha, s):
    ws = _ws(lib.wctb200_wct_workspace_bytes(c, nc, 0))
    out = U.act_alloc(nc, h, w, c)
    _capi.check(lib.wctb200_wct_apply(content.data_ptr(), nc, h, w, c, state.data_ptr(), ns, float(alpha), s["eps_cov"],
                                      s["eps_eig"], s["thresh"], s["readd"], out.data_ptr(), None, ws.data_ptr(), ws.numel(),
                                      U.stream()))
    return out


def _case(c, case, sem, seed=0):
    rc, rs = CASES[case]
    H = W = 64
    x = _gauss(1, H, W, c, 10 + seed, None if rc is None else int(rc * c))
    y = _gauss(1, H, W, c, 20 + seed, None if rs is None else int(rs * c), lo=0.3, hi=3.0, offset=0.6)
    content, style = U.act_from_numpy(x), U.act_from_numpy(y)
    xs = U.act_to_numpy(content, 1, H, W, c).astype(np.float64)       # the values the kernels read
    ys = U.act_to_numpy(style, 1, H, W, c).astype(np.float64)
    return content, style, xs, ys, H, W


def _run_case(c, case, sem, alpha=0.8):
    lib = U.lib()
    s = SEMANTICS[sem]
    content, style, xs, ys, H, W = _case(c, case, sem)
    state = _prepare(lib, style, 1, H, W, c, s)
    out, k = _ost(lib, content, 1, H, W, c, state, 1, alpha, s)
    got = U.act_to_numpy(out, 1, H, W, c).astype(np.float64)
    ref, info = O.ost(xs, ys, alpha, sem, return_info=True)
    return got, ref, k, info, (lib, content, state, xs, ys, H, W, s)


# ------------------------------------------------------------------------------------------------------------- C ABI
@pytest.mark.parametrize("c", [64, 128, 256, 512])
@pytest.mark.parametrize("sem", ["tf", "np"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_ost_apply_vs_fp64(c, sem, case):
    got, ref, k, info, _ = _run_case(c, case, sem)
    err = float(np.abs(got - ref).max())
    print("ost C=%d %s %s: max-abs %.2e  k_out %s (oracle k_c %d k_s %d)" % (c, sem, case, err, k.tolist(), info["k_c"], info["k_s"]))
    assert err <= 1e-3
    assert k[0] == info["k_c"]
    if case == "full" and c >= 128:
        assert k[2] == 1 and k[3] == 1 and k[1] == 0 and k[4] == 0          # Newton-Schulz for W_c and for B^1/2
    if case == "style_rank_deficient":
        assert k[3] == 0 and k[4] > 0                                       # B is singular: the eigensolver
    if case == "content_rank_deficient":
        assert k[0] == c // 2
    U.check_device()


@pytest.mark.parametrize("c", [64, 128, 256, 512])
@pytest.mark.parametrize("sem", ["tf", "np"])
def test_fast_path_off_agrees(c, sem):
    """Case (a) with the matrix-function fast path switched off: both roots by the eigensolver, same bound, and within it
    of the fast path."""
    lib = U.lib()
    fast, ref, _, _, _ = _run_case(c, "full", sem)
    lib.wctb200_debug_set_matfun(0, 0)
    try:
        slow, _, k, _, _ = _run_case(c, "full", sem)
    finally:
        lib.wctb200_debug_set_matfun(1, 0)
    assert k[2] == 0 and k[3] == 0 and k[1] > 0 and k[4] > 0
    assert np.abs(slow - ref).max() <= 1e-3
    assert np.abs(slow - fast).max() <= 1e-3
    U.check_device()


@pytest.mark.parametrize("c", [64, 256, 512])
@pytest.mark.parametrize("sem", ["tf", "np"])
def test_ost_properties(c, sem):
    """At alpha = 1 the output covariance is the style's, and OST moves the features less than WCT."""
    got, _, _, _, (lib, content, state, xs, ys, H, W, s) = _run_case(c, "full", sem, alpha=1.0)
    f = got.reshape(-1, c)
    cov_out = np.cov(f, rowvar=False)
    cov_s = np.cov(ys.reshape(-1, c), rowvar=False) + s["eps_cov"] * np.eye(c)
    rel = np.linalg.norm(cov_out - cov_s) / np.linalg.norm(cov_s)
    wct = U.act_to_numpy(_wct(lib, content, 1, H, W, c, state, 1, 1.0, s), 1, H, W, c).astype(np.float64)
    x = xs.reshape(-1, c)
    cost_ost = float(((f - x) ** 2).sum(1).mean())
    cost_wct = float(((wct.reshape(-1, c) - x) ** 2).sum(1).mean())
    print("C=%d %s: output covariance rel. Frobenius %.2e; mean |out - x|^2 OST %.4g, WCT %.4g" % (c, sem, rel, cost_ost, cost_wct))
    assert rel <= 1e-3
    assert cost_ost < cost_wct


@pytest.mark.parametrize("c", [64, 128, 256, 512])
@pytest.mark.parametrize("shared", [True, False], ids=["shared_style", "per_frame_styles"])
def test_batch_equals_single_frames(c, shared):
    lib = U.lib()
    s = SEMANTICS["tf"]
    nc, H, W, Hs, Ws = 3, 24, 40, 28, 30
    xs = np.concatenate([_gauss(1, H, W, c, 30 + i) for i in range(nc)])
    ys = np.concatenate([_gauss(1, Hs, Ws, c, 40 + i, rank=c // 2 if i == 1 else None) for i in range(nc)])
    content = U.act_from_numpy(xs)
    ns = 1 if shared else nc
    style = U.act_from_numpy(ys[:ns])
    state = _prepare(lib, style, ns, Hs, Ws, c, s)
    out, k = _ost(lib, content, nc, H, W, c, state, ns, 0.7, s)
    batch = planes(out, nc, H, W, c)
    for i in range(nc):
        st_i = state if shared else _prepare(lib, frame_copy(style, i, nc, Hs, Ws, c), 1, Hs, Ws, c, s)
        o1, k1 = _ost(lib, frame_copy(content, i, nc, H, W, c), 1, H, W, c, st_i, 1, 0.7, s)
        assert_bits(batch[:, i:i + 1], planes(o1, 1, H, W, c), "ost frame %d" % i)
        assert k[i::nc].tolist() == k1.tolist()
    U.check_device()


@pytest.mark.parametrize("c", [64, 128, 256, 512])
@pytest.mark.parametrize("nc", [1, 3])
@pytest.mark.parametrize("sem", ["tf", "np"])
def test_transform_from_whole_record_equals_apply(c, nc, sem):
    lib = U.lib()
    s = SEMANTICS[sem]
    H, W, Hs, Ws = 23, 31, 19, 27
    content = U.act_from_numpy(np.concatenate([_gauss(1, H, W, c, 50 + i) for i in range(nc)]))
    state = _prepare(lib, U.act_from_numpy(_gauss(1, Hs, Ws, c, 60)), 1, Hs, Ws, c, s)
    ref, kref = _ost(lib, content, nc, H, W, c, state, 1, 0.7, s)
    offs = [ctypes.c_size_t() for _ in range(4)]
    rec = torch.zeros(lib.wctb200_stats_record_layout(c, nc, 0, *[ctypes.byref(o) for o in offs]), dtype=torch.uint8, device="cuda")
    _capi.check(lib.wctb200_wct_stats_rect(content.data_ptr(), nc, H, W, c, 0, 0, H, W, rec.data_ptr(), U.stream()))
    om, ob, ok = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_size_t()
    tr = _ws(lib.wctb200_wct_transform_layout(c, nc, ctypes.byref(om), ctypes.byref(ob), ctypes.byref(ok)))
    ws = _ws(lib.wctb200_ost_workspace_bytes(c, nc))
    _capi.check(lib.wctb200_ost_transform_from_stats(rec.data_ptr(), nc, c, state.data_ptr(), 1, 0.7, s["eps_cov"], s["eps_eig"],
                                                     s["thresh"], s["readd"], tr.data_ptr(), ws.data_ptr(), ws.numel(), U.stream()))
    out = U.act_alloc(nc, H, W, c)
    _capi.check(lib.wctb200_wct_transform_apply(content.data_ptr(), nc, H, W, c, tr.data_ptr(), out.data_ptr(), U.stream()))
    assert_bits(planes(out, nc, H, W, c), planes(ref, nc, H, W, c), "ost transform from record")
    k = tr[ok.value:ok.value + 8 * nc].view(torch.int32).cpu().numpy()
    assert np.array_equal(k, kref[:2 * nc])
    U.check_device()


def test_rejections():
    lib = U.lib()
    s = SEMANTICS["tf"]
    c, H, W = 64, 8, 8
    content = U.act_from_numpy(_gauss(3, H, W, c, 1))
    state = _prepare(lib, U.act_from_numpy(_gauss(2, H, W, c, 2)), 2, H, W, c, s)
    ws = _ws(lib.wctb200_ost_workspace_bytes(c, 3))
    out = U.act_alloc(3, H, W, c)

    def call(C, nc, ns, nbytes):
        return lib.wctb200_ost_apply(content.data_ptr(), nc, H, W, C, state.data_ptr(), ns, 1.0, s["eps_cov"], s["eps_eig"],
                                     s["thresh"], s["readd"], out.data_ptr(), None, ws.data_ptr(), nbytes, U.stream())
    assert lib.wctb200_ost_workspace_bytes(96, 1) == 0
    assert call(96, 1, 1, ws.numel()) == _capi.EINVAL
    assert call(c, 3, 2, ws.numel()) == _capi.EINVAL
    assert call(c, 3, 1, ws.numel() - 1) == _capi.EWS
    assert lib.wctb200_ost_transform_from_stats(None, 1, c, state.data_ptr(), 1, 1.0, 0.0, 0.0, 1e-5, 0, ws.data_ptr(),
                                                ws.data_ptr(), ws.numel(), U.stream()) == _capi.EINVAL
    U.check_device()


# ------------------------------------------------------------------------------------------------------------ pipeline
@pytest.fixture(scope="module")
def weights():
    return make_synthetic_weights(42)


def _u8(n, H, W, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, H, W, 3), dtype=np.uint8)


@pytest.mark.parametrize("sem", ["tf", "np"])
def test_teacher_forced_levels(weights, sem):
    """Every level from the device's own level input: its encoding, OST and decode in fp64 against the device's."""
    eng = Engine(weights, ALL, semantics=sem)
    content, style = _u8(1, 128, 128, 100), _u8(1, 144, 144, 101)
    cap = {}
    eng.stylize(torch.from_numpy(content).cuda(), torch.from_numpy(style).cuda(), alpha=0.8, want_info=True, capture=cap, ost=True)
    eng.check_device()
    sfe = nets.encode(nets.preprocess(style).astype(np.float64), weights, ALL, np.float64)
    worst = 0.0
    for i, relu in enumerate(ALL):
        x = cap["level_input"][i].cpu().numpy().astype(np.float64)
        cf = nets.encode(x, weights, [relu], np.float64)[relu]
        f, info = O.ost(cf, sfe[relu], 0.8, sem, return_info=True)
        assert eng.last_info[i].cpu().numpy()[0] == info["k_c"]
        e_t = np.abs(eng.act_to_f32(cap["transformed"][i]).cpu().numpy() - f).max()
        y = nets.decode(np.asarray(f, dtype=np.float64), weights, relu, np.float64)
        if i < len(ALL) - 1:
            y = np.clip(y, 0, 1)
        e_out = np.abs(cap["level_output"][i].cpu().numpy() - y).max()
        print("%s %s: transform %.2e  level output %.2e  k_out %s" % (sem, relu, e_t, e_out, eng.last_info[i].cpu().numpy().tolist()))
        worst = max(worst, e_t, e_out)
    assert worst <= 1e-3


# Per-level transform error of OST relative to WCT's on the same device features: OST adds the products of S_c, B and M and
# a second matrix root to WCT's W_c, so it may carry a few times WCT's rounding error, not orders of magnitude more.
# Measured on an H100 at the free-running inputs below: at most 7.6x (relu3_1, np, B^1/2 by Newton-Schulz).
OST_OVER_WCT = 10.0


@pytest.mark.parametrize("sem", ["tf", "np"])
@pytest.mark.parametrize("fast", [1, 0], ids=["fast_path", "eigensolver"])
def test_teacher_forced_on_free_running_inputs(weights, sem, fast):
    """At every level of the free-running inputs, the device's OST transform of its own content feature against the fp64
    oracle, next to WCT's error on the same feature: within OST_OVER_WCT times WCT's error (floor 1e-4)."""
    content, style = _u8(1, 128, 128, 1000), _u8(1, 128, 128, 7)
    sfe = nets.encode(nets.preprocess(style).astype(np.float64), weights, ALL, np.float64)
    lib = U.lib()
    errs = {}
    lib.wctb200_debug_set_matfun(fast, 0)
    try:
        for ost in (True, False):
            eng = Engine(weights, ALL, semantics=sem)
            cap = {}
            eng.stylize(torch.from_numpy(content).cuda(), torch.from_numpy(style).cuda(), alpha=0.8, capture=cap, ost=ost)
            eng.check_device()
            for i, relu in enumerate(ALL):
                cf = eng.act_to_f32(cap["content_feat"][i]).cpu().numpy().astype(np.float64)
                if ost:
                    f = O.ost(cf, sfe[relu], 0.8, sem)
                else:
                    p = O.SEMANTICS[sem]
                    f = ref_ops.wct_generic(cf, sfe[relu], 0.8, eps_cov=p["eps_cov"], eps_eig=p["eps_eig"],
                                            readd_content_mean=p["readd_content_mean"])
                errs[(relu, ost)] = float(np.abs(eng.act_to_f32(cap["transformed"][i]).cpu().numpy() - f).max())
    finally:
        lib.wctb200_debug_set_matfun(1, 0)
    for relu in ALL:
        print("%s %s %s: OST %.2e  WCT %.2e" % (sem, "fast" if fast else "jacobi", relu, errs[(relu, True)], errs[(relu, False)]))
        assert errs[(relu, True)] <= max(1e-4, OST_OVER_WCT * errs[(relu, False)]), relu


def test_free_running_vs_oracle(weights):
    content, style = _u8(1, 128, 128, 1000), _u8(1, 128, 128, 7)
    o64 = O.pipeline_ost(content[0], style[0], weights, ALL, alpha=0.8, semantics="np", dtype=np.float64)
    o32 = O.pipeline_ost(content[0], style[0], weights, ALL, alpha=0.8, semantics="np", dtype=np.float32)
    bound = max(1e-3, FREE_RUN_NOISE_FACTOR * float(np.abs(o32 - o64).max()))
    eng = Engine(weights, ALL, semantics="np")
    got = eng.stylize(torch.from_numpy(content).cuda(), torch.from_numpy(style).cuda(), alpha=0.8, ost=True).cpu().numpy()
    err = float(np.abs(got - o64).max())
    print("free-running OST 128^2: vs fp64 oracle %.3e (bound %.3e)" % (err, bound))
    assert err <= bound


# -------------------------------------------------------------------------------------------------------------- engine
def test_prepared_and_saved_styles_equal_image(weights, tmp_path):
    wct = WCT(relu_targets=ALL, weights=weights)
    c, s = _u8(2, 96, 80, 1), _u8(1, 64, 72, 2)
    ref = wct.predict_batch(c, s, alpha=0.8, ost=True)
    ps = wct.prepare_style(s[0])
    assert np.array_equal(wct.predict_batch(c, ps, alpha=0.8, ost=True), ref)
    path = str(tmp_path / "one.wctstyle")
    ps.save(path)
    assert np.array_equal(wct.predict_batch(c, wct.load_style(path), alpha=0.8, ost=True), ref)
    s2 = _u8(2, 64, 72, 3)                                         # one style per frame
    assert np.array_equal(wct.predict_batch(c, wct.prepare_style(s2), alpha=0.8, ost=True),
                          wct.predict_batch(c, s2, alpha=0.8, ost=True))
    assert not np.array_equal(ref, wct.predict_batch(c, s, alpha=0.8))            # OST is not WCT


def test_passes_groups_and_outputs(weights):
    wct = WCT(relu_targets=ALL, weights=weights, semantics="np")
    c, s = _u8(4, 80, 96, 4), _u8(1, 64, 64, 5)
    one = wct.predict_batch(c, s, alpha=0.7, ost=True)
    assert np.array_equal(wct.predict_batch(c, s, alpha=0.7, ost=True, passes=2), wct.predict_batch(one, s, alpha=0.7, ost=True))
    eng = wct.engine
    g0 = eng.groups
    eng.groups = 2
    try:
        two = wct.predict_batch(c, s, alpha=0.7, ost=True)
    finally:
        eng.groups = g0
    assert np.array_equal(two, one)
    assert np.array_equal(np.concatenate([wct.predict_batch(c[i:i + 1], s, alpha=0.7, ost=True) for i in range(4)]), one)
    u8, f = wct.predict_batch(c, s, alpha=0.7, ost=True, return_float=True)
    assert np.array_equal(u8, one) and f.dtype == np.float32
    dev = wct.predict_batch(c, s, alpha=0.7, ost=True, return_device=True)
    assert np.array_equal(dev.cpu().numpy(), one)
    assert np.array_equal(wct.predict(c[0], s[0], alpha=0.7, ost=True), one[0])


def test_tiles(weights):
    wct = WCT(relu_targets=ALL, weights=weights)
    c, s = _u8(1, 160, 192, 1), _u8(1, 128, 144, 2)
    ref_u8, ref_f = wct.predict_batch(c, s, alpha=0.8, ost=True, return_float=True)
    got_u8, got_f = wct.predict_batch(c, s, alpha=0.8, ost=True, return_float=True, tile_size=256)
    assert np.array_equal(got_u8, ref_u8) and np.array_equal(got_f.view(np.uint32), ref_f.view(np.uint32))


def test_many_tiles_teacher_forced_1024(weights):
    eng = Engine(weights, ALL, semantics="tf")
    c = torch.from_numpy(_u8(1, 1024, 1024, 5)).cuda()
    s = torch.from_numpy(_u8(1, 512, 512, 6)).cuda()
    cap = {}
    eng.stylize(c, s, alpha=0.8, capture=cap, ost=True)
    ps = eng.prepare_call(s)
    torch.cuda.synchronize()
    worst = {}
    for i, lvl in enumerate(eng.model.levels):
        got = eng.tiled_level(cap["level_input"][i], i, ps.wct[lvl.relu_target], 0.8, False, 256, clip=i < len(ALL) - 1, ost=True)
        worst[lvl.relu_target] = float((got - cap["level_output"][i]).abs().max())
    print("teacher-forced OST tiled (T = 256) vs untiled, 1024^2: %s" % worst)
    assert max(worst.values()) <= TF_TILED_BOUND, worst
    eng.check_device()


def test_swap_level_is_untouched(weights):
    """With swap_targets=["relu3_1"] the swap level takes the same input with and without OST (it is the first level) and
    gives the same bytes; the next level uses OST."""
    targets = ["relu3_1", "relu2_1", "relu1_1"]
    eng = Engine(make_synthetic_weights(3, relu_targets=targets), targets, semantics="tf")
    c = torch.from_numpy(_u8(2, 128, 128, 7)).cuda()
    s = torch.from_numpy(_u8(1, 128, 128, 8)).cuda()
    cap_o, cap_w = {}, {}
    eng.stylize(c, s, alpha=0.8, capture=cap_o, swap_targets=["relu3_1"], ost=True)
    eng.stylize(c, s, alpha=0.8, capture=cap_w, swap_targets=["relu3_1"])
    assert torch.equal(cap_o["transformed"][0].buf, cap_w["transformed"][0].buf)
    assert torch.equal(cap_o["level_output"][0], cap_w["level_output"][0])
    assert not torch.equal(cap_o["transformed"][1].buf, cap_w["transformed"][1].buf)
    eng.check_device()


def test_temporal_runs(weights):
    wct = WCT(relu_targets=["relu3_1", "relu1_1"], weights=make_synthetic_weights(1, relu_targets=["relu3_1", "relu1_1"]))
    c, s = _u8(3, 64, 64, 1), _u8(1, 64, 64, 2)
    st = wct.temporal_state(0.5)
    out = wct.predict_batch(c, s, ost=True, temporal=st)
    assert out.shape == (3, 64, 64, 3)
    assert np.array_equal(out[0], wct.predict_batch(c[:1], s, ost=True)[0])     # the first frame of a clip is unchanged


@pytest.mark.parametrize("kw", [dict(adain=True), dict(content_mask=np.zeros((8, 8), np.uint8)), dict(style_weights=[1.0])],
                         ids=["adain", "content_mask", "style_weights"])
def test_rejected_combinations(kw):
    wct = WCT(relu_targets=["relu3_1", "relu1_1"], weights=make_synthetic_weights(1, relu_targets=["relu3_1", "relu1_1"]))
    c, s = _u8(1, 64, 64, 1), _u8(1, 64, 64, 2)
    styles = [s[0]] if ("content_mask" in kw or "style_weights" in kw) else s
    with pytest.raises(ValueError):
        wct.predict_batch(c, styles, ost=True, **kw)
    with pytest.raises(ValueError):
        wct.predict(c[0], styles if isinstance(styles, list) else s[0], ost=True, **kw)
    with pytest.raises(ValueError):
        wct.predict_batch(c, [s[0]], content_mask=np.zeros((8, 8), np.uint8), style_masks=[np.zeros((8, 8), np.uint8)], ost=True)
