"""Tiled stylisation on the GPU (DESIGN.md §3.3.7): statistics of a rectangle, the fold of records, transforms from a
record, the halos, and ``predict(tile_size=)`` against the untiled call, the fp64 oracle and itself at other tile sizes."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import nets
from tests import gpu_util as U
from tests import tiles_ref as R
from tests.test_gpu_invariance import assert_bits, feats, planes
from wct_tf_b200 import _capi
from wct_tf_b200.engine import SEMANTICS, Engine
from wct_tf_b200.model import RELU_LEVEL, tile_grid, tile_halos
from wct_tf_b200.wct import WCT
from wct_tf_b200.weights import make_synthetic_weights

pytestmark = pytest.mark.gpu
ALL = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]
FREE_RUN_NOISE_FACTOR = 3          # tests/test_gpu_pipeline.py: the free-running bound, a multiple of the oracle's fp32 noise
# Teacher-forced tiled vs untiled level: the two runs differ only in the order in which the level's statistics are summed
# (fp32 products per 4096-pixel slot, fp64 above).  Each is within the fp32 summation error of the fp64 statistics, which the
# teacher-forced parity tests bound at <= 1e-3 of the fp64 oracle for the whole level output; a different split of the same
# sum moves the fp32 partials by the same order of unit roundoffs, and tiles only regroup them, so their difference is a
# tenth of that bound.
TF_TILED_BOUND = 1e-4


def _ws(nbytes):
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device="cuda")


def _record(C, N, diag):
    lib = U.lib()
    offs = [ctypes.c_size_t() for _ in range(4)]
    nbytes = lib.wctb200_stats_record_layout(C, N, int(diag), *[ctypes.byref(o) for o in offs])
    return torch.zeros(nbytes, dtype=torch.uint8, device="cuda"), [o.value for o in offs]


def _read_record(buf, offs, C, N, diag):
    raw = buf.cpu().numpy()

    def arr(o, count):
        return raw[o:o + 8 * count].view(np.float64)
    n, t, s = arr(offs[0], N), arr(offs[1], N * C).reshape(N, C), arr(offs[2], N * C).reshape(N, C)
    S = arr(offs[3], N * C * (1 if diag else C)).reshape((N, C) if diag else (N, C, C))
    return [dict(n=n[i], t=t[i], s=s[i], S=S[i]) for i in range(N)]


def _rect(act, N, H, W, C, y0, x0, h, w, diag, buf=None, offs=None):
    if buf is None:
        buf, offs = _record(C, N, diag)
    fn = U.lib().wctb200_adain_stats_rect if diag else U.lib().wctb200_wct_stats_rect
    _capi.check(fn(act.data_ptr(), N, H, W, C, y0, x0, h, w, buf.data_ptr(), U.stream()))
    return buf, offs


RECTS = {"whole": lambda H, W: (0, 0, H, W), "top_left": lambda H, W: (0, 0, 11, 17), "bottom_right": lambda H, W: (H - 9, W - 33, 9, 33),
         "interior": lambda H, W: (5, 7, 20, 30), "left_strip": lambda H, W: (0, 0, H, 1), "bottom_row": lambda H, W: (H - 1, 3, 1, 40)}


# ------------------------------------------------------------------------------------------------- statistics of a rect
@pytest.mark.parametrize("c", [64, 128, 256, 512])
@pytest.mark.parametrize("rect", sorted(RECTS))
def test_rect_statistics_vs_fp64(c, rect):
    N, H, W = 2, 37, 45
    x = feats(N, H, W, c, 3)
    act = U.act_from_numpy(x)
    xs = U.act_to_numpy(act, N, H, W, c).astype(np.float64)         # the SPF16 values the kernels read
    y0, x0, h, w = RECTS[rect](H, W)
    for diag in (False, True):
        buf, offs = _rect(act, N, H, W, c, y0, x0, h, w, diag)
        for i, r in enumerate(_read_record(buf, offs, c, N, diag)):
            px = xs[i, y0:y0 + h, x0:x0 + w].reshape(-1, c)
            assert r["n"] == h * w
            scale = np.abs(px).max() ** 2 * len(px)
            if diag:
                mean, var = R.moments(r)
                np.testing.assert_allclose(mean, px.mean(0), atol=1e-6 * np.abs(px).max())
                assert np.abs(var * r["n"] - px.var(0) * r["n"]).max() <= 1e-6 * scale
            else:
                mean, cov = R.covariance(r)
                np.testing.assert_allclose(mean, px.mean(0), atol=1e-6 * np.abs(px).max())
                if len(px) >= 2:
                    ref = np.cov(px, rowvar=False) * (len(px) - 1)
                    assert np.abs(cov * (r["n"] - 1) - ref).max() <= 1e-6 * scale
    U.check_device()


@pytest.mark.parametrize("c", [64, 128, 256, 512])
def test_whole_map_record_is_todays_covariance(c):
    """The record of the whole map, finalised by the expressions of k_cov_sums / k_cov_finalize (restated in float64
    here), gives wctb200_covariance's fp32 mean and covariance bit for bit: same split, same samples, same sums."""
    lib = U.lib()
    N, H, W = 2, 41, 67
    act = U.act_from_numpy(feats(N, H, W, c, 9))
    mean = torch.empty((N, c), dtype=torch.float32, device="cuda")
    cov = torch.empty((N, c, c), dtype=torch.float32, device="cuda")
    _capi.check(lib.wctb200_covariance(act.data_ptr(), N, H, W, c, 0.0, mean.data_ptr(), cov.data_ptr(), U.stream()))
    buf, offs = _rect(act, N, H, W, c, 0, 0, H, W, False)
    for i, r in enumerate(_read_record(buf, offs, c, N, False)):
        n = r["n"]
        m = (r["t"].astype(np.float32).astype(np.float64) + r["s"] / n).astype(np.float32)
        S = np.triu(r["S"]) + np.triu(r["S"], 1).T
        G = ((S - np.outer(r["s"], r["s"]) / n) / (n - 1)).astype(np.float32)
        assert np.array_equal(m.view(np.uint32), mean[i].cpu().numpy().view(np.uint32))
        assert np.array_equal(G.view(np.uint32), cov[i].cpu().numpy().view(np.uint32))


@pytest.mark.parametrize("diag", [False, True], ids=["cov", "moments"])
def test_accumulate_one_record_is_identity(diag):
    lib = U.lib()
    c, N, H, W = 128, 2, 30, 50
    act = U.act_from_numpy(feats(N, H, W, c, 4))
    b, offs = _rect(act, N, H, W, c, 3, 4, 20, 40, diag)
    a, _ = _record(c, N, diag)
    _capi.check(lib.wctb200_stats_accumulate(a.data_ptr(), b.data_ptr(), c, N, int(diag), U.stream()))
    assert torch.equal(a, b)


@pytest.mark.parametrize("c", [64, 256, 512])
@pytest.mark.parametrize("diag", [False, True], ids=["cov", "moments"])
def test_merged_records_vs_fp64_union(c, diag):
    """Tiles of a map with a strong gradient (shifts far apart), folded in tile order, against fp64 of the whole map."""
    lib = U.lib()
    N, H, W = 1, 70, 90
    rng = np.random.default_rng(6)
    yy, xx = np.mgrid[0:H, 0:W]
    x = (rng.standard_normal((N, H, W, c)) * 0.2 + (yy * 0.05 + xx * 0.03)[None, ..., None] * rng.uniform(0.5, 2, c)).astype(np.float32)
    act = U.act_from_numpy(x)
    xs = U.act_to_numpy(act, N, H, W, c).astype(np.float64).reshape(-1, c)
    acc, offs = _record(c, N, diag)
    part, _ = _record(c, N, diag)
    for y0, y1, x0, x1 in tile_grid(H, W, 32):
        _rect(act, N, H, W, c, y0, x0, y1 - y0, x1 - x0, diag, part, offs)
        _capi.check(lib.wctb200_stats_accumulate(acc.data_ptr(), part.data_ptr(), c, N, int(diag), U.stream()))
    r = _read_record(acc, offs, c, N, diag)[0]
    assert r["n"] == H * W
    # fp32 summation error: unit roundoff times the slot length (<= 4096 pixels) of sums of terms bounded by max|x - t|^2
    bound = 6e-8 * 4096 * (np.abs(xs - xs.mean(0)).max() ** 2)
    if diag:
        mean, var = R.moments(r)
        np.testing.assert_allclose(mean, xs.mean(0), atol=bound)
        assert np.abs(var - xs.var(0)).max() <= bound
    else:
        mean, cov = R.covariance(r)
        np.testing.assert_allclose(mean, xs.mean(0), atol=bound)
        assert np.abs(cov - np.cov(xs, rowvar=False)).max() <= bound


# ------------------------------------------------------------------------------------------------- transforms from a record
@pytest.mark.parametrize("c", [64, 128, 256, 512])
@pytest.mark.parametrize("nc", [1, 3])
@pytest.mark.parametrize("sem", ["tf", "np"])
def test_wct_transform_from_whole_record_equals_apply(c, nc, sem):
    lib = U.lib()
    s = SEMANTICS[sem]
    H, W, Hs, Ws = 23, 31, 19, 27
    content = U.act_from_numpy(feats(nc, H, W, c, 1))
    style = U.act_from_numpy(feats(1, Hs, Ws, c, 2, offset=0.5))
    state = _ws(lib.wctb200_wct_style_state_bytes(c, 1))
    ws = _ws(lib.wctb200_wct_workspace_bytes(c, nc, 1))
    _capi.check(lib.wctb200_wct_style_prepare(style.data_ptr(), 1, Hs, Ws, c, s["eps_cov"], s["eps_eig"], s["thresh"],
                                              state.data_ptr(), ws.data_ptr(), ws.numel(), U.stream()))
    ref = U.act_alloc(nc, H, W, c)
    kref = torch.zeros(2 * (nc + 1), dtype=torch.int32, device="cuda")
    _capi.check(lib.wctb200_wct_apply(content.data_ptr(), nc, H, W, c, state.data_ptr(), 1, 0.7, s["eps_cov"], s["eps_eig"],
                                      s["thresh"], s["readd"], ref.data_ptr(), kref.data_ptr(), ws.data_ptr(), ws.numel(), U.stream()))
    rec, _ = _rect(content, nc, H, W, c, 0, 0, H, W, False)
    om, ob, ok = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_size_t()
    tr = _ws(lib.wctb200_wct_transform_layout(c, nc, ctypes.byref(om), ctypes.byref(ob), ctypes.byref(ok)))
    _capi.check(lib.wctb200_wct_transform_from_stats(rec.data_ptr(), nc, c, state.data_ptr(), 1, 0.7, s["eps_cov"], s["eps_eig"],
                                                     s["thresh"], s["readd"], tr.data_ptr(), ws.data_ptr(), ws.numel(), U.stream()))
    out = U.act_alloc(nc, H, W, c)
    _capi.check(lib.wctb200_wct_transform_apply(content.data_ptr(), nc, H, W, c, tr.data_ptr(), out.data_ptr(), U.stream()))
    assert_bits(planes(out, nc, H, W, c), planes(ref, nc, H, W, c), "wct transform from record")
    k = tr[ok.value:ok.value + 8 * nc].view(torch.int32).cpu().numpy()
    kr = kref.cpu().numpy()
    assert np.array_equal(k[:nc], kr[:nc]) and np.array_equal(k[nc:2 * nc], kr[nc + 1:2 * nc + 1])
    U.check_device()


@pytest.mark.parametrize("c", [64, 128, 256, 512])
@pytest.mark.parametrize("nc", [1, 3])
def test_adain_transform_from_whole_record_equals_apply(c, nc):
    lib = U.lib()
    H, W, Hs, Ws = 23, 31, 19, 27
    content = U.act_from_numpy(feats(nc, H, W, c, 1))
    style = U.act_from_numpy(feats(1, Hs, Ws, c, 2, offset=0.5))
    state = _ws(lib.wctb200_adain_style_state_bytes(c, 1))
    _capi.check(lib.wctb200_adain_style_prepare(style.data_ptr(), 1, Hs, Ws, c, state.data_ptr(), U.stream()))
    ref = U.act_alloc(nc, H, W, c)
    ws = _ws(lib.wctb200_wct_workspace_bytes(c, nc, 0))
    _capi.check(lib.wctb200_adain_apply(content.data_ptr(), nc, H, W, c, state.data_ptr(), 1, 0.7, 1e-5, ref.data_ptr(),
                                        ws.data_ptr(), ws.numel(), U.stream()))
    rec, _ = _rect(content, nc, H, W, c, 0, 0, H, W, True)
    tr = _ws(lib.wctb200_adain_transform_layout(c, nc, None, None, None, None))
    _capi.check(lib.wctb200_adain_transform_from_stats(rec.data_ptr(), nc, c, state.data_ptr(), 1, 1e-5, tr.data_ptr(), U.stream()))
    out = U.act_alloc(nc, H, W, c)
    _capi.check(lib.wctb200_adain_transform_apply(content.data_ptr(), nc, H, W, c, tr.data_ptr(), 0.7, out.data_ptr(), U.stream()))
    assert_bits(planes(out, nc, H, W, c), planes(ref, nc, H, W, c), "adain transform from record")


def test_bad_arguments_are_einval():
    lib = U.lib()
    act = U.act_from_numpy(feats(1, 8, 8, 64, 1))
    buf, _ = _record(64, 1, False)
    for args in [(0, 0, 9, 8), (-1, 0, 4, 4), (0, 5, 4, 4), (0, 0, 0, 4)]:
        assert lib.wctb200_wct_stats_rect(act.data_ptr(), 1, 8, 8, 64, *args, buf.data_ptr(), U.stream()) == _capi.EINVAL
    assert lib.wctb200_wct_stats_rect(act.data_ptr(), 1, 8, 8, 64, 0, 0, 4, 4, None, U.stream()) == _capi.EINVAL
    a96 = U.act_from_numpy(feats(1, 8, 8, 96, 1))
    assert lib.wctb200_wct_stats_rect(a96.data_ptr(), 1, 8, 8, 96, 0, 0, 4, 4, buf.data_ptr(), U.stream()) == _capi.EINVAL
    assert lib.wctb200_stats_accumulate(buf.data_ptr(), buf.data_ptr(), 64, 1, 2, U.stream()) == _capi.EINVAL
    assert lib.wctb200_stats_record_layout(64, 0, 0, None, None, None, None) == 0
    assert lib.wctb200_wct_transform_layout(96, 1, None, None, None) == 0
    assert lib.wctb200_wct_transform_from_stats(None, 1, 64, buf.data_ptr(), 1, 1.0, 0.0, 0.0, 1e-5, 0, buf.data_ptr(),
                                                buf.data_ptr(), buf.numel(), U.stream()) == _capi.EINVAL
    U.check_device()


# ------------------------------------------------------------------------------------------------------------------ halos
@pytest.fixture(scope="module")
def weights():
    return make_synthetic_weights(42)


@pytest.fixture(scope="module")
def engine(weights):
    return Engine(weights, ALL, semantics="tf")


def _img(H, W, seed):
    return torch.from_numpy(np.random.default_rng(seed).random((1, H, W, 3), dtype=np.float32)).cuda()


def _interior(act, y0, x0, h, w):
    a = planes(act.buf, act.N, act.H, act.W, act.C)      # [2, N, H+2, W+2, C] raw fp16 bits
    return a[:, :, 1 + y0:1 + y0 + h, 1 + x0:1 + x0 + w]


@pytest.mark.parametrize("relu", ALL)
def test_halos_sufficient_and_needed(engine, relu):
    """On a ragged 1000 x 1496 image with T = 512, at tiles on each border and inside: the relu feature of a crop widened
    by h_A equals the untiled encoding on the interior bit for bit, and the decode of a crop widened by h_B equals the
    untiled decode of the same transformed feature on the interior; one step g less changes an interior value."""
    eng = engine
    lvl = [l for l in eng.model.levels if l.relu_target == relu][0]
    g = 2 ** (RELU_LEVEL[relu] - 1)
    h_a, h_b = tile_halos(relu)
    H, W, T = 1000, 1496, 256
    x = _img(H, W, 11)
    full, _ = eng.encode(x, relu)
    style = torch.from_numpy(np.random.default_rng(3).integers(0, 256, (1, 256, 256, 3), dtype=np.uint8)).cuda()
    ps = eng.prepare_call(style)
    torch.cuda.synchronize()
    C = lvl.channels
    rec = eng.stats_record(C, False)
    eng.stats_rect(full, 0, 0, full.H, full.W, rec, False)
    tr = eng.transform_from_stats(rec, C, ps.wct[relu], 0.8, False)
    # unclipped: a clip to [0, 1] could hide a difference
    dec_full = eng.decode(eng.transform_apply(full, tr, 0.8, False), lvl.index, clip=False).cpu().numpy()
    tiles = tile_grid(H, W, T)
    assert len(tiles) == 24                                                      # 4 rows x 6 columns
    picks = [tiles[0], tiles[8], tiles[5], tiles[18], tiles[-1]]                 # corner, inside, top right, bottom left, corner
    for y0, y1, x0, x1 in picks:
        for halo, what in ((h_a, "encode"), (h_b, "decode")):
            for h, must_match in ((halo, True), (halo - g, False)):
                cy0, cx0 = max(0, y0 - h), max(0, x0 - h)
                cy1, cx1 = min(H, y1 + h), min(W, x1 + h)
                cut = cy0 > 0 or cx0 > 0 or cy1 < H or cx1 < W
                if not must_match and not cut:
                    continue
                f, _ = eng.encode(x[:, cy0:cy1, cx0:cx1].contiguous(), relu)
                fy0, fx0 = y0 // g, x0 // g
                fh, fw = -(-y1 // g) - fy0, -(-x1 // g) - fx0
                if what == "encode":
                    got = _interior(f, fy0 - cy0 // g, fx0 - cx0 // g, fh, fw)
                    ref = _interior(full, fy0, fx0, fh, fw)
                else:
                    d = eng.decode(eng.transform_apply(f, tr, 0.8, False), lvl.index, clip=False).cpu().numpy()
                    oy1, ox1 = g * (fy0 + fh), g * (fx0 + fw)
                    got = d[:, y0 - cy0:oy1 - cy0, x0 - cx0:ox1 - cx0]
                    ref = dec_full[:, y0:oy1, x0:ox1]
                same = np.array_equal(got, ref) if what == "encode" else np.array_equal(got.view(np.uint32), ref.view(np.uint32))
                assert same == must_match, (relu, what, (y0, x0), h, must_match)
    eng.check_device()


# ----------------------------------------------------------------------------------------------------- whole pipeline
def _u8(n, H, W, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, H, W, 3), dtype=np.uint8)


@pytest.mark.parametrize("case", ["tf", "np", "adain", "passes2", "prepared", "reversed", "ragged", "batch3"])
def test_one_tile_equals_untiled(weights, case):
    targets = list(reversed(ALL)) if case == "reversed" else ALL
    wct = WCT(relu_targets=targets, weights=weights, semantics="np" if case == "np" else "tf")
    H, W = (211, 173) if case == "ragged" else (160, 192)
    n = 3 if case == "batch3" else 1
    c, s = _u8(n, H, W, 1), _u8(1, 128, 144, 2)
    kw = dict(alpha=0.8, adain=case == "adain", passes=2 if case == "passes2" else 1, return_float=True)
    if case == "prepared":
        s = wct.prepare_style(s[0])
    ref_u8, ref_f = wct.predict_batch(c, s, **kw)
    got_u8, got_f = wct.predict_batch(c, s, tile_size=256, **kw)
    assert np.array_equal(got_u8, ref_u8)
    assert np.array_equal(got_f.view(np.uint32), ref_f.view(np.uint32))
    if case == "tf":
        assert np.array_equal(wct.predict(c[0], s[0], alpha=0.8, tile_size=1024), wct.predict(c[0], s[0], alpha=0.8))


@pytest.mark.parametrize("adain", [False, True], ids=["wct", "adain"])
def test_many_tiles_teacher_forced_2048(engine, adain):
    """Every level of an untiled 2048^2 run, run again tiled from the same input image with T = 512 and T = 1024."""
    eng = engine
    H = W = 2048
    c = torch.from_numpy(_u8(1, H, W, 5)).cuda()
    s = torch.from_numpy(_u8(1, 512, 512, 6)).cuda()
    cap = {}
    eng.stylize(c, s, alpha=0.8, adain=adain, capture=cap)
    ps = eng.prepare_call(s, adain=adain)
    torch.cuda.synchronize()                 # tiled_level reads the states without waiting for the style stream
    worst = {}
    for i, lvl in enumerate(eng.model.levels):
        x = cap["level_input"][i]
        ref = cap["level_output"][i]
        state = ps.adain[lvl.relu_target] if adain else ps.wct[lvl.relu_target]
        for T in (512, 1024):
            got = eng.tiled_level(x, i, state, 0.8, adain, T, clip=i < len(ALL) - 1)
            assert got.shape == ref.shape
            err = float((got - ref).abs().max())
            worst[(lvl.relu_target, T)] = err
    print("teacher-forced tiled vs untiled, 2048^2 (%s): %s" % ("adain" if adain else "wct", worst))
    assert max(worst.values()) <= TF_TILED_BOUND, worst
    eng.check_device()


@pytest.fixture(scope="module")
def free_run(weights):
    size = 128
    content, style = _u8(1, size, size, 1000), _u8(1, size, size, 7)
    o64 = nets.pipeline(content[0], style[0], weights, ALL, alpha=0.8, semantics="np", dtype=np.float64)
    o32 = nets.pipeline(content[0], style[0], weights, ALL, alpha=0.8, semantics="np", dtype=np.float32)
    return content, style, o64, float(np.abs(o32 - o64).max())


def test_free_running_tiled_vs_oracle(weights, free_run):
    content, style, o64, noise = free_run
    bound = max(1e-3, FREE_RUN_NOISE_FACTOR * noise)
    eng = Engine(weights, ALL, semantics="np")
    outs = {}
    for T in (32, 64):
        outs[T] = eng.stylize_tiled(torch.from_numpy(content).cuda(), torch.from_numpy(style).cuda(), alpha=0.8,
                                    tile_size=T).cpu().numpy()
        err = float(np.abs(outs[T] - o64).max())
        print("free-running tiled T=%d: vs fp64 oracle %.3e (bound %.3e)" % (T, err, bound))
        assert err <= bound
    assert float(np.abs(outs[32] - outs[64]).max()) <= bound


def test_memory_4096(engine):
    eng = engine
    c = torch.from_numpy(_u8(1, 4096, 4096, 8)).cuda()
    ps = eng.prepare_call(torch.from_numpy(_u8(1, 512, 512, 9)).cuda())
    torch.cuda.synchronize()
    peaks = {}
    for name, fn in (("untiled", lambda: eng.stylize(c, ps, alpha=0.8)),
                     ("tiled", lambda: eng.stylize_tiled(c, ps, alpha=0.8, tile_size=1024))):
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = fn()
        torch.cuda.synchronize()
        peaks[name] = torch.cuda.max_memory_allocated() - base
        del out
    print("peak allocated above the resident buffers, 4096^2: untiled %.2f GB, tiled T=1024 %.2f GB"
          % (peaks["untiled"] / 1e9, peaks["tiled"] / 1e9))
    assert peaks["tiled"] <= peaks["untiled"] / 2


def test_beyond_untiled_limit_12288(engine, free_run):
    """A 12288^2 content: the untiled call is rejected (its 64-channel conv geometry exceeds the 32-bit element limit); the
    tiled call completes, and two tile sizes agree within the free-running bound."""
    eng = engine
    _, _, _, noise = free_run
    H = W = 12288
    c = torch.from_numpy(_u8(1, H, W, 12)).cuda()
    ps = eng.prepare_call(torch.from_numpy(_u8(1, 512, 512, 13)).cuda())
    with pytest.raises(_capi.WctB200Error):
        eng.stylize(c, ps, alpha=0.8)
    torch.cuda.synchronize()
    a = eng.stylize_tiled(c, ps, alpha=0.8, tile_size=2048)
    assert a.shape == (1, H, W, 3) and bool(torch.isfinite(a).all())
    b = eng.stylize_tiled(c, ps, alpha=0.8, tile_size=3072)
    err = float((a - b).abs().max())
    print("12288^2 tiled T=2048 vs T=3072: max-abs %.3e" % err)
    assert err <= max(1e-3, FREE_RUN_NOISE_FACTOR * noise)
    eng.check_device()


@pytest.mark.parametrize("kw", [dict(content_mask=np.zeros((8, 8), np.uint8)), dict(style_weights=[1.0]), dict(swap5=True),
                                dict(swap_targets=["relu3_1"]), dict(temporal="state"), dict(tile_size=24), dict(tile_size=-16),
                                dict(tile_size=8.5)],
                         ids=["content_mask", "style_weights", "swap5", "swap_targets", "temporal", "not_multiple", "negative",
                              "float"])
def test_tiled_rejections(weights, kw):
    wct = WCT(relu_targets=["relu3_1", "relu1_1"], weights=make_synthetic_weights(1, relu_targets=["relu3_1", "relu1_1"]))
    kw = dict(kw)
    if kw.get("temporal") == "state":
        kw["temporal"] = wct.temporal_state(0.5)
    kw.setdefault("tile_size", 64)
    c, s = _u8(1, 64, 64, 1), _u8(1, 64, 64, 2)
    with pytest.raises(ValueError):
        wct.predict_batch(c, [s[0]] if ("content_mask" in kw or "style_weights" in kw) else s, **kw)
    with pytest.raises(ValueError):
        wct.predict_batch(c, [s[0]], content_mask=np.zeros((8, 8), np.uint8), style_masks=[np.zeros((8, 8), np.uint8)],
                          tile_size=64)


def test_tiled_synthesize_and_out(weights):
    wct = WCT(relu_targets=["relu3_1", "relu1_1"], weights=make_synthetic_weights(1, relu_targets=["relu3_1", "relu1_1"]))
    s = _u8(1, 64, 64, 2)[0]
    ref = wct.synthesize(s, (96, 80), count=2, seed=3)
    got = wct.synthesize(s, (96, 80), count=2, seed=3, tile_size=512)
    assert np.array_equal(ref, got)
    out = torch.empty((2, 96, 80, 3), dtype=torch.uint8).pin_memory()
    r = wct.synthesize(s, (96, 80), count=2, seed=3, tile_size=32, out=out)
    assert r is out and out.shape == (2, 96, 80, 3)
    dev = wct.synthesize(s, (96, 80), count=2, seed=3, tile_size=32, return_device=True)
    assert torch.equal(dev.cpu(), out)
