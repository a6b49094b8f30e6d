"""Sliced distribution matching (DESIGN.md §3.3.14) on the GPU: the rotation against float64, one step with an exact
(signed-permutation) rotation against the EFDM oracle, a K = 4 chain against ``tests/sliced_ref.py``, byte identity over
workspace sizes, batches, shared styles and runs, offsets past 2^31, and the engine and API paths.

Along a chain of rotations per-pixel equality with the oracle is not well posed: a last-bit difference in a projected
value can swap two adjacent ranks at a later step.  So the chain is compared by its sorted per-channel marginals (which
such a swap does not move) and by a sliced Wasserstein distance over held-out directions; per-pixel equality is asked
only of single steps with exact rotations."""
import gc
import zlib

import numpy as np
import pytest
import torch

from oracle import nets
from tests import gpu_util as U
from tests import sliced_ref as SR
from tests.test_gpu_efdm import _content, _style, _tol, _u8, _ws, act_exact, prepare
from tests.test_gpu_invariance import assert_bits, planes
from wct_tf_b200 import _capi, sliced
from wct_tf_b200.engine import Engine
from wct_tf_b200.wct import WCT
from wct_tf_b200.weights import make_synthetic_weights

pytestmark = pytest.mark.gpu
ALL = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def rot_prepare(style, ns, hs, ws_, c, R, max_segments=1 << 30):
    lib = U.lib()
    state = _ws(lib.wctb200_efdm_style_state_bytes(c, ns, hs, ws_))
    ws = _ws(lib.wctb200_efdm_style_workspace_bytes(c, ns, hs, ws_, max_segments))
    Rd = _dev(R)
    _capi.check(lib.wctb200_efdm_rotated_style_prepare(style.data_ptr(), ns, hs, ws_, c, Rd.data_ptr(), state.data_ptr(),
                                                       ws.data_ptr(), ws.numel(), U.stream()))
    return state


def step(content, src, n, h, w, c, G, state, ns, hs, ws_, alpha=1.0, to_planes=False, max_segments=1 << 30):
    """One sliced step through the C ABI: returns the fp32 planes [n][c][h*w] or the SPF16 output."""
    lib = U.lib()
    ws = _ws(lib.wctb200_efdm_workspace_bytes(c, n, h, w, max_segments))
    Gd = _dev(G)
    if to_planes:
        dst = _ws(lib.wctb200_efdm_planes_bytes(c, n, h, w))
        out = None
    else:
        dst, out = None, U.act_alloc(n, h, w, c)
    _capi.check(lib.wctb200_efdm_sliced_step(content.data_ptr() if content is not None else None,
                                             src.data_ptr() if src is not None else None, n, h, w, c, Gd.data_ptr(),
                                             state.data_ptr(), ns, hs, ws_, float(alpha),
                                             dst.data_ptr() if dst is not None else None,
                                             out.data_ptr() if out is not None else None, ws.data_ptr(), ws.numel(), U.stream()))
    return dst if to_planes else out


def chain(content, style, n, h, w, c, ns, hs, ws_, K, alpha, max_segments=1 << 30):
    """The whole chain of K slices through the C ABI, with every state made up front."""
    Gs = sliced.step_matrices(c, K)
    states = [rot_prepare(style, ns, hs, ws_, c, R) for R in sliced.rotations(c, K)] + [prepare(style, ns, hs, ws_, c)]
    src = None
    for k in range(K + 1):
        last = k == K
        res = step(content, src, n, h, w, c, Gs[k], states[k], ns, hs, ws_, alpha, to_planes=not last,
                   max_segments=max_segments)
        src = res
    return res


def plane_values(buf, n, c, L):
    torch.cuda.synchronize()
    return buf[:n * c * L * 4].view(torch.float32).view(n, c, L).cpu().numpy()


def _fma_bound(G, v):
    """The standard fp32 dot-product bound of y = G v, element by element: C 2^-23 sum_j |G_cj| |v_j|."""
    C = G.shape[0]
    return C * 2.0 ** -23 * (np.abs(v).astype(np.float64) @ np.abs(G).astype(np.float64).T)


@pytest.mark.parametrize("c", [64, 128, 256, 512])
def test_rotation_vs_fp64(c):
    """k_efdm_rotate_keys: 1x1 styles (one value per channel, so the state is R v element by element) from the SPF16
    layout; a 37x41 style's sorted values per channel; and the planes layout, which must give the SPF16 layout's bytes."""
    rng = np.random.default_rng(c)
    R = sliced.rotations(c, 1)[0]
    ns = 300
    style, v = act_exact(rng.standard_normal((ns, 1, 1, c)) * rng.uniform(0.2, 3.0, c))
    got = rot_prepare(style, ns, 1, 1, c, R)[:ns * c * 4].view(torch.float32).view(ns, c).cpu().numpy()
    v = v.reshape(ns, c).astype(np.float64)
    ref = v @ R.astype(np.float64).T
    err = np.abs(got - ref)
    bound = _fma_bound(R, v)
    print("C=%d: max |R v - fp64| %.3e, max ratio to the bound %.3f" % (c, err.max(), (err / bound).max()))
    assert np.all(err <= bound)
    # a larger style: the sorted values of each channel against the sorted fp64 projections, within the channel's bound
    hs, ws_ = 37, 41
    style2, v2 = act_exact(np.maximum(rng.standard_normal((1, hs, ws_, c)), 0))
    st = rot_prepare(style2, 1, hs, ws_, c, R)[:c * hs * ws_ * 4].view(torch.float32).view(c, hs * ws_).cpu().numpy()
    v2 = v2.reshape(-1, c).astype(np.float64)
    ref2 = np.sort(v2 @ R.astype(np.float64).T, axis=0).T
    assert np.all(np.abs(st - ref2) <= _fma_bound(R, v2).max(axis=0)[:, None])
    # the planes layout: the same values as fp32 channel-major planes give the same step bytes as the SPF16 layout
    n, h, w = 2, 21, 19
    x = np.maximum(rng.standard_normal((n, h, w, c)), 0).astype(np.float32)
    content, xv = act_exact(x)
    pl = _dev(xv.reshape(n, h * w, c).transpose(0, 2, 1))
    state = prepare(style2, 1, hs, ws_, c)
    a = step(content, None, n, h, w, c, R, state, 1, hs, ws_, to_planes=True)
    b = step(None, pl, n, h, w, c, R, state, 1, hs, ws_, to_planes=True)
    torch.cuda.synchronize()
    assert torch.equal(a, b), "planes and SPF16 input layouts differ"


def _signed_perm(c, seed):
    rng = np.random.default_rng(seed)
    G = np.zeros((c, c), np.float32)
    G[np.arange(c), rng.permutation(c)] = rng.choice([-1.0, 1.0], c)
    return G


@pytest.mark.parametrize("c,kind,alpha", [(64, "ties", 1.0), (128, "negative", 0.7), (256, "distinct", 0.6)])
def test_signed_permutation_steps_vs_efdm_oracle(c, kind, alpha):
    """Two steps with signed-permutation G (exact in fp32): SPF16 -> planes -> SPF16 blended with the content, on the
    spaced inputs of test_gpu_efdm.py, against the EFDM oracle at EFDM's tolerance."""
    n, h, w, hs, ws_ = 2, 29, 33, 27, 31
    rng = np.random.default_rng(zlib.crc32(("%d%s" % (c, kind)).encode()))
    content = U.act_from_numpy(_content(rng, n, h, w, c, kind))
    x = U.act_to_numpy(content, n, h, w, c).reshape(n, -1, c).astype(np.float64)
    style, s = act_exact(_style(rng, 1, hs, ws_, c, 0.3))
    s = s.reshape(-1, c).astype(np.float64)
    G1, G2 = _signed_perm(c, 1), _signed_perm(c, 2)
    R2 = G2 @ G1          # the basis of step 2: a signed permutation too, exact
    st1 = rot_prepare(style, 1, hs, ws_, c, G1)
    st2 = rot_prepare(style, 1, hs, ws_, c, R2)
    m1 = step(content, None, n, h, w, c, G1, st1, 1, hs, ws_, to_planes=True)
    out = step(content, m1, n, h, w, c, G2, st2, 1, hs, ws_, alpha)
    got1 = plane_values(m1, n, c, h * w).transpose(0, 2, 1)
    got = U.act_to_numpy(out, n, h, w, c).reshape(n, -1, c)
    tol = _tol(float(np.abs(s).max()), float(np.abs(x).max()))
    for i in range(n):
        ref1 = SR.step(x[i], G1, s @ G1.astype(np.float64).T)
        ref = SR.step(ref1, G2, s @ R2.astype(np.float64).T, alpha, blend_with=x[i])
        e1, e2 = float(np.abs(got1[i] - ref1).max()), float(np.abs(got[i] - ref).max())
        print("C=%d %s frame %d: step 1 %.3e, step 2 %.3e (tolerance %.3e)" % (c, kind, i, e1, e2, tol))
        assert e1 <= tol and e2 <= tol


def sorted_marginal_error(got, ref, tol):
    """Per channel, the device's sorted values against the oracle's [Nc, C]: the largest error beyond ``tol`` and the share
    of values in runs the rounding merged.  Ranks are unstable along the chain, so the sorted values are what is well posed, with one
    exception: projected values that round to the same fp32 number form a run in the device's sort that the float64
    oracle does not see, and all of a run take the mean of its ranks' quantiles.  Such a run is held to the oracle's
    range over its ranks; every other rank to ``tol``."""
    worst, tied = 0.0, 0
    for j in range(got.shape[1]):
        g, r = np.sort(got[:, j]), np.sort(ref[:, j])
        start = np.flatnonzero(np.concatenate([[True], g[1:] != g[:-1]]))
        end = np.concatenate([start[1:], [len(g)]])
        for a, b in zip(start, end):
            if b - a == 1:
                worst = max(worst, abs(g[a] - r[a]) - tol)
            else:                           # a run; one the oracle has too (equal style quantiles) is no merge
                if r[b - 1] - r[a] > tol:
                    tied += b - a
                worst = max(worst, r[a] - tol - g[a], g[a] - r[b - 1] - tol)
    return worst, tied / got.size


def _mixture(rng, n, h, w, c, scale=1.0):
    """ReLU'd mixture of two correlated Gaussians: non-Gaussian, with exact zeros and correlated channels."""
    A = rng.standard_normal((c, c)) / np.sqrt(c)
    z = rng.standard_normal((n, h * w, c)) @ A.T
    z[:, : h * w // 2] += 1.5 * rng.standard_normal(c)
    return (scale * np.maximum(z, 0)).reshape(n, h, w, c).astype(np.float32)


@pytest.mark.parametrize("c", [64, 128])
def test_chain_k4_vs_oracle(c):
    """K = 4 on the device's own input: per channel the sorted output matches the oracle's within EFDM's tolerance, and the
    held-out sliced-W1 to the style is within 1 % of the oracle's."""
    K, n, h, w, hs, ws_ = 4, 1, 48, 40, 44, 46
    rng = np.random.default_rng(c + 7)
    content = U.act_from_numpy(_mixture(rng, n, h, w, c))
    x = U.act_to_numpy(content, n, h, w, c)
    style, s = act_exact(_mixture(np.random.default_rng(c + 8), 1, hs, ws_, c, 1.7))
    out = chain(content, style, n, h, w, c, 1, hs, ws_, K, 1.0)
    got = U.act_to_numpy(out, n, h, w, c).reshape(-1, c)
    ref = SR.sliced_efdm(x, s, K).reshape(-1, c)
    tol = _tol(float(np.abs(s).max()), float(np.abs(x).max()))
    e = float(np.abs(np.sort(got, 0) - np.sort(ref, 0)).max())
    over, tied = sorted_marginal_error(got, ref, tol)
    dirs = SR.held_out_directions(c, 256)
    sw_got, sw_ref = SR.sliced_w1(got, s.reshape(-1, c), dirs), SR.sliced_w1(ref, s.reshape(-1, c), dirs)
    sw0 = SR.sliced_w1(x.reshape(-1, c), s.reshape(-1, c), dirs)
    print("C=%d K=%d: sorted marginals max %.3e, beyond tolerance %.3e outside ties (tolerance %.3e), %.4f%% tied; "
          "sliced-W1 device %.5f oracle %.5f (content %.5f)" % (c, K, e, over, tol, 100 * tied, sw_got, sw_ref, sw0))
    assert over <= 0 and tied <= 0.001
    assert abs(sw_got - sw_ref) <= 0.01 * sw_ref


def _chain_bytes(name, n, shared, max_segments=1 << 30, frames=None):
    c, h, w, hs, ws_, K, alpha = 128, 26, 30, 22, 24, 2, 0.8
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    x = _mixture(rng, n, h, w, c)
    ns = 1 if shared else n
    s = _mixture(np.random.default_rng(5), ns, hs, ws_, c, 1.5)
    if frames is not None:
        x = x[frames]
        s = s if shared else s[frames]
        n, ns = len(frames), (1 if shared else len(frames))
    content = U.act_from_numpy(x)
    style, _ = act_exact(s)
    return planes(chain(content, style, n, h, w, c, ns, hs, ws_, K, alpha, max_segments), n, h, w, c)


def test_byte_identity():
    full = _chain_bytes("bytes", 3, False)
    assert_bits(_chain_bytes("bytes", 3, False), full, "two runs")
    for segs in (1, 5, 100):                 # chunks that start and end inside a 64-channel rotation block
        assert_bits(_chain_bytes("bytes", 3, False, max_segments=segs), full, "%d segments per chunk" % segs)
    for i in range(3):
        assert_bits(_chain_bytes("bytes", 3, False, frames=[i])[:, 0], full[:, i], "frame %d alone" % i)
    shared = _chain_bytes("bytes", 3, True)
    c, h, w, hs, ws_ = 128, 26, 30, 22, 24
    x = _mixture(np.random.default_rng(zlib.crc32(b"bytes")), 3, h, w, c)
    s = np.repeat(_mixture(np.random.default_rng(5), 1, hs, ws_, c, 1.5), 3, axis=0)
    content = U.act_from_numpy(x)
    style, _ = act_exact(s)
    rep = planes(chain(content, style, 3, h, w, c, 3, hs, ws_, 2, 0.8), 3, h, w, c)
    assert_bits(rep, shared, "a shared style against the same style repeated per frame")


def test_alpha_zero_and_rejections():
    lib = U.lib()
    c, n, h, w = 64, 2, 6, 5
    content = U.act_from_numpy(np.random.default_rng(1).standard_normal((n, h, w, c)).astype(np.float32))
    style, _ = act_exact(np.ones((1, 3, 3, c), np.float32))
    state = prepare(style, 1, 3, 3, c)
    G = np.eye(c, dtype=np.float32)
    out = step(content, None, n, h, w, c, G, state, 1, 3, 3, alpha=0.0)
    assert_bits(planes(out, n, h, w, c), planes(content, n, h, w, c), "alpha = 0")
    ws = _ws(lib.wctb200_efdm_workspace_bytes(c, n, h, w, 1))
    Gd = _dev(G)
    dst = _ws(lib.wctb200_efdm_planes_bytes(c, n, h, w))
    o = U.act_alloc(n, h, w, c)

    def call(cnt, src, C, ns, alpha, pl, out_, g=Gd):
        return lib.wctb200_efdm_sliced_step(cnt, src, n, h, w, C, g.data_ptr() if g is not None else None, state.data_ptr(), ns,
                                            3, 3, alpha, pl, out_, ws.data_ptr(), ws.numel(), U.stream())
    assert call(content.data_ptr(), None, c, 1, 1.0, dst.data_ptr(), None) == 0
    assert call(content.data_ptr(), None, c, 1, 1.0, None, o.data_ptr()) == 0
    assert call(None, None, c, 1, 1.0, dst.data_ptr(), None) == _capi.EINVAL                 # no input
    assert call(content.data_ptr(), None, c, 1, 1.0, dst.data_ptr(), o.data_ptr()) == _capi.EINVAL   # two outputs
    assert call(None, dst.data_ptr(), c, 1, 1.0, None, o.data_ptr()) == _capi.EINVAL         # a blend needs the content
    assert call(content.data_ptr(), None, c, 1, 1.0, dst.data_ptr(), None, g=None) == _capi.EINVAL
    assert call(content.data_ptr(), None, 32, 1, 1.0, dst.data_ptr(), None) == _capi.EINVAL  # C % 64
    assert call(content.data_ptr(), None, c, 3, 1.0, dst.data_ptr(), None) == _capi.EINVAL   # Ns not in {1, N}
    assert call(content.data_ptr(), None, c, 1, float("inf"), None, o.data_ptr()) == _capi.EINVAL
    assert lib.wctb200_efdm_planes_bytes(96, n, h, w) == 0
    assert lib.wctb200_efdm_rotated_style_prepare(style.data_ptr(), 1, 3, 3, c, None, state.data_ptr(), ws.data_ptr(),
                                                  ws.numel(), U.stream()) == _capi.EINVAL
    torch.cuda.synchronize()


def test_large_offsets_frame_2_alone():
    """K = 1 at relu1_1 on three 3584^2 frames: frame 2's elements lie past 2^31 in the SPF16 planes and in the fp32 plane
    buffer; its bytes equal the frame alone.  (The sort's keys are per chunk, here 16 segments.)"""
    n, h, w, c = 3, 3584, 3584, 64
    from tests.test_gpu_large_offsets import act_of, pl
    gc.collect()
    torch.cuda.empty_cache()
    buf = U.act_alloc(n, h, w, c, poison=False)
    dst = pl(buf, n, h, w, c)
    for i in range(n):
        g = torch.Generator(device="cuda").manual_seed(40 + i)
        x = torch.relu(torch.randn(1, h, w, c, generator=g, device="cuda") - 0.3 * (i + 1))
        one = act_of(x)
        dst[:, i:i + 1].copy_(pl(one, 1, h, w, c))
        del one, x
    style, _ = act_exact(_mixture(np.random.default_rng(3), 1, 300, 280, c))
    assert 2 * c * h * w < 2 ** 31 < 3 * c * h * w
    out = chain(buf, style, n, h, w, c, 1, 300, 280, 1, 1.0, max_segments=16)
    last = pl(out, n, h, w, c)[:, 2:3].clone()
    del out
    gc.collect()
    torch.cuda.empty_cache()
    one_in = U.act_alloc(1, h, w, c, poison=False)
    pl(one_in, 1, h, w, c).copy_(pl(buf, n, h, w, c)[:, 2:3])
    del buf
    gc.collect()
    torch.cuda.empty_cache()
    one = chain(one_in, style, 1, h, w, c, 1, 300, 280, 1, 1.0, max_segments=64)
    U.check_device()
    assert torch.equal(pl(one, 1, h, w, c), last), "frame 2 of 3 at 3584^2 differs from the frame alone"
    del one, last, one_in
    gc.collect()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------ engine and API
@pytest.fixture(scope="module")
def weights():
    return make_synthetic_weights(42)


def _style_feats(eng, style_u8):
    x = torch.empty(style_u8.shape, dtype=torch.float32, device="cuda")
    t = torch.from_numpy(style_u8).cuda()
    _capi.check(U.lib().wctb200_image_u8_to_f32(t.data_ptr(), t.numel(), x.data_ptr(), U.stream()))
    _, feats = eng.encode(x, eng.model.deepest_target, taps=eng.model.style_taps)
    return feats


def test_slices_zero_is_efdm(weights):
    eng = Engine(weights, ALL)
    c, s = torch.from_numpy(_u8(2, 96, 80, 1)).cuda(), torch.from_numpy(_u8(1, 64, 72, 2)).cuda()
    cap0, cap1 = {}, {}
    a = eng.stylize(c, s, alpha=0.8, efdm=True, capture=cap0)
    b = eng.stylize(c, s, alpha=0.8, efdm=True, efdm_slices=0, capture=cap1)
    for i in range(len(ALL)):
        assert torch.equal(cap0["transformed"][i].buf, cap1["transformed"][i].buf), ALL[i]
    assert torch.equal(a, b)
    eng.check_device()


def test_teacher_forced_levels(weights):
    """At every level of a five-level 128^2 run with K = 3 at alpha = 1, the sorted marginals of the device's transform of
    its own content feature against its own style feature are within EFDM's tolerance of the oracle's, and the level's
    decode is within 1e-3 of fp64."""
    K = 3
    eng = Engine(weights, ALL)
    content, style = _u8(1, 128, 128, 100), _u8(1, 144, 144, 101)
    cap = {}
    eng.stylize(torch.from_numpy(content).cuda(), torch.from_numpy(style).cuda(), alpha=1.0, capture=cap, efdm=True,
                efdm_slices=K)
    sf = _style_feats(eng, style)
    eng.check_device()
    for i, relu in enumerate(ALL):
        x = eng.act_to_f32(cap["content_feat"][i]).cpu().numpy()
        s = eng.act_to_f32(sf[relu]).cpu().numpy()
        C = x.shape[-1]
        ref = SR.sliced_efdm(x, s, K).reshape(-1, C)
        got = eng.act_to_f32(cap["transformed"][i]).cpu().numpy()
        tol = _tol(float(np.abs(s).max()), float(np.abs(x).max()))
        e_t, tied = sorted_marginal_error(got.reshape(-1, C), ref, tol)
        y = nets.decode(got.astype(np.float64), weights, relu, np.float64)
        if i < len(ALL) - 1:
            y = np.clip(y, 0, 1)
        e_out = float(np.abs(cap["level_output"][i].cpu().numpy() - y).max())
        print("%s: sorted marginals beyond tolerance %.2e outside ties (tolerance %.2e), %.4f%% tied  level output %.2e"
              % (relu, e_t, tol, 100 * tied, e_out))
        assert e_t <= 0 and tied <= 0.001 and e_out <= 1e-3


def test_held_out_sliced_w1_below_efdm(weights):
    """On real encoder features of a 256^2 content at alpha = 1, the sliced-W1 to the style over held-out directions is
    lower at K = 8 than EFDM's at every level with at least as many positions as channels (WCT's printed beside them).
    relu5_1 has 256 positions for 512 channels: there EFDM's distance is already at the floor the finite samples leave
    (measured on an H100: EFDM 0.06786, K = 8 0.06788), and K = 8 is held to within 0.5 % of it."""
    eng = Engine(weights, ALL)
    content, style = _u8(1, 256, 256, 3), _u8(1, 256, 256, 4)
    cf_all, sf = _style_feats(eng, content), _style_feats(eng, style)
    for relu in ALL:
        cf, s_act = cf_all[relu], sf[relu]
        C = cf.C
        s = eng.act_to_f32(s_act).cpu().numpy().reshape(-1, C)
        dirs = SR.held_out_directions(C, 256)
        st = dict(eng.efdm_prepare(s_act), slices=8, rot=None)
        d = {}
        for name in ("content", "efdm", "sliced8", "wct"):
            if name == "content":
                f = cf
            elif name == "efdm":
                f, _ = eng.efdm_apply(cf, st, 1, 1.0)
            elif name == "sliced8":
                f, _ = eng.efdm_sliced_apply(cf, st, 1, 1.0, s_act)
            else:
                f, _ = eng.transform(cf, s_act, 1.0, False)
            d[name] = SR.sliced_w1(eng.act_to_f32(f).cpu().numpy().reshape(-1, C), s, dirs)
        print("%s: held-out sliced-W1 content %.4g  efdm %.4g  sliced K=8 %.4g  wct %.4g"
              % (relu, d["content"], d["efdm"], d["sliced8"], d["wct"]))
        if cf.H * cf.W >= C:
            assert d["sliced8"] < d["efdm"]
        else:
            assert d["sliced8"] <= 1.005 * d["efdm"]
    eng.check_device()


def test_options(weights):
    """passes (a shared or per-frame style prepared once per call), groups, swap levels, seamless, synthesize, temporal
    and return_float; a shared style gives the bytes of the same style per frame."""
    wct = WCT(relu_targets=ALL, weights=weights)
    eng = wct.engine
    c, s, s3 = _u8(3, 64, 80, 4), _u8(1, 64, 64, 5), _u8(3, 64, 64, 6)
    kw = dict(alpha=0.8, efdm=True, efdm_slices=2)
    one = wct.predict_batch(c, s, **kw)
    assert not np.array_equal(one, wct.predict_batch(c, s, alpha=0.8, efdm=True))
    assert np.array_equal(wct.predict_batch(c, np.repeat(s, 3, axis=0), **kw), one)
    for i in range(3):
        assert np.array_equal(wct.predict_batch(c[i:i + 1], s, **kw)[0], one[i])
    assert np.array_equal(wct.predict_batch(c, s, passes=2, **kw), wct.predict_batch(one, s, **kw))
    per = wct.predict_batch(c, s3, **kw)
    assert np.array_equal(wct.predict_batch(c, s3, passes=2, **kw), wct.predict_batch(per, s3, **kw))
    g0 = eng.groups
    eng.groups = 2
    try:
        assert np.array_equal(wct.predict_batch(c, s, **kw), one)
        assert np.array_equal(wct.predict_batch(c, s3, **kw), per)
    finally:
        eng.groups = g0
    u8, f = wct.predict_batch(c, s, return_float=True, **kw)
    assert np.array_equal(u8, one) and f.dtype == np.float32
    assert np.array_equal(wct.predict(c[0], s[0], **kw), one[0])
    # swap levels still swap; the other levels run the chain
    cap = {}
    sw = eng.stylize(torch.from_numpy(c[:1]).cuda(), torch.from_numpy(s).cuda(), swap_targets=["relu5_1"], capture=cap, **kw)
    assert sw.shape[0] == 1
    from wct_tf_b200.device_image import noise_u8
    tex = wct.synthesize(s[0], (64, 96), count=2, seed=5, **kw)
    assert np.array_equal(tex, wct.predict_batch(noise_u8(2, 64, 96, seed=5, device=eng.device), s[0], **kw))
    sl = eng.stylize(torch.from_numpy(c[:1]).cuda(), torch.from_numpy(s).cuda(), seamless="xy", **kw)
    assert torch.isfinite(sl).all()
    st = wct.temporal_state(0.5)
    out = wct.predict_batch(c, s, temporal=st, **kw)
    assert np.array_equal(out[0], one[0])
    eng.check_device()


@pytest.mark.parametrize("bad", [-1, 33, 2.0, True, "4"])
def test_rejections_before_any_launch(weights, bad):
    wct = WCT(relu_targets=["relu3_1", "relu1_1"], weights=make_synthetic_weights(1, relu_targets=["relu3_1", "relu1_1"]))
    c, s = _u8(1, 32, 32, 1), _u8(1, 32, 32, 2)
    n0 = wct.engine.launches
    with pytest.raises(ValueError, match="efdm_slices"):
        wct.predict_batch(c, s, efdm=True, efdm_slices=bad)
    with pytest.raises(ValueError, match="efdm_slices needs efdm"):
        wct.predict_batch(c, s, efdm_slices=2)
    with pytest.raises(ValueError, match="efdm"):
        wct.predict_batch(c, s, efdm=True, efdm_slices=2, adain=True)
    with pytest.raises(ValueError, match="efdm_slices"):
        wct.engine.stylize(torch.from_numpy(c).cuda(), torch.from_numpy(s).cuda(), efdm=True, efdm_slices=bad)
    assert wct.engine.launches == n0
    eng = wct.engine
    ps = eng.prepare_call(torch.from_numpy(s).cuda(), efdm=True, efdm_slices=2)
    with pytest.raises(ValueError, match="efdm_slices"):
        eng.stylize(torch.from_numpy(c).cuda(), ps, efdm=True, efdm_slices=3)
