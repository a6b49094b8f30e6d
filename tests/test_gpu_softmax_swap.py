"""The softmax style swap (DESIGN.md §3.3.17) on the device.

1. C-ABI accuracy: at C in {64,128,256,512}, (P,S) in {(3,1),(5,2)}, Nc in {1,3} and temperatures from near-hard to
   near-uniform, the swapped feature (read back from the workspace) is within 1e-3 of the float64 oracle evaluated on the
   device's own whitened content and style; with rank-deficient content and a padded last patch block.
2. Invariance: every workspace size from the minimum (one block) to one chunk gives the same bytes; frame i of a batch
   equals that frame alone, bit for bit.
3. The hard limit: at tau = 1e-4 and 1e-7 the swapped feature equals the hard apply's within fp32 rounding, and the
   coloured output within 1e-5 of its largest value, wherever every covering anchor has a z-margin above 50 tau; the
   output is finite everywhere.
4. Labels: uniform labels give the unlabelled softmax bytes; block labels with a label absent from the style match the
   masked oracle.
5. Engine: teacher-forced five-level runs with the softmax swap at relu5_1 and relu3_1; the default workspace policy at
   relu3_1 at 512^2 gives the one-chunk bytes; a prepared style gives the image style's bytes; ss_temperature=None gives
   the bytes of leaving it out; bad temperatures are WCTB200_EINVAL.
"""
import ctypes

import numpy as np
import pytest
import torch

from oracle import nets, ref_ops
from tests import gpu_util as U
from tests import softmax_swap_ref as SR
from tests import swap_labels_ref as SLR
from tests.test_gpu_invariance import assert_bits, frame_copy, planes
from wct_tf_b200 import _capi
from wct_tf_b200.engine import Engine
from wct_tf_b200.weights import make_synthetic_weights

pytestmark = pytest.mark.gpu
TF = (1e-8, 1e-5)
ALL = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]
GATE = 1e-3
BLOCK = 256
# content h=w, style h=w per (patch, stride): 289 patches (cout_pad 320: a full block and a padded one) and 361 (384)
GEOM = {(3, 1): (18, 19), (5, 2): (21, 41)}


def _ws(nbytes):
    return torch.full((max(int(nbytes), 1),), 255, dtype=torch.uint8, device="cuda")   # 0xffff: an fp16 NaN


def _layout(c, nc, hc, wc, hs, ws_, p, s):
    """Where the apply leaves its stages (wctb200_debug_style_swap_layout; the softmax workspace begins with that layout)."""
    out = (ctypes.c_longlong * 11)()
    _capi.check(U.lib().wctb200_debug_style_swap_layout(c, nc, hc, wc, hs, ws_, p, s, out))
    keys = ("n_patches", "cout_pad", "ho", "wo", "feat", "norms", "wsplit", "wc_feat", "scores", "idx", "ss_feat")
    return dict(zip(keys, [int(v) for v in out]))


def _fp16_planes(buf, off, n, h, w, c):
    nb = 2 * n * (h + 2) * (w + 2) * c * 2
    return buf[off:off + nb].view(torch.float16).view(2, n, h + 2, w + 2, c).cpu().numpy()


def _setup(c, p, s, nc, seed, hc, hs, dead=0):
    lib = U.lib()
    rng = np.random.default_rng(seed)
    content = np.maximum(rng.standard_normal((nc, hc, hc, c)) + 0.3, 0).astype(np.float32)
    if dead:
        content[..., :dead] = 0.0                         # rank-deficient: dead channels
    style = np.maximum(rng.standard_normal((1, hs, hs, c)) + 0.4, 0).astype(np.float32)
    cin, sin = U.act_from_numpy(content), U.act_from_numpy(style)
    state = _ws(lib.wctb200_style_swap_state_bytes(c, hs, hs, p, s))
    pws = _ws(lib.wctb200_style_swap_prepare_workspace_bytes(c, hs, hs, p, s))
    _capi.check(lib.wctb200_style_swap_prepare(sin.data_ptr(), hs, hs, c, p, s, *TF, state.data_ptr(), None, pws.data_ptr(),
                                               pws.numel(), U.stream()))
    L = _layout(c, nc, hc, hc, hs, hs, p, s)
    full = lib.wctb200_style_swap_softmax_workspace_bytes(c, nc, hc, hc, hs, hs, p, s)
    least = lib.wctb200_style_swap_softmax_min_workspace_bytes(c, nc, hc, hc, hs, hs, p, s)
    return dict(lib=lib, c=c, p=p, s=s, nc=nc, hc=hc, hs=hs, cin=cin, state=state, L=L, full=full, least=least)


def _softmax(d, tau, nbytes=None, cl=None, sl=None, alpha=0.6, cin=None, nc=None):
    """The softmax apply through the C-ABI; returns (rc, output planes, k_out, workspace)."""
    lib, c, p, s, hc, hs = d["lib"], d["c"], d["p"], d["s"], d["hc"], d["hs"]
    nc = d["nc"] if nc is None else nc
    cin = d["cin"] if cin is None else cin
    aws = _ws(d["full"] if nbytes is None else nbytes)
    out = U.act_alloc(nc, hc, hc, c)
    kout = torch.full((nc + 1,), -7, dtype=torch.int32, device="cuda")
    lab = (None, 0, 0, 0, None, 0, 0)
    lbuf = None
    if cl is not None:
        lbuf = _ws(lib.wctb200_style_swap_labels_workspace_bytes(cl.shape[0], hc, hc, hs, hs, p, s))
        lab = (cl.data_ptr(), cl.shape[0], cl.shape[1], cl.shape[2], sl.data_ptr(), sl.shape[-2], sl.shape[-1])
    rc = lib.wctb200_style_swap_apply_softmax(cin.data_ptr(), nc, hc, hc, c, d["state"].data_ptr(), hs, hs, p, s, alpha, *TF,
                                              float(tau), *lab, out.data_ptr(), kout.data_ptr(), aws.data_ptr(), aws.numel(),
                                              None if lbuf is None else lbuf.data_ptr(), 0 if lbuf is None else lbuf.numel(),
                                              U.stream())
    if rc:
        return rc, None, None, None
    U.check_device()
    torch.cuda.synchronize()
    return rc, planes(out, nc, hc, hc, c), kout.cpu().numpy(), aws


def _hard(d, nbytes=None, alpha=0.6):
    lib, c, p, s, hc, hs, nc = d["lib"], d["c"], d["p"], d["s"], d["hc"], d["hs"], d["nc"]
    aws = _ws(lib.wctb200_style_swap_apply_workspace_bytes(c, nc, hc, hc, hs, hs, p, s) if nbytes is None else nbytes)
    out = U.act_alloc(nc, hc, hc, c)
    _capi.check(lib.wctb200_style_swap_apply(d["cin"].data_ptr(), nc, hc, hc, c, d["state"].data_ptr(), hs, hs, p, s, alpha, *TF,
                                             out.data_ptr(), None, aws.data_ptr(), aws.numel(), U.stream()))
    U.check_device()
    torch.cuda.synchronize()
    return planes(out, nc, hc, hc, c), aws


def _merged(pl):
    """fp32 values of SPF16 planes given as int16 bits [2][n][h+2][w+2][c] or fp16 [2][...]: interior only."""
    f = pl.view(np.float16) if pl.dtype == np.int16 else pl
    return (f[0].astype(np.float64) + f[1].astype(np.float64))[:, 1:-1, 1:-1]


def _device_inputs(d, aws):
    """The device's whitened content [nc,hc,hc,C] and whitened style [hs,hs,C], float64."""
    c, nc, hc, hs, L = d["c"], d["nc"], d["hc"], d["hs"], d["L"]
    wc = _merged(_fp16_planes(aws, L["wc_feat"], nc, hc, hc, c))
    ws = _merged(_fp16_planes(d["state"], L["feat"], 1, hs, hs, c))[0]
    return wc, ws


def _swapped(d, aws):
    return _merged(_fp16_planes(aws, d["L"]["ss_feat"], d["nc"], d["hc"], d["hc"], d["c"]))


def _err(got, ref):
    return np.abs(got - ref).max() / max(1.0, np.abs(ref).max())


# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nc", [1, 3])
@pytest.mark.parametrize("ps", list(GEOM), ids=lambda v: "p%ds%d" % v)
@pytest.mark.parametrize("c", [64, 128, 256, 512])
def test_accuracy_against_the_oracle(c, ps, nc):
    p, s = ps
    hc, hs = GEOM[ps]
    d = _setup(c, p, s, nc, c + 5 * p + nc, hc, hs, dead=c // 4 if c == 128 else 0)
    assert d["L"]["cout_pad"] > BLOCK                     # two blocks, the last one padded
    worst = 0.0
    for tau in (3e-3, 0.05, 1.0, 100.0):
        rc, _, k, aws = _softmax(d, tau)
        assert rc == 0, d["lib"].wctb200_last_error().decode()
        wc, ws = _device_inputs(d, aws)
        got = _swapped(d, aws)
        for i in range(nc):
            ref = SR.style_swap_softmax(wc[i], ws, p, s, tau)
            e = _err(got[i], ref)
            worst = max(worst, e)
            assert e <= GATE, "C %d p%d s%d frame %d tau %g: %.2e" % (c, p, s, i, tau, e)
    print("softmax swap C %d p%d s%d Nc %d: worst %.2e" % (c, p, s, nc, worst))


def _sizes(d):
    """Workspace sizes from one block to one chunk: each whole number of blocks, a ragged size and the full one."""
    col = 2 * 2 * d["nc"] * (d["hc"] + 2) * (d["hc"] + 2)
    nblk = -(-d["L"]["cout_pad"] // BLOCK)
    sizes = {"%d_blocks" % k: d["least"] + (k - 1) * BLOCK * col for k in range(1, nblk)}
    sizes["ragged"] = d["least"] + BLOCK * col + 4096
    sizes["full"] = d["full"]
    return sizes


@pytest.mark.parametrize("c", [128, 512])
def test_every_workspace_size_and_batch_gives_the_same_bytes(c):
    d = _setup(c, 3, 1, 3, 41 + c, 18, 40)                # 1444 patches: six blocks, the last one padded
    rc, ref, kref, _ = _softmax(d, 0.05)
    assert rc == 0, d["lib"].wctb200_last_error().decode()
    for name, nbytes in _sizes(d).items():
        rc, got, k, _ = _softmax(d, 0.05, nbytes)
        assert rc == 0, d["lib"].wctb200_last_error().decode()
        assert_bits(got, ref, "C %d workspace %s" % (c, name))
        assert np.array_equal(k, kref)
    rc, _, _, _ = _softmax(d, 0.05, d["least"] - 1)
    assert rc == _capi.EWS
    for i in range(3):
        one = frame_copy(d["cin"], i, 3, 18, 18, c)
        for nbytes in (None, "least"):
            dd = dict(d, full=d["lib"].wctb200_style_swap_softmax_workspace_bytes(c, 1, 18, 18, 40, 40, 3, 1))
            n = dd["full"] if nbytes is None else d["lib"].wctb200_style_swap_softmax_min_workspace_bytes(c, 1, 18, 18, 40, 40, 3, 1)
            rc, got, _, _ = _softmax(dd, 0.05, n, cin=one, nc=1)
            assert rc == 0
            assert_bits(got[:, 0], ref[:, i], "C %d frame %d alone (%s)" % (c, i, nbytes or "full"))


@pytest.mark.parametrize("tau", [1e-4, 1e-7])
@pytest.mark.parametrize("ps", list(GEOM), ids=lambda v: "p%ds%d" % v)
def test_small_temperature_is_the_hard_apply(ps, tau):
    p, s = ps
    hc, hs = GEOM[ps]
    d = _setup(256, p, s, 2, 77 + p, hc, hs)
    rc, got, _, aws = _softmax(d, tau)
    assert rc == 0
    ref, hws = _hard(d)
    wc, ws = _device_inputs(d, aws)
    g, r = _merged(got), _merged(ref)
    gs, rs = _swapped(d, aws), _swapped(d, hws)
    assert np.isfinite(g).all() and np.isfinite(gs).all()          # every weight <= 1, at any tau
    # fp32 rounding: the fold sums the <= P*P weighted patches on the tensor cores (truncating adds) and stores SPF16, the
    # gather sums them in fp32; both are within 9 * 2^-23 + 2^-22 + 9 * 2^-24 (< 2e-6) of the mean |patch value|
    bound = 4e-6 * np.abs(ws).max()
    checked = 0
    for i in range(2):
        _, inf = SR.style_swap_softmax(wc[i], ws, p, s, tau, return_info=True)
        top2 = np.sort(inf["z"], axis=2)[..., -2:]
        bad = (top2[..., 1] - top2[..., 0]) <= 50 * tau
        ok = np.ones((hc, hc), bool)
        for y, x in np.argwhere(bad):
            ok[y * s:y * s + p, x * s:x * s + p] = False
        checked += ok.sum()
        e = np.abs(gs[i][ok] - rs[i][ok]).max()
        assert e <= bound, "frame %d swapped feature: %.2e > %.2e" % (i, e, bound)
        e_out = np.abs(g[i][ok] - r[i][ok]).max()
        assert e_out <= 1e-5 * max(1.0, np.abs(r[i]).max()), "frame %d output: %.2e" % (i, e_out)
        print("p%d s%d tau %g frame %d: swapped feature %.2e (bound %.2e), coloured output %.2e"
              % (p, s, tau, i, e, bound, e_out))
    # random features have near-flat scores: at tau = 1e-4 only a few pixels clear the 50 tau margin
    print("p%d s%d tau %g: %d margin pixels of %d" % (p, s, tau, checked, 2 * hc * hc))
    assert checked >= (8 if tau >= 1e-4 else hc * hc)


def _blocks(h, w, labels, seed, cells=4):
    rng = np.random.default_rng(seed)
    grid = rng.choice(np.asarray(labels, np.uint8), (cells, cells))
    return np.ascontiguousarray(grid[np.arange(h) * cells // h][:, np.arange(w) * cells // w])


@pytest.mark.parametrize("ps", list(GEOM), ids=lambda v: "p%ds%d" % v)
def test_labels(ps):
    p, s = ps
    hc, hs = GEOM[ps]
    d = _setup(128, p, s, 3, 91 + p, hc, hs)
    rc, ref, _, _ = _softmax(d, 0.05)
    assert rc == 0
    cl = torch.full((3, 2 * hc + 1, hc + 3), 5, dtype=torch.uint8, device="cuda")
    sl = torch.full((7, 5), 5, dtype=torch.uint8, device="cuda")
    for name, nbytes in (("full", d["full"]), ("least", d["least"])):
        rc, got, _, _ = _softmax(d, 0.05, nbytes, cl, sl)
        assert rc == 0, d["lib"].wctb200_last_error().decode()
        assert_bits(got, ref, "uniform labels (%s)" % name)
    # block labels: content 0..3, style 0..2 (label 3 absent: those anchors take every patch)
    cl_np = np.stack([_blocks(hc, hc, range(4), 10 + i) for i in range(3)])
    sl_np = _blocks(hs, hs, range(3), 20)
    cl, sl = torch.from_numpy(cl_np).cuda(), torch.from_numpy(sl_np).cuda()
    rc, full_bits, _, aws = _softmax(d, 0.05, None, cl, sl)
    assert rc == 0
    rc, least_bits, _, _ = _softmax(d, 0.05, d["least"], cl, sl)
    assert_bits(least_bits, full_bits, "block labels, least workspace")
    wc, ws = _device_inputs(d, aws)
    got = _swapped(d, aws)
    plab = SLR.patch_labels(sl_np, hs, hs, p, s)
    for i in range(3):
        allowed = SLR.allowed(SLR.anchor_labels(cl_np[i], hc, hc, p, s), plab)
        assert (~allowed).any()
        e = _err(got[i], SR.style_swap_softmax(wc[i], ws, p, s, 0.05, allowed))
        assert e <= GATE, "frame %d: %.2e" % (i, e)


def test_bad_temperatures_are_einval():
    d = _setup(64, 3, 1, 1, 5, 18, 19)
    for tau in (0.0, -1.0, float("nan"), float("inf"), 1e-40):        # 1e-40: a subnormal float32, no finite 1/tau
        rc, _, _, _ = _softmax(d, tau)
        assert rc == _capi.EINVAL, tau


# ------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def weights():
    return make_synthetic_weights(0, relu_targets=ALL)


def _imgs(n, h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, h, w, 3), dtype=np.uint8)


@pytest.mark.parametrize("relu", ["relu5_1", "relu3_1"])
def test_teacher_forced_pipeline(weights, relu):
    """Every level of one engine run against the float64 oracle on the device's level input (WCT at the other levels):
    the transformed feature relative to its largest value (at least 1), the level output absolutely."""
    eng = Engine(weights, ALL, semantics="tf")
    content, style = _imgs(1, 256, 256, 1000), _imgs(1, 256, 256, 7)
    cap = {}
    eng.stylize(torch.from_numpy(content).cuda(), torch.from_numpy(style).cuda(), alpha=0.8, want_info=True, capture=cap,
                swap_targets=[relu], ss_alpha=0.6, ss_temperature=0.05)
    eng.check_device()
    sfe = nets.encode(nets.preprocess(style).astype(np.float64), weights, ALL, np.float64)
    worst = 0.0
    for i, r in enumerate(ALL):
        x = cap["level_input"][i].cpu().numpy().astype(np.float64)
        cfo = nets.encode(x, weights, [r], np.float64)[r]
        if r == relu:
            f = SR.wct_style_swap_softmax(cfo, sfe[r], 0.6, 0.05, 3, 1)
        else:
            f = ref_ops.wct_tf(cfo, sfe[r], 0.8)
        e_t = _err(eng.act_to_f32(cap["transformed"][i]).cpu().numpy(), f)
        y = nets.decode(np.asarray(f, dtype=np.float64), weights, r, np.float64)
        if i < len(ALL) - 1:
            y = np.clip(y, 0, 1)
        e_out = np.abs(cap["level_output"][i].cpu().numpy() - y).max()
        print("softmax swap at %s, %s: transform %.2e  level output %.2e" % (relu, r, e_t, e_out))
        worst = max(worst, e_t, e_out)
    assert worst <= GATE


def test_engine_identities(weights, monkeypatch):
    from wct_tf_b200 import engine as E
    eng = Engine(weights, ALL, semantics="tf")
    c, s = torch.from_numpy(_imgs(2, 512, 512, 3)).cuda(), torch.from_numpy(_imgs(1, 512, 512, 4)).cuda()
    kw = dict(alpha=0.8, swap_targets=["relu3_1"], ss_alpha=0.6)
    # relu3_1 of two 512^2 frames: 15 876 patches, about 2.2 GB of scores -- chunked under the default policy
    policy = eng.stylize(c, s, ss_temperature=0.05, **kw).cpu()
    monkeypatch.setattr(E, "SWAP_WORKSPACE_BYTES", 1 << 40)
    one_chunk = eng.stylize(c, s, ss_temperature=0.05, **kw).cpu()
    monkeypatch.setattr(E, "SWAP_WORKSPACE_BYTES", 1 << 30)
    assert torch.equal(policy, one_chunk)
    ps = eng.prepare_call(s, swap_targets=["relu3_1"])
    assert torch.equal(eng.stylize(c, ps, ss_temperature=0.05, **kw).cpu(), policy)
    assert torch.equal(eng.stylize(c, s, ss_temperature=None, **kw).cpu(), eng.stylize(c, s, **kw).cpu())
    assert not torch.equal(eng.stylize(c, s, **kw).cpu(), policy)
    with pytest.raises(ValueError, match="ss_temperature needs"):
        eng.stylize(c, s, alpha=0.8, ss_temperature=0.05)
