"""The balanced style swap (DESIGN.md §3.3.18) on the device.

1. C-ABI accuracy: at C in {64,128,256,512}, (P,S) in {(3,1),(5,2)}, Nc in {1,3}, tau in {0.01, 0.05, 1} and T in
   {1, 4, 16}, the swapped feature (read back from the workspace) is within 1e-3 of the largest whitened style value of
   the float64 oracle evaluated on the device's own whitened content and style, and the column sums within 1e-3 of the
   oracle's largest.
2. T = 0 is the softmax apply: its bytes and its launch count.
3. Invariance: every workspace size from one block to one chunk gives the same bytes and column sums; frame i of a batch
   equals that frame alone, bit for bit; T in {1, 4}, with and without labels.
4. Identical rows: a periodic content with stride = patch; after one iteration the column sums are the targets and the
   output the uniform patch mean, within fp32 rounding.
5. Labels: uniform labels give the unlabelled bytes; block labels with a label absent from the style match the masked
   oracle.  A bad iteration count is WCTB200_EINVAL.
6. Engine: teacher-forced five-level runs with the balanced swap at relu5_1 and relu3_1; a prepared style gives the image
   style's bytes; ss_balance=0 gives the softmax bytes; the default workspace policy at relu3_1 at 512^2 gives the
   one-chunk bytes.
"""
import numpy as np
import pytest
import torch

from oracle import nets, ref_ops
from tests import balanced_swap_ref as BR
from tests import gpu_util as U
from tests import softmax_swap_ref as SR
from tests import swap_labels_ref as SLR
from tests.test_gpu_invariance import assert_bits, frame_copy, planes
from tests.test_gpu_softmax_swap import (ALL, BLOCK, GATE, GEOM, TF, _blocks, _device_inputs, _err, _imgs, _merged, _setup,
                                         _softmax, _swapped, _ws, weights)  # noqa: F401
from wct_tf_b200 import _capi
from wct_tf_b200.engine import Engine

pytestmark = pytest.mark.gpu
ABLK = 256


def _bsetup(c, p, s, nc, seed, hc, hs, dead=0):
    d = _setup(c, p, s, nc, seed, hc, hs, dead)
    lib = d["lib"]
    d["bfull"] = lib.wctb200_style_swap_balanced_workspace_bytes(c, nc, hc, hc, hs, hs, p, s)
    d["bleast"] = lib.wctb200_style_swap_balanced_min_workspace_bytes(c, nc, hc, hc, hs, hs, p, s)
    return d


def _balanced(d, tau, iters, nbytes=None, cl=None, sl=None, alpha=0.6, cin=None, nc=None, cols=True):
    """The balanced apply through the C-ABI; returns (rc, output planes, k_out, workspace, column sums [nc, n_p])."""
    lib, c, p, s, hc, hs = d["lib"], d["c"], d["p"], d["s"], d["hc"], d["hs"]
    nc = d["nc"] if nc is None else nc
    cin = d["cin"] if cin is None else cin
    aws = _ws(d["bfull"] if nbytes is None else nbytes)
    out = U.act_alloc(nc, hc, hc, c)
    kout = torch.full((nc + 1,), -7, dtype=torch.int32, device="cuda")
    col = torch.full((nc, d["L"]["n_patches"]), float("nan"), dtype=torch.float32, device="cuda") if cols else None
    lab = (None, 0, 0, 0, None, 0, 0)
    lbuf = None
    if cl is not None:
        lbuf = _ws(lib.wctb200_style_swap_labels_workspace_bytes(cl.shape[0], hc, hc, hs, hs, p, s))
        lab = (cl.data_ptr(), cl.shape[0], cl.shape[1], cl.shape[2], sl.data_ptr(), sl.shape[-2], sl.shape[-1])
    rc = lib.wctb200_style_swap_apply_balanced(cin.data_ptr(), nc, hc, hc, c, d["state"].data_ptr(), hs, hs, p, s, alpha, *TF,
                                               float(tau), int(iters), *lab, out.data_ptr(), kout.data_ptr(),
                                               None if col is None else col.data_ptr(), aws.data_ptr(), aws.numel(),
                                               None if lbuf is None else lbuf.data_ptr(), 0 if lbuf is None else lbuf.numel(),
                                               U.stream())
    if rc:
        return rc, None, None, None, None
    U.check_device()
    torch.cuda.synchronize()
    return rc, planes(out, nc, hc, hc, c), kout.cpu().numpy(), aws, None if col is None else col.cpu().numpy()


def _oracle_case(wc, ws, p, s):
    """(scores, norms, K) of one frame for BR.balanced_weights."""
    _, inf = ref_ops.style_swap(wc[None], ws[None], p, s, return_info=True)
    return inf["scores"], SR.anchor_norms(wc, p, s), p * p * wc.shape[2]


# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nc", [1, 3])
@pytest.mark.parametrize("ps", list(GEOM), ids=lambda v: "p%ds%d" % v)
@pytest.mark.parametrize("c", [64, 128, 256, 512])
def test_accuracy_against_the_oracle(c, ps, nc):
    p, s = ps
    hc, hs = GEOM[ps]
    d = _bsetup(c, p, s, nc, c + 5 * p + nc, hc, hs, dead=c // 4 if c == 128 else 0)
    assert d["L"]["cout_pad"] > BLOCK                     # two blocks, the last one padded
    worst_f = worst_c = 0.0
    cases = None
    for tau in (0.01, 0.05, 1.0):
        for T in (1, 4, 16):
            rc, _, _, aws, col = _balanced(d, tau, T)
            assert rc == 0, d["lib"].wctb200_last_error().decode()
            if cases is None:
                wc, ws = _device_inputs(d, aws)
                cases = [_oracle_case(wc[i], ws, p, s) for i in range(nc)]
                scale = np.abs(ws).max()
            got = _swapped(d, aws)
            for i in range(nc):
                w, cref, _, _, _ = BR.balanced_weights(*cases[i], tau, T)
                ref = BR.paste(w, ws, hc, hc, p, s)
                e_f = np.abs(got[i] - ref).max() / scale
                e_c = np.abs(col[i] - cref).max() / np.abs(cref).max()
                worst_f, worst_c = max(worst_f, e_f), max(worst_c, e_c)
                assert e_f <= GATE, "C %d p%d s%d frame %d tau %g T %d: feature %.2e" % (c, p, s, i, tau, T, e_f)
                assert e_c <= GATE, "C %d p%d s%d frame %d tau %g T %d: column sums %.2e" % (c, p, s, i, tau, T, e_c)
    print("balanced swap C %d p%d s%d Nc %d: worst feature %.2e, column sums %.2e" % (c, p, s, nc, worst_f, worst_c))


@pytest.mark.parametrize("labelled", [False, True])
def test_zero_iterations_are_the_softmax_apply(labelled):
    d = _bsetup(128, 3, 1, 3, 61, 18, 40)
    lib, geom = d["lib"], (128, 3, 18, 18, 40, 40, 3, 1)
    cl = sl = None
    if labelled:
        cl = torch.from_numpy(np.stack([_blocks(18, 18, range(4), 30 + i) for i in range(3)])).cuda()
        sl = torch.from_numpy(_blocks(40, 40, range(3), 40)).cuda()
    for soft_bytes, bal_bytes in ((d["full"], d["bfull"]), (d["least"], d["bleast"])):
        rc, ref, kref, _ = _softmax(d, 0.05, soft_bytes, cl, sl)
        assert rc == 0
        rc, got, k, _, _ = _balanced(d, 0.05, 0, bal_bytes, cl, sl, cols=False)
        assert rc == 0, lib.wctb200_last_error().decode()
        assert_bits(got, ref, "T = 0")
        assert np.array_equal(k, kref)
        assert (lib.wctb200_style_swap_balanced_launches(*geom, bal_bytes, int(labelled), 0, 0)
                == lib.wctb200_style_swap_softmax_launches(*geom, soft_bytes, int(labelled)))
    # the column sums of T = 0 are the softmax plan's; T adds its passes to the count
    n1 = lib.wctb200_style_swap_balanced_launches(*geom, d["bfull"], 0, 1, 0)
    n0 = lib.wctb200_style_swap_balanced_launches(*geom, d["bfull"], 0, 0, 0)
    assert n1 - n0 == 1 + 3 + 1 and lib.wctb200_style_swap_balanced_launches(*geom, d["bfull"], 0, 0, 1) == n0 + 2


def _bsizes(d):
    """Workspace sizes from one block to one chunk: each whole number of blocks, a ragged size and the full one."""
    nablk = -(-d["L"]["ho"] * d["L"]["wo"] // ABLK)
    col = 2 * 2 * d["nc"] * (d["hc"] + 2) * (d["hc"] + 2) + d["nc"] * nablk * 8
    nblk = -(-d["L"]["cout_pad"] // BLOCK)
    sizes = {"%d_blocks" % k: d["bleast"] + (k - 1) * BLOCK * col for k in range(1, nblk)}
    sizes["ragged"] = d["bleast"] + BLOCK * col + 4096
    sizes["full"] = d["bfull"]
    return sizes


@pytest.mark.parametrize("labelled", [False, True], ids=["free", "labels"])
@pytest.mark.parametrize("T", [1, 4])
def test_every_workspace_size_and_batch_gives_the_same_bytes(T, labelled):
    c, nc, hc, hs = 128, 3, 18, 40                          # 1444 patches: six blocks, the last one padded
    d = _bsetup(c, 3, 1, nc, 43 + T, hc, hs)
    lib = d["lib"]
    cl = sl = None
    if labelled:
        cl_np = np.stack([_blocks(hc, hc, range(4), 50 + i) for i in range(nc)])
        cl, sl = torch.from_numpy(cl_np).cuda(), torch.from_numpy(_blocks(hs, hs, range(3), 60)).cuda()
    rc, ref, kref, _, cref = _balanced(d, 0.05, T, None, cl, sl)
    assert rc == 0, lib.wctb200_last_error().decode()
    chunks = set()
    for name, nbytes in _bsizes(d).items():
        rc, got, k, _, col = _balanced(d, 0.05, T, nbytes, cl, sl)
        assert rc == 0, lib.wctb200_last_error().decode()
        assert_bits(got, ref, "T %d workspace %s" % (T, name))
        assert np.array_equal(k, kref) and np.array_equal(col.view(np.int32), cref.view(np.int32)), name
        chunks.add(lib.wctb200_style_swap_balanced_launches(c, nc, hc, hc, hs, hs, 3, 1, nbytes, int(labelled), T, 1))
    assert len(chunks) >= 4                               # the sizes run in 6, 3, 2 and 1 chunks
    rc, _, _, _, _ = _balanced(d, 0.05, T, d["bleast"] - 1, cl, sl)
    assert rc == _capi.EWS
    for i in range(nc):
        one = frame_copy(d["cin"], i, nc, hc, hc, c)
        for which in ("full", "least"):
            fn = (lib.wctb200_style_swap_balanced_workspace_bytes if which == "full"
                  else lib.wctb200_style_swap_balanced_min_workspace_bytes)
            dd = dict(d, bfull=fn(c, 1, hc, hc, hs, hs, 3, 1))
            rc, got, _, _, col = _balanced(dd, 0.05, T, None, None if cl is None else cl[i:i + 1].contiguous(), sl,
                                           cin=one, nc=1)
            assert rc == 0
            assert_bits(got[:, 0], ref[:, i], "T %d frame %d alone (%s)" % (T, i, which))
            assert np.array_equal(col[0].view(np.int32), cref[i].view(np.int32))


@pytest.mark.parametrize("tau", [0.05, 1.0])
def test_identical_rows_balance_in_one_iteration(tau):
    """Content of period 3 and 3 x 3 patches at stride 3: every anchor sees the same window, so every row of the plan is
    the same; one column step makes it uniform."""
    c, p, s, hc, hs = 128, 3, 3, 18, 19
    rng = np.random.default_rng(5)
    tile = np.maximum(rng.standard_normal((3, 3, c)) + 0.3, 0)
    content = np.tile(tile, (hc // 3, hc // 3, 1))[None].astype(np.float32)
    d = _bsetup(c, p, s, 1, 9, hc, hs)
    d["cin"] = U.act_from_numpy(content)
    rc, _, _, aws, col0 = _balanced(d, tau, 0)
    assert rc == 0
    rc, _, _, aws, col = _balanced(d, tau, 1)
    assert rc == 0
    na, npat = d["L"]["ho"] * d["L"]["wo"], d["L"]["n_patches"]
    target = na / npat
    e0 = np.abs(col0 - target).max() / target
    e1 = np.abs(col - target).max() / target
    _, ws = _device_inputs(d, aws)
    want = SR.uniform_swap(ws, hc, hc, p, s)
    e_f = np.abs(_swapped(d, aws)[0] - want).max() / np.abs(ws).max()
    print("identical rows, tau %g: column error %.2e at T = 0, %.2e at T = 1; feature %.2e" % (tau, e0, e1, e_f))
    assert e0 > 1e-3 or tau >= 1.0
    assert e1 <= 2e-5 and e_f <= 2e-5


@pytest.mark.parametrize("ps", list(GEOM), ids=lambda v: "p%ds%d" % v)
def test_labels(ps):
    p, s = ps
    hc, hs = GEOM[ps]
    d = _bsetup(128, p, s, 3, 93 + p, hc, hs)
    rc, ref, _, _, cref = _balanced(d, 0.05, 4)
    assert rc == 0
    cl = torch.full((3, 2 * hc + 1, hc + 3), 5, dtype=torch.uint8, device="cuda")
    sl = torch.full((7, 5), 5, dtype=torch.uint8, device="cuda")
    for name, nbytes in (("full", d["bfull"]), ("least", d["bleast"])):
        rc, got, _, _, col = _balanced(d, 0.05, 4, nbytes, cl, sl)
        assert rc == 0, d["lib"].wctb200_last_error().decode()
        assert_bits(got, ref, "uniform labels (%s)" % name)
        assert np.array_equal(col.view(np.int32), cref.view(np.int32))
    # block labels: content 0..3, style 0..2 (label 3 absent: those anchors take every patch)
    cl_np = np.stack([_blocks(hc, hc, range(4), 10 + i) for i in range(3)])
    sl_np = _blocks(hs, hs, range(3), 20)
    cl, sl = torch.from_numpy(cl_np).cuda(), torch.from_numpy(sl_np).cuda()
    rc, _, _, aws, col = _balanced(d, 0.05, 4, None, cl, sl)
    assert rc == 0
    wc, ws = _device_inputs(d, aws)
    got = _swapped(d, aws)
    plab = SLR.patch_labels(sl_np, hs, hs, p, s)
    for i in range(3):
        allowed = SLR.allowed(SLR.anchor_labels(cl_np[i], hc, hc, p, s), plab)
        assert (~allowed).any()
        w, cs, _, _, _ = BR.balanced_weights(*_oracle_case(wc[i], ws, p, s), 0.05, 4, allowed)
        e_f = np.abs(got[i] - BR.paste(w, ws, hc, hc, p, s)).max() / np.abs(ws).max()
        e_c = np.abs(col[i] - cs).max() / np.abs(cs).max()
        assert e_f <= GATE and e_c <= GATE, "frame %d: %.2e %.2e" % (i, e_f, e_c)


def test_bad_iterations_are_einval():
    d = _bsetup(64, 3, 1, 1, 5, 18, 19)
    for T in (-1, 257, 1 << 20):
        rc, _, _, _, _ = _balanced(d, 0.05, T)
        assert rc == _capi.EINVAL, T
        assert d["lib"].wctb200_style_swap_balanced_launches(64, 1, 18, 18, 19, 19, 3, 1, d["bfull"], 0, T, 0) == 0
    rc, _, _, _, _ = _balanced(d, 0.0, 4)
    assert rc == _capi.EINVAL
    rc, _, _, _, _ = _balanced(d, 0.05, 256)
    assert rc == 0


# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("relu", ["relu5_1", "relu3_1"])
def test_teacher_forced_pipeline(weights, relu):  # noqa: F811
    """Every level of one engine run against the float64 oracle on the device's level input (WCT at the other levels):
    the transformed feature relative to its largest value (at least 1), the level output absolutely."""
    eng = Engine(weights, ALL, semantics="tf")
    content, style = _imgs(1, 256, 256, 1000), _imgs(1, 256, 256, 7)
    cap = {}
    eng.stylize(torch.from_numpy(content).cuda(), torch.from_numpy(style).cuda(), alpha=0.8, want_info=True, capture=cap,
                swap_targets=[relu], ss_alpha=0.6, ss_temperature=0.05, ss_balance=4)
    eng.check_device()
    sfe = nets.encode(nets.preprocess(style).astype(np.float64), weights, ALL, np.float64)
    worst = 0.0
    for i, r in enumerate(ALL):
        x = cap["level_input"][i].cpu().numpy().astype(np.float64)
        cfo = nets.encode(x, weights, [r], np.float64)[r]
        if r == relu:
            f = BR.wct_style_swap_balanced(cfo, sfe[r], 0.6, 0.05, 4, 3, 1)
        else:
            f = ref_ops.wct_tf(cfo, sfe[r], 0.8)
        e_t = _err(eng.act_to_f32(cap["transformed"][i]).cpu().numpy(), f)
        y = nets.decode(np.asarray(f, dtype=np.float64), weights, r, np.float64)
        if i < len(ALL) - 1:
            y = np.clip(y, 0, 1)
        e_out = np.abs(cap["level_output"][i].cpu().numpy() - y).max()
        print("balanced swap at %s, %s: transform %.2e  level output %.2e" % (relu, r, e_t, e_out))
        worst = max(worst, e_t, e_out)
    assert worst <= GATE


def test_engine_identities(weights, monkeypatch):  # noqa: F811
    from wct_tf_b200 import engine as E
    eng = Engine(weights, ALL, semantics="tf")
    c, s = torch.from_numpy(_imgs(2, 512, 512, 3)).cuda(), torch.from_numpy(_imgs(1, 512, 512, 4)).cuda()
    kw = dict(alpha=0.8, swap_targets=["relu3_1"], ss_alpha=0.6, ss_temperature=0.05)
    # relu3_1 of two 512^2 frames: 15 876 patches, about 2.2 GB of scores -- chunked under the default policy
    policy = eng.stylize(c, s, ss_balance=2, **kw).cpu()
    monkeypatch.setattr(E, "SWAP_WORKSPACE_BYTES", 1 << 40)
    one_chunk = eng.stylize(c, s, ss_balance=2, **kw).cpu()
    monkeypatch.undo()
    assert torch.equal(policy, one_chunk)
    ps = eng.prepare_call(s, swap_targets=["relu3_1"])
    assert torch.equal(eng.stylize(c, ps, ss_balance=2, **kw).cpu(), policy)
    soft = eng.stylize(c, s, **kw).cpu()
    assert torch.equal(eng.stylize(c, s, ss_balance=0, **kw).cpu(), soft)
    assert not torch.equal(soft, policy)
    with pytest.raises(ValueError, match="ss_balance needs ss_temperature"):
        eng.stylize(c, s, alpha=0.8, swap_targets=["relu3_1"], ss_balance=2)
