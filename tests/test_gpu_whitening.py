"""GPU: stage B of a WCT level -- the whitening matrix W_c and the colouring matrix C_s, from either solver (one-sided
Jacobi, wct.cu; Newton-Schulz, matfun_tc.cu) -- against float64 in the eigenbasis of the fp32 covariance the solvers
receive, on rotated, graded spectra.  Metric, bound and its derivation: tests/whitening_ref.py.

W_c is read through the public API: a statistics record with covariance Q diag(lam) Q^T, a style state with C_s = I and
alpha = 1 give M = W_c, and the transform's readback (M_hi + M_lo) 2^-e is W_c as stored.  Each call is a batch of frames
with different spectra, some of which the Newton-Schulz guard accepts and some it must reject, so the per-matrix routing
between the two solvers (`ok` / `skip`) is exercised inside one call.  The `tail` frames put a graded run of kept
eigenvalues under 3.16e-6 lambda_max, where k_jacobi's null floor once froze them (whitening_ref, test_whitening_cpu)."""
import ctypes

import numpy as np
import pytest
import torch

from tests import gpu_util as U
from tests import whitening_ref as R
from tests.test_gpu_apply import read_transform, transform_offsets, write_record, write_style_state
from tests.test_gpu_tiles import _read_record, _rect
from wct_tf_b200 import _capi

pytestmark = pytest.mark.gpu

# the frames of one call.  Guard: accepted only with lam_min > 1.01 thresh and convergence within 16 iterations (cond
# up to ~5e3 .. 1e4), so graded_1e2 / _1e3 / _5e3 and near_guard_2 are candidates for the fast path, the rest must go to
# the eigensolver.
FRAMES = [("graded_%g" % c, (lambda C, c=c, i=i: R.graded(C, c, seed=C + i))) for i, c in enumerate((1e2, 1e3, 5e3, 3e4, 1e5))]
FRAMES += [("tail_%g" % l, (lambda C, l=l, i=i: R.tail(C, l, seed=C + 5 + i))) for i, l in enumerate((1.0, 30.0, 300.0))]
FRAMES += [("cut", lambda C: R.cut(C, seed=C + 8)), ("cut_rank", lambda C: R.cut(C, seed=C + 9, rank=C // 2 + 3)),
           ("clustered", lambda C: R.clustered(C, seed=C + 10))]
FRAMES += [("near_guard_%g" % f, (lambda C, f=f, i=i: R.near_guard(C, f, seed=C + 11 + i)))
           for i, f in enumerate((0.9, 1.0, 1.02, 1.1, 2.0))]


@pytest.fixture(params=[0, 1], ids=["jacobi", "newton_schulz"])
def matfun(request):
    lib = U.lib()
    lib.wctb200_debug_set_matfun(request.param, 0)
    yield request.param
    lib.wctb200_debug_set_matfun(1, 0)


def _whiten(C, recs, sem):
    """W_c of every record through wctb200_wct_transform_from_stats (C_s = I, alpha = 1): (W [N,C,C] float64, k slot)."""
    lib = U.lib()
    s = R.SEMANTICS[sem]
    N = len(recs)
    rec = write_record(np.array([r[0] for r in recs]), np.zeros((N, C)), np.stack([r[1] for r in recs]),
                       np.stack([r[2] for r in recs]))
    state = write_style_state(np.zeros((1, C), np.float32), np.eye(C, dtype=np.float32)[None], C)
    ws = torch.empty(lib.wctb200_wct_workspace_bytes(C, N, 0), dtype=torch.uint8, device="cuda")
    tr = torch.full((transform_offsets(C, N)[0],), 255, dtype=torch.uint8, device="cuda")
    _capi.check(lib.wctb200_wct_transform_from_stats(rec.data_ptr(), N, C, state.data_ptr(), 1, 1.0, s["eps_cov"],
                                                     s["eps_eig"], R.THRESH, s["readd"], tr.data_ptr(), ws.data_ptr(),
                                                     ws.numel(), U.stream()))
    U.check_device()
    M, _, kk = read_transform(tr, C, N)
    return M, kk


def _k_decided(lam):
    """No eigenvalue within 5 % of the cut (near_guard_1.0 / _1.02 put one there on purpose)."""
    return np.abs(lam - R.THRESH).min() >= 0.05 * R.THRESH


@pytest.mark.parametrize("sem", ["tf", "np"])
@pytest.mark.parametrize("C", [64, 128, 256, 512])
def test_whitening_against_fp64(C, sem, matfun):
    """k_c equals the float64 count on the fp32 covariance exactly wherever no eigenvalue sits at the cut; the sweep slot
    is 0 exactly where the fast path ran (never with the knob off or at C = 64), and every matrix it accepted has
    lam_min > thresh; Ew within the bound of the solver that ran, on every entry fp32 determines."""
    s = R.SEMANTICS[sem]
    specs = [(name, fn(C)) for name, fn in FRAMES]
    recs = [R.record_of(Q, lam) for _, (Q, lam) in specs]
    M, kk = _whiten(C, recs, sem)
    N = len(specs)
    fails, accepted, rejected = [], [], []
    for f, (name, _) in enumerate(specs):
        S32 = R.sigma32(*recs[f], s["eps_cov"])
        lam, E = R.eig(S32)
        k_ref = int((lam > R.THRESH).sum())
        fast = kk[N + f] == 0
        where = "%s (cond %.2g, lam_min/thresh %.3g)" % (name, lam.max() / max(lam.min(), 1e-30), lam.min() / R.THRESH)
        (accepted if fast else rejected).append(where)
        if fast:
            assert matfun and C >= 128, "%s: sweep slot 0 with the fast path off" % name
            assert lam.min() > R.THRESH, "%s: the guard accepted a matrix with lam_min = %.3g" % (name, lam.min())
        if _k_decided(lam):
            assert kk[f] == k_ref, "%s: k_c %d, float64 %d" % (name, kk[f], k_ref)
        elif kk[f] != k_ref:
            print("C=%d %s %s: k %d, float64 %d (eigenvalue at the cut)" % (C, sem, name, kk[f], k_ref))
            continue
        b, m = R.whitening_bound(lam, R.THRESH, "newton_schulz" if fast else "jacobi", np.abs(M[f]).max())
        r, excl = R.worst_ratio(R.whitening_error(M[f], S32, s["eps_eig"], basis=(lam, E)), b, m)
        print("C=%d %s matfun=%d %-16s %s k %d sweeps %2d: worst Ew / bound %.3g (%d entries not determined by fp32)" % (
            C, sem, matfun, name, "fast  " if fast else "jacobi", kk[f], kk[N + f], r, excl))
        if r > 1.0:
            fails.append((name, round(r, 3)))
            U.dump("fail_whiten_C%d_%s_%d_%s" % (C, sem, matfun, name), M=M[f], S32=S32)
    print("C=%d %s matfun=%d: fast path took %s; eigensolver took %s" % (C, sem, matfun, accepted or "none", rejected))
    if matfun and C >= 128:
        assert accepted, "the fast path took none of the well-conditioned frames"
    assert not fails, fails


@pytest.mark.parametrize("C", [64, 256, 512])
def test_sigma32_is_the_library_covariance(C):
    """A whole-map record through wctb200_wct_stats_rect, finalised by whitening_ref.sigma32, gives wctb200_covariance's
    fp32 covariance bit for bit (eps_cov included): the metric's Sigma32 is what the solvers receive."""
    lib = U.lib()
    N, H, W = 2, 33, 40
    rng = np.random.default_rng(C)
    x = (rng.standard_normal((N, H, W, C)) @ (rng.standard_normal((C, C)) / np.sqrt(C)) + 0.5).astype(np.float32)
    act = U.act_from_numpy(x)
    mean = torch.empty((N, C), dtype=torch.float32, device="cuda")
    cov = torch.empty((N, C, C), dtype=torch.float32, device="cuda")
    _capi.check(lib.wctb200_covariance(act.data_ptr(), N, H, W, C, 1e-8, mean.data_ptr(), cov.data_ptr(), U.stream()))
    buf, offs = _rect(act, N, H, W, C, 0, 0, H, W, False)
    for i, r in enumerate(_read_record(buf, offs, C, N, False)):
        got = R.sigma32(r["n"], r["s"], r["S"], 1e-8)
        assert np.array_equal(got.view(np.uint32), cov[i].cpu().numpy().view(np.uint32)), i


def _designed_map(Q, lam, HW, seed):
    """[HW, C] features whose float64 covariance is Q diag(lam) Q^T: U diag(sqrt((HW - 1) lam)) Q^T + mean, U with
    orthonormal columns orthogonal to the ones vector."""
    C = len(lam)
    rng = np.random.default_rng(seed)
    Z = rng.standard_normal((HW, C))
    Z -= Z.mean(0)
    Uo, _ = np.linalg.qr(Z)
    return Uo * np.sqrt((HW - 1) * lam) @ Q.T + rng.uniform(-1.0, 1.0, C)


@pytest.mark.parametrize("sem", ["tf", "np"])
@pytest.mark.parametrize("C,H,W", [(256, 128, 128), (512, 32, 32)])
def test_colouring_against_fp64(C, H, W, sem, matfun):
    """C_s of wctb200_wct_style_prepare on maps of designed spectra at level sizes (relu4_1 of 1024^2, relu5_1 of 512^2),
    against the eigenbasis of wctb200_covariance of the same stored map (prepare and covariance share cov_tc): k_s exact,
    Ec within the bound on the kept block, dropped directions within theirs."""
    lib = U.lib()
    s = R.SEMANTICS[sem]
    specs = [("graded_1e3", R.graded(C, 1e3, seed=C + 20)), ("tail_30", R.tail(C, 30.0, seed=C + 21)),
             ("cut", R.cut(C, seed=C + 22))]
    Ns = len(specs)
    x = np.stack([_designed_map(Q, lam, H * W, C + i).reshape(H, W, C) for i, (_, (Q, lam)) in enumerate(specs)])
    act = U.act_from_numpy(x.astype(np.float32))
    cov = torch.empty((Ns, C, C), dtype=torch.float32, device="cuda")
    mean = torch.empty((Ns, C), dtype=torch.float32, device="cuda")
    _capi.check(lib.wctb200_covariance(act.data_ptr(), Ns, H, W, C, s["eps_cov"], mean.data_ptr(), cov.data_ptr(), U.stream()))
    state = torch.empty(lib.wctb200_wct_style_state_bytes(C, Ns), dtype=torch.uint8, device="cuda")
    ws = torch.empty(lib.wctb200_wct_workspace_bytes(C, 0, Ns), dtype=torch.uint8, device="cuda")
    _capi.check(lib.wctb200_wct_style_prepare(act.data_ptr(), Ns, H, W, C, s["eps_cov"], s["eps_eig"], R.THRESH,
                                              state.data_ptr(), ws.data_ptr(), ws.numel(), U.stream()))
    U.check_device()
    o = [ctypes.c_size_t() for _ in range(3)]
    lib.wctb200_wct_style_state_layout(C, Ns, *[ctypes.byref(v) for v in o])
    raw = state.cpu().numpy()
    Cs = raw[o[1].value:o[1].value + Ns * C * C * 4].view(np.float32).reshape(Ns, C, C).astype(np.float64)
    kk = raw[o[2].value:o[2].value + 2 * Ns * 4].view(np.int32)
    covs = cov.cpu().numpy()
    fails = []
    for f, (name, _) in enumerate(specs):
        lam, E = R.eig(covs[f])
        k_ref = int((lam > R.THRESH).sum())
        assert kk[f] == k_ref, "%s: k_s %d, float64 %d" % (name, kk[f], k_ref)
        fast = kk[Ns + f] == 0
        solver = "newton_schulz" if fast else "jacobi"
        Ec, drop = R.colouring_error(Cs[f], covs[f], s["eps_eig"], basis=(lam, E))
        b, m, bd = R.colouring_bound(lam, R.THRESH, solver, np.abs(Cs[f]).max())
        r, excl = R.worst_ratio(Ec, b, m)
        rd = float((drop / bd).max()) if drop.size else 0.0
        print("C=%d %dx%d %s matfun=%d %-10s %s k %d sweeps %2d: worst Ec / bound %.3g, dropped %.3g (%d excluded)" % (
            C, H, W, sem, matfun, name, solver, kk[f], kk[Ns + f], r, rd, excl))
        if r > 1.0 or rd > 1.0:
            fails.append((name, round(r, 3), round(rd, 3)))
            U.dump("fail_colour_C%d_%s_%d_%s" % (C, sem, matfun, name), Cs=Cs[f], S32=covs[f])
    assert not fails, fails
