"""The labelled style swap (DESIGN.md §3.3.13) without a GPU: the oracle (tests/swap_labels_ref.py) against the plain swap,
its arg-max rule, and the validation of ``swap_labels`` in options.py, ``WCT.predict_batch`` / ``predict`` /
``synthesize`` through a stub engine."""
import numpy as np
import pytest
import torch

from oracle import ref_ops
from tests import swap_labels_ref as SL
from tests.test_options_cpu import StubEngine, stub  # noqa: F401  (the stub fixture)
from wct_tf_b200 import options
from wct_tf_b200.prepared import PreparedStyle


def _feats(seed, hc, hs, c=8):
    rng = np.random.default_rng(seed)
    content = np.maximum(rng.standard_normal((1, hc, hc, c)) + 0.3, 0)
    style = np.maximum(rng.standard_normal((1, hs, hs, c)) + 0.4, 0)
    return content, style


@pytest.mark.parametrize("p,s", [(3, 1), (5, 2)])
def test_uniform_labels_are_the_plain_swap(p, s):
    content, style = _feats(1, 13, 11)
    ref = ref_ops.wct_style_swap(content, style, 0.6, p, s)
    for lab in (0, 7):
        got = SL.wct_style_swap_labels(content, style, 0.6, np.full((5, 9), lab, np.uint8), np.full((3, 4), lab, np.uint8), p, s)
        assert np.array_equal(got, ref)


def test_label_sampling_rule():
    lab = np.arange(6 * 8, dtype=np.uint8).reshape(6, 8)
    # a 6 x 8 style feature with its own map: patch (py, px) of P = 3, S = 1 reads the map at (py + 1, px + 1)
    assert np.array_equal(SL.patch_labels(lab, 6, 8, 3, 1), lab[1:5, 1:7].reshape(-1))
    assert np.array_equal(SL.anchor_labels(lab, 6, 8, 5, 1), lab[2:4, 2:6])
    # P = 5, S = 2 on a 7 x 9 grid from a 14 x 18 map: anchor (y, x) at (2y + 2, 2x + 2) on the grid, (4y + 5, 4x + 5) on the map
    big = np.arange(14 * 18, dtype=np.int64).reshape(14, 18)
    assert np.array_equal(SL.anchor_labels(big, 7, 9, 5, 2), big[5:10:4, 5:14:4])


def test_anchors_take_their_own_label():
    """Block labels with a label the style lacks: a present label's anchors take only patches of that label (their first
    maximum among them), an absent label's the unconstrained arg-max."""
    content, style = _feats(2, 16, 14)
    cl = np.zeros((16, 16), np.uint8)
    cl[:, 8:] = 1
    cl[12:, :] = 5                   # absent from the style
    sl = np.zeros((14, 14), np.uint8)
    sl[7:, :] = 1
    sl[:3, :3] = 2                   # a label of the style the content lacks
    _, info = SL.wct_style_swap_labels(content, style, 0.6, cl, sl, 3, 1, return_info=True)
    idx, alab, plab, sc = info["idx"], info["anchor_labels"], info["patch_labels"], info["scores"]
    assert set(np.unique(alab)) == {0, 1, 5} and set(np.unique(plab)) == {0, 1, 2}
    for y in range(idx.shape[0]):
        for x in range(idx.shape[1]):
            lab = alab[y, x]
            if lab in plab:
                own = np.flatnonzero(plab == lab)
                assert plab[idx[y, x]] == lab
                assert idx[y, x] == own[np.argmax(sc[y, x, own])]
            else:
                assert idx[y, x] == info["free_idx"][y, x]
    assert (alab == 5).any() and (idx != info["free_idx"]).any()


def test_masked_argmax_ties_go_low():
    scores = np.array([[[1.0, 3.0, 3.0, 3.0]]])
    assert SL.masked_argmax(scores, np.array([[1]]), np.array([0, 2, 1, 1]))[0, 0] == 2
    assert SL.masked_argmax(scores, np.array([[4]]), np.array([0, 2, 1, 1]))[0, 0] == 1


# ------------------------------------------------------------------------------------------------------------ validation
def _maps(cshape=(8, 8), sshape=(6, 6), dtype=np.uint8):
    return np.zeros(cshape, dtype), np.zeros(sshape, dtype)


@pytest.mark.parametrize("value,swap,n,ns,match", [
    (_maps(), False, 1, 1, "needs swap5 / swap_targets"),
    (_maps()[0], True, 1, 1, "must be a pair"),
    (list(_maps()) + [None], True, 1, 1, "must be a pair"),
    (_maps(dtype=np.int32), True, 1, 1, "must be uint8"),
    ((np.zeros((8, 8), np.uint8), np.zeros((6, 6), np.float32)), True, 1, 1, "style labels must be uint8"),
    (_maps(cshape=(3, 8, 8)), True, 2, 1, r"content labels must be .* N = 1 or 2"),
    (_maps(cshape=(8,)), True, 1, 1, "content labels must be"),
    (_maps(cshape=(1, 2, 8, 8)), True, 1, 1, "content labels must be"),
    (_maps(sshape=(2, 6, 6)), True, 2, 1, "style labels must be"),
    (_maps(sshape=(3, 6, 6)), True, 2, 2, "style labels must be"),
    (_maps(cshape=(0, 8)), True, 1, 1, "must not be empty"),
    (_maps(sshape=(6, 0)), True, 1, 1, "must not be empty"),
])
def test_check_swap_labels_rejects(value, swap, n, ns, match):
    with pytest.raises(ValueError, match=match):
        options.check_swap_labels(value, swap, n, ns)


def test_check_swap_labels_accepts():
    c, s = options.check_swap_labels(_maps(), True, 3)
    assert c.shape == (1, 8, 8) and s.shape == (1, 6, 6)
    c, s = options.check_swap_labels((np.zeros((3, 8, 8), np.uint8), np.zeros((3, 6, 6), np.uint8)), True, 3, 3)
    assert c.shape == (3, 8, 8) and s.shape == (3, 6, 6)
    c, s = options.check_swap_labels([torch.zeros(8, 8, dtype=torch.uint8), torch.zeros(6, 6, dtype=torch.uint8)], True, 1)
    assert isinstance(c, torch.Tensor) and c.shape == (1, 8, 8)
    assert "swap_labels" not in options.SPELLINGS


def _imgs(n, h, w, seed=0):
    return np.random.default_rng(seed).integers(0, 256, (n, h, w, 3), dtype=np.uint8)


def test_api_passes_labels_to_the_engine(stub):  # noqa: F811
    c, s = _imgs(2, 32, 32), _imgs(1, 16, 16, 1)
    cl = np.arange(32 * 32, dtype=np.int64).reshape(32, 32).astype(np.uint8)
    sl = np.ones((16, 16), np.uint8)
    stub.engine.prepare_call = lambda a, **kw: a          # passes > 1 prepare the style once
    stub.predict_batch(c, s, swap_targets=["relu3_1"], swap_labels=(cl, sl), passes=2)
    (m0, _, kw0), (m1, _, kw1) = stub.engine.calls
    got_c, got_s = kw0["swap_labels"]
    assert isinstance(got_c, torch.Tensor) and got_c.dtype == torch.uint8 and got_c.shape == (1, 32, 32)
    assert np.array_equal(got_c[0].numpy(), cl) and np.array_equal(got_s[0].numpy(), sl)
    assert kw1["swap_labels"] is None and kw1["swap_targets"] is None        # the labels act in the first pass only
    stub.engine.calls.clear()
    stub.predict(c[0], s[0], swap5=True, swap_labels=(cl, sl))
    assert stub.engine.calls[0][2]["swap_labels"] is not None and stub.engine.calls[0][2]["swap5"]
    stub.engine.calls.clear()
    per = _imgs(2, 16, 16, 2)
    stub.predict_batch(c, per, swap_targets=["relu3_1"], swap_labels=(np.stack([cl, cl]), np.stack([sl, sl])))
    assert stub.engine.calls[0][2]["swap_labels"][1].shape == (2, 16, 16)
    stub.engine.calls.clear()
    stub.predict_batch(c, PreparedStyle(1, {}, ["relu5_1"]), swap5=True, swap_labels=(cl, sl))
    assert stub.engine.calls[0][2]["swap_labels"] is not None


def test_api_crops_a_content_sized_map_with_the_content(stub, monkeypatch):  # noqa: F811
    """With a stride the content is centre-cropped for the swap; a map of the content's size is cropped the same way, a map
    of another size is passed whole."""
    from wct_tf_b200 import wct as W
    stub.ss_stride = 2
    monkeypatch.setattr(W.WCT, "swap_fit", lambda self, contents, *a: torch.as_tensor(contents)[:, 2:30, 2:30])
    c, s = _imgs(1, 32, 32), _imgs(1, 16, 16, 1)
    cl = np.arange(32 * 32, dtype=np.int64).reshape(32, 32).astype(np.uint8)
    stub.predict_batch(c, s, swap_targets=["relu3_1"], swap_labels=(cl, np.zeros((4, 4), np.uint8)))
    got = stub.engine.calls[0][2]["swap_labels"][0]
    assert np.array_equal(got[0].numpy(), cl[2:30, 2:30])
    stub.engine.calls.clear()
    other = cl[:16, :20].copy()
    stub.predict_batch(c, s, swap_targets=["relu3_1"], swap_labels=(other, np.zeros((4, 4), np.uint8)))
    assert np.array_equal(stub.engine.calls[0][2]["swap_labels"][0][0].numpy(), other)


@pytest.mark.parametrize("kw,match", [
    (dict(), "needs swap5 / swap_targets"),
    (dict(swap_targets=["relu3_1"], adain=True, content_mask=np.zeros((8, 8), np.uint8)), "content_mask"),
    (dict(swap_targets=["relu3_1"], labels_dtype=np.int16), "uint8"),
    (dict(swap_targets=["relu3_1"], n_content_maps=3), "content labels"),
    (dict(swap_targets=["relu3_1"], n_style_maps=2), "style labels"),
])
def test_api_rejects_before_device_work(stub, kw, match):  # noqa: F811
    kw = dict(kw)
    dt = kw.pop("labels_dtype", np.uint8)
    cl = np.zeros((kw.pop("n_content_maps", 1), 8, 8), dt)
    sl = np.zeros((kw.pop("n_style_maps", 1), 8, 8), np.uint8)
    styles = [_imgs(1, 16, 16)[0]] if "content_mask" in kw else _imgs(1, 16, 16)
    with pytest.raises(ValueError, match=match):
        stub.predict_batch(_imgs(2, 32, 32), styles, swap_labels=(cl, sl), **kw)
    assert stub.engine.calls == []


def test_synthesize_passes_labels(stub, monkeypatch):  # noqa: F811
    from wct_tf_b200 import device_image
    monkeypatch.setattr(device_image, "noise_u8", lambda n, h, w, seed=0, first_index=0, device=None: torch.zeros(
        (n, h, w, 3), dtype=torch.uint8))
    lab = (np.zeros((8, 8), np.uint8), np.zeros((8, 8), np.uint8))
    stub.synthesize(_imgs(1, 16, 16), (32, 48), count=3, swap_targets=["relu3_1"], swap_labels=lab)
    assert stub.engine.calls[0][2]["swap_labels"][0].shape == (1, 8, 8)
