"""Coarse-to-fine stylisation (DESIGN.md §3.3.16) without a GPU: the options rules and their messages in the three
vocabularies, the fine-target checks and defaults, the coarse size rule at its edges, the join oracle against torch's
bilinear interpolation, and the two-stage call WCT.predict_batch makes (a stub engine and host stand-ins for the image
steps record it)."""
import contextlib

import numpy as np
import pytest
import torch

from tests import coarse_ref as R
from wct_tf_b200 import device_image as D
from wct_tf_b200 import options
from wct_tf_b200 import wct as W
from wct_tf_b200.model import coarse_size
from wct_tf_b200.prepared import PreparedStyle

ALL = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]
VOCABS = [options.API, options.ENGINE, options.CLI]


# ------------------------------------------------------------------------------------------------------------ options
@pytest.mark.parametrize("other,why", [("swap", "patch grid"), ("seamless", "wraps"), ("mst", "own level chain")])
@pytest.mark.parametrize("vocab", [options.API, options.CLI], ids=["api", "cli"])
def test_rejected_combinations_name_both(other, why, vocab):
    with pytest.raises(ValueError) as e:
        options.check({"coarse_to_fine", other}, vocab)
    msg = str(e.value)
    assert vocab["coarse_to_fine"] in msg and vocab[other] in msg and why in msg


@pytest.mark.parametrize("other", sorted(set(options.SPELLINGS) - {"swap", "seamless", "mst"}) + ["luminance_only"])
def test_every_other_option_combines(other):
    needs = dict(options.NEEDS).get(other, ())
    options.check({"coarse_to_fine", other} | set(needs[:1]), options.API)


def test_spellings():
    assert options.API["coarse_to_fine"] == "coarse_to_fine"
    assert options.ENGINE["coarse_to_fine"] is None
    assert options.CLI["coarse_to_fine"] == "--coarse-to-fine"
    assert "coarse_to_fine" not in options.SPELLINGS           # the engine's part is levels=, not an option of its own


def test_fine_target_defaults():
    assert options.check_coarse_to_fine(4, None, ALL) == (4, ("relu3_1", "relu2_1", "relu1_1"))
    assert options.check_coarse_to_fine(np.int64(2), None, ["relu4_1", "relu1_1"]) == (2, ("relu1_1",))
    with pytest.raises(ValueError, match="none of the default fine targets"):
        options.check_coarse_to_fine(2, None, ["relu5_1", "relu4_1"])


def test_fine_targets_run_in_the_models_order():
    assert options.check_coarse_to_fine(2, ["relu1_1", "relu4_1"], ALL) == (2, ("relu4_1", "relu1_1"))
    assert options.check_coarse_to_fine(16, "relu2_1", ALL) == (16, ("relu2_1",))
    assert options.check_levels(["relu1_1", "relu5_1"], ALL) == ("relu5_1", "relu1_1")


@pytest.mark.parametrize("f", [0, 1, 17, -2, 2.0, 4.5, True, "4", None])
def test_factor_range(f):
    with pytest.raises(ValueError, match="coarse_to_fine" if f is not None else "needs coarse_to_fine"):
        options.check_coarse_to_fine(f, None if f is not None else ["relu1_1"], ALL)


@pytest.mark.parametrize("fine,msg", [([], "at least one"), (["relu6_1"], "not a relu target"),
                                      (["relu3_1"], "not a relu target"), (["relu1_1", "relu1_1"], "more than once")])
def test_bad_fine_targets(fine, msg):
    with pytest.raises(ValueError, match=msg):
        options.check_coarse_to_fine(2, fine, ["relu4_1", "relu1_1"])


def test_messages_in_the_cli_vocabulary():
    with pytest.raises(ValueError, match="--fine-targets needs --coarse-to-fine"):
        options.check_coarse_to_fine(None, ["relu1_1"], ALL, options.CLI)
    with pytest.raises(ValueError, match="--coarse-to-fine must be an integer factor in 2..16"):
        options.check_coarse_to_fine(1, None, ALL, options.CLI)
    with pytest.raises(ValueError, match="--fine-targets: relu9_1"):
        options.check_coarse_to_fine(2, ["relu9_1"], ALL, options.CLI)


# ---------------------------------------------------------------------------------------------------------- size rule
@pytest.mark.parametrize("g", [1, 2, 4, 8, 16])
@pytest.mark.parametrize("f", [2, 3, 4, 5, 8, 16])
def test_size_rule_matches_the_oracle(f, g):
    for n in list(range(1, 3 * f * g + 3)) + [g * f - 1, g * f, g * f + 1, 1000, 1496, 4096, 12288]:
        assert coarse_size(n, n + 7, f, g) == R.coarse_size(n, n + 7, f, g)


def test_size_rule_edges():
    g = 16
    assert coarse_size(5, 9, 2, g) == (16, 16)                  # H < g: one g, larger than the frame
    assert coarse_size(31, 33, 2, g) == (16, 16)                # g f - 1, g f + 1
    assert coarse_size(47, 48, 2, g) == (16, 32)                # 1.47 rounds down, 1.5 up
    assert coarse_size(1000, 1496, 4, g) == (256, 368)          # non-square
    assert coarse_size(4096, 4096, 4, g) == (1024, 1024)
    h, w = coarse_size(777, 1234, 3, g)
    assert h % g == 0 and w % g == 0 and abs(h - 777 / 3) <= g / 2 and abs(w - 1234 / 3) <= g / 2


# ------------------------------------------------------------------------------------------------------------ oracle
@pytest.mark.parametrize("hw,coarse", [((1000, 1496), (256, 368)), ((10, 12), (16, 16)), ((40, 50), (16, 16)),
                                       ((1, 37), (16, 16)), ((37, 1), (16, 16)), ((64, 64), (16, 16)), ((96, 128), (48, 64))])
def test_oracle_is_bilinear_interpolation(hw, coarse):
    rng = np.random.default_rng(hw[0] * 7 + hw[1])
    d = rng.integers(0, 256, (2,) + coarse + (3,), dtype=np.uint8)
    s = rng.integers(0, 256, (2,) + coarse + (3,), dtype=np.uint8)
    got = R.upsampled_delta(d, s, *hw)
    delta = torch.from_numpy(s.astype(np.float32) - d.astype(np.float32)).permute(0, 3, 1, 2)
    want = torch.nn.functional.interpolate(delta, size=hw, mode="bilinear", align_corners=False).permute(0, 2, 3, 1).numpy()
    # |delta| <= 255.  torch may round the scale n_in / n_out differently: one float32 ulp of it moves a source coordinate
    # by up to n_in ulps of 1, each worth up to 2 |delta| after the two interpolations; plus a few roundings of the result
    assert np.abs(got - want).max() <= 255 * (2 * max(coarse) + 8) * 2.0 ** -23


def test_oracle_join_rounds_half_to_even_and_clips():
    c = np.array([[[[10, 0, 255]]]], np.uint8)
    d = np.zeros((1, 1, 1, 3), np.uint8)
    s = np.array([[[[0, 5, 200]]]], np.uint8)
    assert R.join(c, d, s).tolist() == [[[[10, 5, 255]]]]
    # a constant difference passes unchanged; a zero difference returns the content
    c = np.random.default_rng(1).integers(0, 256, (1, 9, 11, 3), dtype=np.uint8)
    assert np.array_equal(R.join(c, d.repeat(4, 1).repeat(4, 2), d.repeat(4, 1).repeat(4, 2)), c)
    up = R.join(np.full((1, 9, 11, 3), 100, np.uint8), np.full((1, 4, 4, 3), 50, np.uint8), np.full((1, 4, 4, 3), 57, np.uint8))
    assert (up == 107).all()


# -------------------------------------------------------------------------------------------------- the call it makes
class _Level(object):
    def __init__(self, relu):
        self.relu_target = relu


class StubEngine(object):
    """Records every stylize / stylize_tiled call and the style sides it prepares."""
    device = "cpu"

    def __init__(self):
        self.calls, self.prepared = [], []
        self.model = type("Model", (), dict(levels=[_Level(r) for r in ALL], relu_targets=ALL, deepest_target="relu5_1"))()

    def swap_levels(self, swap5=False, swap_targets=None):
        return ()

    def prepare_call(self, style, **kw):
        ps = PreparedStyle(style.shape[0], {}, ALL)
        self.prepared.append((ps, kw))
        return ps

    def stylize(self, c, s, **kw):
        self.calls.append(("stylize", tuple(c.shape), s, kw))
        return torch.full(c.shape, 7.0)

    def stylize_tiled(self, c, s, **kw):
        self.calls.append(("stylize_tiled", tuple(c.shape), s, kw))
        return torch.full(c.shape, 7.0)

    def to_u8(self, x):
        return x.to(torch.uint8)

    def check_device(self):
        pass


@pytest.fixture
def stub(monkeypatch):
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    joins = []

    def imresize(x, hw):
        return torch.zeros((x.shape[0],) + tuple(hw) + (3,), dtype=torch.uint8)

    def coarse_join(c, d, s):
        joins.append((tuple(c.shape), tuple(d.shape), tuple(s.shape)))
        return c.clone()
    monkeypatch.setattr(D, "imresize", imresize)
    monkeypatch.setattr(D, "coarse_join", coarse_join)
    m = W.WCT.__new__(W.WCT)
    m.ss_patch_size, m.ss_stride, m.verbose = 3, 1, False
    m.engine = StubEngine()
    m.model = m.engine.model
    m.joins = joins
    return m


@pytest.mark.parametrize("tiled", [False, True])
def test_two_stages_with_one_style_side(stub, tiled):
    c = np.zeros((2, 100, 130, 3), np.uint8)
    s = np.zeros((1, 20, 20, 3), np.uint8)
    kw = dict(tile_size=64) if tiled else {}
    stub.predict_batch(c, s, coarse_to_fine=2, passes=2, return_device=True, **kw)
    method = "stylize_tiled" if tiled else "stylize"
    assert len(stub.engine.prepared) == 1                      # prepared once for both stages and both passes
    ps = stub.engine.prepared[0][0]
    h, w = coarse_size(100, 130, 2, 16)
    fine = ("relu3_1", "relu2_1", "relu1_1")
    want = [(method, (2, h, w, 3), ps, None), (method, (2, 100, 130, 3), ps, fine)] * 2
    assert [(m, shape, st, kw.get("levels")) for m, shape, st, kw in stub.engine.calls] == want
    assert stub.joins == [((2, 100, 130, 3), (2, h, w, 3), (2, h, w, 3))] * 2


def test_fine_targets_reach_the_fine_stage(stub):
    c = np.zeros((1, 64, 64, 3), np.uint8)
    s = np.zeros((1, 20, 20, 3), np.uint8)
    stub.predict_batch(c, s, coarse_to_fine=4, fine_targets=["relu1_1", "relu2_1"], return_device=True)
    assert [kw.get("levels") for _, _, _, kw in stub.engine.calls] == [None, ("relu2_1", "relu1_1")]
    assert [shape for _, shape, _, _ in stub.engine.calls] == [(1, 16, 16, 3), (1, 64, 64, 3)]


def test_off_is_one_untouched_call(stub):
    c = np.zeros((1, 64, 64, 3), np.uint8)
    s = np.zeros((1, 20, 20, 3), np.uint8)
    stub.predict_batch(c, s, return_device=True)
    assert len(stub.engine.calls) == 1 and stub.engine.calls[0][3].get("levels") is None
    assert stub.engine.prepared == [] and stub.joins == []


@pytest.mark.parametrize("kw,msg", [(dict(swap5=True), "swap"), (dict(seamless="x"), "seamless"), (dict(mst=2), "mst"),
                                    (dict(fine_targets=["relu1_1"], coarse_to_fine=None), "fine_targets needs"),
                                    (dict(coarse_to_fine=1), "2..16"), (dict(fine_targets=["relu1_1", "relu1_1"]), "more than once")])
def test_rejected_before_device_work(stub, kw, msg):
    c = np.zeros((1, 64, 64, 3), np.uint8)
    s = np.zeros((1, 20, 20, 3), np.uint8)
    kw = dict(dict(coarse_to_fine=2), **kw)
    with pytest.raises(ValueError, match=msg):
        stub.predict_batch(c, s, return_device=True, **kw)
    assert stub.engine.calls == [] and stub.joins == []
