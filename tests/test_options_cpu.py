"""The table of options that combine (wct_tf_b200/options.py): its verdict on every pair, and that stylize.py,
WCT.predict_batch and WCT.predict follow it.  No GPU needed (a stub engine records what reaches it)."""
import contextlib
import itertools

import numpy as np
import pytest
import torch

import stylize
from tests.test_tiles_cpu import _base
from wct_tf_b200 import options
from wct_tf_b200 import temporal as T
from wct_tf_b200 import wct as W
from wct_tf_b200.engine import Engine
from wct_tf_b200.prepared import PreparedStyle

OPTIONS = sorted(options.SPELLINGS)
_SOFT = ("strength_map", "content_weights", "mask_feather")
# every pair of options that does not combine, or of which one needs an option the other is not
REJECTED = {frozenset(p) for p in
            [("efdm", b) for b in ("adain", "ost", "mst", "content_mask", "style_masks", "content_weights", "mask_feather",
                                   "strength_map", "style_weights", "tile_size", "prepared")]
            + [("mst", b) for b in ("adain", "ost", "content_mask", "style_masks", "style_weights", "swap", "tile_size",
                                    "seamless", "prepared", "per_frame_styles")]
            + [(a, b) for a in _SOFT for b in ("style_weights", "swap", "mst", "tile_size")]
            + [(a, b) for a in ("content_weights", "mask_feather") for b in ("adain", "ost")]
            + [("ost", b) for b in ("adain", "content_mask", "style_masks", "style_weights")]
            + [("tile_size", b) for b in ("content_mask", "style_masks", "style_weights", "swap", "temporal")]
            + [("seamless", "swap"), ("seamless", "temporal"), ("style_weights", "content_mask"), ("style_weights", "swap"),
               ("content_mask", "adain"), ("content_mask", "swap"), ("temporal", "return_float"),
               ("content_weights", "content_mask")]}
NEEDS = {"mask_feather": {"content_mask"}, "style_masks": {"content_mask", "content_weights"}}


def _pairs():
    return [(a,) for a in OPTIONS] + list(itertools.combinations(OPTIONS, 2))


def _expected_ok(combo):
    s = set(combo)
    if len(s) == 2 and frozenset(s) in REJECTED:
        return False
    return all(not (a in s and not s & want) for a, want in NEEDS.items())


def _table_ok(combo, vocab=options.API):
    try:
        options.check(set(combo), vocab)
        return True
    except ValueError:
        return False


@pytest.mark.parametrize("combo", _pairs(), ids="+".join)
def test_table_verdict(combo):
    assert _table_ok(combo) == _expected_ok(combo)


# ---------------------------------------------------------------------------------------------------- stylize.py flags
_CLI_ARGS = {"adain": ["--adain"], "ost": ["--ost"], "efdm": ["--efdm"], "mst": ["--mst", "2"], "swap": ["--swap5"],
             "content_mask": ["--content-mask", "m.png"], "style_masks": ["--style-masks", "ma.png", "mb.png"],
             "style_weights": [], "content_weights": ["--mask-weights", "wa.png", "wb.png"],
             "mask_feather": ["--mask-feather", "2"], "strength_map": ["--strength-map", "g.png"],
             "tile_size": ["--tile-size", "64"], "seamless": ["--seamless", "x"], "prepared": []}


def _cli_argv(tmp_path, combo):
    ext = ".wctstyle" if "prepared" in combo else ".png"
    argv = _base(tmp_path)
    if "content_mask" in combo or "content_weights" in combo:
        argv += ["--mask-styles", "a" + ext, "b" + ext]
    if "style_weights" in combo:
        argv += ["--interp-styles", "a" + ext, "b" + ext, "--interp-weights", "1", "1"]
    if argv == _base(tmp_path):
        argv += ["--style-path", "s" + ext]
    return argv + sum((_CLI_ARGS[o] for o in combo), [])


@pytest.mark.parametrize("combo", [c for c in _pairs() if all(o in _CLI_ARGS for o in c)], ids="+".join)
def test_stylize_flags_follow_the_table(tmp_path, combo, capsys):
    argv = _cli_argv(tmp_path, combo)
    if _table_ok(combo):
        stylize.parse_args(argv)
        return
    with pytest.raises(SystemExit):
        stylize.parse_args(argv)
    err = capsys.readouterr().err
    if frozenset(combo) in REJECTED:
        assert all(options.CLI[o] in err for o in combo)
    else:
        assert any(options.CLI[o] + " needs " in err for o in combo if o in NEEDS)


# ---------------------------------------------------------------------------------------- WCT.predict / predict_batch
ALL = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]
API_OPTIONS = ["adain", "ost", "efdm", "mst", "swap5", "swap_targets", "content_mask", "style_masks", "style_weights",
               "content_weights", "mask_feather", "strength_map", "tile_size", "seamless", "temporal", "return_float",
               "prepared", "per_frame_styles"]


class _Level(object):
    def __init__(self, relu):
        self.relu_target = relu


class StubEngine(object):
    """Records every stylize / stylize_tiled call: (method, style argument, keyword arguments)."""
    device = "cpu"

    def __init__(self):
        self.calls = []
        self.model = type("Model", (), dict(levels=[_Level(r) for r in ALL]))()

    swap_levels = Engine.swap_levels

    def stylize(self, c, s, **kw):
        self.calls.append(("stylize", s, kw))
        return torch.zeros(c.shape, dtype=torch.float32)

    def stylize_tiled(self, c, s, **kw):
        self.calls.append(("stylize_tiled", s, kw))
        return torch.zeros(c.shape, dtype=torch.float32)

    def to_u8(self, x):
        return x.to(torch.uint8)

    def check_device(self):
        pass


@pytest.fixture
def stub(monkeypatch):
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    stabilized = []
    monkeypatch.setattr(T, "stabilize_", lambda state, c, out: stabilized.append(state))
    empty = torch.empty
    monkeypatch.setattr(torch, "empty", lambda *a, pin_memory=False, **k: empty(*a, **k))
    m = W.WCT.__new__(W.WCT)
    m.ss_patch_size, m.ss_stride, m.verbose = 3, 1, False
    m.engine = StubEngine()
    m.model = m.engine.model
    m.stabilized = stabilized
    return m


def _call(combo, n):
    """(content [n,32,32,3], styles, predict_batch keywords) of a call with the options ``combo``."""
    rng = np.random.default_rng(0)
    c = rng.integers(0, 256, (n, 32, 32, 3), dtype=np.uint8)
    s = rng.integers(0, 256, (1, 16, 16, 3), dtype=np.uint8)
    listed = any(o in combo for o in ("content_mask", "style_weights", "content_weights"))
    if "prepared" in combo:
        styles = [PreparedStyle(1, {}, ALL)] * 2 if listed else PreparedStyle(n if "per_frame_styles" in combo else 1, {}, ALL)
    elif listed:
        styles = [s[0], s[0]]
    elif "per_frame_styles" in combo:
        styles = rng.integers(0, 256, (n, 16, 16, 3), dtype=np.uint8)
    else:
        styles = s
    values = dict(mst=2, swap_targets=["relu3_1"], content_mask=np.zeros((8, 8), np.uint8),
                  style_masks=[None, np.zeros((8, 8), np.uint8)], style_weights=[1.0, 2.0],
                  content_weights=np.full((2, 8, 8), 0.25, np.float32), mask_feather=2.0,
                  strength_map=np.full((8, 8), 0.5, np.float32), tile_size=64, seamless="x")
    kw = {}
    for o in combo:
        if o == "temporal":
            kw[o] = T.TemporalState(0.5)
        elif o not in ("prepared", "per_frame_styles"):
            kw[o] = values.get(o, True)
    return c, styles, kw


def _reached(o, method, style, kw):
    """Whether the option ``o`` of the call reached the engine call (method, style, kw)."""
    if o == "tile_size":
        return method == "stylize_tiled" and kw["tile_size"] == 64
    if o == "prepared":
        styles = kw.get("region_styles") or kw.get("interp_styles") or [style]
        return all(isinstance(x, PreparedStyle) for x in styles)
    if o == "per_frame_styles":
        styles = kw.get("region_styles") or kw.get("interp_styles")
        return len(styles) == 2 if styles else (style.n if isinstance(style, PreparedStyle) else style.shape[0]) == 2
    name = {"content_mask": "labels", "style_masks": "region_masks", "style_weights": "interp_weights"}.get(o, o)
    return kw.get(name) is not None and kw.get(name) is not False


def _api_combos(single):
    skip = {"temporal", "return_float", "per_frame_styles"} if single else set()
    return [c for c in [(o,) for o in API_OPTIONS] + list(itertools.combinations(API_OPTIONS, 2)) if not skip & set(c)]


def _canonical(combo):
    return tuple(sorted({"swap" if o in ("swap5", "swap_targets") else o for o in combo}))


@pytest.mark.parametrize("single", [False, True], ids=["predict_batch", "predict"])
def test_api_follows_the_table(stub, single):
    for combo in _api_combos(single):
        stub.engine.calls.clear()
        del stub.stabilized[:]
        c, styles, kw = _call(combo, 1 if single else 2)
        ok = _table_ok(_canonical(combo)) and set(combo) != {"swap5", "swap_targets"}
        if not ok:
            with pytest.raises(ValueError):
                if single:
                    stub.predict(c[0], styles[0] if isinstance(styles, np.ndarray) else styles, **kw)
                else:
                    stub.predict_batch(c, styles, return_device=True, **kw)
            assert stub.engine.calls == [], combo
            continue
        if single:
            stub.predict(c[0], styles[0] if isinstance(styles, np.ndarray) else styles, **kw)
        else:
            out = stub.predict_batch(c, styles, return_device=True, **kw)
            assert isinstance(out, tuple) == ("return_float" in combo)
        assert len(stub.engine.calls) == 1, combo
        method, style, ekw = stub.engine.calls[0]
        for o in combo:
            if o == "temporal":
                assert stub.stabilized == [kw["temporal"]]
            elif o != "return_float":
                assert _reached(o, method, style, ekw), (combo, o)
