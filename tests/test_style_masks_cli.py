"""CLI style masks (stylize.py --style-masks): flag errors, mask quantisation, one load per repeated path and the call the
driver makes; no GPU needed (fake WCT)."""
import numpy as np
import pytest
from PIL import Image

import stylize
from tests.regions_ref import mask_regions


def _base(tmp_path):
    return ["--relu-targets", "relu1_1", "--synthetic-weights", "1", "--content-path", str(tmp_path / "c.png"),
            "--out-path", str(tmp_path / "out")]


@pytest.mark.parametrize("argv", [
    ["--mask-styles", "a.png", "--style-masks", "m.png"],                                           # no --content-mask
    ["--content-mask", "m.png", "--mask-styles", "a.png", "b.png", "--style-masks", "m.png"],       # one mask per style
    ["--content-mask", "m.png", "--mask-styles", "a.png", "--style-masks", "m.png", "n.png"],
    ["--content-mask", "m.png", "--mask-styles", "a.png", "--style-masks", "m.png", "--crop-size", "256"],
    ["--content-mask", "m.png", "--mask-styles", "a.wctstyle", "--style-masks", "m.png"],           # prepared styles
])
def test_style_mask_flag_errors(tmp_path, argv):
    with pytest.raises(SystemExit):
        stylize.parse_args(_base(tmp_path) + argv)


def test_style_mask_flags_accepted_and_default_off(tmp_path):
    a = stylize.parse_args(["--relu-targets", "relu1_1"])
    assert a.style_masks is None
    a = stylize.parse_args(_base(tmp_path) + ["--content-mask", "m.png", "--mask-styles", "a.png", "a.png", "--style-masks",
                                              "s.png", "s.png", "--style-size", "300"])
    assert a.style_masks == ["s.png", "s.png"] and a.style_size == 300


def _write(tmp_path):
    Image.fromarray(np.full((8, 12, 3), 10, np.uint8)).save(str(tmp_path / "c.png"))
    for name, v in (("painting", 50), ("sea", 90)):
        Image.fromarray(np.full((6, 6, 3), v, np.uint8)).save(str(tmp_path / (name + ".png")))
    mask = np.zeros((8, 12), np.uint8)
    mask[4:] = 200
    Image.fromarray(mask, mode="L").save(str(tmp_path / "m.png"))
    smask = np.tile(np.arange(0, 256, 43, dtype=np.uint8), (6, 1))              # every grey level of a 6-wide ramp
    Image.fromarray(smask, mode="L").save(str(tmp_path / "sm.png"))
    return mask, smask


class _HostImageOps(object):
    to_device = staticmethod(lambda img, device=None: np.asarray(img))
    to_host = staticmethod(lambda img: np.asarray(img))
    resize_to = staticmethod(lambda img, size: img)


def _fake(calls):
    class FakeWCT(object):
        class engine(object):
            device = None

        def predict_batch(self, contents, styles, alpha=1, content_mask=None, return_device=False, **kw):
            calls.append((list(styles), np.asarray(content_mask).copy(), alpha, kw))
            c = np.asarray(contents)
            return (c[None] if c.ndim == 3 else c) + 1
    return FakeWCT()


def test_style_masked_run_loads_each_path_once_and_names_output(tmp_path, monkeypatch):
    mask, smask = _write(tmp_path)
    from wct_tf_b200 import imageio
    loads = []
    get_img = imageio.get_img
    monkeypatch.setattr(imageio, "get_img", lambda p: (loads.append(p), get_img(p))[1])
    read_mask = stylize.read_mask
    mask_reads = []
    monkeypatch.setattr(stylize, "read_mask", lambda p, R: (mask_reads.append(p), read_mask(p, R))[1])
    calls = []
    p, sm = str(tmp_path / "painting.png"), str(tmp_path / "sm.png")
    argv = _base(tmp_path) + ["--content-mask", str(tmp_path / "m.png"), "--mask-styles", p, p, "--style-masks", sm, sm,
                              "--alpha", "0.7", "--passes", "2"]
    n = stylize.main(argv, model_factory=lambda a: _fake(calls), image_ops=_HostImageOps)
    assert n == 1
    out = tmp_path / "out" / "c_painting+painting.png"
    assert out.exists()
    assert np.array_equal(np.asarray(Image.open(str(out))), np.full((8, 12, 3), 12, np.uint8))   # two passes
    assert loads.count(p) == 1 and mask_reads.count(sm) == 1
    assert len(calls) == 2
    for styles, m, alpha, kw in calls:
        assert styles[0] is styles[1] and int(np.asarray(styles[0])[0, 0, 0]) == 50 and alpha == 0.7
        assert np.array_equal(m, mask_regions(mask, 2))
        assert set(kw) == {"style_masks"}
        s0, s1 = kw["style_masks"]
        assert s0 is s1 and np.array_equal(s0, mask_regions(smask, 2))            # quantised like the content mask
        assert s0.dtype == np.uint8


def test_distinct_style_masks_are_passed_in_order(tmp_path):
    _, smask = _write(tmp_path)
    Image.fromarray(255 - smask, mode="L").save(str(tmp_path / "sm2.png"))
    calls = []
    argv = _base(tmp_path) + ["--content-mask", str(tmp_path / "m.png"), "--mask-styles", str(tmp_path / "painting.png"),
                              str(tmp_path / "sea.png"), "--style-masks", str(tmp_path / "sm.png"), str(tmp_path / "sm2.png")]
    stylize.main(argv, model_factory=lambda a: _fake(calls), image_ops=_HostImageOps)
    styles, _, _, kw = calls[0]
    assert [int(np.asarray(s)[0, 0, 0]) for s in styles] == [50, 90]
    s0, s1 = kw["style_masks"]
    assert np.array_equal(s0, mask_regions(smask, 2)) and np.array_equal(s1, mask_regions(255 - smask, 2))
