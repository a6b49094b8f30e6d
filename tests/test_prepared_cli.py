"""The CLI with prepared styles (.wctstyle), driven with stand-in models: parser rules, one load per file per run, output
names, ``--concat`` from the stored image, and the batched style swap of the video driver.  No GPU needed."""
import numpy as np
import pytest
from PIL import Image

import prepare_styles
import stylize
import stylize_video as V


class Prepared(object):
    """stand-in for a PreparedStyle: an id and the stored style image"""
    def __init__(self, value):
        self.n, self.image = 1, np.full((1, 6, 6, 3), value, np.uint8)


class FakeModel(object):
    class engine(object):
        device = None

    def __init__(self):
        self.loads, self.calls = [], []

    def load_style(self, path):
        self.loads.append(path)
        return Prepared(100 + len(self.loads))

    def prepare_style(self, img):
        model = self

        class Saver(object):
            def save(self, path):
                model.calls.append(("save", path, int(np.asarray(img)[0, 0, 0])))
        return Saver()

    def predict_batch(self, contents, styles, alpha=1, adain=False, passes=1, swap5=False, ss_alpha=None, **kw):
        c = np.asarray(contents)
        c = c[None] if c.ndim == 3 else c
        self.calls.append(("predict", [int(x[0, 0, 0]) for x in c], styles, passes, swap5, ss_alpha))
        return c + 1


class HostImageOps(object):
    to_device = staticmethod(lambda img, device=None: np.asarray(img))
    to_host = staticmethod(lambda img: np.asarray(img))
    resize_to = staticmethod(lambda img, size: img)
    center_crop = staticmethod(lambda img, size: img[:size, :size])
    concat_with_style = staticmethod(lambda style, result: np.hstack([np.repeat(np.asarray(style)[:1], result.shape[0], 0), result]))


def _png(path, value, hw=(8, 12)):
    Image.fromarray(np.full(hw + (3,), value, dtype=np.uint8)).save(str(path))
    return str(path)


def _touch(path):
    path.write_bytes(b"")
    return str(path)


def test_parser_rules(tmp_path):
    a, b, img = _touch(tmp_path / "a.wctstyle"), _touch(tmp_path / "b.wctstyle"), _png(tmp_path / "s.png", 1)
    base = ["--relu-targets", "relu1_1", "--content-path", "c.png", "--out-path", "o"]
    stylize.parse_args(base + ["--style-path", a])
    stylize.parse_args(base + ["--interp-styles", a, b, "--interp-weights", "1", "1"])
    stylize.parse_args(["--relu-targets", "relu1_1", "--content-path", "c.png", "--out-path", "o", "--content-mask", "m.png",
                        "--mask-styles", a, b])
    for extra in (["--style-path", a, "--style-size", "256"], ["--style-path", a, "--crop-size", "256"],
                  ["--style-path", a, "--keep-colors"], ["--interp-styles", a, img, "--interp-weights", "1", "1"]):
        with pytest.raises(SystemExit):
            stylize.parse_args(base + extra)
    mixed = tmp_path / "mixed"
    mixed.mkdir()
    _touch(mixed / "x.wctstyle")
    _png(mixed / "y.png", 2)
    with pytest.raises(SystemExit):
        stylize.parse_args(base + ["--style-path", str(mixed)])
    vbase = ["--relu-targets", "relu1_1", "--in-path", "x", "--out-path", "y"]
    V.parse_args(vbase + ["--style-path", a])
    for extra in (["--style-path", a, "--style-size", "64"], ["--interp-styles", a, img, "--interp-weights", "1", "1"]):
        with pytest.raises(SystemExit):
            V.parse_args(vbase + extra)


def test_each_file_loaded_once_names_and_concat(tmp_path):
    contents = tmp_path / "contents"
    contents.mkdir()
    for i in (1, 2, 3):
        _png(contents / ("c%d.png" % i), 10 * i)
    styles = tmp_path / "styles"
    styles.mkdir()
    _touch(styles / "starry.wctstyle")
    _touch(styles / "wave.wctstyle")
    model = FakeModel()
    out = tmp_path / "out"
    n = stylize.main(["--relu-targets", "relu1_1", "--content-path", str(contents), "--style-path", str(styles), "--out-path",
                      str(out), "--passes", "2", "--concat"], model_factory=lambda a: model, image_ops=HostImageOps)
    assert n == 6
    assert sorted(model.loads) == sorted(str(styles / f) for f in ("starry.wctstyle", "wave.wctstyle"))   # once per file
    predicts = [c for c in model.calls if c[0] == "predict"]
    assert len(predicts) == 12                                         # 3 contents x 2 styles x 2 passes
    assert all(isinstance(c[2], Prepared) for c in predicts)
    res = np.array(Image.open(str(out / "c2_starry.png")))
    assert res.shape == (8, 6 + 12, 3) and res[0, -1, 0] == 22         # 20 + two passes
    assert res[0, 0, 0] in (101, 102)                                  # --concat shows the stored style image
    assert (out / "c3_wave.png").exists()
    # interpolation and masks read their files once as well
    model2 = FakeModel()
    stylize.main(["--relu-targets", "relu1_1", "--content-path", str(contents), "--interp-styles", str(styles / "starry.wctstyle"),
                  str(styles / "wave.wctstyle"), "--interp-weights", "1", "3", "--out-path", str(out)],
                 model_factory=lambda a: model2, image_ops=HostImageOps)
    assert len(model2.loads) == 2 and (out / "c1_starry-0.25+wave-0.75.png").exists()


def test_prepare_styles_writes_one_file_per_style(tmp_path):
    styles = tmp_path / "styles"
    styles.mkdir()
    _png(styles / "a.png", 5)
    _png(styles / "b.jpg", 7)
    model = FakeModel()
    n = prepare_styles.main(["--relu-targets", "relu1_1", "--style-path", str(styles), "--out-path", str(tmp_path / "p"),
                             "--crop-size", "4"], model_factory=lambda a: model, image_ops=HostImageOps)
    assert n == 2
    saves = sorted((c[1], c[2]) for c in model.calls if c[0] == "save")
    assert saves == [(str(tmp_path / "p" / "a.wctstyle"), 5), (str(tmp_path / "p" / "b.wctstyle"), 7)]


def test_video_batches_swap5_frames(tmp_path):
    frames = tmp_path / "clip"
    frames.mkdir()
    for i in (1, 2, 3, 4):
        _png(frames / ("frame_%d.png" % i), i)
    _png(frames / "frame_5.png", 5, hw=(16, 12))                      # ragged: per frame
    style = _png(tmp_path / "style.png", 200, hw=(6, 6))
    model = FakeModel()
    out = tmp_path / "out"
    n = V.main(["--relu-targets", "relu5_1", "--in-path", str(frames), "--style-path", style, "--out-path", str(out), "--batch",
                "2", "--swap5", "--ss-alpha", "0.4"], wct_factory=lambda a: model, image_ops=HostImageOps)
    assert n == 5
    calls = [c for c in model.calls if c[0] == "predict"]
    assert [c[1] for c in calls] == [[1, 2], [3, 4], [5]]
    assert all(c[4] and c[5] == 0.4 for c in calls)                   # the batched calls swap, with --ss-alpha
    # a prepared style is read once for the whole clip
    model2 = FakeModel()
    pstyle = _touch(tmp_path / "starry.wctstyle")
    V.main(["--relu-targets", "relu5_1", "--in-path", str(frames), "--style-path", pstyle, "--out-path", str(out), "--batch", "2",
            "--swap5", "--concat"], wct_factory=lambda a: model2, image_ops=HostImageOps)
    assert model2.loads == [pstyle]
    assert all(isinstance(c[2], Prepared) for c in model2.calls if c[0] == "predict")
    assert (out / "clip_starry_frames" / "frame_3.png").exists()
