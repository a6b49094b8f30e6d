"""Prepared styles without a GPU: encoder fingerprints and the checks of a ``.wctstyle`` file."""
import numpy as np
import pytest

from wct_tf_b200 import prepared as P
from wct_tf_b200.engine import SEMANTICS
from wct_tf_b200.weights import make_synthetic_weights

ALL = ["relu5_1", "relu4_1", "relu3_1", "relu2_1", "relu1_1"]
TF = {k: SEMANTICS["tf"][k] for k in P.SEMANTIC_KEYS}


def test_fingerprints_follow_the_encoder_only():
    a, b = make_synthetic_weights(1), make_synthetic_weights(2)
    fa = P.encoder_fingerprints(a["vgg"], ALL)
    assert sorted(fa) == sorted(ALL) and len(set(fa.values())) == 5
    assert P.encoder_fingerprints(make_synthetic_weights(1)["vgg"], ALL) == fa          # equal encoders
    mixed = dict(b, vgg=a["vgg"])                                                       # other decoders, same encoder
    assert P.encoder_fingerprints(mixed["vgg"], ALL) == fa
    assert P.encoder_fingerprints(a["vgg"], ["relu2_1"]) == {"relu2_1": fa["relu2_1"]}  # a subset of the targets
    fb = P.encoder_fingerprints(b["vgg"], ALL)
    assert all(fa[r] != fb[r] for r in ALL)
    # a change in conv4_1 leaves the levels below it alone
    c = make_synthetic_weights(1)
    layer = next(l for l in c["vgg"] if l["name"] == "conv4_1")
    layer["bias"] = np.asarray(layer["bias"]) + 1.0
    fc = P.encoder_fingerprints(c["vgg"], ALL)
    assert [fc[r] == fa[r] for r in ALL] == [False, False, True, True, True]


def _file(tmp_path, fp, **over):
    arrays = dict(format=np.array(P.FORMAT), version=np.array(P.VERSION), image=np.zeros((1, 8, 8, 3), np.uint8),
                  targets=np.array(["relu2_1", "relu1_1"]), **{k: np.array(v) for k, v in TF.items()})
    for r, c in (("relu2_1", 128), ("relu1_1", 64)):
        arrays.update({"%s/fingerprint" % r: np.array(fp[r]), "%s/wct_mean" % r: np.zeros((1, c), np.float32),
                       "%s/wct_cs" % r: np.zeros((1, c, c), np.float32), "%s/wct_k" % r: np.zeros((1, 2), np.int32),
                       "%s/adain_mean" % r: np.zeros((1, c), np.float32), "%s/adain_var" % r: np.zeros((1, c), np.float32)})
    arrays.update(over)
    path = str(tmp_path / "s.wctstyle")
    with open(path, "wb") as f:
        np.savez(f, **arrays)
    return path


def test_file_checks_name_the_field(tmp_path):
    w = make_synthetic_weights(3)
    fp = P.encoder_fingerprints(w["vgg"], ["relu2_1", "relu1_1"])
    path = _file(tmp_path, fp)
    data = P.read_file(path)
    P.check_file(data, path, TF, ["relu2_1", "relu1_1"], fp)
    P.check_file(data, path, TF, ["relu1_1"], fp)                                      # a subset of the targets
    with pytest.raises(ValueError, match="targets"):
        P.check_file(data, path, TF, ["relu3_1"], dict(fp, relu3_1="x"))
    with pytest.raises(ValueError, match="eps_cov"):
        P.check_file(data, path, {k: SEMANTICS["np"][k] for k in P.SEMANTIC_KEYS}, ["relu1_1"], fp)
    with pytest.raises(ValueError, match="eps_eig"):
        P.check_file(data, path, dict(TF, eps_eig=1e-5), ["relu1_1"], fp)
    other = P.encoder_fingerprints(make_synthetic_weights(4)["vgg"], ["relu2_1", "relu1_1"])
    with pytest.raises(ValueError, match="relu1_1/fingerprint"):
        P.check_file(data, path, TF, ["relu1_1"], other)
    with pytest.raises(ValueError, match="version"):
        P.read_file(_file(tmp_path, fp, version=np.array(2)))
    with pytest.raises(ValueError, match="format"):
        P.read_file(_file(tmp_path, fp, format=np.array("other")))
    # the container is read without pickles: an object array is refused
    with pytest.raises(ValueError):
        P.read_file(_file(tmp_path, fp, image=np.array([None, 1], dtype=object)))
