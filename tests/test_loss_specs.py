"""CPU checks of the loss codes at the interface: the header's b2g_loss, engine.LOSSES and the Java facade's LossFunction codes agree, the spec's
activation reaches b2g_layer_desc for the losses that apply one, the default discriminator builders produce the same specs and descriptors as
before the loss options existed, and loss specs round-trip through a checkpoint."""
import json
import os
import re

import numpy as np
import pytest

from gan_deeplearning4j_b200 import engine, models as m

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("XENT", "MCXENT", "MSE", "L1", "L2", "MAE", "HINGE", "SQUARED_HINGE", "WASSERSTEIN")
JAVA = {"XENT": 0, "MCXENT": 1, "MSE": 2, "L1": 3, "L2": 4, "MEAN_ABSOLUTE_ERROR": 5, "HINGE": 6, "SQUARED_HINGE": 7, "WASSERSTEIN": 8}


def test_loss_codes_agree_across_header_engine_and_java():
    src = open(os.path.join(ROOT, "include", "b200gan.h")).read()
    body = re.search(r"typedef enum \{([^}]*)\} b2g_loss;", src).group(1)
    header = {k: int(v) for k, v in re.findall(r"B2G_LOSS_(\w+) = (\d+)", body)}
    assert header == {n: i for i, n in enumerate(NAMES)}
    assert {k.upper(): v for k, v in engine.LOSSES.items()} == header
    jsrc = open(os.path.join(ROOT, "java/src/main/java/org/nd4j/linalg/lossfunctions/LossFunctions.java")).read()
    assert dict((k, int(v)) for k, v in re.findall(r"\b([A-Z_0-9]+)\((\d+)\)", jsrc)) == JAVA
    assert "ordinal()" not in jsrc
    kernels = open(os.path.join(ROOT, "gan_deeplearning4j_b200/csrc/kernels.h")).read()
    body = re.search(r"enum Loss \{([^}]*)\}", kernels).group(1)
    assert {k: int(v) for k, v in re.findall(r"LOSS_(\w+) = (\d+)", body)} == {k: v for k, v in header.items() if v >= 2}
    layers = "java/src/main/java/org/deeplearning4j/nn/conf/layers/"
    for cls, t in (("OutputLayer", 7), ("LossLayer", 8)):
        jl = open(os.path.join(ROOT, layers + cls + ".java")).read()
        assert f"l.type = {t}; l.loss = f.code; l.act = 0;" in jl, cls       # the code, and identity unless .activation(..) says otherwise


@pytest.mark.parametrize("loss", ["mse", "l1", "l2", "mae", "hinge", "squared_hinge", "wasserstein"])
def test_activation_reaches_the_descriptor(loss):
    for t in ("output", "loss"):
        d = engine.layer_desc({"type": t, "name": "o", "n_out": 2, "loss": loss, "activation": "lrelu", "alpha": 0.3})
        assert (d.type, d.loss, d.act) == (engine.LAYER_TYPES[t], engine.LOSSES[loss], engine.ACTS["lrelu"]) and d.act_alpha == np.float32(0.3)
    assert engine.layer_desc({"type": "output", "name": "o", "n_out": 2, "loss": loss}).act == 0
    with pytest.raises(KeyError):
        engine.layer_desc({"type": "output", "name": "o", "n_out": 2, "loss": "kld"})


def _desc_bytes(specs):
    return [bytes(memoryview(engine.layer_desc(s))) for s in specs]


def test_default_builders_produce_todays_specs():
    for size in (16, 64):
        ds = m.dcgan_discriminator(size, 8, 3)
        assert ds[-1] == {"type": "loss", "name": "dis_loss"}
        assert ds == m.dcgan_discriminator(size, 8, 3, loss="xent", out_activation="identity")
        assert _desc_bytes(ds) == _desc_bytes(m.dcgan_discriminator(size, 8, 3, loss="xent"))
    for dropout in (None, 0.5):
        ms = m.mlp_discriminator(256, 64, dropout=dropout)
        assert set(ms[-1]) == {"type", "name", "n_out", "updater"} and ms[-1]["n_out"] == 1
        assert _desc_bytes(ms) == _desc_bytes(m.mlp_discriminator(256, 64, dropout=dropout, loss="xent", out_activation="identity"))
    ls = m.dcgan_discriminator(16, 8, 3, loss="mse")
    assert ls[-1] == {"type": "loss", "name": "dis_loss", "loss": "mse", "activation": "identity"} and ls[:-1] == m.dcgan_discriminator(16, 8, 3)[:-1]
    ws = m.mlp_discriminator(256, 64, loss="wasserstein", out_activation="tanh")
    d = engine.layer_desc(ws[-1])
    assert (d.loss, d.act) == (8, 1)
    with pytest.raises(ValueError):
        m.dcgan_discriminator(16, 8, 3, loss="xent", out_activation="sigmoid")        # XENT implies its sigmoid


def test_test_hook_struct_appends_the_loss_field():
    from gan_deeplearning4j_b200 import _lib
    f = [n for n, _ in _lib.TestEwOpts._fields_]
    assert f[-2:] == ["kernel", "loss"] and _lib.TestEwOpts.loss.offset >= _lib.TestEwOpts.kernel.offset + 64
    assert engine.EW_OPS["loss"] == 10


def test_loss_specs_round_trip_through_a_checkpoint(tmp_path):
    from gan_deeplearning4j_b200 import serializer as sz
    specs = [{"type": "dense", "name": "d1", "n_out": 5, "activation": "tanh", "updater": m.adam(1e-3)},
             {"type": "output", "name": "out", "n_out": 7, "loss": "mse", "activation": "sigmoid", "updater": m.adam(1e-3)}]
    specs2 = m.dcgan_discriminator(16, 8, 3, loss="hinge", out_activation="tanh")
    rng = np.random.default_rng(0)
    for sp in (specs, specs2):
        p = rng.standard_normal(11).astype(np.float32); u = rng.standard_normal(22).astype(np.float32)

        class FakeNet:
            def __init__(self): self.p, self.u = p.copy(), u.copy()
            def params(self): return self.p
            def updater_state(self): return self.u
            def num_params(self): return self.p.size
            def set_params(self, v): self.p = np.asarray(v, np.float32).copy()
            def set_updater_state(self, v): self.u = np.asarray(v, np.float32).copy()
        path = tmp_path / "ckpt.zip"
        sz.save_net(FakeNet(), path, sp, (6,))
        got = sz.read_model(path)
        assert got["specs"] == json.loads(json.dumps(sp))          # tuples come back as lists
        assert _desc_bytes(got["specs"]) == _desc_bytes(sp)
