"""CPU checks of the activation codes at the interface: the header's b2g_activation, kernels.h, engine.ACTS and the Java facade's Activation agree;
spec -> b2g_layer_desc codes and the per-kind alpha defaults; the builders' activation arguments, whose defaults give today's specs."""
import os
import re

import numpy as np
import pytest

from gan_deeplearning4j_b200 import engine, models as m
from oracle import dl4j_oracle as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("IDENTITY", "TANH", "SIGMOID", "RELU", "LRELU", "ELU", "SELU", "SOFTPLUS", "SOFTSIGN", "HARDTANH", "HARDSIGMOID", "RELU6", "SWISH", "CUBE",
         "RATIONALTANH", "RECTIFIEDTANH", "THRESHOLDEDRELU")
JAVA = "java/src/main/java/"


def test_codes_agree_across_header_kernels_engine_and_java():
    src = open(os.path.join(ROOT, "include", "b200gan.h")).read()
    body = re.search(r"typedef enum \{([^}]*)\} b2g_activation;", src).group(1)
    header = {k: int(v) for k, v in re.findall(r"B2G_ACT_(\w+) = (\d+)", body)}
    assert header == {n: i for i, n in enumerate(NAMES)}
    assert {k.upper(): v for k, v in engine.ACTS.items()} == header
    assert {k: v for k, v in engine.ACTS.items() if v >= 5} == o.ACT_CODES
    kernels = open(os.path.join(ROOT, "gan_deeplearning4j_b200/csrc/kernels.h")).read()
    body = re.search(r"enum Act \{([^}]*)\}", kernels).group(1)
    assert {k: int(v) for k, v in re.findall(r"ACT_(\w+) = (\d+)", body)} == header
    jsrc = open(os.path.join(ROOT, JAVA, "org/nd4j/linalg/activations/Activation.java")).read()
    java = {k: int(v) for k, v in re.findall(r"\b([A-Z_0-9]+)\((\d+)\)", jsrc)}
    assert java == {("LEAKYRELU" if k == "LRELU" else k): v for k, v in header.items()}


def test_java_parameterized_activations_and_default_alpha():
    for cls, kind in (("ActivationELU", "ELU"), ("ActivationThresholdedReLU", "THRESHOLDEDRELU")):
        jsrc = open(os.path.join(ROOT, JAVA, f"org/nd4j/linalg/activations/impl/{cls}.java")).read()
        assert f"Activation.{kind}.code" in jsrc and "this(1.0)" in jsrc and "implements IActivation" in jsrc
    layer = open(os.path.join(ROOT, JAVA, "org/deeplearning4j/nn/conf/layers/Layer.java")).read()
    assert "public T activation(IActivation a)" in layer
    assert "!alphaSet && (a == Activation.ELU.code || a == Activation.THRESHOLDEDRELU.code) ? 1.0f : alpha" in layer


@pytest.mark.parametrize("kind", o.EXT_ACTS)
def test_spec_to_descriptor(kind):
    for t in ("conv2d", "deconv2d", "dense", "activation"):
        d = engine.layer_desc({"type": t, "name": "l", "n_out": 2, "activation": kind})
        assert d.act == o.ACT_CODES[kind] and d.act_alpha == np.float32(o.ACT_ALPHA_DEFAULTS.get(kind, 0.01))
        d = engine.layer_desc({"type": t, "name": "l", "n_out": 2, "activation": kind, "alpha": 0.3})
        assert d.act == o.ACT_CODES[kind] and d.act_alpha == np.float32(0.3)
    for t in ("output", "loss"):
        d = engine.layer_desc({"type": t, "name": "o", "n_out": 2, "loss": "mse", "activation": kind})
        assert (d.loss, d.act) == (2, o.ACT_CODES[kind])
    # LeakyReLU keeps its 0.01 default
    assert engine.layer_desc({"type": "dense", "name": "l", "n_out": 2, "activation": "lrelu"}).act_alpha == np.float32(0.01)


def test_builders_take_the_activation_and_default_to_todays_specs():
    assert m.dcgan_generator(16, 12, 8, 3) == m.dcgan_generator(16, 12, 8, 3, activation="relu", out_activation="tanh")
    assert m.dcgan_discriminator(16, 8, 3) == m.dcgan_discriminator(16, 8, 3, activation="lrelu", alpha=0.2)
    assert m.mlp_generator(12, 32, 16) == m.mlp_generator(12, 32, 16, activation="relu", out_activation="tanh")
    assert m.mlp_discriminator(16, 32) == m.mlp_discriminator(16, 32, activation="lrelu", alpha=0.2)
    assert m.dcgan_discriminator(16, 8, 3)[0]["alpha"] == 0.2 and m.dcgan_discriminator(16, 8, 3)[0]["activation"] == "lrelu"
    g = m.dcgan_generator(16, 12, 8, 3, activation="elu", out_activation="hardtanh")
    assert [s["activation"] for s in g if s["type"] == "activation"] == ["elu", "elu"] and g[-1]["activation"] == "hardtanh"
    assert all("alpha" not in s for s in g)                      # layer_desc fills ELU's 1.0
    d = m.dcgan_discriminator(16, 8, 3, activation="selu")
    assert d[0]["activation"] == "selu" and "alpha" not in d[0] and d[3]["activation"] == "selu"
    mg = m.mlp_generator(12, 32, 16, activation="swish")
    assert [s["activation"] for s in mg] == ["swish", "swish", "tanh"]
    md = m.mlp_discriminator(16, 32, activation="elu", alpha=0.5)
    assert md[0]["activation"] == "elu" and engine.layer_desc(md[0]).act_alpha == np.float32(0.5)


def test_test_hook_ops():
    assert engine.EW_OPS["act_ext_fwd"] == 11 and engine.EW_OPS["act_ext_bwd"] == 12
    src = open(os.path.join(ROOT, "include", "b200gan.h")).read()
    assert "B2G_EW_ACT_EXT_FWD = 11, B2G_EW_ACT_EXT_BWD = 12" in src
