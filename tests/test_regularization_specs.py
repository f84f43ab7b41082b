"""Regularization in the layer specs: the global builder's coefficients and each layer's own (engine.resolve_regularization), argument
errors, the oracle's net_from_specs, a checkpoint's specs, and the names across the header, Python, the JNI shim and the Java facade."""
import copy
import os
import re

import numpy as np
import pytest

from gan_deeplearning4j_b200 import _lib, engine, models as m, serializer
from oracle import dl4j_oracle as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REG = {"l1": 1e-3, "l2": 1e-4, "l1_bias": 2e-3, "l2_bias": 3e-4}


def specs():
    return [{"type": "conv2d", "name": "c1", "n_out": 4, "kernel": (3, 3), "stride": (2, 2), "padding": (1, 1), "updater": m.adam(1e-3),
             "frozen": True},
            {"type": "conv2d", "name": "c2", "n_out": 4, "kernel": (3, 3), "updater": m.adam(1e-3), "l1": 5e-3, "l2": 0.0},
            {"type": "batchnorm", "name": "bn", "updater": m.adam(1e-3)},
            {"type": "cnn_to_ff", "name": "flat"},
            {"type": "dense", "name": "fc", "n_out": 6, "updater": m.adam(1e-3), "l2_bias": 0.5},
            {"type": "output", "name": "out", "n_out": 1, "updater": m.adam(1e-3)}]


def test_global_fills_what_a_layer_does_not_set():
    s = engine.resolve_regularization(specs(), REG)
    assert engine.spec_regularization(s[1]) == dict(REG, l1=5e-3, l2=0.0)          # its own l1 and l2 win
    assert engine.spec_regularization(s[4]) == dict(REG, l2_bias=0.5)
    assert engine.spec_regularization(s[5]) == REG
    assert not any(k in s[0] for k in REG)                                          # frozen: not given the global values
    assert not any(k in s[2] for k in REG) and not any(k in s[3] for k in REG)      # BatchNorm and parameterless layers never
    plain = specs()
    assert engine.resolve_regularization(copy.deepcopy(plain), None) == plain
    assert engine.layer_desc(s[5]).l2 == np.float32(REG["l2"])                      # the global l2 reaches the desc
    assert engine.layer_desc(s[1]).l2 == 0.0


@pytest.mark.parametrize("bad", [-1e-6, float("nan"), float("inf"), -float("inf")])
@pytest.mark.parametrize("key", ["l1", "l2", "l1_bias", "l2_bias"])
def test_bad_values_are_refused(key, bad):
    with pytest.raises(ValueError):
        engine.check_regularization({key: bad})
    with pytest.raises(ValueError):
        engine.resolve_regularization(specs(), {key: bad})
    if key != "l2":                       # a spec's own l2 is the desc's, passed on as before
        with pytest.raises(ValueError):
            engine.resolve_regularization([dict(specs()[4], **{key: bad})])


def test_unknown_key_and_zero():
    with pytest.raises(ValueError):
        engine.check_regularization({"l3": 1.0})
    assert engine.check_regularization({"l1": 0, "l2_bias": 1}) == {"l1": 0.0, "l2_bias": 1.0}
    r = engine.regularization_struct(REG)
    assert [getattr(r, k) for k in engine.REGULARIZATION_KEYS] == [np.float32(REG[k]) for k in engine.REGULARIZATION_KEYS]


def test_oracle_reads_the_spec_keys():
    s = engine.resolve_regularization(specs(), REG)
    net = o.net_from_specs(s, (3, 8, 8))
    for name in ("c1", "c2", "fc", "out"):
        l, sp = net.layer(name), next(x for x in s if x["name"] == name)
        l1, l1_bias, l2_bias = net.layer_regularization.get(name, (0.0, 0.0, 0.0))
        assert (l1, l.l2, l1_bias, l2_bias) == tuple(float(sp.get(k, 0.0)) for k in engine.REGULARIZATION_KEYS)
        assert net.reg_coefs(l, "W") == (l1, l.l2) and net.reg_coefs(l, "b") == (l1_bias, l2_bias)
    assert net.layer("c1").frozen


def test_checkpoint_carries_the_specs(tmp_path):
    s = engine.resolve_regularization(specs(), REG)
    onet = o.net_from_specs(s, (3, 8, 8))
    path = str(tmp_path / "reg.zip")
    serializer.write_model(path, s, (3, 8, 8), onet.params_flat().astype(np.float32))
    back = serializer.read_model(path)["specs"]
    for a, c in zip(s, back):
        assert engine.spec_regularization(a) == engine.spec_regularization(c), a["name"]
    again = o.net_from_specs(back, (3, 8, 8))
    onet.set_params_flat(onet.params_flat())
    again.set_params_flat(onet.params_flat())
    assert again.calc_l1() == onet.calc_l1() and again.calc_l2() == onet.calc_l2() and onet.calc_l1() > 0


def test_names_agree_across_header_python_jni_and_java():
    hdr = open(os.path.join(ROOT, "include", "b200gan.h")).read()
    fields = re.search(r"typedef struct \{ float ([^;]*); \} b2g_regularization;", hdr).group(1)
    assert [f.strip() for f in fields.split(",")] == list(engine.REGULARIZATION_KEYS) == [f for f, _ in _lib.Regularization._fields_]
    for fn in ("b2g_net_set_regularization", "b2g_net_get_regularization", "b2g_net_calc_regularization"):
        assert fn in hdr and fn in _lib.PROTOTYPES
    jni = open(os.path.join(ROOT, "jni", "b200gan_jni.cpp")).read()
    native = open(os.path.join(ROOT, "java", "src", "main", "java", "org", "deeplearning4j", "b200", "Native.java")).read()
    for n in ("netSetRegularization", "netCalcRegularization"):
        assert f"FN({n})" in jni and f"native int {n}(" in native
    java = os.path.join(ROOT, "java", "src", "main", "java", "org", "deeplearning4j", "nn")
    for rel in (("conf", "layers", "Layer.java"), ("conf", "NeuralNetConfiguration.java"), ("transferlearning", "FineTuneConfiguration.java")):
        src = open(os.path.join(java, *rel)).read()
        for b in ("l1", "l1Bias", "l2Bias"):
            assert re.search(rf"public \w+ {b}\(double v\)", src), (rel, b)
    tl = open(os.path.join(java, "transferlearning", "TransferLearning.java")).read()
    assert ".l1(ft.l1).l1Bias(ft.l1Bias).l2Bias(ft.l2Bias)" in tl
