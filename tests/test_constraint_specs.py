"""The plumbing of the weight constraints: which parameters weights / bias / all reach per layer type, the kind names across the C header,
Python and Java, the JNI symbols, the checkpoint's layer specs, and argument checks that need no GPU.  CPU only."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from gan_deeplearning4j_b200 import engine as e
from gan_deeplearning4j_b200 import models as m
from gan_deeplearning4j_b200 import serializer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JAVA = os.path.join(ROOT, "java/src/main/java/org/deeplearning4j")


@pytest.mark.parametrize("spec,weights,bias,all_", [
    ({"type": "conv2d"}, ["W"], ["b"], ["b", "W"]),
    ({"type": "conv2d", "has_bias": False}, ["W"], [], ["W"]),
    ({"type": "deconv2d"}, ["W"], ["b"], ["b", "W"]),
    ({"type": "dense"}, ["W"], ["b"], ["b", "W"]),
    ({"type": "output"}, ["W"], ["b"], ["b", "W"]),
    ({"type": "batchnorm"}, [], [], ["gamma", "beta", "mean", "var"]),
    ({"type": "dense", "frozen": True}, [], [], []),
    ({"type": "activation"}, [], [], []),
    ({"type": "dropout"}, [], [], []),
])
def test_targets_per_layer_type(spec, weights, bias, all_):
    assert e.constraint_params(spec, "weights") == weights
    assert e.constraint_params(spec, "bias") == bias
    assert e.constraint_params(spec, "all") == all_
    with pytest.raises(ValueError):
        e.constraint_params(spec, "params")


def test_list_order_all_then_weights_then_bias():
    a, w1, w2, bb = m.unit_norm((0,), on="all"), m.max_norm(1, (0,)), m.non_negative(), m.max_norm(2, (1,), on="bias")
    r = e.resolve_constraints({"type": "dense", "constraints": [bb, w1, a, w2]})
    assert r == {"b": [a, bb], "W": [a, w1, w2]}


def test_builders_and_struct():
    c = m.min_max_norm(0.5, 2.0, (1, 2, 3), rate=0.25, on="all")
    assert c == {"constraint": "min_max_norm", "min": 0.5, "max": 2.0, "rate": 0.25, "dims": [1, 2, 3], "on": "all"}
    s = e.constraint_struct(c)
    assert (s.kind, s.dims_mask, s.max_norm, s.min_norm, s.rate) == (1, 0b1110, 2.0, 0.5, 0.25)
    assert e.constraint_struct(m.max_norm(3.0, ())).dims_mask == 0
    with pytest.raises(ValueError):
        e.constraint_struct({"constraint": "spectral"})


def test_kind_names_agree_across_header_python_and_java():
    src = open(os.path.join(ROOT, "include", "b200gan.h")).read()
    body = re.search(r"typedef enum \{([^}]*)\} b2g_constraint_kind;", src).group(1)
    header = {k.lower(): int(v) for k, v in re.findall(r"B2G_CONSTRAINT_(\w+) = (\d+)", body)}
    assert header == e.CONSTRAINT_KINDS == {"max_norm": 0, "min_max_norm": 1, "unit_norm": 2, "non_negative": 3}
    for cls, kind in (("MaxNorm", 0), ("MinMaxNorm", 1), ("UnitNorm", 2), ("NonNegative", 3)):
        java = open(os.path.join(JAVA, "nn/conf/constraint", cls + "Constraint.java")).read()
        assert f"public int kind() {{ return {kind}; }}" in java
    assert "public MaxNormConstraint(double maxNorm, int... dimensions)" in open(os.path.join(JAVA, "nn/conf/constraint/MaxNormConstraint.java")).read()
    # the Java facade states the same targets as constraint_params
    cg = open(os.path.join(JAVA, "nn/graph/ComputationGraph.java")).read()
    assert 'if (gemm && on.equals("weights")) return new String[] { "W" };' in cg
    assert 'if (gemm && on.equals("all")) return l.hasBias != 0 ? new String[] { "b", "W" } : new String[] { "W" };' in cg
    assert 'if (l.type == 2 && on.equals("all")) return new String[] { "gamma", "beta", "mean", "var" };' in cg
    assert "if (per.isEmpty()) per = constraintsByParam(l, conf.b.g.constrainAll, conf.b.g.constrainW, conf.b.g.constrainB);" in cg
    for name in ("constrainWeights", "constrainBias", "constrainAllParameters"):
        assert f"public T {name}(LayerConstraint... c)" in open(os.path.join(JAVA, "nn/conf/layers/Layer.java")).read()
        assert f"public Builder {name}(LayerConstraint... c)" in open(os.path.join(JAVA, "nn/conf/NeuralNetConfiguration.java")).read()


@pytest.fixture(scope="module")
def lib():
    import gan_deeplearning4j_b200 as b
    if not os.path.exists(b.LIB_PATH):
        sys.path.insert(0, ROOT)
        import __graft_entry__
        __graft_entry__.build()
    return b.load()


def test_entry_points_and_jni_symbols_exported(lib):
    assert hasattr(lib, "b2g_net_set_constraints") and hasattr(lib, "b2g_net_apply_constraints")
    out = subprocess.run(["nm", "-D", "--defined-only", os.path.join(ROOT, "gan_deeplearning4j_b200", "lib", "libb200gan.so")], capture_output=True, text=True).stdout
    native = open(os.path.join(JAVA, "b200/Native.java")).read()
    for sym in ("netSetConstraints", "netApplyConstraints"):
        assert "Java_org_deeplearning4j_b200_Native_" + sym in out
        assert f"public static native int {sym}(" in native


def test_null_net_is_refused(lib):
    assert lib.b2g_net_set_constraints(None, b"a", b"W", None, 0) == -1
    assert lib.b2g_net_apply_constraints(None) == -1


def test_checkpoint_carries_the_constraints(tmp_path):
    specs = [{"type": "dense", "name": "a", "n_in": 3, "n_out": 2, "constraints": [m.max_norm(1.5, (0,)), m.non_negative(on="bias")]},
             {"type": "batchnorm", "name": "bn", "constraints": [m.min_max_norm(0.1, 2.0, (1,), rate=0.5, on="all")]}]
    serializer.write_model(tmp_path / "c.zip", specs, (3,), np.zeros(6 + 4 * 2, np.float32))
    back = serializer.read_model(tmp_path / "c.zip")["specs"]
    assert [sp["constraints"] for sp in back] == [sp["constraints"] for sp in specs]
    assert e.resolve_constraints(back[0]) == e.resolve_constraints(specs[0])
