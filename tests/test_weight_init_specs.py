"""Weight initialization's host-side plumbing (b2g_weight_init in include/b200gan.h): the scheme and distribution numbers agree across the
header, the Python dicts, the oracle's restatement and the Java facade; the builders refuse what the engine refuses, before any library call; a checkpoint round-trips the settings; the symbols are exported and
bound.  No GPU needed."""
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import dl4j_oracle as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JAVA = os.path.join(ROOT, "java", "src", "main", "java", "org", "deeplearning4j")


def _header():
    with open(os.path.join(ROOT, "include", "b200gan.h")) as f:
        return f.read()


def _read(*parts):
    with open(os.path.join(JAVA, *parts)) as f:
        return f.read()


def test_scheme_numbers_agree_across_header_python_and_java():
    from gan_deeplearning4j_b200 import engine
    body = re.search(r"typedef enum \{([^}]*)\} b2g_weight_init_scheme;", _header()).group(1)
    header = {k.lower(): int(v) for k, v in re.findall(r"B2G_WI_(\w+) = (\d+)", body)}
    assert header == {s: i for i, s in enumerate(o.SCHEMES)} == engine.WEIGHT_INIT_SCHEMES
    java = re.search(r"enum WeightInit \{([^}]*)\}", _read("nn", "weights", "WeightInit.java")).group(1)
    assert [w.strip().lower() for w in java.split(",")] == list(o.SCHEMES)


def test_distribution_numbers_agree_across_header_python_and_java():
    from gan_deeplearning4j_b200 import engine
    h = _header()
    body = re.search(r"typedef enum \{([^}]*)\} b2g_distribution_kind;", h).group(1)
    assert re.findall(r"B2G_DIST_(\w+) = (\d+)", body) == [("NORMAL", "0"), ("UNIFORM", "1")]     # weight noise's two, then the rest
    header = {k.lower(): int(v) for k, v in re.findall(r"B2G_DIST_(\w+) = (\d+)", h)}
    assert header == {d: i for i, d in enumerate(o.DISTRIBUTIONS)}
    assert {k: v[0] for k, v in engine.INIT_DISTRIBUTIONS.items()} == header
    # weight noise keeps its two
    assert {k: v[0] for k, v in engine.DISTRIBUTIONS.items()} == {"normal": 0, "uniform": 1}
    classes = {"NormalDistribution": 0, "UniformDistribution": 1, "TruncatedNormalDistribution": 2, "LogNormalDistribution": 3,
               "BinomialDistribution": 4, "ConstantDistribution": 5, "OrthogonalDistribution": 6}
    for cls, code in classes.items():
        assert int(re.search(r"int kind\(\) \{ return (\d+); \}", _read("nn", "conf", "distribution", cls + ".java")).group(1)) == code, cls
    assert "extends NormalDistribution" in _read("nn", "conf", "distribution", "GaussianDistribution.java")


def test_java_builders_reach_the_native_call():
    """weightInit / dist / biasInit on both builders; ComputationGraph.init resolving them per conv, deconv, dense and output layer (the
    layer's own field, else the global builder's) and making one named netInitWeights call per layer, never a layer-NULL call that would
    hand the global settings to layers overriding them (a global DISTRIBUTION whose dist is set per layer, a global IDENTITY that the convs
    override); the 20-byte b2g_weight_init layout (scheme, dist, a, b, bias_init)."""
    nnc = _read("nn", "conf", "NeuralNetConfiguration.java")
    layer = _read("nn", "conf", "layers", "Layer.java")
    for src in (nnc, layer):
        for m in ("weightInit(WeightInit w)" if src is nnc else "weightInit(org.deeplearning4j.nn.weights.WeightInit w)",
                  "dist(org.deeplearning4j.nn.conf.distribution.Distribution d)", "biasInit(double b)"):
            assert m in src, m
    assert "public Builder weightInit(WeightInit w) { return this; }" not in nnc
    assert "c.weightInit = weightInit; c.dist = dist; c.biasInit = biasInit;" in layer
    cg = _read("nn", "graph", "ComputationGraph.java")
    init = cg[cg.index("public void init()"):cg.index("static String[] constrainedParams")]
    assert "initWeights(null" not in init and init.count("initWeights(") == 1
    call = init[init.index("initWeights(l.name,"):]
    call = call[:call.index(";")]
    for field in ("weightInit", "dist", "biasInit"):
        assert f"l.{field} != null ? l.{field} : g.{field}" in call, field
    loop = init[init.index("for (Layer l : layers)"):init.index("initWeights(l.name,")]
    assert "l.type == 0 || l.type == 1 || l.type == 3 || l.type == 7" in loop and "global ||" in loop
    assert "Native.netInitWeights(" in cg and "Native.direct(20)" in cg
    assert re.search(r"putInt\(0, .*ordinal\(\)\)\.putInt\(4, .*kind\(\)\)\.putFloat\(8, .*\n\s*\.putFloat\(12, .*\)\.putFloat\(16, ", cg)
    assert "public static native int netInitWeights(long net, long layerNameAddr, long weightInitAddr);" in _read("b200", "Native.java")
    with open(os.path.join(ROOT, "jni", "b200gan_jni.cpp")) as f:
        assert "b2g_net_init_weights(P(b2g_net*, net), P(const char*, layerNameAddr), P(const b2g_weight_init*, wiAddr))" in f.read()


def test_struct_layout_matches_the_header():
    from gan_deeplearning4j_b200 import _lib
    import ctypes as C
    assert C.sizeof(_lib.WeightInit) == 20
    assert [f[0] for f in _lib.WeightInit._fields_] == ["scheme", "dist", "a", "b", "bias_init"]
    body = re.search(r"typedef struct \{([^}]*)\} b2g_weight_init;", _header()).group(1)
    assert re.findall(r"(int32_t|float) ([\w, ]+);", body) == [("int32_t", "scheme"), ("int32_t", "dist"), ("float", "a, b"), ("float", "bias_init")]


def test_symbols_are_exported_and_bound():
    from gan_deeplearning4j_b200 import _lib
    assert "b2g_net_init_weights" in _lib.PROTOTYPES
    lib = os.path.join(ROOT, "gan_deeplearning4j_b200", "lib", "libb200gan.so")
    if not os.path.exists(lib):
        pytest.skip("library not built")
    out = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True).stdout
    for sym in ("b2g_net_init_weights", "Java_org_deeplearning4j_b200_Native_netInitWeights"):
        assert re.search(r"\b%s\b" % sym, out), sym


def test_models_and_structs():
    from gan_deeplearning4j_b200 import engine, models as m
    wi = m.weight_init("distribution", m.normal(0, 0.02), bias_init=0.1)
    assert wi == {"weight_init": "distribution", "distribution": {"distribution": "normal", "mean": 0.0, "std": 0.02}, "bias_init": 0.1}
    s = engine.weight_init_struct(wi)
    assert (s.scheme, s.dist, s.a, s.b, s.bias_init) == (0, 0, 0.0, np.float32(0.02), np.float32(0.1))
    assert m.truncated_normal(0.5, 0.1) == {"distribution": "truncated_normal", "mean": 0.5, "std": 0.1}
    assert m.log_normal(-1, 0.5) == {"distribution": "log_normal", "mean": -1.0, "std": 0.5}
    assert m.binomial(5, 0.25) == {"distribution": "binomial", "n_trials": 5, "p": 0.25} == m.binomial(5.0, 0.25)
    for bad in (2.5, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            m.binomial(bad, 0.5)
    assert m.constant(0.75) == {"distribution": "constant", "value": 0.75}
    for dist, code, a, b in ((m.uniform(-1, 2), 1, -1, 2), (m.truncated_normal(0.5, 0.1), 2, 0.5, 0.1), (m.log_normal(-1, 0.5), 3, -1, 0.5),
                             (m.binomial(5, 0.25), 4, 5, 0.25), (m.constant(0.75), 5, 0.75, 0)):
        s = engine.weight_init_struct(m.weight_init("distribution", dist))
        assert (s.scheme, s.dist, s.a, s.b) == (0, code, np.float32(a), np.float32(b)), dist
    for name, code in engine.WEIGHT_INIT_SCHEMES.items():
        if name != "distribution":
            s = engine.weight_init_struct(m.weight_init(name))
            assert (s.scheme, s.bias_init) == (code, 0.0)


@pytest.mark.parametrize("wi", [
    {"weight_init": "kaiming"}, {"weight_init": "distribution"},
    {"weight_init": "distribution", "distribution": {"distribution": "gamma", "a": 1}},
    {"weight_init": "distribution", "distribution": {"distribution": "orthogonal", "gain": 1.0}},
    {"weight_init": "distribution", "distribution": {"distribution": "normal", "mean": 0.0, "std": -0.1}},
    {"weight_init": "distribution", "distribution": {"distribution": "log_normal", "mean": 0.0, "std": -1.0}},
    {"weight_init": "distribution", "distribution": {"distribution": "truncated_normal", "mean": float("nan"), "std": 1.0}},
    {"weight_init": "distribution", "distribution": {"distribution": "uniform", "lower": 1.0, "upper": 0.5}},
    {"weight_init": "distribution", "distribution": {"distribution": "binomial", "n_trials": 70000, "p": 0.5}},
    {"weight_init": "distribution", "distribution": {"distribution": "binomial", "n_trials": 2.5, "p": 0.5}},
    {"weight_init": "distribution", "distribution": {"distribution": "binomial", "n_trials": 3, "p": 1.5}},
    {"weight_init": "distribution", "distribution": {"distribution": "constant", "value": float("inf")}},
    {"weight_init": "xavier", "bias_init": float("nan")},
], ids=lambda w: str(w.get("distribution", w)))
def test_builders_refuse_what_the_engine_refuses(wi):
    from gan_deeplearning4j_b200 import engine, models as m
    with pytest.raises(ValueError):
        engine.weight_init_struct(wi)
    if "weight_init" in wi and wi["weight_init"] in engine.WEIGHT_INIT_SCHEMES:
        with pytest.raises(ValueError):
            m.weight_init(wi["weight_init"], wi.get("distribution"), wi.get("bias_init", 0.0))


def test_identity_refused_on_convolutions_and_non_square_dense_specs():
    from gan_deeplearning4j_b200 import engine
    wi = {"weight_init": "identity"}
    for spec in ({"type": "conv2d", "name": "c", "n_in": 4, "n_out": 4, "kernel": (1, 1)}, {"type": "deconv2d", "name": "d", "n_in": 4, "n_out": 4},
                 {"type": "dense", "name": "f", "n_in": 4, "n_out": 5}):
        with pytest.raises(ValueError):
            engine.weight_init_struct(wi, spec)
    assert engine.weight_init_struct(wi, {"type": "output", "name": "o", "n_in": 4, "n_out": 4}).scheme == 13


def test_net_refuses_before_any_native_call():
    """Net validates every layer's weight_init before b2g_net_create: a bad one raises ValueError with no library call (the context's library
    here is a stand-in that fails the test if touched)."""
    from gan_deeplearning4j_b200 import engine, models as m

    class Untouchable:
        def __getattr__(self, name):
            raise AssertionError(f"library called: {name}")

    class Ctx:
        lib, h = Untouchable(), None
    with pytest.raises(ValueError):
        engine.Net(Ctx(), [{"type": "conv2d", "name": "c", "n_in": 1, "n_out": 1, "kernel": (1, 1)}], (1, 4, 4), 4, weight_init={"weight_init": "identity"})
    specs = m.mlp_discriminator(8, 4)
    bad = [dict(s, weight_init={"weight_init": "distribution"}) if s["type"] == "output" else s for s in specs]
    with pytest.raises(ValueError):
        engine.Net(Ctx(), bad, (8,), 4)


def test_checkpoint_round_trips_the_specs(tmp_path):
    from gan_deeplearning4j_b200 import models as m, serializer
    wi = m.weight_init("distribution", m.truncated_normal(0, 0.02), 0.01)
    specs = [dict(s, weight_init=wi) if s["type"] in ("dense", "output") else s for s in m.mlp_discriminator(8, 4)]
    path = str(tmp_path / "ck.zip")
    serializer.write_model(path, specs, (8,), np.arange(4, dtype=np.float32), None, {"dropout_pass": 0})
    assert serializer.read_model(path)["specs"] == specs
