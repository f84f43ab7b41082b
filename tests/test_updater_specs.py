"""CPU checks of the updater kinds at the interface: the enum values agree across the C header, engine.UPDATERS and the Java facade's kind()s,
the JNI entry of b2g_net_updater_state_size is exported, the builders carry DL4J's defaults into b2g_layer_desc, the learning-rate rule excludes
AdaDelta (and NoOp), and updater specs of every kind round-trip through a checkpoint with the three-slot state."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from gan_deeplearning4j_b200 import engine, models as m

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("SGD", "RMSPROP", "ADAM", "NOOP", "NESTEROVS", "ADAGRAD", "ADAMAX", "NADAM", "AMSGRAD", "ADADELTA")
JAVA = {"Sgd": 0, "RmsProp": 1, "Adam": 2, "NoOp": 3, "Nesterovs": 4, "AdaGrad": 5, "AdaMax": 6, "Nadam": 7, "AMSGrad": 8, "AdaDelta": 9}


def test_enum_values_agree_across_header_engine_and_java():
    src = open(os.path.join(ROOT, "include", "b200gan.h")).read()
    body = re.search(r"typedef enum \{([^}]*)\} b2g_updater;", src).group(1)
    header = {k: int(v) for k, v in re.findall(r"B2G_UPD_(\w+) = (\d+)", body)}
    assert header == {n: i for i, n in enumerate(NAMES)}
    assert {k.upper(): v for k, v in engine.UPDATERS.items()} == header
    jdir = os.path.join(ROOT, "java/src/main/java/org/nd4j/linalg/learning/config")
    for cls, kind in JAVA.items():
        jsrc = open(os.path.join(jdir, cls + ".java")).read()
        assert f"public int kind() {{ return {kind}; }}" in jsrc, cls
        assert f"public class {cls} implements IUpdater" in jsrc, cls


@pytest.fixture(scope="module")
def lib():
    import gan_deeplearning4j_b200 as b
    if not os.path.exists(b.LIB_PATH):
        sys.path.insert(0, ROOT)
        import __graft_entry__
        __graft_entry__.build()
    return b.load()


def test_state_size_entry_point_and_jni_symbol(lib):
    import gan_deeplearning4j_b200 as b
    assert "b2g_net_updater_state_size" in b.PROTOTYPES and lib.b2g_net_updater_state_size.restype is C.c_int32
    out = subprocess.run(["nm", "-D", "--defined-only", b.LIB_PATH], capture_output=True, text=True).stdout
    assert "Java_org_deeplearning4j_b200_Native_netUpdaterStateSize" in out
    native = open(os.path.join(ROOT, "java/src/main/java/org/deeplearning4j/b200/Native.java")).read()
    assert "public static native int netUpdaterStateSize(" in native
    graph = open(os.path.join(ROOT, "java/src/main/java/org/deeplearning4j/nn/graph/ComputationGraph.java")).read()
    assert "2 * (int) numParams()" not in graph and "Native.netUpdaterStateSize" in graph


def _desc(u):
    d = engine.layer_desc({"type": "dense", "name": "d", "n_out": 2, "updater": u})
    return d.updater, d.lr, d.beta1, d.beta2, d.eps


def test_builders_carry_dl4js_defaults():
    f = lambda *v: tuple(float(np.float32(x)) for x in v)
    assert _desc(m.nesterovs()) == (4,) + f(0.1, 0.9, 0.0, 0.0)                      # Nesterovs(lr 0.1, momentum 0.9)
    assert _desc(m.adagrad()) == (5,) + f(0.1, 0.0, 0.0, 1e-6)                       # AdaGrad(lr 0.1, eps 1e-6)
    for kind, code in (("adamax", 6), ("nadam", 7), ("amsgrad", 8)):
        assert _desc(getattr(m, kind)()) == (code,) + f(1e-3, 0.9, 0.999, 1e-8), kind
    assert _desc(m.adadelta()) == (9,) + f(0.0, 0.95, 0.0, 1e-6)                     # AdaDelta(rho 0.95, eps 1e-6): no lr
    assert _desc(m.noop())[0] == 3
    assert _desc(m.nesterovs(0.02, 0.5)) == (4,) + f(0.02, 0.5, 0.0, 0.0)
    assert _desc(m.adadelta(0.9, 1e-5)) == (9,) + f(0.0, 0.9, 0.0, 1e-5)
    sched = m.step_schedule(0.2, 0.5, 10)
    for kind in ("nesterovs", "adagrad", "adamax", "nadam", "amsgrad"):
        assert _desc(getattr(m, kind)(sched))[1] == np.float32(0.2), kind       # a schedule's value at 0
    with pytest.raises(TypeError):
        m.adadelta(lr=0.1)
    jdir = os.path.join(ROOT, "java/src/main/java/org/nd4j/linalg/learning/config")
    jsrc = {c: open(os.path.join(jdir, c + ".java")).read() for c in JAVA}
    assert "DEFAULT_NESTEROV_LEARNING_RATE = 0.1, DEFAULT_NESTEROV_MOMENTUM = 0.9" in jsrc["Nesterovs"]
    assert "DEFAULT_ADAGRAD_LEARNING_RATE = 0.1, DEFAULT_ADAGRAD_EPSILON = 1e-6" in jsrc["AdaGrad"]
    assert "DEFAULT_ADADELTA_RHO = 0.95, DEFAULT_ADADELTA_EPSILON = 1e-6" in jsrc["AdaDelta"]
    for c in ("AdaMax", "Nadam", "AMSGrad"):
        assert f"DEFAULT_{c.upper()}_LEARNING_RATE = 1e-3, DEFAULT_{c.upper()}_BETA1_MEAN_DECAY = 0.9, DEFAULT_{c.upper()}_BETA2_VAR_DECAY = 0.999, " \
               f"DEFAULT_{c.upper()}_EPSILON = 1e-8" in jsrc[c], c
        assert f"public {c}(ISchedule learningRateSchedule)" in jsrc[c], c
    assert "ISchedule" not in jsrc["AdaDelta"] and "ISchedule" not in jsrc["NoOp"]


def test_learning_rate_rule_excludes_adadelta_and_noop():
    specs = [{"type": "dense", "name": k, "n_out": 2, "updater": getattr(m, k)()} for k in ("nesterovs", "adagrad", "adamax", "nadam", "amsgrad")]
    specs += [{"type": "dense", "name": "dd", "n_out": 2, "updater": m.adadelta()}, {"type": "batchnorm", "name": "bn", "updater": m.adadelta()},
              {"type": "dense", "name": "nop", "n_out": 2, "updater": m.noop()}]
    assert [engine.layer_has_lr(s) for s in specs] == [True] * 5 + [False] * 3
    const = [engine.constant_lr((s.get("updater") or {}).get("lr", 0.0)) for s in specs]
    sched = m.exponential_schedule(1e-2, 0.9)
    engine.follow_lr_schedule(specs, const, sched)
    assert all(s["updater"]["lr"] == sched for s in specs[:5])
    assert all("lr" not in s["updater"] for s in specs[5:])          # the all-layers form skips them
    graph = open(os.path.join(ROOT, "java/src/main/java/org/deeplearning4j/nn/graph/ComputationGraph.java")).read()
    assert "l.updater.kind() != 3 && l.updater.kind() != 9" in graph


def test_specs_and_three_slot_state_round_trip_through_a_checkpoint(tmp_path):
    from gan_deeplearning4j_b200 import serializer as sz
    specs = [{"type": "dense", "name": "d1", "n_out": 4, "updater": m.amsgrad(m.map_schedule({0: 1e-3, 5: 5e-4}))},
             {"type": "batchnorm", "name": "bn", "updater": m.adagrad(0.05, 1e-7)},
             {"type": "dense", "name": "d2", "n_out": 4, "updater": m.nesterovs(0.01, 0.8)},
             {"type": "dense", "name": "d3", "n_out": 4, "updater": m.adamax()},
             {"type": "dense", "name": "d4", "n_out": 4, "updater": m.nadam(2e-3, 0.85)},
             {"type": "output", "name": "out", "n_out": 1, "updater": m.adadelta(0.9)}]
    rng = np.random.default_rng(0)
    p = rng.standard_normal(97).astype(np.float32); u = rng.standard_normal(3 * 97).astype(np.float32)

    class FakeNet:            # the part of the Net interface the checkpoint wrappers use
        def __init__(self): self.p, self.u = p.copy(), u.copy()
        def params(self): return self.p
        def updater_state(self): return self.u
        def num_params(self): return self.p.size
        def set_params(self, v): self.p = np.asarray(v, np.float32).copy()
        def set_updater_state(self, v): self.u = np.asarray(v, np.float32).copy()
    path = tmp_path / "ckpt.zip"
    sz.save_net(FakeNet(), path, specs, (6,), meta={"iteration": 11})
    other = FakeNet(); other.p[:] = 0; other.u = np.zeros(3 * 97, np.float32)
    got = sz.restore_into(other, path)
    assert got["specs"] == specs
    assert np.array_equal(other.u, u) and np.array_equal(other.p, p)
    assert [engine.layer_desc(s).updater for s in got["specs"]] == [8, 5, 4, 6, 7, 9]
    assert "[state0 | state1 | state2]" in sz.__doc__
