"""CPU checks of the learning-rate schedules: the oracle's restatement against hand-computed values at and around the
boundaries, identity schedules leave the oracle bit-identical, the updater-spec builders, and the boundary (header enums, ctypes layout of
b2g_lr_schedule against the C compiler, bound and exported symbols)."""
import copy
import ctypes as C
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest


from gan_deeplearning4j_b200 import models as m
from oracle import dl4j_oracle as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_exponential_and_inverse():
    e = m.exponential_schedule(0.1, 0.9)
    assert o.value(e, 0) == 0.1 and o.value(e, 1) == 0.1 * 0.9 and o.value(e, 3) == 0.1 * 0.9 ** 3
    inv = m.inverse_schedule(0.2, 0.5, 2.0)
    assert o.value(inv, 0) == 0.2 and o.value(inv, 2) == 0.2 / 4.0 and o.value(inv, 6) == 0.2 / 16.0
    assert o.lr_at(e, 3, 0) == np.float32(0.1 * 0.9 ** 3) and o.lr_at(e, 3, 0).dtype == np.float32


def test_sigmoid_at_and_around_its_step_size():
    s = m.sigmoid_schedule(0.4, 2.0, 10)
    assert o.value(s, 10) == 0.2                                   # exactly half at i = stepSize
    assert o.value(s, 9) == 0.4 / (1 + math.exp(2.0)) < 0.2 < o.value(s, 11) == 0.4 / (1 + math.exp(-2.0))
    assert o.value(s, 0) < o.value(s, 5) < o.value(s, 10) < o.value(s, 100) <= 0.4


def test_step_at_multiples_of_step():
    s = m.step_schedule(0.08, 0.5, 3)
    assert [o.value(s, i) for i in range(10)] == [0.08] * 3 + [0.04] * 3 + [0.02] * 3 + [0.01]
    frac = m.step_schedule(1.0, 0.1, 2.5)                          # step is a double: floor(i / 2.5)
    assert [o.value(frac, i) for i in range(8)] == [1.0, 1.0, 1.0, 0.1, 0.1, 0.1 ** 2, 0.1 ** 2, 0.1 ** 2]


def test_map_at_and_between_keys():
    s = m.map_schedule({10: 0.01, 0: 0.1, 3: 0.05})
    assert s["values"] == [[0, 0.1], [3, 0.05], [10, 0.01]]       # sorted [key, value] pairs (JSON-safe)
    assert [o.value(s, i) for i in (0, 1, 2, 3, 4, 9, 10, 11, 10 ** 6)] == [0.1, 0.1, 0.1, 0.05, 0.05, 0.05, 0.01, 0.01, 0.01]
    assert m.map_schedule([(0, 1.0), (5, 2.0)])["values"] == [[0, 1.0], [5, 2.0]]


def test_type_selects_the_counter():
    it, ep = m.step_schedule(1.0, 0.5, 1), m.step_schedule(1.0, 0.5, 1, type="epoch")
    assert o.lr_at(it, 3, 1) == np.float32(0.125) and o.lr_at(ep, 3, 1) == np.float32(0.5)


def _mlp(lr):
    return [{"type": "dense", "name": "d1", "n_out": 16, "activation": "tanh", "updater": m.adam(lr), "l2": 1e-3},
            {"type": "dense", "name": "d2", "n_out": 8, "activation": "lrelu", "alpha": 0.2, "updater": m.rmsprop(lr)},
            {"type": "output", "name": "out", "n_out": 1, "updater": m.sgd(lr)}]


@pytest.mark.parametrize("identity", ["exponential", "map"])
def test_identity_schedules_leave_the_oracle_bit_identical(identity):
    lr = float(np.float32(3e-3))         # the engine's constant lr is fp32; a schedule's value is rounded to fp32 too
    sched = m.exponential_schedule(lr, 1.0) if identity == "exponential" else m.map_schedule({0: lr})
    plain = o.net_from_specs(_mlp(lr), (5,), seed=4)
    specs = copy.deepcopy(_mlp(lr))
    for s in specs:
        s["updater"]["lr"] = sched
    wrapped = o.net_from_specs(specs, (5,), seed=4)
    assert set(wrapped.schedules) == {"d1", "d2", "out"}
    rng = np.random.default_rng(0)
    for _ in range(4):
        x, y = rng.uniform(-1, 1, (6, 5)), rng.uniform(0, 1, (6, 1))
        assert plain.fit(x, y) == wrapped.fit(x, y)
        assert np.array_equal(plain.params_flat(), wrapped.params_flat())
    for k in plain.state:
        for a, b in zip(plain.state[k], wrapped.state[k]):
            assert np.array_equal(a, b)


def test_wrapped_oracle_uses_the_scheduled_rate_per_update():
    """SGD with a StepSchedule: each update moves the output bias by exactly lr_i * g (no l2 on biases)."""
    sched = m.step_schedule(0.5, 0.5, 2)
    specs = [{"type": "output", "name": "out", "n_out": 1, "updater": m.sgd(sched)}]
    net = o.net_from_specs(specs, (3,), seed=2)
    rng = np.random.default_rng(1)
    for it in range(5):
        x, y = rng.uniform(-1, 1, (4, 3)), rng.uniform(0, 1, (4, 1))
        b0 = net.layers[0].params["b"].copy()
        net.compute_gradient_and_score(x, y)
        g = net.layers[0].grads["b"] / 4
        net.apply_update(4)
        np.testing.assert_allclose(b0 - net.layers[0].params["b"], float(np.float32(0.5 * 0.5 ** (it // 2))) * g, rtol=1e-12)
    net.set_lr_schedule(None, "out")
    assert net.iteration == 5
    net.compute_gradient_and_score(x, y); net.apply_update(4)
    assert net.learning_rate("out") == 0.5                      # back to the constant lr


def test_epoch_schedules_follow_the_epoch_word():
    specs = [{"type": "output", "name": "out", "n_out": 1, "updater": m.sgd(m.map_schedule({0: 0.1, 2: 0.01}, type="epoch"))}]
    net = o.net_from_specs(specs, (3,), seed=2)
    x, y = np.ones((2, 3)), np.ones((2, 1))
    lrs = []
    for ep in (0, 1, 2, 5, 0):
        net.set_epoch(ep)
        lrs.append(net.learning_rate("out"))
        net.compute_gradient_and_score(x, y); net.apply_update(2)
    assert lrs == [float(np.float32(v)) for v in (0.1, 0.1, 0.01, 0.01, 0.1)]


def test_updater_specs_take_a_schedule_and_layer_desc_writes_a_float():
    from gan_deeplearning4j_b200.engine import constant_lr, layer_desc, schedule_struct
    s = m.step_schedule(2e-4, 0.5, 1000)
    u = m.adam(lr=s)
    assert u["lr"] is s
    d = layer_desc({"type": "dense", "name": "d", "n_out": 4, "updater": u})
    assert d.lr == np.float32(2e-4)
    assert constant_lr(m.map_schedule({0: 0.25, 4: 1.0})) == 0.25 and constant_lr(0.5) == 0.5
    st, arrays = schedule_struct(m.map_schedule({0: 0.25, 4: 1.0}, type="epoch"))
    assert (st.kind, st.type, st.n_map) == (5, 1, 2) and [st.map_keys[i] for i in range(2)] == [0, 4] and st.map_values[1] == 1.0
    for bad in ({"schedule": "poly", "initial": 1.0}, {"schedule": "step", "type": "minibatch"}):
        with pytest.raises(ValueError):
            schedule_struct(bad)


def _header_enum(name, prefix):
    src = open(os.path.join(ROOT, "include", "b200gan.h")).read()
    body = re.search(r"typedef enum \{([^}]*)\} " + name + ";", src).group(1)
    return {k: int(v) for k, v in re.findall(prefix + r"(\w+) = (\d+)", body)}


def test_kind_and_type_values_match_header_and_java():
    from gan_deeplearning4j_b200.engine import SCHEDULE_KINDS, SCHEDULE_TYPES
    kinds = _header_enum("b2g_schedule_kind", "B2G_SCHED_")
    assert kinds == {"NONE": 0, "EXPONENTIAL": 1, "INVERSE": 2, "SIGMOID": 3, "STEP": 4, "MAP": 5}
    assert {k.upper(): v for k, v in SCHEDULE_KINDS.items()} == {k: v for k, v in kinds.items() if k != "NONE"}
    assert _header_enum("b2g_schedule_type", "B2G_SCHED_") == {"ITERATION": 0, "EPOCH": 1}
    assert SCHEDULE_TYPES == {"iteration": 0, "epoch": 1}
    jdir = os.path.join(ROOT, "java/src/main/java/org/nd4j/linalg/schedule")
    names = re.search(r"enum ScheduleType \{\s*([^;}]*)", open(os.path.join(jdir, "ScheduleType.java")).read()).group(1)
    assert names.replace(" ", "").replace("\n", "").split(",") == ["ITERATION", "EPOCH"]
    for cls, kind in (("ExponentialSchedule", 1), ("InverseSchedule", 2), ("SigmoidSchedule", 3), ("StepSchedule", 4), ("MapSchedule", 5)):
        src = open(os.path.join(jdir, cls + ".java")).read()
        assert f"public int kind() {{ return {kind}; }}" in src, cls
    assert not os.path.exists(os.path.join(jdir, "PolySchedule.java"))


@pytest.fixture(scope="module")
def lib():
    import gan_deeplearning4j_b200 as b
    if not os.path.exists(b.LIB_PATH):
        sys.path.insert(0, ROOT)
        import __graft_entry__
        __graft_entry__.build()
    return b.load()


def test_entry_points_bound_and_jni_symbols_exported(lib):
    import gan_deeplearning4j_b200 as b
    for n in ("b2g_net_set_lr_schedule", "b2g_net_get_learning_rate", "b2g_net_get_epoch", "b2g_net_set_epoch"):
        assert hasattr(lib, n) and n in b.PROTOTYPES
        assert getattr(lib, n).restype is C.c_int32
    out = subprocess.run(["nm", "-D", "--defined-only", os.path.join(ROOT, "gan_deeplearning4j_b200", "lib", "libb200gan.so")], capture_output=True, text=True).stdout
    native = open(os.path.join(ROOT, "java/src/main/java/org/deeplearning4j/b200/Native.java")).read()
    for n in ("netSetLrSchedule", "netGetLearningRate", "netGetEpoch", "netSetEpoch"):
        assert f"Java_org_deeplearning4j_b200_Native_{n}" in out
        assert f"public static native int {n}(" in native


def test_schedule_struct_layout_matches_the_c_header(tmp_path):
    from gan_deeplearning4j_b200 import _lib
    prog = tmp_path / "layout.c"
    fields = ("kind", "type", "initial", "gamma", "power", "step", "decay_rate", "n_map", "map_keys", "map_values")
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200gan.h"\nint main(){printf("%zu' + " %zu" * len(fields) + '\\n", sizeof(b2g_lr_schedule)'
                    + "".join(f", offsetof(b2g_lr_schedule,{f})" for f in fields) + ");return 0;}")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True).stdout.split()]
    S = _lib.LrSchedule
    assert got == [C.sizeof(S)] + [getattr(S, f).offset for f in fields]
    assert got == [72, 0, 4, 8, 16, 24, 32, 40, 48, 56, 64]     # the layout the Java facade writes into a direct ByteBuffer
