"""CPU checks that the layer specs a checkpoint writes follow the engine's learning rate through schedule changes: the constant lr a layer
returns to when its schedule is cleared is its creation-time one, a schedule's constant lr is its value at 0 for every kind (as the Java
facade's updaters write it), and layers without an updater spec are recorded like the engine treats them (Sgd)."""
import copy
import math

import numpy as np

from gan_deeplearning4j_b200 import engine, models as m
from oracle import dl4j_oracle as o


def _schedules():
    return [m.exponential_schedule(0.1, 0.9), m.inverse_schedule(0.2, 0.5, 2.0), m.sigmoid_schedule(0.4, 2.0, 10), m.step_schedule(0.08, 0.5, 3),
            m.map_schedule({0: 0.1, 3: 0.05}), m.map_schedule({0: 0.3}, type="epoch")]


def test_constant_lr_is_the_value_at_zero_for_every_kind():
    for s in _schedules():
        assert engine.constant_lr(s) == engine.schedule_value(s, 0) == o.value(s, 0), s
    assert engine.constant_lr(m.sigmoid_schedule(0.4, 2.0, 10)) == 0.4 / (1 + math.exp(20.0))      # not `initial`
    assert engine.layer_desc({"type": "dense", "name": "d", "n_out": 2, "updater": m.sgd(m.sigmoid_schedule(0.4, 0.5, 1))}).lr == \
        np.float32(0.4 / (1 + math.exp(0.5)))
    for s in _schedules():
        for i in (0, 1, 2, 3, 7, 10, 11, 250):
            assert engine.schedule_value(s, i) == o.value(s, i), (s, i)


def _specs():
    return [{"type": "dense", "name": "d1", "n_out": 4, "updater": m.adam(1e-2)},
            {"type": "dense", "name": "d2", "n_out": 4, "updater": m.rmsprop(m.step_schedule(3e-3, 0.5, 2))},
            {"type": "batchnorm", "name": "bn"},                                       # no updater: Sgd with lr 0
            {"type": "activation", "name": "act", "activation": "relu", "updater": m.sgd(0.5)},   # no parameters
            {"type": "dense", "name": "fz", "n_out": 4, "updater": m.sgd(0.5), "frozen": True},
            {"type": "dense", "name": "nop", "n_out": 4, "updater": {"kind": "noop"}},
            {"type": "output", "name": "out", "n_out": 1, "updater": m.sgd(m.sigmoid_schedule(0.4, 2.0, 10))}]


def test_layer_rule():
    assert [engine.layer_has_lr(s) for s in _specs()] == [True, True, True, False, False, False, True]


def test_clearing_writes_back_the_creation_time_constant():
    specs = copy.deepcopy(_specs())
    const = [engine.constant_lr((s.get("updater") or {}).get("lr", 0.0)) for s in specs]
    untouched = {i: copy.deepcopy(specs[i]) for i in (3, 4, 5)}
    e = m.exponential_schedule(2e-2, 0.8)
    engine.follow_lr_schedule(specs, const, e)
    for i in (0, 1, 2, 6):
        assert specs[i]["updater"]["lr"] == e and specs[i]["updater"]["lr"] is not e
    assert specs[2]["updater"]["kind"] == "sgd"                       # recorded the way the engine treats it
    engine.follow_lr_schedule(specs, const, None, "d1")
    assert specs[0]["updater"]["lr"] == 1e-2                          # its creation-time lr, not the cleared schedule's value at 0
    engine.follow_lr_schedule(specs, const, None)
    assert [specs[i]["updater"]["lr"] for i in (0, 1, 2, 6)] == [1e-2, 3e-3, 0.0, 0.4 / (1 + math.exp(20.0))]
    for i, s in untouched.items():
        assert specs[i] == s


def test_a_named_layer_is_the_first_of_its_name():
    specs = [{"type": "dense", "name": "x", "n_out": 4, "updater": m.sgd(0.1)}, {"type": "dense", "name": "x", "n_out": 4, "updater": m.sgd(0.2)}]
    engine.follow_lr_schedule(specs, [0.1, 0.2], m.map_schedule({0: 1.0}), "x")
    assert specs[0]["updater"]["lr"] == m.map_schedule({0: 1.0}) and specs[1]["updater"]["lr"] == 0.2


class _Lib:
    """Stands in for libb200gan: accepts every schedule (argument checks are the GPU tests' business)."""

    def b2g_net_set_lr_schedule(self, h, layer, s):
        self.calls = getattr(self, "calls", 0) + 1
        return 0


def test_net_set_lr_schedule_keeps_the_specs_in_step():
    net = engine.Net.__new__(engine.Net)
    net.lib, net.h = _Lib(), None
    net.specs = copy.deepcopy(_specs())
    net.lr_constants = [engine.constant_lr((s.get("updater") or {}).get("lr", 0.0)) for s in net.specs]
    net.set_lr_schedule(m.exponential_schedule(2e-2, 0.8))
    net.set_lr_schedule(None)
    assert net.lib.calls == 2
    assert net.specs[0]["updater"]["lr"] == 1e-2 and net.specs[1]["updater"]["lr"] == 3e-3
