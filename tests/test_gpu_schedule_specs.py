"""The layer specs a checkpoint writes against the learning rate the engine uses, through schedule set / clear, on the GPU: after every change
a net rebuilt from the checkpoint's specs uses the same learning rate in every layer, and Python's rule for which layers have a learning rate
is the engine's."""
import math

import numpy as np
import pytest

from gan_deeplearning4j_b200 import engine
from helpers import b200

pytestmark = pytest.mark.gpu


def _specs():
    from gan_deeplearning4j_b200 import models as m
    return [{"type": "dense", "name": "fz", "n_out": 8, "updater": m.sgd(0.5), "frozen": True},                # FrozenLayer
            {"type": "dense", "name": "d1", "n_out": 16, "activation": "tanh", "updater": m.adam(1e-2)},
            {"type": "dense", "name": "d2", "n_out": 16, "activation": "tanh", "updater": m.rmsprop(m.sigmoid_schedule(3e-3, 0.5, 4))},
            {"type": "batchnorm", "name": "bn"},                                                    # no updater spec: Sgd, lr 0
            {"type": "activation", "name": "act", "activation": "relu", "updater": m.sgd(0.5)},    # no parameters
            {"type": "dense", "name": "nop", "n_out": 8, "updater": {"kind": "noop"}},
            {"type": "output", "name": "out", "n_out": 1, "updater": m.sgd(m.step_schedule(0.1, 0.5, 1))}]


def _rates(b, net):
    out = {}
    for s in net.specs:
        try:
            out[s["name"]] = net.learning_rate(s["name"])
        except b.B200GanError as e:
            assert e.code == -1
            out[s["name"]] = None
    return out


def test_layer_rule_matches_the_engine(b200):
    b, ctx = b200
    net = b.Net(ctx, _specs(), (8,), max_batch=4)
    got = _rates(b, net)
    assert {k: v is not None for k, v in got.items()} == {s["name"]: engine.layer_has_lr(s) for s in _specs()}
    net.close()


def test_checkpoint_specs_follow_set_and_clear(b200, tmp_path):
    b, ctx = b200
    from gan_deeplearning4j_b200 import models as m, serializer
    net = b.Net(ctx, _specs(), (8,), max_batch=4, seed=3)
    rng = np.random.default_rng(0)
    x, y = rng.uniform(-1, 1, (4, 8)), rng.uniform(0, 1, (4, 1))
    plan = [(m.exponential_schedule(2e-2, 0.8), None), (None, "d1"), (m.map_schedule({0: 1e-3, 2: 4e-3}, type="epoch"), "d2"), (None, None),
            (m.inverse_schedule(5e-3, 0.1, 1.0), None), (None, "out"), (None, None)]
    for k, (sched, layer) in enumerate(plan):
        net.set_lr_schedule(sched, layer)
        net.set_epoch(k)
        net.fit(x, y)
        path = str(tmp_path / f"ckpt{k}.zip")
        net.save(path)
        saved = serializer.read_model(path)
        rebuilt = b.Net(ctx, saved["specs"], (8,), max_batch=4)
        rebuilt.restore(path)
        assert _rates(b, rebuilt) == _rates(b, net), (k, sched, layer)
        for s in saved["specs"]:          # a constant in the spec is exactly the rate the engine uses
            lr = (s.get("updater") or {}).get("lr")
            if engine.layer_has_lr(s) and not engine.is_schedule(lr):
                assert np.float32(lr) == net.learning_rate(s["name"]), (k, s["name"], lr)
        rebuilt.close()
    # everything cleared: every layer is back at its creation-time constant, which a sigmoid-scheduled layer takes as its value at 0
    assert _rates(b, net) == {"d1": np.float32(1e-2), "d2": np.float32(3e-3 / (1 + math.exp(2.0))), "bn": 0.0, "act": None, "fz": None, "nop": None,
                              "out": np.float32(0.1)}
    net.close()
