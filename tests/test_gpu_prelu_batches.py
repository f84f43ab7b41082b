"""PReLU nets trained at batches below max_batch, where the backward's row groups outnumber those of a max_batch pass (max_batch 65, batch 64:
64 groups against 33), against the oracle's restatement; and a 1x1 convolutional map declared [C, 1, 1] by inputShape, whose H and W shared
axes are accepted."""
import numpy as np
import pytest

from gan_deeplearning4j_b200 import models as m
from helpers import b200, compare_params_and_state, push_params, randomize  # noqa: F401
from oracle import dl4j_oracle as o

pytestmark = pytest.mark.gpu
TOL = 1e-3
LR = 2e-3


def _oracle(specs, shape, seed):
    rng = np.random.default_rng(seed)
    onet = o.net_from_specs(specs, shape, seed=2)
    randomize(onet, rng)
    for l in onet.layers:
        if isinstance(l, o.PReLU):
            l.params["W"] = rng.uniform(-0.3, 0.6, l.alpha_shape)
    return onet, rng


def _fit(b, ctx, specs, shape, max_batch, batches, seed=7):
    onet, rng = _oracle(specs, shape, seed)
    bnet = b.Net(ctx, specs, shape, max_batch=max_batch, precision=b.FP32)
    push_params(onet, bnet)
    bounds = {s["name"]: 2 * LR + 2e-3 for s in specs if s.get("updater")}
    for it, n in enumerate(batches):
        x, y = rng.uniform(-1, 1, (n,) + shape), rng.uniform(0, 1, (n, 1))
        so, sb = onet.fit(x, y), bnet.fit(x, y)
        assert abs(so - sb) < TOL * max(1.0, abs(so)), (it, n, so, sb)
        compare_params_and_state(onet, bnet, (it, n), TOL, bounds)
    bnet.close()


@pytest.mark.parametrize("axes", [(), (1,)])
def test_fit_below_max_batch(b200, axes):
    b, ctx = b200
    u = lambda: m.adam(LR)
    specs = [{"type": "dense", "name": "d1", "n_out": 32, "updater": u()}, dict(m.prelu(axes, "p1"), updater=u(), l1=1e-3, l2=1e-2),
             {"type": "output", "name": "out", "n_out": 1, "updater": u()}]
    _fit(b, ctx, specs, (12,), 65, [64, 65, 34, 1, 64])


def test_conv_map_below_max_batch(b200):
    """M = 4 * 4 * 8 = 128 row elements: max_batch 65 holds 33 groups, batch 34 runs 34."""
    b, ctx = b200
    u = lambda: m.adam(LR)
    specs = [{"type": "conv2d", "name": "c1", "n_out": 8, "kernel": (3, 3), "stride": (2, 2), "padding": (1, 1), "updater": u()},
             dict(m.prelu((), "p1"), updater=u()), dict(m.prelu((2, 3), "p2"), updater=u()), {"type": "cnn_to_ff", "name": "flat"},
             {"type": "output", "name": "out", "n_out": 1, "updater": u()}]
    _fit(b, ctx, specs, (3, 8, 8), 65, [34, 64, 65])


def test_one_by_one_map_with_input_shape(b200):
    b, ctx = b200
    u = lambda: m.adam(LR)
    head = [{"type": "cnn_to_ff", "name": "flat"}, {"type": "output", "name": "out", "n_out": 1, "updater": u()}]
    conv = {"type": "conv2d", "name": "c1", "n_out": 6, "kernel": (4, 4), "stride": (1, 1), "padding": (0, 0), "updater": u()}
    for axes in ((2, 3), (1, 2, 3), (3,)):
        _fit(b, ctx, [conv, dict(m.prelu(axes, "p1", input_shape=(6, 1, 1)), updater=u())] + head, (3, 4, 4), 8, [8, 5])
    with pytest.raises(b.B200GanError) as e:         # without inputShape a 1x1 map is a feed-forward input: axis 1 only
        b.Net(ctx, [conv, dict(m.prelu((2, 3), "p1"), updater=u())] + head, (3, 4, 4), max_batch=4)
    assert e.value.code == -1
