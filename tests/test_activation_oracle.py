"""CPU checks of the oracle's float64 restatement of b2g_activation codes 5-16: finite differences at GradientCheckUtil's
tolerances, hand-computed values at and beside every boundary, float64 torch where torch has the same function, the quirk flags' reach, and the
restatement through oracle layers and a loss (existing kinds unchanged)."""
import numpy as np
import pytest

from helpers import randomize
from oracle import dl4j_oracle as o

# GradientCheckUtil (DL4J): epsilon 1e-6, max relative error 1e-3, min absolute error 1e-8
EPS, MAX_REL, MIN_ABS = 1e-6, 1e-3, 1e-8
KINKS = {"elu": [0.0], "selu": [0.0], "hardtanh": [-1.0, 1.0], "hardsigmoid": [-2.5, 2.5], "relu6": [0.0, 6.0], "rectifiedtanh": [0.0],
         "thresholdedrelu": [1.0], "rationaltanh": [0.0]}


def _points(kind, rng):
    z = np.concatenate([rng.uniform(-8, 8, 400), rng.uniform(-1.5, 1.5, 200), [-30.0, -12.0, 12.0, 30.0]])
    for k in KINKS.get(kind, []):
        z = z[np.abs(z - k) > 10 * EPS]
    return z


@pytest.mark.parametrize("kind", o.EXT_ACTS)
def test_finite_differences(kind):
    rng = np.random.default_rng(o.ACT_CODES[kind])
    z = _points(kind, rng)
    num = (o.forward(kind, z + EPS) - o.forward(kind, z - EPS)) / (2 * EPS)
    ana = o.derivative(kind, z)
    d = np.abs(num - ana)
    rel = d / np.maximum(np.abs(num) + np.abs(ana), 1e-300)
    assert np.all((rel <= MAX_REL) | (d <= MIN_ABS)), (kind, z[np.argmax(rel)], rel.max())


@pytest.mark.parametrize("kind", ("elu", "thresholdedrelu"))
def test_finite_differences_with_alpha(kind):
    z = _points("selu", np.random.default_rng(3))
    z = z[np.abs(z - 0.37) > 10 * EPS]
    num = (o.forward(kind, z + EPS, 0.37) - o.forward(kind, z - EPS, 0.37)) / (2 * EPS)
    ana = o.derivative(kind, z, 0.37)
    assert np.all((np.abs(num - ana) <= MAX_REL * (np.abs(num) + np.abs(ana))) | (np.abs(num - ana) <= MIN_ABS))


L, S = o.SELU_LAMBDA, o.SELU_ALPHA
# (kind, alpha, z, f(z), f'(z)) at and beside the boundaries, by hand
HAND = [
    ("elu", None, 0.0, 0.0, 1.0), ("elu", None, -1.0, np.e ** -1 - 1, np.e ** -1), ("elu", 0.5, -2.0, 0.5 * (np.e ** -2 - 1), 0.5 * np.e ** -2),
    ("elu", None, 1.0, 1.0, 1.0),
    ("selu", None, 0.0, 0.0, L * S), ("selu", None, 1.0, L, L), ("selu", None, -1.0, L * S * (np.e ** -1 - 1), L * S * np.e ** -1),
    ("softplus", None, 0.0, np.log(2.0), 0.5), ("softplus", None, 100.0, 100.0, 1.0), ("softplus", None, -100.0, np.exp(-100.0), np.exp(-100.0)),
    ("softsign", None, 0.0, 0.0, 1.0), ("softsign", None, 1.0, 0.5, 0.25), ("softsign", None, -3.0, -0.75, 1 / 16),
    ("hardtanh", None, 1.0, 1.0, 1.0), ("hardtanh", None, -1.0, -1.0, 1.0), ("hardtanh", None, 1.5, 1.0, 0.0), ("hardtanh", None, -1.5, -1.0, 0.0),
    ("hardtanh", None, 0.0, 0.0, 1.0),
    ("hardsigmoid", None, 2.5, 1.0, 0.2), ("hardsigmoid", None, -2.5, 0.0, 0.2), ("hardsigmoid", None, 2.6, 1.0, 0.0),
    ("hardsigmoid", None, -2.6, 0.0, 0.0), ("hardsigmoid", None, 0.0, 0.5, 0.2), ("hardsigmoid", None, 1.0, 0.7, 0.2),
    ("relu6", None, 0.0, 0.0, 0.0), ("relu6", None, 6.0, 6.0, 0.0), ("relu6", None, 5.5, 5.5, 1.0), ("relu6", None, 6.5, 6.0, 0.0),
    ("relu6", None, 0.5, 0.5, 1.0), ("relu6", None, -0.5, 0.0, 0.0),
    ("swish", None, 0.0, 0.0, 0.5), ("swish", None, 100.0, 100.0, 1.0), ("swish", None, -100.0, -100.0 * np.exp(-100.0), -99.0 * np.exp(-100.0)),
    ("cube", None, -2.0, -8.0, 12.0), ("cube", None, 0.0, 0.0, 0.0),
    ("rationaltanh", None, 0.0, 0.0, 1.7159 * 2 / 3), ("rationaltanh", None, 1.5, 1.7159 * (1 - 1 / (3 + 1.41645)),
                                                        1.7159 * 2 / 3 * (1 + 2 + 4 * 1.41645) / (3 + 1.41645) ** 2),
    ("rationaltanh", None, -1.5, -1.7159 * (1 - 1 / (3 + 1.41645)), 1.7159 * 2 / 3 * (1 + 2 + 4 * 1.41645) / (3 + 1.41645) ** 2),
    ("rectifiedtanh", None, 0.0, 0.0, 0.0), ("rectifiedtanh", None, -1.0, 0.0, 0.0), ("rectifiedtanh", None, 1.0, np.tanh(1.0), 1 - np.tanh(1.0) ** 2),
    ("thresholdedrelu", None, 1.0, 0.0, 0.0), ("thresholdedrelu", None, 1.5, 1.5, 1.0), ("thresholdedrelu", None, 0.5, 0.0, 0.0),
    ("thresholdedrelu", 2.0, 2.0, 0.0, 0.0), ("thresholdedrelu", 2.0, 2.25, 2.25, 1.0), ("thresholdedrelu", -1.0, -0.5, -0.5, 1.0),
]


@pytest.mark.parametrize("kind,alpha,z,f,df", HAND)
def test_hand_computed_boundaries(kind, alpha, z, f, df):
    assert o.forward(kind, np.array([z]), alpha)[0] == pytest.approx(f, rel=1e-12, abs=1e-300)
    assert o.derivative(kind, np.array([z]), alpha)[0] == pytest.approx(df, rel=1e-12, abs=1e-300)


def test_no_overflow_where_the_function_is_finite():
    z = np.array([-1e4, -700.0, -100.0, 100.0, 700.0, 1e4])
    for kind in o.EXT_ACTS:
        assert np.all(np.isfinite(o.forward(kind, z))) and np.all(np.isfinite(o.derivative(kind, z))), kind


@pytest.mark.parametrize("kind,fn", [("elu", "elu"), ("selu", "selu"), ("softplus", "softplus"), ("softsign", "softsign"),
                                     ("hardtanh", "hardtanh"), ("relu6", "relu6"), ("swish", "silu")])
def test_torch_float64_cross_check(kind, fn):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(11)
    z = _points(kind, rng)
    t = torch.tensor(z, dtype=torch.float64, requires_grad=True)
    y = getattr(torch.nn.functional, fn)(t)
    y.sum().backward()
    np.testing.assert_allclose(o.forward(kind, z), y.detach().numpy(), rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(o.derivative(kind, z), t.grad.numpy(), rtol=1e-12, atol=1e-15)


def test_quirk_flags_move_only_their_boundaries():
    z = np.array([-2.5, -1.0, 0.0, 1.0, 2.5, 6.0, 3.0])
    base = {k: o.derivative(k, z) for k in ("hardtanh", "hardsigmoid", "relu6")}
    for field, kind, moved in (("hardtanh_closed", "hardtanh", [1, 3]), ("hardsigmoid_closed", "hardsigmoid", [0, 4]), ("relu6_open", "relu6", [2, 5])):
        q = o.Quirks(**{field: not getattr(o.DEFAULT_QUIRKS, field)})
        d = o.derivative(kind, z, q=q)
        changed = np.nonzero(d != base[kind])[0].tolist()
        assert changed == moved, (field, changed)
    with pytest.raises(ValueError):
        o.forward("thresholdedrelu", z, q=o.Quirks(thresholded_relu_in_beta3=False))


@pytest.mark.parametrize("kind", o.EXT_ACTS)
def test_net_gradient_through_layers_and_loss(kind):
    """Dense(kind) -> ActivationLayer(kind) -> Output(MSE on kind): the oracle net's parameter gradients against finite differences."""
    specs = [{"type": "dense", "name": "d1", "n_out": 5, "activation": kind},
             {"type": "activation", "name": "a1", "activation": "tanh"},
             {"type": "dense", "name": "d2", "n_out": 4},
             {"type": "activation", "name": "a2", "activation": kind},
             {"type": "output", "name": "out", "n_out": 3, "loss": "mse", "activation": kind}]
    net = o.net_from_specs(specs, (6,), seed=4)
    rng = np.random.default_rng(5)
    randomize(net, rng)          # non-zero biases: a row whose hidden units are all 0 would otherwise sit on the kink at z = 0
    x, y = rng.uniform(-1.2, 1.2, (7, 6)), rng.uniform(-1, 1, (7, 3))
    p0 = net.params_flat().copy()
    net.compute_gradient_and_score(x, y)
    grads = net.grads_flat().copy()          # minibatch sums: the derivative of the summed score
    score = lambda p: (net.set_params_flat(p), net.compute_gradient_and_score(x, y))[1] * x.shape[0]
    for j in np.random.default_rng(6).choice(p0.size, 12, replace=False):
        d = np.zeros_like(p0); d[j] = EPS
        num = (score(p0 + d) - score(p0 - d)) / (2 * EPS)
        ana = grads[j]
        assert abs(num - ana) <= MAX_REL * (abs(num) + abs(ana)) or abs(num - ana) <= 1e-6, (kind, j, num, ana)
    net.set_params_flat(p0)
