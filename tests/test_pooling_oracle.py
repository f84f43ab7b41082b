"""CPU checks of the oracle's float64 restatement of SubsamplingLayer AVG / SUM / PNORM and GlobalPoolingLayer: finite differences at
GradientCheckUtil's tolerances for every kind alone and inside conv -> pool -> dense -> output nets, hand-computed answers at the recalled
points (padded AVG corner, zero p-norm window, global MAX tie), float64 torch where torch has the same pooling, and the quirk flags' reach."""
import numpy as np
import pytest

from helpers import randomize
from oracle import dl4j_oracle as o

# GradientCheckUtil (DL4J): epsilon 1e-6, max relative error 1e-3, min absolute error 1e-8
EPS, MAX_REL, MIN_ABS = 1e-6, 1e-3, 1e-8

# (kernel, stride, padding, H, W): overlapping windows (k > s), padding, odd H / W, stride larger than the kernel
GEOMS = [((2, 2), (2, 2), (0, 0), 6, 6), ((3, 3), (2, 2), (1, 1), 7, 5), ((3, 2), (1, 2), (2, 1), 5, 6), ((2, 3), (3, 1), (1, 0), 7, 7)]
POOL2D = [("avg", 2), ("sum", 2), ("pnorm", 1), ("pnorm", 2), ("pnorm", 3)]


def _x(rng, shape):
    """Values bounded away from 0 (p = 1's sign kink, zero windows) with random signs."""
    return rng.uniform(0.3, 1.5, shape) * rng.choice([-1.0, 1.0], shape)


def _fd_check(f, x, grad, rng, n=40):
    for j in rng.choice(x.size, min(n, x.size), replace=False):
        d = np.zeros_like(x); d.flat[j] = EPS
        num = (f(x + d) - f(x - d)) / (2 * EPS)
        ana = grad.flat[j]
        assert abs(num - ana) <= MAX_REL * (abs(num) + abs(ana)) or abs(num - ana) <= MIN_ABS, (j, num, ana)


@pytest.mark.parametrize("geom", range(len(GEOMS)))
@pytest.mark.parametrize("kind,p", POOL2D)
def test_pool2d_finite_differences(kind, p, geom):
    k, s, pad, h, w = GEOMS[geom]
    rng = np.random.default_rng(geom * 10 + p)
    x = _x(rng, (2, 3, h, w))
    y = o.pool2d_forward(kind, x, k, s, pad, p)
    wgt = rng.standard_normal(y.shape)
    loss = lambda v: float((wgt * o.pool2d_forward(kind, v, k, s, pad, p)).sum())
    _fd_check(loss, x, o.pool2d_backward(kind, x, y, wgt, k, s, pad, p), rng)


@pytest.mark.parametrize("kind,p", [("max", 2), ("avg", 2), ("sum", 2), ("pnorm", 1), ("pnorm", 2), ("pnorm", 3)])
def test_global_finite_differences(kind, p):
    seed = o.POOL_CODES[kind] * 5 + p
    rng = np.random.default_rng(seed)
    x = _x(rng, (3, 4, 5, 3))                    # continuous values: no ties
    y, idx = o.global_forward(kind, x, p)
    wgt = rng.standard_normal(y.shape)
    loss = lambda v: float((wgt * o.global_forward(kind, v, p)[0]).sum())
    _fd_check(loss, x, o.global_backward(kind, x, y, idx, wgt, p), np.random.default_rng(seed))


def _net_specs(kind):
    if kind == "global":
        return lambda pool, p: [{"type": "conv2d", "name": "c1", "n_out": 4, "kernel": (3, 3), "stride": (1, 1), "padding": (1, 1), "activation": "tanh"},
                                {"type": "global_pooling", "name": "g", "pooling": pool, "pnorm": p},
                                {"type": "dense", "name": "d1", "n_out": 5, "activation": "tanh"},
                                {"type": "output", "name": "out", "n_out": 3, "loss": "mse"}]
    return lambda pool, p: [{"type": "conv2d", "name": "c1", "n_out": 4, "kernel": (3, 3), "stride": (1, 1), "padding": (1, 1), "activation": "tanh"},
                            {"type": "subsampling", "name": "s", "pooling": pool, "kernel": (3, 3), "stride": (2, 2), "padding": (1, 1), "pnorm": p},
                            {"type": "cnn_to_ff", "name": "ff"},
                            {"type": "dense", "name": "d1", "n_out": 5, "activation": "tanh"},
                            {"type": "output", "name": "out", "n_out": 3, "loss": "mse"}]


@pytest.mark.parametrize("layer,pool,p", [("sub", "avg", 2), ("sub", "sum", 2), ("sub", "pnorm", 2), ("sub", "pnorm", 3),
                                          ("global", "max", 2), ("global", "avg", 2), ("global", "sum", 2), ("global", "pnorm", 1), ("global", "pnorm", 3)])
def test_net_gradient_through_pooling(layer, pool, p):
    """conv -> pool -> dense -> output(MSE): the oracle net's parameter gradients against finite differences."""
    specs = _net_specs(layer)(pool, p)
    net = o.net_from_specs(specs, (2, 7, 5), seed=4, flat_input=False)
    rng = np.random.default_rng(5 + p)
    randomize(net, rng)
    x, y = rng.uniform(-1, 1, (3, 2, 7, 5)), rng.uniform(-1, 1, (3, 3))
    p0 = net.params_flat().copy()
    net.compute_gradient_and_score(x, y)
    grads = net.grads_flat().copy()
    score = lambda q: (net.set_params_flat(q), net.compute_gradient_and_score(x, y))[1] * x.shape[0]
    for j in np.random.default_rng(6).choice(p0.size, 16, replace=False):
        d = np.zeros_like(p0); d[j] = EPS
        num = (score(p0 + d) - score(p0 - d)) / (2 * EPS)
        assert abs(num - grads[j]) <= MAX_REL * (abs(num) + abs(grads[j])) or abs(num - grads[j]) <= 1e-6, (layer, pool, j, num, grads[j])
    net.set_params_flat(p0)


def test_oracle_net_shapes_follow_the_pooling_layers():
    specs = _net_specs("sub")("avg", 2)
    net = o.net_from_specs(specs, (2, 7, 5), flat_input=False)
    out, acts = net.forward(np.ones((2, 2, 7, 5)), True, collect=True)
    assert acts[1].shape == (2, 4, 4, 3) and acts[2].shape == (2, 48) and out.shape == (2, 3)
    net = o.net_from_specs(_net_specs("global")("sum", 2), (2, 7, 5), flat_input=False)
    assert net.forward(np.ones((2, 2, 7, 5)), True, collect=True)[1][1].shape == (2, 4)


# ------------------------------------------------------------------ hand-computed answers ----------------------------------------------
def test_avg_padded_corner_divides_by_the_whole_window():
    """2x2 window, stride 2, padding 1 on a 2x2 map: each corner window holds one input element and three zeros; y = x / 4, not x / 1."""
    x = np.array([1.0, 2.0, 3.0, 4.0]).reshape(1, 1, 2, 2)
    y = o.pool2d_forward("avg", x, (2, 2), (2, 2), (1, 1))
    np.testing.assert_array_equal(y, x / 4)
    dx = o.pool2d_backward("avg", x, y, np.ones_like(y), (2, 2), (2, 2), (1, 1))
    np.testing.assert_array_equal(dx, np.full_like(x, 0.25))
    q = o.Quirks(avg_include_pad_in_divisor=False)
    np.testing.assert_array_equal(o.pool2d_forward("avg", x, (2, 2), (2, 2), (1, 1), q=q), x)


@pytest.mark.parametrize("p", [1, 2, 3])
def test_pnorm_zero_window_is_floored(p):
    """An all-zero window (after a ReLU): y = 0 and dx = 0, where the unfloored formula gives 0 / 0."""
    x = np.zeros((1, 1, 2, 2)); x[0, 0, 1, 1] = 0.0
    y = o.pool2d_forward("pnorm", x, (2, 2), (2, 2), (0, 0), p)
    assert y.ravel().tolist() == [0.0]
    dx = o.pool2d_backward("pnorm", x, y, np.full_like(y, 3.0), (2, 2), (2, 2), (0, 0), p)
    assert np.array_equal(dx, np.zeros_like(x))
    yg, _ = o.global_forward("pnorm", x, p)
    assert np.array_equal(o.global_backward("pnorm", x, yg, None, np.ones_like(yg), p), np.zeros_like(x))
    if p >= 2:
        with np.errstate(invalid="ignore", divide="ignore"):
            bad = o.global_backward("pnorm", x, yg, None, np.ones_like(yg), p, o.Quirks(pnorm_denominator_floor=False))
        assert np.isnan(bad).all()          # DL4J's GlobalPoolingLayer, as recalled


def test_pnorm_hand_values():
    x = np.array([3.0, -4.0, 0.0, 0.0]).reshape(1, 1, 2, 2)
    y = o.pool2d_forward("pnorm", x, (2, 2), (2, 2), (0, 0), 2)
    assert y.item() == 5.0
    dx = o.pool2d_backward("pnorm", x, y, np.ones_like(y), (2, 2), (2, 2), (0, 0), 2)
    np.testing.assert_allclose(dx.ravel(), [0.6, -0.8, 0.0, 0.0], rtol=1e-15)
    y1 = o.pool2d_forward("pnorm", x, (2, 2), (2, 2), (0, 0), 1)
    assert y1.item() == 7.0
    np.testing.assert_array_equal(o.pool2d_backward("pnorm", x, y1, np.ones_like(y1), (2, 2), (2, 2), (0, 0), 1).ravel(), [1.0, -1.0, 0.0, 0.0])


def test_global_max_tie_goes_to_the_first_maximum():
    x = np.array([1.0, 3.0, 3.0, 2.0]).reshape(1, 1, 2, 2)
    y, idx = o.global_forward("max", x)
    assert y.item() == 3.0 and idx.item() == 1
    np.testing.assert_array_equal(o.global_backward("max", x, y, idx, np.array([[5.0]])).ravel(), [0.0, 5.0, 0.0, 0.0])
    q = o.Quirks(global_max_first_tie=False)
    y2, idx2 = o.global_forward("max", x, q=q)
    assert idx2.item() == 2


# ------------------------------------------------------------------ float64 torch ----------------------------------------------------
@pytest.mark.parametrize("geom", [g for g, (k, _, pad, _, _) in enumerate(GEOMS) if 2 * pad[0] <= k[0] and 2 * pad[1] <= k[1]])
def test_torch_avg_pool2d_count_include_pad(geom):
    """(torch's avg_pool2d takes padding up to half the kernel)"""
    torch = pytest.importorskip("torch")
    k, s, pad, h, w = GEOMS[geom]
    rng = np.random.default_rng(geom)
    x = rng.standard_normal((2, 3, h, w))
    t = torch.tensor(x, requires_grad=True)
    y = torch.nn.functional.avg_pool2d(t, k, s, pad, count_include_pad=True)
    e = rng.standard_normal(tuple(y.shape))
    y.backward(torch.tensor(e))
    ref = o.pool2d_forward("avg", x, k, s, pad)
    np.testing.assert_allclose(ref, y.detach().numpy(), rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(o.pool2d_backward("avg", x, ref, e, k, s, pad), t.grad.numpy(), rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize("p", [1, 2, 3])
def test_torch_lp_pool2d_on_non_negative_inputs(p):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(p)
    x = rng.uniform(0.1, 2.0, (2, 3, 7, 6))
    t = torch.tensor(x, requires_grad=True)
    y = torch.nn.functional.lp_pool2d(t, float(p), (3, 2), (2, 2))
    e = rng.standard_normal(tuple(y.shape))
    y.backward(torch.tensor(e))
    ref = o.pool2d_forward("pnorm", x, (3, 2), (2, 2), (0, 0), p)
    np.testing.assert_allclose(ref, y.detach().numpy(), rtol=1e-10)
    np.testing.assert_allclose(o.pool2d_backward("pnorm", x, ref, e, (3, 2), (2, 2), (0, 0), p), t.grad.numpy(), rtol=1e-8, atol=1e-12)


@pytest.mark.parametrize("kind", ["avg", "max", "sum"])
def test_torch_global_pooling(kind):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(7)
    x = rng.standard_normal((3, 5, 4, 6))
    t = torch.tensor(x, requires_grad=True)
    y = {"avg": lambda v: torch.nn.functional.adaptive_avg_pool2d(v, 1).flatten(1), "max": lambda v: v.amax((2, 3)), "sum": lambda v: v.sum((2, 3))}[kind](t)
    e = rng.standard_normal(tuple(y.shape))
    y.backward(torch.tensor(e))
    ref, idx = o.global_forward(kind, x)
    np.testing.assert_allclose(ref, y.detach().numpy(), rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(o.global_backward(kind, x, ref, idx, e), t.grad.numpy(), rtol=1e-12, atol=1e-15)


def test_quirk_flag_moves_only_padded_windows():
    rng = np.random.default_rng(3)
    x = rng.standard_normal((1, 2, 5, 5))
    a = o.pool2d_forward("avg", x, (3, 3), (1, 1), (1, 1))
    b = o.pool2d_forward("avg", x, (3, 3), (1, 1), (1, 1), q=o.Quirks(avg_include_pad_in_divisor=False))
    changed = np.abs(a - b) > 0
    assert not changed[:, :, 1:-1, 1:-1].any() and changed[:, :, 0, :].all() and changed[:, :, :, -1].all()
