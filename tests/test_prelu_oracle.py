"""PReLULayer on the CPU: the oracle's restatement against finite differences at GradientCheckUtil's tolerances for every shared-axes mask,
in nets around it (conv -> PReLU -> dense, conv -> BatchNorm -> PReLU, PReLU first, a residual block of PReLUs) and against float64
torch.autograd; known answers at the signed zeros and NaN; hand-computed updates with l1 / l2 and a schedule on alpha; the spec builders and
their refusals."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gan_deeplearning4j_b200 import engine, models as m
from oracle import dl4j_oracle as o

# GradientCheckUtil: epsilon 1e-6, max relative error 1e-3, min absolute error 1e-8
EPS, MAX_REL, MIN_ABS = 1e-6, 1e-3, 1e-8
CONV_MASKS = [(), (1,), (2,), (3,), (1, 2), (1, 3), (2, 3), (1, 2, 3)]


def _randomize_alpha(net, rng):
    for l in net.layers:
        if isinstance(l, o.PReLU):
            l.params["W"] = rng.uniform(-0.5, 0.8, l.alpha_shape)
        elif l.has_params:
            for p, shape, _ in l.param_specs():
                if p in ("b", "beta"):
                    l.params[p] = 0.1 * rng.standard_normal(shape)


def _grad_check(net, x, y):
    """Every parameter's analytic gradient of score * mb against central differences of the score (GradientCheckUtil's rule: relative error
    within MAX_REL unless both are below MIN_ABS).  BatchNorm's running statistics have pseudo-gradients and are skipped."""
    mb = x.shape[0]
    net.compute_gradient_and_score(x, y)
    checked = 0
    for l in net.layers:
        if not l.has_params:
            continue
        for p, _, _ in l.param_specs():
            if p in l.noop_names():
                continue
            g = l.grads[p].ravel()
            v = l.params[p].reshape(-1)
            for i in range(v.size):
                old = v[i]
                v[i] = old + EPS; sp = net.compute_gradient_and_score(x, y)
                v[i] = old - EPS; sm = net.compute_gradient_and_score(x, y)
                v[i] = old
                num = (sp - sm) / (2 * EPS) * mb
                err = abs(num - g[i]) / max(abs(num) + abs(g[i]), 1e-300)
                assert err < MAX_REL or abs(num - g[i]) < MIN_ABS, (l.name, p, i, num, g[i])
                checked += 1
    net.compute_gradient_and_score(x, y)
    return checked


def _net(specs, shape, seed=3):
    rng = np.random.default_rng(seed)
    net = o.net_from_specs(specs, shape, seed=2)
    _randomize_alpha(net, rng)
    return net, rng


def _prelu(axes, name="p", **kw):
    return dict(m.prelu(axes, name), updater=m.sgd(0.1), **kw)


@pytest.mark.parametrize("axes", CONV_MASKS)
def test_finite_differences_conv_prelu_dense(axes):
    specs = [{"type": "conv2d", "name": "c1", "n_out": 3, "kernel": (3, 3), "stride": (1, 1), "padding": (1, 1), "updater": m.sgd(0.1)},
             _prelu(axes), {"type": "cnn_to_ff", "name": "f"}, {"type": "dense", "name": "d", "n_out": 4, "activation": "tanh", "updater": m.sgd(0.1)},
             {"type": "output", "name": "out", "n_out": 1, "updater": m.sgd(0.1)}]
    net, rng = _net(specs, (2, 4, 3))
    assert net.layers[2].alpha_shape == tuple(1 if a in axes else d for a, d in zip((1, 2, 3), (3, 4, 3)))
    x, y = rng.uniform(-1, 1, (3, 2, 4, 3)), rng.uniform(0, 1, (3, 1))
    assert _grad_check(net, x, y) > 0


@pytest.mark.parametrize("axes", [(), (1,)])
def test_finite_differences_feed_forward(axes):
    specs = [{"type": "dense", "name": "d1", "n_out": 5, "updater": m.sgd(0.1)}, _prelu(axes),
             {"type": "output", "name": "out", "n_out": 1, "updater": m.sgd(0.1)}]
    net, rng = _net(specs, (4,))
    x, y = rng.uniform(-1, 1, (4, 4)), rng.uniform(0, 1, (4, 1))
    assert _grad_check(net, x, y) > 0


def test_finite_differences_batchnorm_first_layer_and_residual():
    u = lambda: m.sgd(0.1)
    convbn = [{"type": "conv2d", "name": "c1", "n_out": 3, "kernel": (3, 3), "stride": (1, 1), "padding": (1, 1), "has_bias": False, "updater": u()},
              {"type": "batchnorm", "name": "bn", "updater": u()}, _prelu((2, 3)), {"type": "cnn_to_ff", "name": "f"},
              {"type": "output", "name": "out", "n_out": 1, "updater": u()}]
    first = [_prelu((), "p0"), {"type": "cnn_to_ff", "name": "f"}, {"type": "output", "name": "out", "n_out": 1, "updater": u()}]
    res = ([{"type": "conv2d", "name": "stem", "n_out": 3, "kernel": (3, 3), "stride": (1, 1), "padding": (1, 1), "updater": u()}, _prelu((2, 3), "stem_act")] +
           m.residual_block("r", 3, "stem_act", activation="prelu") + [{"type": "cnn_to_ff", "name": "f"}, {"type": "output", "name": "out", "n_out": 1, "updater": u()}])
    assert sum(s["type"] == "prelu" for s in res) == 3
    for specs in (convbn, first, res):
        net, rng = _net(specs, (2, 4, 4))
        x, y = rng.uniform(-1, 1, (3, 2, 4, 4)), rng.uniform(0, 1, (3, 1))
        assert _grad_check(net, x, y) > 0


@pytest.mark.parametrize("axes", CONV_MASKS)
def test_float64_autograd(axes):
    rng = np.random.default_rng(len(axes) + 10 * sum(axes))
    l = o.PReLU((3, 4, 5), axes)
    l.init(rng, np.float64)
    l.params["W"] = rng.uniform(-0.5, 0.8, l.alpha_shape)
    x, e = rng.uniform(-1, 1, (2, 3, 4, 5)), rng.standard_normal((2, 3, 4, 5))
    y = l.forward(x, True); dx = l.backward(e)
    xt = torch.tensor(x, requires_grad=True); at = torch.tensor(l.params["W"], requires_grad=True)
    yt = F.prelu(xt, at.reshape(-1)) if axes == (2, 3) else torch.where(xt < 0, at[None] * xt, xt)
    yt.backward(torch.tensor(e))
    np.testing.assert_allclose(y, yt.detach().numpy(), rtol=1e-13, atol=1e-15)
    np.testing.assert_allclose(dx, xt.grad.numpy(), rtol=1e-13, atol=1e-15)
    np.testing.assert_allclose(l.grads["W"], at.grad.numpy(), rtol=1e-12, atol=1e-14)


def test_known_answers_signed_zero_and_nan():
    l = o.PReLU((6,), ())
    l.init(np.random.default_rng(0), np.float64)
    l.params["W"] = np.full(6, 0.25)
    x = np.array([[0.0, -0.0, -2.0, 3.0, np.nan, -4.0]])
    y = l.forward(x, True)
    assert y[0, 0] == 0 and not np.signbit(y[0, 0]) and y[0, 1] == 0 and np.signbit(y[0, 1])
    assert y[0, 2] == -0.5 and y[0, 3] == 3.0 and np.isnan(y[0, 4]) and y[0, 5] == -1.0
    dx = l.backward(np.array([[1.0, 2.0, 4.0, 5.0, 6.0, 8.0]]))
    np.testing.assert_array_equal(dx, [[1.0, 2.0, 1.0, 5.0, 6.0, 2.0]])
    np.testing.assert_array_equal(l.grads["W"], [0.0, 0.0, -8.0, 0.0, 0.0, -32.0])


def test_new_prelu_is_a_relu():
    net = o.net_from_specs([_prelu((1,)), {"type": "output", "name": "out", "n_out": 1, "updater": m.sgd(0.1)}], (5,), seed=1)
    assert np.all(net.layers[0].params["W"] == 0) and net.layers[0].alpha_shape == (1,)
    x = np.linspace(-2, 2, 10).reshape(2, 5)
    np.testing.assert_array_equal(net.layers[0].forward(x, True), np.maximum(x, 0))


@pytest.mark.parametrize("l1,l2", [(0.0, 0.0), (2e-3, 0.0), (0.0, 1e-2), (2e-3, 1e-2)])
def test_hand_computed_update_with_l1_l2(l1, l2):
    lr, mb = 0.1, 2
    specs = [dict(_prelu((), l1=l1, l2=l2), updater=m.sgd(lr)), {"type": "output", "name": "out", "n_out": 1, "updater": m.sgd(0.0)}]
    net = o.net_from_specs(specs, (3,), seed=1)
    a0 = np.array([0.3, -0.2, 0.0])
    net.layers[0].params["W"] = a0.copy()
    x, y = np.array([[-1.0, -2.0, 3.0], [-0.5, 1.0, -1.0]]), np.array([[1.0], [0.0]])
    score = net.compute_gradient_and_score(x, y)
    g = net.layers[0].grads["W"].copy()
    want_score_reg = 0.5 * l2 * float((a0 ** 2).sum()) + l1 * float(np.abs(a0).sum())
    assert abs(net.l2_score() - want_score_reg) < 1e-15
    net.apply_update(mb)
    want = a0 - (lr * g / mb + l2 * a0 + l1 * np.sign(a0))
    np.testing.assert_allclose(net.layers[0].params["W"], want, rtol=0, atol=1e-15)
    assert score > 0


def test_schedule_value_on_the_prelu_layer():
    sched = m.exponential_schedule(0.1, 0.5)
    specs = [dict(m.prelu((), "p"), updater=m.sgd(sched)), {"type": "output", "name": "out", "n_out": 1, "updater": m.sgd(0.0)}]
    net = o.net_from_specs(specs, (2,), seed=1)
    assert net.schedules == {"p": sched}
    x, y = np.array([[-1.0, -2.0]]), np.array([[1.0]])
    for it in range(3):
        a0 = net.layers[0].params["W"].copy()
        net.compute_gradient_and_score(x, y)
        g = net.layers[0].grads["W"].copy()
        assert net.learning_rate("p") == np.float32(0.1 * 0.5 ** it)
        net.apply_update(1)
        np.testing.assert_allclose(net.layers[0].params["W"], a0 - float(np.float32(0.1 * 0.5 ** it)) * g, rtol=0, atol=1e-15)


def test_frozen_prelu_passes_dx_without_slope_gradient():
    specs = [{"type": "dense", "name": "d1", "n_out": 4, "updater": m.sgd(0.1)}, dict(_prelu(()), frozen=True),
             {"type": "output", "name": "out", "n_out": 1, "updater": m.sgd(0.1)}]
    net, rng = _net(specs, (3,))
    x, y = rng.uniform(-1, 1, (4, 3)), rng.uniform(0, 1, (4, 1))
    net.compute_gradient_and_score(x, y)
    assert "W" not in net.layers[1].grads and np.abs(net.layers[0].grads["W"]).max() > 0
    a0 = net.layers[1].params["W"].copy()
    net.apply_update(4)
    np.testing.assert_array_equal(net.layers[1].params["W"], a0)


def test_spec_builder_and_desc():
    s = m.prelu((3, 2, 2), "act", input_shape=(8, 4, 4))
    assert s == {"type": "prelu", "name": "act", "shared_axes": [2, 3], "input_shape": [8, 4, 4]}
    d = engine.layer_desc(dict(s, updater=m.adam(1e-3), l2=1e-4))
    assert (d.type, d.act, d.pre_c, d.pre_h, d.pre_w, d.updater) == (17, 6, 8, 4, 4, engine.UPDATERS["adam"]) and abs(d.l2 - 1e-4) < 1e-9
    d = engine.layer_desc(m.prelu((1,), "ff", input_shape=(10,)))
    assert (d.act, d.pre_c, d.pre_h, d.pre_w) == (1, 10, 0, 0)
    assert engine.layer_desc(m.prelu()).act == 0
    assert engine.layer_has_lr(dict(m.prelu(), updater=m.adam())) and not engine.layer_has_lr(dict(m.prelu(), updater=m.adam(), frozen=True))


def test_refusals():
    for bad in ((0,), (4,), (-1,)):
        with pytest.raises(ValueError):
            m.prelu(bad)
    with pytest.raises(ValueError):
        engine.layer_desc(m.prelu(input_shape=(2, 3)))
    for scheme in ("xavier", "relu", "identity"):
        with pytest.raises(ValueError):
            engine.weight_init_struct(m.weight_init(scheme), m.prelu(name="p"))
    for scheme in ("zero", "ones"):
        engine.weight_init_struct(m.weight_init(scheme), m.prelu(name="p"))
    engine.weight_init_struct(m.weight_init("distribution", m.normal(0.25, 0.01)), m.prelu(name="p"))
    with pytest.raises(ValueError):
        o.PReLU((5,), (2,))


def test_dcgan_prelu_specs_resolve_and_count():
    for residual in (False, True):
        gs = m.dcgan_generator(16, 12, 8, 3, activation="prelu", residual=residual)
        ds = m.dcgan_discriminator(16, 8, 3, activation="prelu", residual=residual)
        for specs, shape in ((gs, (12,)), (ds, (3, 16, 16))):
            assert not any(s["type"] == "activation" for s in specs)
            assert all(s["shared_axes"] == [2, 3] and s["updater"]["kind"] == "adam" for s in specs if s["type"] == "prelu")
            engine.resolve_vertices(specs)
            base = m.dcgan_generator(16, 12, 8, 3, residual=residual) if shape == (12,) else m.dcgan_discriminator(16, 8, 3, residual=residual)
            assert m.forward_macs(specs, shape) == m.forward_macs(base, shape)
            net = o.net_from_specs(specs, shape, seed=1)
            assert sum(isinstance(l, o.PReLU) for l in net.layers) == sum(s["type"] == "prelu" for s in specs)
        assert ds[0].get("activation", "identity") == "identity" and ds[1]["name"] == "dis_act_1" and ds[1]["type"] == "prelu"


def test_oracle_gan_step_trains_both_nets_slopes():
    gs, ds = m.dcgan_generator(16, 12, 8, 3, lr=2e-3, activation="prelu"), m.dcgan_discriminator(16, 8, 3, lr=2e-3, activation="prelu")
    G = o.net_from_specs(gs, (12,), seed=1); D = o.net_from_specs(ds, (3, 16, 16), seed=2)
    rng = np.random.default_rng(4)
    _randomize_alpha(G, rng); _randomize_alpha(D, rng)
    before = {(net_i, l.name): l.params["W"].copy() for net_i, net in enumerate((G, D)) for l in net.layers if isinstance(l, o.PReLU)}
    r = o.gan_step(G, D, *[a.astype(np.float64) for a in o.synthetic_batch(4, 16, 3, 12, seed=3)])
    assert np.isfinite([r["loss_d_real"], r["loss_d_fake"], r["loss_g"]]).all()
    for (net_i, name), w in before.items():
        assert not np.array_equal((G, D)[net_i].layer(name).params["W"], w), name


def test_checkpoint_specs_round_trip(tmp_path):
    from gan_deeplearning4j_b200 import serializer
    ds = m.dcgan_discriminator(16, 8, 3, activation="prelu") + [dict(m.prelu((1,), "extra", input_shape=(4,)), l1=1e-3, frozen=True)]
    net = o.net_from_specs(ds[:-1], (3, 16, 16), seed=1)
    serializer.write_model(tmp_path / "d.zip", ds, (3, 16, 16), net.params_flat().astype(np.float32))
    back = serializer.read_model(tmp_path / "d.zip")
    assert back["specs"] == [json_like(s) for s in ds]
    assert [engine.layer_desc(s, v).act for s, v in zip(back["specs"], engine.resolve_vertices(back["specs"]))] == \
           [engine.layer_desc(s, v).act for s, v in zip(ds, engine.resolve_vertices(ds))]


def json_like(spec):
    import json
    return json.loads(json.dumps(spec))
