"""CPU checks of the oracle's restatement of DL4J's MSE, L1, L2, MAE, Hinge, SquaredHinge and Wasserstein losses: finite differences
with GradientCheckUtil's tolerances for every (loss, activation) pair (on the loss alone and through a small net on the unchanged oracle),
hand-computed answers including the kinks, a float64 torch.autograd cross-check, and the reach of the Wasserstein quirk flag."""
import zlib

import numpy as np
import pytest

from oracle import dl4j_oracle as o

ACTS = o.ACTS
EPS, MAX_REL, MIN_ABS = 1e-6, 1e-3, 1e-8          # GradientCheckUtil


def _rng(*parts):
    return np.random.default_rng(zlib.crc32(repr(parts).encode()))


def _away_from_kinks(loss, act, rng, shape, alpha=0.2):
    """z and labels whose a - y, 1 - y a and z all stay >= 1e-2 from 0, where L1 / MAE / the hinges and ReLU / LeakyReLU have kinks."""
    while True:
        z = rng.uniform(-2, 2, shape)
        y = rng.choice([-1.0, 1.0], shape) if loss in ("hinge", "squared_hinge") else rng.uniform(-1, 1, shape)
        a = o.act_forward(act, z, alpha)
        if np.abs(z).min() > 1e-2 and np.abs(a - y).min() > 1e-2 and np.abs(1 - y * a).min() > 1e-2:
            return z, y


def _check_fd(analytic, numeric, what):
    d = np.abs(analytic - numeric)
    rel = d / np.maximum(np.abs(analytic) + np.abs(numeric), 1e-300)
    bad = (rel > MAX_REL) & (d > MIN_ABS)
    assert not bad.any(), (what, float(rel[bad].max()))


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("loss", o.LOSSES)
def test_finite_differences_on_the_loss(loss, act):
    rng = _rng("loss", loss, act)
    z, y = _away_from_kinks(loss, act, rng, (5, 3))
    _, g = o.score_and_grad(loss, act, 0.2, z, y)
    num = np.zeros_like(z)
    for i in np.ndindex(z.shape):
        zp, zm = z.copy(), z.copy(); zp[i] += EPS; zm[i] -= EPS
        num[i] = (o.score_and_grad(loss, act, 0.2, zp, y)[0] - o.score_and_grad(loss, act, 0.2, zm, y)[0]) / (2 * EPS)
    _check_fd(g, num, (loss, act))


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("loss", o.LOSSES)
def test_finite_differences_through_the_oracle_net(loss, act):
    """Dense(tanh) -> OutputLayer(loss, act, nOut = 3): the oracle's compute_gradient_and_score on its Output layer, every parameter."""
    rng = _rng("net", loss, act)
    specs = [{"type": "dense", "name": "d", "n_out": 4, "activation": "tanh"},
             {"type": "output", "name": "out", "n_out": 3, "loss": loss, "activation": act, "alpha": 0.2}]
    net = o.net_from_specs(specs, (3,), seed=3)
    assert isinstance(net.layers[-1], o.Output) and net.layers[-1].loss_act == act
    x = rng.uniform(-1, 1, (4, 3))
    for _ in range(100):              # labels away from the kinks at the net's own outputs
        _, y = _away_from_kinks(loss, "identity", rng, (4, 3))
        a = net.output(x)
        if np.abs(a - y).min() > 1e-2 and np.abs(1 - y * a).min() > 1e-2 and np.abs(net.layers[-1]._z).min() > 1e-2:
            break
    net.compute_gradient_and_score(x, y)
    g = net.grads_flat().copy()
    p0 = net.params_flat().copy()
    num = np.zeros_like(p0)
    for i in range(p0.size):
        for sgn in (1, -1):
            p = p0.copy(); p[i] += sgn * EPS; net.set_params_flat(p)
            num[i] += sgn * net.compute_gradient_and_score(x, y) * x.shape[0] / (2 * EPS)      # score = sum / mb
    net.set_params_flat(p0)
    _check_fd(g, num, (loss, act))


def test_hand_computed_answers_and_kinks():
    z = np.array([[0.5, -1.0, 2.0]]); y = np.array([[1.0, -1.0, 0.0]])
    s, g = o.score_and_grad("mse", "identity", 0.0, z, y)
    assert s == pytest.approx((0.25 + 0 + 4) / 3) and np.allclose(g, [[2 * -0.5 / 3, 0, 4 / 3]])
    s, g = o.score_and_grad("l2", "identity", 0.0, z, y)
    assert s == pytest.approx(4.25) and np.allclose(g, [[-1, 0, 4]])
    s, g = o.score_and_grad("l1", "identity", 0.0, z, y)                  # a = y in the middle: sign(0) = 0
    assert s == pytest.approx(2.5) and np.array_equal(g, [[-1, 0, 1]])
    s, g = o.score_and_grad("mae", "identity", 0.0, z, y)
    assert s == pytest.approx(2.5 / 3) and np.allclose(g, [[-1 / 3, 0, 1 / 3]])
    zh = np.array([[1.0, 0.5, -1.0, 3.0]]); yh = np.array([[1.0, 1.0, -1.0, -1.0]])   # margins 0 (kink), 0.5, 0 (kink), 4
    s, g = o.score_and_grad("hinge", "identity", 0.0, zh, yh)
    assert s == pytest.approx(4.5) and np.array_equal(g, [[0, -1, 0, 1]])
    s, g = o.score_and_grad("squared_hinge", "identity", 0.0, zh, yh)
    assert s == pytest.approx(16.25) and np.allclose(g, [[0, -1, 0, 8]])
    s, g = o.score_and_grad("wasserstein", "identity", 0.0, zh, yh)
    assert s == pytest.approx((1 + 0.5 + 1 - 3) / 4) and np.allclose(g, yh / 4)
    s, g = o.score_and_grad("mse", "sigmoid", 0.0, np.array([[0.0]]), np.array([[1.0]]))   # a = 0.5, act' = 0.25
    assert s == pytest.approx(0.25) and g[0, 0] == pytest.approx(2 * -0.5 * 0.25)
    s, g = o.score_and_grad("hinge", "tanh", 0.0, np.array([[0.0]]), np.array([[1.0]]))      # a = 0, margin 1, act' = 1
    assert s == pytest.approx(1.0) and g[0, 0] == pytest.approx(-1.0)
    s, g = o.score_and_grad("l1", "lrelu", 0.2, np.array([[-1.0]]), np.array([[0.0]]))      # a = -0.2: sign -1, act' = alpha
    assert s == pytest.approx(0.2) and g[0, 0] == pytest.approx(-0.2)


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("loss", o.LOSSES)
def test_torch_autograd_float64(loss, act):
    import torch
    rng = _rng("torch", loss, act)
    z, y = _away_from_kinks(loss, act, rng, (6, 4))
    s, g = o.score_and_grad(loss, act, 0.2, z, y)
    zt, yt = torch.tensor(z, dtype=torch.float64, requires_grad=True), torch.tensor(y, dtype=torch.float64)
    a = {"identity": lambda t: t, "tanh": torch.tanh, "sigmoid": torch.sigmoid, "relu": torch.relu,
         "lrelu": lambda t: torch.nn.functional.leaky_relu(t, 0.2)}[act](zt)
    n = z.shape[1]
    st = {"mse": lambda: ((a - yt) ** 2).sum() / n, "l2": lambda: ((a - yt) ** 2).sum(), "l1": lambda: (a - yt).abs().sum(),
          "mae": lambda: (a - yt).abs().sum() / n, "hinge": lambda: torch.clamp(1 - yt * a, min=0).sum(),
          "squared_hinge": lambda: (torch.clamp(1 - yt * a, min=0) ** 2).sum(), "wasserstein": lambda: (yt * a).sum() / n}[loss]()
    st.backward()
    assert s == pytest.approx(st.item(), rel=1e-12, abs=1e-14)
    np.testing.assert_allclose(g, zt.grad.numpy(), rtol=1e-10, atol=1e-14)


def test_wasserstein_quirk_reaches_only_wasserstein_at_n_out_above_one():
    rng = np.random.default_rng(0)
    off = o.Quirks(wasserstein_per_output=False)
    for n_out in (1, 3):
        z, y = rng.uniform(-1, 1, (4, n_out)), rng.uniform(-1, 1, (4, n_out))
        for loss in o.LOSSES:
            for act in ACTS:
                a, b = o.score_and_grad(loss, act, 0.2, z, y), o.score_and_grad(loss, act, 0.2, z, y, off)
                same = a[0] == b[0] and np.array_equal(a[1], b[1])
                assert same == (loss != "wasserstein" or n_out == 1), (loss, act, n_out)
    s_on, g_on = o.score_and_grad("wasserstein", "identity", 0, z, y)
    s_off, g_off = o.score_and_grad("wasserstein", "identity", 0, z, y, off)
    assert s_off == pytest.approx(3 * s_on) and np.allclose(g_off, 3 * g_on)


def test_loss_layer_runs_the_oracle_gan_step():
    """The DCGAN discriminator ending in LossLayer(hinge): the oracle's gan_step runs on it and reports its losses."""
    from gan_deeplearning4j_b200 import models as m
    size, z, nf, n = 16, 12, 8, 4
    gs, ds = m.dcgan_generator(size, z, nf, 3), m.dcgan_discriminator(size, nf, 3, loss="hinge")
    G = o.net_from_specs(gs, (z,), seed=1); D = o.net_from_specs(ds, (3, size, size), seed=2)
    assert isinstance(D.layers[-1], o.LossLayer) and not isinstance(G.layers[-1], (o.LossLayer, o.Output))
    x, zd, zg, _, _, _ = [a.astype(np.float64) for a in o.synthetic_batch(n, size, 3, z, seed=3)]
    ones = np.ones((n, 1))
    r = o.gan_step(G, D, x, zd, zg, ones, -ones, ones)
    logits = D.layers[-1]._z.reshape(n, 1)                           # the G pass's logits
    assert r["loss_g"] == pytest.approx(np.maximum(0, 1 - logits).sum() / n)
    assert all(np.isfinite(r[k]) for k in ("loss_d_real", "loss_d_fake", "loss_g"))
