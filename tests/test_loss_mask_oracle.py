"""The oracle's weighted / masked losses on the CPU: finite differences for every (loss, activation) pair on OutputLayer,
LossLayer, a CnnLossLayer on an odd map and a conv -> CnnLossLayer net; float64 torch for one-hot MCXENT and for XENT; hand-computed two-row
answers; all-ones weights and mask reproduce the unweighted oracle bit for bit; the refusals; the spec key and a checkpoint round trip."""
import copy

import numpy as np
import pytest

from gan_deeplearning4j_b200 import models as m
from gan_deeplearning4j_b200 import serializer
from oracle import dl4j_oracle as o

ACTS = ("identity", "tanh", "sigmoid", "softplus")
PAIRS = [("xent", "identity"), ("mcxent", "identity")] + [(l, a) for l in ("mse", "l1", "l2", "mae") for a in ACTS] + \
        [(l, a) for l in ("hinge", "squared_hinge", "wasserstein") for a in ("identity", "tanh")]


def _labels(loss, rng, shape, axis=1):
    if loss == "mcxent":
        k = rng.integers(0, shape[axis], np.prod(shape) // shape[axis])
        y = np.moveaxis(np.eye(shape[axis])[k].reshape(tuple(np.delete(shape, axis)) + (shape[axis],)), -1, axis)
        return np.ascontiguousarray(y)
    if loss == "xent":
        return rng.uniform(0, 1, shape)
    if loss in ("hinge", "squared_hinge"):
        return rng.choice([-1.0, 1.0], shape)
    return rng.uniform(-1, 1, shape)


def _weights(loss, rng, c):
    return None if loss in o.DEFAULT_QUIRKS.weightless_losses else rng.uniform(0.2, 2.0, c)


def _masks(loss, rng, rows_shape, full_shape):
    """A 0/1 per-row mask, a fractional per-row one and (not MCXENT) a fractional per-output one."""
    out = [rng.integers(0, 2, rows_shape).astype(np.float64), rng.uniform(0, 1, rows_shape)]
    if loss != "mcxent":
        out.append(rng.uniform(0, 1, full_shape))
    return out


def _fd_check(f, z, g, eps=1e-6, max_rel=1e-3, min_abs=1e-8):
    """GradientCheckUtil: central differences of f at every element of z against g (relative error max_rel, absolute floor min_abs)."""
    zf = z.ravel()
    for i in range(zf.size):
        old = zf[i]
        zf[i] = old + eps; sp = f(z)
        zf[i] = old - eps; sm = f(z)
        zf[i] = old
        num, ana = (sp - sm) / (2 * eps), g.ravel()[i]
        if abs(num - ana) < min_abs:
            continue
        assert abs(num - ana) / max(abs(num), abs(ana)) < max_rel, (i, num, ana)


def _avoid_kinks(loss, z, y, act):
    """L1 / MAE / hinge kinks: keep every element away from them so that central differences are smooth."""
    a = o.forward(act, z, 0.01) if act in o.EXT_ACTS else o.act_forward(act, z, 0.01)
    if loss in ("l1", "mae"):
        return np.all(np.abs(a - y) > 1e-3)
    if loss in ("hinge", "squared_hinge"):
        return np.all(np.abs(1 - y * a) > 1e-3)
    return True


@pytest.mark.parametrize("loss,act", PAIRS)
@pytest.mark.parametrize("kind", ["output", "loss", "cnn_loss"])
def test_finite_differences_on_the_logits(kind, loss, act):
    """dz of the weighted / masked loss against central differences of its score, for every mask kind, on the three loss-bearing layers (the
    CnnLossLayer on an odd 3x5 map)."""
    if kind == "loss" and loss == "mcxent":
        pytest.skip("MCXENT is an OutputLayer / CnnLossLayer loss")
    rng = np.random.default_rng(len(loss) * 7 + len(act) + len(kind))
    c = 1 if loss == "xent" and kind != "cnn_loss" else 3
    n, h, w = 3, 3, 5
    if kind == "cnn_loss":
        layer, zshape = o.CnnLossLayer("cl", loss=loss, activation=act), (n, c, h, w)
        rows_shape, full_shape = (n, 1, h, w), (n, c, h, w)
    else:
        layer = o.LossLayer("l", loss=loss, activation=act) if kind == "loss" else o.Output(4, c, loss=loss, activation=act)
        zshape, rows_shape, full_shape = (n, c), (n, 1), (n, c)
        if loss == "mcxent":
            layer = o.OutputSoftmax(4, c)
    for attempt in range(20):
        z = rng.uniform(-2, 2, zshape); y = _labels(loss, rng, zshape)
        if _avoid_kinks(loss, z, y, act):
            break
    wts = _weights(loss, rng, c)
    for mk in _masks(loss, rng, rows_shape, full_shape) + [None]:
        def score(zz):
            layer._z = zz
            return layer.score_and_eps(y, wts, mk)[0]
        layer._z = z
        _, g = layer.score_and_eps(y, wts, mk)
        _fd_check(score, z.copy(), g)


@pytest.mark.parametrize("loss", ["xent", "mcxent", "mse", "l2"])
def test_finite_differences_conv_to_cnn_loss_net(loss):
    """conv -> conv -> CnnLossLayer on an odd map, weighted and masked: the net's parameter gradients against central
    differences of its score."""
    c = 3
    specs = [{"type": "conv2d", "name": "c1", "n_out": 4, "kernel": (3, 3), "stride": (1, 1), "padding": (1, 1), "activation": "tanh",
              "updater": m.sgd(0.1)},
             {"type": "conv2d", "name": "c2", "n_out": c, "kernel": (1, 1), "stride": (1, 1), "padding": (0, 0), "activation": "identity",
              "updater": m.sgd(0.1)},
             m.cnn_loss(loss, "tanh" if loss in ("mse", "l2") else "identity", name="cl", loss_weights=[0.5, 1.5, 1.0])]
    rng = np.random.default_rng(11)
    net = o.net_from_specs(specs, (2, 3, 5), seed=2, flat_input=False)
    x = rng.uniform(-1, 1, (2, 2, 3, 5)); y = _labels(loss, rng, (2, c, 3, 5))
    mk = rng.uniform(0, 1, (2, 1, 3, 5))
    net.compute_gradient_and_score(x, y, mask=mk)
    g = net.grads_flat().copy()
    p0 = net.params_flat().copy()

    def score(p):
        net.set_params_flat(p)
        return net.compute_gradient_and_score(x, y, mask=mk)
    _fd_check(score, p0.copy(), g / 2)          # the gradient is the minibatch sum; the score its mean
    net.set_params_flat(p0)


def test_mcxent_one_hot_against_torch_cross_entropy():
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(3)
    n, c = 7, 5
    z = rng.uniform(-3, 3, (n, c)); k = rng.integers(0, c, n); y = np.eye(c)[k]
    w = rng.uniform(0.2, 2.0, c); mk = rng.uniform(0, 1, (n, 1))
    zt = torch.tensor(z, requires_grad=True)
    l = torch.nn.functional.cross_entropy(zt, torch.tensor(k), weight=torch.tensor(w), reduction="none")
    (l * torch.tensor(mk[:, 0])).sum().backward()
    s, g = o.rows_score_and_grad("mcxent", None, None, z, y, w, mk)
    assert abs(s - float((l * torch.tensor(mk[:, 0])).sum().detach())) < 1e-12 * max(1, abs(s))
    assert np.allclose(g, zt.grad.numpy(), rtol=1e-12, atol=1e-14)
    # the plain weighted form, reduction="sum"
    zt.grad = None
    torch.nn.functional.cross_entropy(zt, torch.tensor(k), weight=torch.tensor(w), reduction="sum").backward()
    s2, g2 = o.rows_score_and_grad("mcxent", None, None, z, y, w, None)
    assert np.allclose(g2, zt.grad.numpy(), rtol=1e-12, atol=1e-14)


def test_xent_with_logits_against_torch():
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(4)
    z = rng.uniform(-3, 3, (6, 2)); y = rng.uniform(0, 1, (6, 2)); w = np.array([0.3, 1.7]); mk = rng.uniform(0, 1, (6, 2))
    zt = torch.tensor(z, requires_grad=True)
    l = torch.nn.functional.binary_cross_entropy_with_logits(zt, torch.tensor(y), weight=torch.tensor(w[None, :] * mk), reduction="sum")
    l.backward()
    s, g = o.rows_score_and_grad("xent", None, None, z, y, w, mk, o.Quirks(xent_clip_eps=0.0))
    assert abs(s - float(l)) < 1e-12 * abs(s)
    assert np.allclose(g, zt.grad.numpy(), rtol=1e-12, atol=1e-14)


def test_hand_computed_two_rows():
    # MSE, nOut 2, identity: a = z.  Row scores (a - y)^2 / 2 per element, weights (2, 0.5), row mask (1, 0.5).
    z = np.array([[1.0, 2.0], [0.0, -1.0]]); y = np.array([[0.0, 0.0], [1.0, 1.0]])
    w = np.array([2.0, 0.5]); mk = np.array([[1.0], [0.5]])
    s, g = o.rows_score_and_grad("mse", "identity", 0.0, z, y, w, mk)
    # row 0: 2*1 + 0.5*4 = 4; row 1: 0.5 * (2*1 + 0.5*4) = 2; sum 6, / nOut = 3
    assert s == 3.0
    # dz = w m 2 (a - y) / 2
    assert np.array_equal(g, np.array([[2.0, 1.0], [-1.0, -0.5]]))
    # MCXENT, two classes, equal logits: p = 0.5.  Row 0 label class 0, row 1 label class 1; weights (3, 1); row 1 masked out.
    z = np.zeros((2, 2)); y = np.array([[1.0, 0.0], [0.0, 1.0]]); w = np.array([3.0, 1.0]); mk = np.array([[1.0], [0.0]])
    s, g = o.rows_score_and_grad("mcxent", None, None, z, y, w, mk)
    assert abs(s - 3 * np.log(2)) < 1e-15
    # row 0: p * (sum w y = 3) - w y = (1.5 - 3, 1.5 - 0)
    assert np.array_equal(g, np.array([[-1.5, 1.5], [0.0, 0.0]]))


@pytest.mark.parametrize("loss", ["xent", "mcxent", "mse", "l1", "l2", "mae", "hinge", "squared_hinge", "wasserstein"])
def test_all_ones_reproduce_the_oracle_bit_for_bit(loss):
    """All-ones weights (where the loss takes them) and an all-ones mask give the unweighted oracle's score and gradients bit for bit (MCXENT
    on one-hot labels)."""
    specs = [{"type": "conv2d", "name": "c1", "n_out": 3, "kernel": (3, 3), "stride": (1, 1), "padding": (1, 1), "activation": "identity",
              "updater": m.adam(0.01)},
             m.cnn_loss(loss, "identity" if loss in ("xent", "mcxent") else "tanh", name="cl")]
    rng = np.random.default_rng(9)
    x = rng.uniform(-1, 1, (2, 2, 3, 5)); y = _labels(loss, rng, (2, 3, 3, 5))
    ref = o.net_from_specs(specs, (2, 3, 5), seed=2, flat_input=False)
    wspecs = copy.deepcopy(specs)
    if loss not in o.DEFAULT_QUIRKS.weightless_losses:
        wspecs[-1]["loss_weights"] = [1.0, 1.0, 1.0]
    net = o.net_from_specs(wspecs, (2, 3, 5), seed=2, flat_input=False)
    for it in range(2):
        s0 = ref.fit(x, y)
        s1 = net.fit(x, y, mask=np.ones((2, 1, 3, 5)))
        assert s0 == s1, (loss, it)
        assert np.array_equal(ref.params_flat(), net.params_flat()), (loss, it)


def test_refusals():
    with pytest.raises(NotImplementedError):
        o.check_weights("hinge", [1.0], 1)
    with pytest.raises(NotImplementedError):
        o.check_weights("wasserstein", [1.0], 1)
    with pytest.raises(ValueError):
        o.check_weights("mse", [1.0, 2.0], 3)
    with pytest.raises(ValueError):
        o.check_weights("mse", [1.0, np.inf], 2)
    with pytest.raises(NotImplementedError):
        o.check_mask("mcxent", np.ones((4, 3)), 4, 3)
    with pytest.raises(ValueError):
        o.check_mask("mse", np.ones((4, 2)), 4, 3)
    layer = o.CnnLossLayer("cl", loss="xent"); layer._z = np.zeros((2, 3, 3, 5))
    with pytest.raises(ValueError):
        layer.score_and_eps(np.zeros((2, 3, 3, 5)), None, np.ones((2, 2, 3, 5)))
    with pytest.raises(ValueError):
        o.net_from_specs([{"type": "dense", "name": "d", "n_out": 2, "loss_weights": [1, 1]}, m.cnn_loss("xent")], (4,))


def test_spec_key_and_checkpoint_round_trip(tmp_path):
    spec = m.cnn_loss("mcxent", name="cl", loss_weights=np.array([0.5, 2.0]))
    assert spec["loss_weights"] == [0.5, 2.0] and all(type(v) is float for v in spec["loss_weights"])
    assert "loss_weights" not in m.cnn_loss("mcxent")
    specs = [{"type": "dense", "name": "d", "n_out": 2, "updater": m.sgd(0.1)}, spec]
    path = tmp_path / "net.zip"
    serializer.write_model(path, specs, (4,), np.arange(10, dtype=np.float32))
    got = serializer.read_model(path)
    assert got["specs"][-1]["loss_weights"] == [0.5, 2.0]

    class Stub:                       # what restore_into calls on a net
        def __init__(self):
            self.weights = "unset"
        num_params = staticmethod(lambda: 10)
        set_params = staticmethod(lambda p: None)

        def set_loss_weights(self, w):
            self.weights = w
    s = Stub()
    serializer.restore_into(s, path)
    assert s.weights == [0.5, 2.0]
    specs[-1].pop("loss_weights")
    serializer.write_model(path, specs, (4,), np.arange(10, dtype=np.float32))
    serializer.restore_into(s, path)
    assert s.weights is None


def test_gan_step_masks_reach_each_pass():
    """gan_step hands m_real, m_fake and m_gen to the D update's real and fake passes and to the G update, in that order: zero masks on one
    pass zero its loss, masks of ones reproduce the unmasked step bit for bit, and no mask outlives its step."""
    size, z, n = 8, 4, 3
    gs = m.dcgan_generator(size, z, 4, 3, lr=1e-3)
    ds = m.dcgan_discriminator(size, 4, 3, lr=1e-3, patch=True)
    rng = np.random.default_rng(5)
    G = o.net_from_specs(gs, (z,), seed=1); D = o.net_from_specs(ds, (3, size, size), seed=2)
    data = [a.astype(np.float64) for a in o.synthetic_batch(n, size, 3, z, seed=3)]
    D2, G2 = copy.deepcopy(D), copy.deepcopy(G)
    out = o.net_from_specs(ds, (3, size, size), seed=2).output(data[0])
    maps = [np.broadcast_to(v.reshape(n, 1, 1, 1), (n,) + out.shape[1:]).copy() for v in data[3:]]
    ones = np.ones((n, 1) + out.shape[2:])
    r0 = o.gan_step(copy.deepcopy(G), copy.deepcopy(D), *data[:3], *maps)
    r1 = o.gan_step(copy.deepcopy(G2), copy.deepcopy(D2), *data[:3], *maps, m_real=ones, m_fake=ones, m_gen=ones)
    assert (r0["loss_d_real"], r0["loss_d_fake"], r0["loss_g"]) == (r1["loss_d_real"], r1["loss_d_fake"], r1["loss_g"])
    r2 = o.gan_step(G2, D2, *data[:3], *maps, m_real=ones, m_fake=0 * ones, m_gen=ones)
    assert r2["loss_d_fake"] == 0.0 and r2["loss_d_real"] == r0["loss_d_real"] and r2["loss_g"] != 0.0
    assert o.gan_step(G2, D2, *data[:3], *maps)["loss_d_fake"] != 0.0
