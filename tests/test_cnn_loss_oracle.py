"""CnnLossLayer on the CPU: the oracle's CnnLossLayer against finite differences at GradientCheckUtil's tolerances, alone and in
conv -> [BN ->] act -> conv -> CnnLossLayer nets with odd H / W and in the adversarial step; float64 torch; hand-computed answers on a 2x2
map; the 1x1 map against LossLayer; the layer specs, the PatchGAN discriminator builder and the codes shared with the header."""
import copy
import os
import re

import numpy as np
import pytest

from helpers import randomize
from oracle import dl4j_oracle as o

EPS, MAX_REL, MIN_ABS = 1e-6, 1e-3, 1e-8
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# (loss, activation, label kind)
LOSSES = [("xent", "identity", "prob"), ("mcxent", "identity", "onehot"), ("mse", "tanh", "real"), ("l1", "identity", "real"),
          ("hinge", "identity", "sign"), ("wasserstein", "identity", "sign")]


def _labels(kind, rng, shape):
    if kind == "prob":
        return rng.uniform(0.05, 0.95, shape)
    if kind == "onehot":
        n, c, h, w = shape
        return np.moveaxis(np.eye(c)[rng.integers(0, c, (n, h, w))], -1, 1)
    if kind == "sign":
        return rng.choice([-1.0, 1.0], shape)
    return rng.uniform(-1, 1, shape)


def _layer(loss, act):
    l = o.CnnLossLayer("cl", loss=loss, activation=act)
    l.init(None, np.float64)
    return l


@pytest.mark.parametrize("loss,act,kind", LOSSES)
def test_layer_finite_differences(loss, act, kind):
    rng = np.random.default_rng(len(loss))
    z = rng.uniform(-1.5, 1.5, (2, 3, 5, 3))
    z[np.abs(z) < 0.05] = 0.3            # away from the L1 kink
    y = _labels(kind, rng, z.shape)
    lay = _layer(loss, act)

    def score(v):
        lay.forward(v, True)
        return lay.score_and_eps(y)[0]
    lay.forward(z, True)
    _, g = lay.score_and_eps(y)
    for j in rng.choice(z.size, 30, replace=False):
        d = np.zeros_like(z); d.flat[j] = EPS
        num = (score(z + d) - score(z - d)) / (2 * EPS)
        assert abs(num - g.flat[j]) <= MAX_REL * (abs(num) + abs(g.flat[j])) or abs(num - g.flat[j]) <= MIN_ABS, (loss, j, num, g.flat[j])


def _net(n_out, bn, loss, act):
    mid = [{"type": "conv2d", "name": "c1", "n_out": 4, "kernel": (3, 3), "stride": (1, 1), "padding": (1, 1), "has_bias": not bn}]
    if bn:
        mid.append({"type": "batchnorm", "name": "bn1"})
    mid.append({"type": "activation", "name": "a1", "activation": "lrelu", "alpha": 0.2})
    return mid + [{"type": "conv2d", "name": "c2", "n_out": n_out, "kernel": (3, 3), "stride": (2, 2), "padding": (1, 1)},
                  {"type": "cnn_loss", "name": "cl", "loss": loss, **({} if loss in ("xent", "mcxent") else {"activation": act})}]


@pytest.mark.parametrize("bn", [False, True])
@pytest.mark.parametrize("n_out", [1, 2, 3])
@pytest.mark.parametrize("loss,act,kind", LOSSES)
def test_net_finite_differences(loss, act, kind, n_out, bn):
    """conv -> [BN ->] LeakyReLU -> conv(3x3 s2 p1, O = 1..3) -> CnnLossLayer on a 7x5 input (a 4x3 map): parameter gradients."""
    if loss == "mcxent" and n_out == 1:
        pytest.skip("a softmax over one channel is constant")
    specs = _net(n_out, bn, loss, act)
    net = o.net_from_specs(specs, (2, 7, 5), seed=4, flat_input=False)
    rng = np.random.default_rng(n_out * 7 + bn)
    randomize(net, rng)
    x = rng.uniform(-1, 1, (3, 2, 7, 5))
    y = _labels(kind, rng, (3, n_out, 4, 3))
    p0 = net.params_flat().copy()
    net.compute_gradient_and_score(x, y)
    grads = net.grads_flat().copy()
    score = lambda q: (net.set_params_flat(q), net.compute_gradient_and_score(x, y))[1] * x.shape[0]
    # the BatchNorm running mean / var carry pseudo-gradients, not derivatives of the train-mode score
    trained = np.concatenate([np.full(int(np.prod(sh)), p not in net.layers[li].noop_names()) for li, _, p, sh, _ in net.param_table()])
    for j in np.random.default_rng(6).choice(np.flatnonzero(trained), 16, replace=False):
        d = np.zeros_like(p0); d[j] = EPS
        num = (score(p0 + d) - score(p0 - d)) / (2 * EPS)
        assert abs(num - grads[j]) <= MAX_REL * (abs(num) + abs(grads[j])) or abs(num - grads[j]) <= 1e-6, (loss, n_out, bn, j, num, grads[j])
    net.set_params_flat(p0)


def _patch_gan(loss="xent"):
    from gan_deeplearning4j_b200 import models as m
    size, z, nf = 16, 6, 4
    gs = m.dcgan_generator(size, z, nf, 3, lr=1e-2)
    ds = m.dcgan_discriminator(size, nf, 3, lr=1e-2, loss=loss, patch=True)
    G = o.net_from_specs(gs, (z,), seed=1); D = o.net_from_specs(ds, (3, size, size), seed=2)
    rng = np.random.default_rng(5)
    randomize(G, rng); randomize(D, rng)
    return G, D, z, size


def test_gan_step_generator_gradient_finite_differences():
    """The G step of the adversarial step through a patch D: the generator's gradient of (sum of patch scores) against finite differences of
    that sum in G's parameters (D untouched, both in train mode as in the step)."""
    G, D, z, size = _patch_gan()
    n = 3
    rng = np.random.default_rng(9)
    zg = rng.uniform(-1, 1, (n, z)); y = np.ones((n, 1, 4, 4))

    def loss_of(Gp):
        return D.layers[-1].score_and_eps((D.forward(Gp.forward(zg, train=True), train=True), y)[1])[0]
    G0, D0 = copy.deepcopy(G), copy.deepcopy(D)
    xg = G.forward(zg, train=True); D.forward(xg, train=True)
    _, eps = D.layers[-1].score_and_eps(y)
    eps = D.backward_from_prefix(eps).reshape(xg.shape)
    for l in reversed(G.layers):
        eps = l.backward(eps)
    grads = G.grads_flat().copy()
    p0 = G0.params_flat().copy()
    for j in np.random.default_rng(3).choice(p0.size, 12, replace=False):
        Gp, Gm = copy.deepcopy(G0), copy.deepcopy(G0)
        d = np.zeros_like(p0); d[j] = EPS
        Gp.set_params_flat(p0 + d); Gm.set_params_flat(p0 - d)
        D.__dict__.update(copy.deepcopy(D0).__dict__)
        num = (loss_of(Gp) - loss_of(Gm)) / (2 * EPS)
        assert abs(num - grads[j]) <= MAX_REL * (abs(num) + abs(grads[j])) or abs(num - grads[j]) <= 1e-6, (j, num, grads[j])


def test_gan_step_with_a_patch_discriminator_broadcast_labels():
    """gan_step with per-pixel label maps equal to the per-image value everywhere gives the per-image sums: loss = row scores / N."""
    G, D, z, size = _patch_gan("mse")
    data = list(o.synthetic_batch(4, size, 3, z, seed=3))
    maps = [np.broadcast_to(v.reshape(4, 1, 1, 1), (4, 1, 4, 4)).astype(np.float64) for v in data[3:]]
    r = o.gan_step(G, D, *[v.astype(np.float64) for v in data[:3]], *maps)
    assert np.isfinite([r["loss_d_real"], r["loss_d_fake"], r["loss_g"]]).all()
    # the G loss is the MSE over the 16 patches (1 channel: / C = 1) summed per image, / N
    assert r["loss_g"] > 0


def test_torch_agrees():
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(1)
    z = rng.uniform(-2, 2, (3, 4, 5, 3))
    for loss, act, kind in (("xent", "identity", "prob"), ("mcxent", "identity", "onehot"), ("mse", "identity", "real")):
        y = _labels(kind, rng, z.shape)
        lay = _layer(loss, act); lay.q = o.Quirks(xent_clip_eps=0.0)
        lay.forward(z, True); s, g = lay.score_and_eps(y)
        zt = torch.tensor(z, requires_grad=True); yt = torch.tensor(y)
        if loss == "xent":
            ref = torch.nn.functional.binary_cross_entropy_with_logits(zt, yt, reduction="sum") / 3
        elif loss == "mcxent":
            ref = torch.nn.functional.cross_entropy(zt, yt.argmax(1), reduction="sum") / 3
        else:
            ref = ((zt - yt) ** 2).sum() / (4 * 3)
        ref.backward()
        assert abs(s / 3 - ref.item()) <= 1e-9 * max(1, abs(ref.item())), (loss, s / 3, ref.item())
        assert np.allclose(g / 3, zt.grad.numpy(), rtol=1e-8, atol=1e-12), loss


def test_hand_computed_2x2():
    """N = 1, C = 2, a 2x2 map of zeros: sigmoid 1/2 everywhere, softmax 1/2 per channel."""
    z = np.zeros((1, 2, 2, 2))
    y = np.zeros((1, 2, 2, 2)); y[0, 0] = 1.0           # channel 0 labelled at every pixel
    lay = _layer("xent", "identity"); lay.q = o.Quirks(xent_clip_eps=0.0)
    lay.forward(z, True); s, g = lay.score_and_eps(y)
    assert np.isclose(s, 8 * np.log(2))                 # 8 elements, each log 2
    assert np.allclose(g, 0.5 - y)
    lay = _layer("mcxent", "identity"); lay.forward(z, True); s, g = lay.score_and_eps(y)
    assert np.isclose(s, 4 * np.log(2)) and np.allclose(g, 0.5 - y)       # 4 pixels, each -log 1/2
    lay = _layer("mse", "identity"); lay.forward(z, True); s, g = lay.score_and_eps(y)
    assert np.isclose(s, 4 * 1 / 2) and np.allclose(g, (0 - y) * 2 / 2)    # per pixel (1^2 + 0^2) / C
    lay = o.CnnLossLayer("cl", o.Quirks(cnn_loss_score_per_minibatch=False), loss="mse"); lay.init(None, np.float64)
    lay.forward(z, True); s2, g2 = lay.score_and_eps(y)
    assert np.isclose(s2, s / 4) and np.allclose(g2, g / 4)


@pytest.mark.parametrize("loss,act,kind", [l for l in LOSSES if l[0] != "mcxent"])
def test_1x1_map_equals_loss_layer(loss, act, kind):
    rng = np.random.default_rng(2)
    z = rng.uniform(-1, 1, (5, 3, 1, 1)) if loss != "xent" else rng.uniform(-1, 1, (5, 1, 1, 1))
    y = _labels(kind, rng, z.shape)
    a = _layer(loss, act); b = o.LossLayer("l", loss=loss, activation=act)
    fa, fb = a.forward(z, True), b.forward(z, True)
    assert np.array_equal(fa, fb)
    sa, ga = a.score_and_eps(y); sb, gb = b.score_and_eps(y.reshape(5, -1))
    assert sa == sb and np.array_equal(ga, gb)


def test_rows_are_the_nhwc_buffer():
    a = np.arange(2 * 3 * 2 * 2).reshape(2, 3, 2, 2)
    assert np.array_equal(o.to_rows(a).ravel(), a.transpose(0, 2, 3, 1).ravel())


# ------------------------------------------------------------------ specs ------------------------------------------------------------
def test_codes_match_the_header():
    from gan_deeplearning4j_b200 import engine
    h = open(os.path.join(ROOT, "include", "b200gan.h")).read()
    assert int(re.search(r"B2G_LAYER_CNN_LOSS\s*=\s*(\d+)", h).group(1)) == engine.LAYER_TYPES["cnn_loss"] == 14
    assert int(re.search(r"B2G_EW_CNN_XENT\s*=\s*(\d+)", h).group(1)) == engine.EW_OPS["cnn_xent"] == 13
    assert int(re.search(r"B2G_EW_CNN_SOFTMAX_XENT\s*=\s*(\d+)", h).group(1)) == engine.EW_OPS["cnn_softmax_xent"] == 14
    java = open(os.path.join(ROOT, "java/src/main/java/org/deeplearning4j/nn/conf/layers/CnnLossLayer.java")).read()
    assert re.search(r"TYPE\s*=\s*14", java)


def test_cnn_loss_descs():
    from gan_deeplearning4j_b200 import engine, models as m
    d = engine.layer_desc(m.cnn_loss("mse", "tanh", name="seg"))
    assert (d.type, d.loss, d.act, d.name) == (14, 2, 1, b"seg")
    d = engine.layer_desc(m.cnn_loss("mcxent"))
    assert (d.type, d.loss, d.act) == (14, 1, 0)
    with pytest.raises(ValueError):
        m.cnn_loss("xent", "tanh")
    with pytest.raises(ValueError):
        m.cnn_loss("poisson")


@pytest.mark.parametrize("size,side", [(16, 4), (32, 4), (64, 4), (128, 8)])
def test_patch_discriminator_shapes_and_parameter_counts(size, side):
    from gan_deeplearning4j_b200 import models as m
    nf = 8
    full, patch = m.dcgan_discriminator(size, nf, 3), m.dcgan_discriminator(size, nf, 3, patch=True)
    assert full[:len(patch) - 2] == patch[:-2]
    assert patch[-2]["kernel"] == (3, 3) and patch[-2]["padding"] == (1, 1) and patch[-2]["n_out"] == 1 and patch[-1]["type"] == "cnn_loss"
    D = o.net_from_specs(patch, (3, size, size), flat_input=False)
    out = D.forward(np.zeros((2, 3, size, size)), train=False)
    assert out.shape == (2, 1, side, side)
    ch = patch[-2]["n_in"]
    assert D.num_params() == o.net_from_specs(patch[:-2], (3, size, size), flat_input=False).num_params() + 9 * ch + 1
    if size <= 64:                     # the same trunk as today's head: the 4x4 valid conv (16 ch + 1) becomes the 3x3 one
        assert D.num_params() == o.net_from_specs(full, (3, size, size), flat_input=False).num_params() - 16 * ch + 9 * ch
    with pytest.raises(ValueError):
        m.dcgan_discriminator(size, nf, 3, patch=True, global_pooling="sum")


def test_cnn_loss_must_be_last():
    with pytest.raises(ValueError):
        o.net_from_specs([{"type": "cnn_loss", "name": "a"}, {"type": "cnn_loss", "name": "b"}], (1, 2, 2), flat_input=False)
