"""Pins for the CPU oracle (oracle/dl4j_oracle.py).

The reference holds no golden vectors (parity unpinned, SURVEY.md 8c), so the oracle is pinned by:
  (i)   finite differences with DL4J's own GradientCheckUtil tolerances (eps 1e-6, maxRelError 1e-3,
        minAbsError 1e-8 -- the upstream CNNGradientCheckTest/BNGradientCheckTest settings),
  (ii)  an independent torch.autograd (fp64) cross-check of every op and of the whole DCGAN step,
  (iii) hand-computed known-answer cases for the DL4J-specific quirks,
  (iv)  the parameter counts and flatten orders of the reference's own graphs (J:118-310).
"""
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import pack_deconv_ps, randomize
from oracle import dl4j_oracle as o


def fd_check(net, x, y, eps=1e-6, max_rel=1e-3, min_abs=1e-8, n_probe=60, seed=0, **kw):
    """kw: passed to compute_gradient_and_score (pass_ pins the DropoutLayer masks)."""
    net.compute_gradient_and_score(x, y, **kw)
    mb = x.shape[0]
    g = net.grads_flat() / mb
    # the regularization contributes l2 theta + l1 sign(theta) to d(score)/dtheta; added analytically (DL4J's check includes it via the score)
    p0 = net.params_flat().copy()
    rng = np.random.default_rng(seed)
    table = net.param_table()
    # skip BN mean/var slots (pseudo-gradients are not derivatives)
    mask = np.ones_like(p0, bool)
    l1, l2 = np.zeros_like(p0), np.zeros_like(p0)
    off = 0
    for li, _, p, shape, _ in table:
        n = int(np.prod(shape))
        if p in net.layers[li].noop_names():
            mask[off:off + n] = False
        l1[off:off + n], l2[off:off + n] = net.reg_coefs(net.layers[li], p)
        off += n
    idx = rng.choice(np.flatnonzero(mask), size=min(n_probe, mask.sum()), replace=False)
    worst = 0.0
    for i in idx:
        pp = p0.copy(); pp[i] += eps; net.set_params_flat(pp); sp = net.compute_gradient_and_score(x, y, **kw)
        pm = p0.copy(); pm[i] -= eps; net.set_params_flat(pm); sm = net.compute_gradient_and_score(x, y, **kw)
        num = (sp - sm) / (2 * eps)
        ana = g[i] + l2[i] * p0[i] + l1[i] * np.sign(p0[i])
        if abs(num - ana) < min_abs:
            continue
        rel = abs(num - ana) / (abs(num) + abs(ana))
        worst = max(worst, rel)
        assert rel < max_rel, (i, num, ana, rel)
    net.set_params_flat(p0)
    return worst


def small_cnn(act="tanh"):
    u = o.Sgd(0.1)
    L = [o.BatchNorm(2, updater=u, name="bn0"),
         o.Conv2D(2, 4, (3, 3), (2, 2), (1, 1), act, 0.2, updater=u, l2=1e-3, name="c1"),
         o.MaxPool((2, 2), (1, 1), name="mp"),
         o.Upsample2D(2, name="up"),
         o.Deconv2D(4, 3, (4, 4), (2, 2), (1, 1), "identity", updater=u, name="d1"),
         o.BatchNorm(3, updater=u, name="bn1"), o.ActivationLayer(act, 0.2, name="a1"),
         o.Conv2D(3, 2, (5, 5), (1, 1), (2, 2), "sigmoid", updater=u, name="c2"),
         o.Reshape((2 * 12 * 12,), name="flat"),
         o.Dense(288, 5, act, 0.2, updater=u, l2=1e-3, name="fc"),
         o.Output(5, 1, updater=u, name="out")]
    return o.Net(L, seed=3)


@pytest.mark.parametrize("act", ["tanh", "lrelu", "relu", "sigmoid"])
def test_finite_differences_every_layer(act):
    net = small_cnn(act)
    rng = np.random.default_rng(1)
    x = rng.uniform(-1, 1, (5, 2, 7, 7))
    y = rng.uniform(-0.1, 1.1, (5, 1))
    # perturb BN affine so the checks are not at the gamma=1/beta=0 special point
    for l in net.layers:
        if isinstance(l, o.BatchNorm):
            l.params["gamma"] = rng.uniform(0.5, 1.5, l.n)
            l.params["beta"] = rng.uniform(-0.5, 0.5, l.n)
    fd_check(net, x, y)


def test_finite_differences_of_a_net_composing_the_later_features():
    """One net_from_specs net mixing an ELU conv, AVG subsampling with padding, a DropoutLayer (pinned to one pass), AdaGrad / Nesterovs on a
    step schedule and an MSE output on Softsign: GradientCheckUtil's tolerances, then two fits through the one update pipeline."""
    from gan_deeplearning4j_b200 import models as m
    sched = m.step_schedule(0.05, 0.5, 1)
    specs = [{"type": "conv2d", "name": "c1", "n_out": 4, "kernel": (3, 3), "padding": (1, 1), "activation": "elu", "updater": m.adagrad(sched), "l2": 1e-3},
             {"type": "subsampling", "name": "s", "pooling": "avg", "kernel": (2, 2), "stride": (2, 2), "padding": (1, 1)},
             {"type": "cnn_to_ff", "name": "ff"},
             {"type": "dropout", "name": "drop", "p": 0.7},
             {"type": "dense", "name": "d1", "n_out": 6, "activation": "swish", "updater": m.nesterovs(sched, 0.9)},
             {"type": "output", "name": "out", "n_out": 3, "loss": "mse", "activation": "softsign", "updater": m.adam(1e-2)}]
    net = o.net_from_specs(specs, (2, 5, 5), seed=4, flat_input=False)
    rng = np.random.default_rng(7)
    randomize(net, rng)
    x, y = rng.uniform(-1, 1, (4, 2, 5, 5)), rng.uniform(-1, 1, (4, 3))
    fd_check(net, x, y, pass_=0)
    assert net.dropout_pass() == 0 and net.layers[3].index == 3
    p0 = net.params_flat().copy()
    net.fit(x, y); net.fit(x, y)
    assert net.iteration == 2 and net.dropout_pass() == 2
    assert net.learning_rate("c1") == net.learning_rate("d1") == np.float32(0.0125) and net.learning_rate("out") == 1e-2
    assert len(net.state[(0, "W")]) == 1 and np.all(np.isfinite(net.params_flat())) and not np.any(net.params_flat() == p0)


def test_one_spec_list_mixes_regularization_weight_noise_prelu_scheduled_noise_and_masks():
    """A conv with l1 / l1Bias / l2Bias and additive WeightNoise -> PReLU on shared axes -> scheduled GaussianDropout -> a weighted MCXENT
    output with a labels mask, from one spec list: GradientCheckUtil's tolerances with every draw pinned to one pass (the conv's parameters
    away from l1's kink), and one masked GAN step with it as D moves D's pass counter by two."""
    from gan_deeplearning4j_b200 import models as m
    specs = [{"type": "conv2d", "name": "c", "n_out": 3, "kernel": (3, 3), "padding": (1, 1), "activation": "tanh", "updater": m.sgd(0.1),
              "l1": 1e-2, "l1_bias": 2e-2, "l2_bias": 3e-2, "weight_noise": m.weight_noise(m.normal(0.0, 0.05), apply_to_bias=True)},
             dict(m.prelu((2, 3), "p"), updater=m.sgd(0.1), l1=1e-2, l2=2e-2),
             m.gaussian_dropout(m.exponential_schedule(0.3, 0.5), "gd"),
             {"type": "cnn_to_ff", "name": "f"},
             {"type": "output", "name": "out", "n_out": 3, "loss": "mcxent", "updater": m.sgd(0.1), "loss_weights": [0.5, 1.0, 2.0]}]
    D = o.net_from_specs(specs, (2, 5, 5), seed=4, mask_seed=9)
    rng = np.random.default_rng(8)
    for l in D.layers:
        for p, shape, _ in l.param_specs():
            v = rng.uniform(-0.5, 0.5, shape)
            l.params[p] = v + 0.05 * np.sign(v)
    assert [type(l) for l in D.layers[1:4]] == [o.Conv2D, o.PReLU, o.Dropout] and D.layers[1].weight_noise and D.loss_weights is not None
    n = 4
    x, y = rng.uniform(-1, 1, (n, 2, 5, 5)), np.eye(3)[rng.integers(0, 3, n)]
    mask = rng.uniform(0.2, 1.0, (n, 1))
    fd_check(D, x, y, n_probe=80, pass_=3, mask=mask)
    assert D.dropout_pass() == 0
    G = o.net_from_specs([{"type": "dense", "name": "g", "n_out": 50, "activation": "tanh", "updater": m.sgd(0.1)}], (6,), seed=5)
    D.set_dropout_pass(5)
    masks = [rng.uniform(0.2, 1.0, (n, 1)) for _ in range(3)]
    r = o.gan_step(G, D, x, *rng.uniform(-1, 1, (2, n, 6)), y, y[::-1], y, m_real=masks[0], m_fake=masks[1], m_gen=masks[2])
    assert np.isfinite([r["loss_d_real"], r["loss_d_fake"], r["loss_g"]]).all() and D.dropout_pass() == 7


def test_finite_differences_dcgan_tiny():
    G = o.dcgan_generator(size=16, z=6, nf=4, nc=3)
    D = o.dcgan_discriminator(size=16, nf=4, nc=3)
    rng = np.random.default_rng(2)
    z = rng.uniform(-1, 1, (4, 6))
    y = np.ones((4, 1))
    stacked = o.Net(G.layers + D.layers, seed=0)
    stacked.layers = G.layers + D.layers
    fd_check(stacked, z, y, n_probe=80)


# ------------------------------------------------------------------------------------------------
# torch cross-checks (independent implementation: conv2d/conv_transpose2d/batch_norm/BCE + autograd)
# ------------------------------------------------------------------------------------------------
def test_conv_matches_torch():
    rng = np.random.default_rng(0)
    l = o.Conv2D(3, 5, (4, 4), (2, 2), (1, 1), "lrelu", 0.2, name="c"); l.init(rng, np.float64)
    l.params["b"] = rng.standard_normal(5)
    x = rng.standard_normal((2, 3, 8, 8)); eps = rng.standard_normal((2, 5, 4, 4))
    a = l.forward(x, True); dx = l.backward(eps)
    xt = torch.tensor(x, requires_grad=True); wt = torch.tensor(l.params["W"], requires_grad=True); bt = torch.tensor(l.params["b"], requires_grad=True)
    at = F.leaky_relu(F.conv2d(xt, wt, bt, 2, 1), 0.2); at.backward(torch.tensor(eps))
    np.testing.assert_allclose(a, at.detach().numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(dx, xt.grad.numpy(), rtol=1e-11, atol=1e-12)
    np.testing.assert_allclose(l.grads["W"], wt.grad.numpy(), rtol=1e-11, atol=1e-12)
    np.testing.assert_allclose(l.grads["b"], bt.grad.numpy(), rtol=1e-11, atol=1e-12)


@pytest.mark.parametrize("k,s,p,h", [(4, 2, 1, 5), (4, 1, 0, 1), (5, 2, 2, 4), (3, 1, 1, 6)])
def test_deconv_matches_torch(k, s, p, h):
    rng = np.random.default_rng(0)
    l = o.Deconv2D(3, 4, (k, k), (s, s), (p, p), "tanh", name="d"); l.init(rng, np.float64)
    l.params["b"] = rng.standard_normal(4)
    x = rng.standard_normal((2, 3, h, h))
    a = l.forward(x, True)
    eps = rng.standard_normal(a.shape); dx = l.backward(eps)
    xt = torch.tensor(x, requires_grad=True); wt = torch.tensor(l.params["W"], requires_grad=True); bt = torch.tensor(l.params["b"], requires_grad=True)
    at = torch.tanh(F.conv_transpose2d(xt, wt, bt, s, p)); at.backward(torch.tensor(eps))
    assert a.shape == tuple(at.shape) == (2, 4, s * (h - 1) + k - 2 * p, s * (h - 1) + k - 2 * p)
    np.testing.assert_allclose(a, at.detach().numpy(), rtol=1e-11, atol=1e-12)
    np.testing.assert_allclose(dx, xt.grad.numpy(), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(l.grads["W"], wt.grad.numpy(), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(l.grads["b"], bt.grad.numpy(), rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("shape", [(6, 3, 4, 4), (7, 5)])
def test_batchnorm_matches_torch_and_dl4j_running_stats(shape):
    rng = np.random.default_rng(0)
    c = shape[1]
    l = o.BatchNorm(c, updater=o.Sgd(0.0), name="bn"); net = o.Net([l], seed=0)
    l.params["gamma"] = rng.uniform(0.5, 1.5, c); l.params["beta"] = rng.standard_normal(c)
    x = rng.standard_normal(shape) * 2 + 1; eps = rng.standard_normal(shape)
    y = l.forward(x, True); dx = l.backward(eps)
    xt = torch.tensor(x, requires_grad=True); g = torch.tensor(l.params["gamma"], requires_grad=True); b = torch.tensor(l.params["beta"], requires_grad=True)
    yt = F.batch_norm(xt, None, None, g, b, training=True, eps=1e-5); yt.backward(torch.tensor(eps))
    np.testing.assert_allclose(y, yt.detach().numpy(), rtol=1e-11, atol=1e-12)
    np.testing.assert_allclose(dx, xt.grad.numpy(), rtol=1e-9, atol=1e-11)
    np.testing.assert_allclose(l.grads["gamma"], g.grad.numpy(), rtol=1e-10)
    np.testing.assert_allclose(l.grads["beta"], b.grad.numpy(), rtol=1e-10)
    # DL4J: running var is the BIASED batch variance (torch uses the unbiased one)
    axes = (0, 2, 3) if len(shape) == 4 else (0,)
    mean0, var0 = l.params["mean"].copy(), l.params["var"].copy()
    net.apply_update(shape[0])
    np.testing.assert_allclose(l.params["mean"], 0.9 * mean0 + 0.1 * x.mean(axes), rtol=1e-12)
    np.testing.assert_allclose(l.params["var"], 0.9 * var0 + 0.1 * x.var(axes), rtol=1e-12)
    # inference uses the stored mean/var
    yi = l.forward(x, False)
    bc = (lambda v: v[None, :, None, None]) if len(shape) == 4 else (lambda v: v[None, :])
    np.testing.assert_allclose(yi, bc(l.params["gamma"]) * (x - bc(l.params["mean"])) / np.sqrt(bc(l.params["var"]) + 1e-5) + bc(l.params["beta"]), rtol=1e-12)


def test_maxpool_upsample_match_torch():
    rng = np.random.default_rng(0)
    x = rng.standard_normal((2, 3, 6, 6))
    mp = o.MaxPool((2, 2), (1, 1)); y = mp.forward(x, True)
    eps = rng.standard_normal(y.shape); dx = mp.backward(eps)
    xt = torch.tensor(x, requires_grad=True); yt = F.max_pool2d(xt, 2, 1); yt.backward(torch.tensor(eps))
    np.testing.assert_allclose(y, yt.detach().numpy()); np.testing.assert_allclose(dx, xt.grad.numpy())
    up = o.Upsample2D(2); y = up.forward(x, True); eps = rng.standard_normal(y.shape); dx = up.backward(eps)
    xt = torch.tensor(x, requires_grad=True); yt = F.interpolate(xt, scale_factor=2, mode="nearest"); yt.backward(torch.tensor(eps))
    np.testing.assert_allclose(y, yt.detach().numpy()); np.testing.assert_allclose(dx, xt.grad.numpy())


def test_maxpool_tie_goes_to_first_in_window():
    x = np.zeros((1, 1, 2, 2)); mp = o.MaxPool((2, 2), (1, 1)); mp.forward(x, True)
    dx = mp.backward(np.ones((1, 1, 1, 1)))
    assert dx[0, 0].tolist() == [[1.0, 0.0], [0.0, 0.0]]


def _torch_dcgan(G, D):
    """Rebuild the oracle's DCGAN nets as plain torch functions over the same parameter arrays."""
    def run(net, x, params):
        a = x
        for li, l in enumerate(net.layers):
            if isinstance(l, o.Reshape):
                a = a.reshape((a.shape[0],) + l.to_shape)
            elif isinstance(l, o.Deconv2D):
                a = F.conv_transpose2d(a, params[(id(net), li, "W")], params.get((id(net), li, "b")), l.s, l.p)
                a = torch.tanh(a) if l.activation == "tanh" else a
            elif isinstance(l, o.Conv2D):
                a = F.conv2d(a, params[(id(net), li, "W")], params.get((id(net), li, "b")), l.s, l.p)
                a = F.leaky_relu(a, l.alpha) if l.activation == "lrelu" else a
            elif isinstance(l, o.BatchNorm):
                a = F.batch_norm(a, None, None, params[(id(net), li, "gamma")], params[(id(net), li, "beta")], True, eps=l.eps)
            elif isinstance(l, o.ActivationLayer):
                a = F.relu(a) if l.activation == "relu" else F.leaky_relu(a, l.alpha)
            elif isinstance(l, o.LossLayer):
                pass
        return a
    params = {}
    for net in (G, D):
        for li, l in enumerate(net.layers):
            if l.has_params:
                for p, _, _ in l.param_specs():
                    if p not in ("mean", "var"):
                        params[(id(net), li, p)] = torch.tensor(l.params[p], requires_grad=True)
    return run, params


def test_dcgan_step_gradients_match_torch_autograd():
    q = o.Quirks(xent_clip_eps=0.0)
    G = o.dcgan_generator(size=16, z=8, nf=4, quirks=q); D = o.dcgan_discriminator(size=16, nf=4, quirks=q)
    x, z_d, z_g, y_r, y_f, y_g = [a.astype(np.float64) for a in o.synthetic_batch(6, 16, 3, 8)]
    run, P = _torch_dcgan(G, D)
    # D gradients, real and fake minibatches separately (separate BN batch statistics)
    xf = G.forward(z_d, True)
    zr = run(D, torch.tensor(x), P).reshape(-1, 1); zf = run(D, torch.tensor(xf), P).reshape(-1, 1)
    loss = F.binary_cross_entropy_with_logits(zr, torch.tensor(y_r), reduction="sum") + F.binary_cross_entropy_with_logits(zf, torch.tensor(y_f), reduction="sum")
    loss.backward()
    D.compute_gradient_and_score(x, y_r); g1 = {(li, p): l.grads[p].copy() for li, l in enumerate(D.layers) if l.has_params for p in l.grads}
    D.compute_gradient_and_score(xf, y_f)
    for li, l in enumerate(D.layers):
        if l.has_params:
            for p, _, _ in l.param_specs():
                if p in ("mean", "var"):
                    continue
                np.testing.assert_allclose(g1[(li, p)] + l.grads[p], P[(id(D), li, p)].grad.numpy(), rtol=1e-8, atol=1e-10)
    # G gradients through D
    for v in P.values():
        v.grad = None
    out = run(D, run(G, torch.tensor(z_g), P), P).reshape(-1, 1)
    F.binary_cross_entropy_with_logits(out, torch.tensor(y_g), reduction="sum").backward()
    Gc, Dc = copy.deepcopy(G), copy.deepcopy(D)
    for l in Gc.layers:
        if l.updater is not None:
            l.updater = o.Sgd(1.0)     # so that params_before - params_after = grad / mb
    for l in Dc.layers:
        if l.updater is not None:
            l.updater = o.Sgd(0.0)     # D weights stay put, so torch's G gradient sees the same D
    before = {(li, p): l.params[p].copy() for li, l in enumerate(Gc.layers) if l.has_params for p, _, _ in l.param_specs()}
    dbefore = Dc.params_flat().copy()
    r = o.gan_step(Gc, Dc, x, z_d, z_g, y_r, y_f, y_g)
    for li, l in enumerate(Gc.layers):
        if l.has_params:
            for p, _, _ in l.param_specs():
                if p in ("mean", "var"):
                    continue
                np.testing.assert_allclose((before[(li, p)] - l.params[p]) * 6, P[(id(G), li, p)].grad.numpy(), rtol=1e-6, atol=1e-9)
    assert np.isfinite(r["loss_g"])
    changed = np.flatnonzero(dbefore != Dc.params_flat())      # only BN running stats moved (NoOp pseudo-gradients)
    table = [(n, p) for li, n, p, sh, _ in Dc.param_table() for _ in range(int(np.prod(sh)))]
    assert len(changed) > 0 and all(table[i][1] in ("mean", "var") for i in changed)


# ------------------------------------------------------------------------------------------------
# Known-answer cases for the DL4J-specific behaviour
# ------------------------------------------------------------------------------------------------
def test_kat_conv_1x1x3x3():
    l = o.Conv2D(1, 1, (2, 2), (1, 1), (0, 0), "identity"); l.init(np.random.default_rng(0), np.float64)
    l.params["W"] = np.array([[[[1., 2.], [3., 4.]]]]); l.params["b"] = np.array([0.5])
    x = np.arange(9.).reshape(1, 1, 3, 3)
    y = l.forward(x, True)
    # cross-correlation (no flip): y[0,0] = 0*1+1*2+3*3+4*4 + .5 = 27.5
    assert y[0, 0].tolist() == [[27.5, 37.5], [57.5, 67.5]]


def test_kat_batchnorm_two_samples():
    l = o.BatchNorm(1); l.init(np.random.default_rng(0), np.float64)
    y = l.forward(np.array([[1.0], [3.0]]), True)          # mu=2, biased var=1
    np.testing.assert_allclose(y[:, 0], [-1 / np.sqrt(1 + 1e-5), 1 / np.sqrt(1 + 1e-5)], rtol=1e-14)


def test_kat_rmsprop_reference_settings_is_sign_sgd():
    # RmsProp(lr, 1e-8, 1e-8): the reference passes rmsDecay=1e-8 (J:133) => cache ~ g^2 => update ~ lr*sign(g)
    l = o.Dense(1, 1, updater=o.RmsProp(0.002, 1e-8, 1e-8), has_bias=False)
    net = o.Net([l]); l.params["W"] = np.array([[1.0]]); l.grads["W"] = np.array([[3.0]])
    c0 = net.state[(0, "W")][0].copy(); assert c0[0, 0] == 1e-8      # cache initialised to epsilon
    net.apply_update(1)
    c = 1e-8 * 1e-8 + (1 - 1e-8) * 9.0
    np.testing.assert_allclose(l.params["W"], [[1.0 - 0.002 * 3.0 / (np.sqrt(c) + 1e-8)]], rtol=1e-15)
    assert abs((1.0 - l.params["W"][0, 0]) - 0.002) < 1e-9


def test_kat_adam_dl4j_form():
    l = o.Dense(1, 1, updater=o.Adam(1e-3, 0.9, 0.999, 1e-8), has_bias=False)
    net = o.Net([l]); l.params["W"] = np.array([[0.0]]); l.grads["W"] = np.array([[2.0]])
    net.apply_update(1)
    m, v = 0.2, 0.004
    alpha = 1e-3 * np.sqrt(1 - 0.999) / (1 - 0.9)
    np.testing.assert_allclose(l.params["W"], [[-alpha * m / (np.sqrt(v) + 1e-8)]], rtol=1e-14)


def test_kat_update_order_divide_clip_updater_l2():
    l = o.Dense(1, 1, updater=o.Sgd(0.5), l2=0.1, has_bias=False)
    net = o.Net([l], grad_clip=1.0); l.params["W"] = np.array([[2.0]]); l.grads["W"] = np.array([[30.0]])
    net.apply_update(10)      # 30/10 = 3 -> clip 1 -> 0.5*1 -> +0.1*2 (not lr-scaled) => W = 2 - 0.7
    np.testing.assert_allclose(l.params["W"], [[1.3]], rtol=1e-15)
    # "frozen" = lr 0 still decays the weights (SURVEY.md 8a row a9)
    l.updater = o.Sgd(0.0); l.grads["W"] = np.array([[30.0]]); net.apply_update(10)
    np.testing.assert_allclose(l.params["W"], [[1.3 - 0.13]], rtol=1e-15)


def test_kat_xent_clip_at_saturated_logits():
    z = np.array([[40.0], [-40.0], [0.0]]); y = np.array([[0.0], [1.0], [1.0]])
    s, g = o.xent_score_and_grad(z, y, 1e-5)
    np.testing.assert_allclose(s, -2 * np.log(1e-5) - np.log(0.5), rtol=1e-12)
    assert abs(g[2, 0] - (-0.5)) < 1e-15
    s2, g2 = o.xent_score_and_grad(z, y, 0.0)                    # BCE-with-logits: no clip
    np.testing.assert_allclose(s2, 40 + 40 + np.log(2), rtol=1e-12)
    np.testing.assert_allclose(g2[:, 0], [1.0, -1.0, -0.5], atol=1e-15)
    # soft labels outside [0,1] (J:405-421) are accepted
    s3, g3 = o.xent_score_and_grad(np.array([[0.3]]), np.array([[1.07]]), 0.0)
    assert abs(g3[0, 0] - (1 / (1 + np.exp(-0.3)) - 1.07)) < 1e-15


def test_reference_graph_parameter_counts_and_flatten_order():
    d = o.reference_discriminator(); g = o.reference_generator(); gan, ng = o.reference_gan()
    assert (d.num_params(), g.num_params(), gan.num_params()) == (1388293, 6663433, 8051726)   # SURVEY.md App. A
    names = [(n, p) for _, n, p, _, _ in d.param_table()]
    assert names[:6] == [("dis_batch_layer_1", "gamma"), ("dis_batch_layer_1", "beta"), ("dis_batch_layer_1", "mean"),
                         ("dis_batch_layer_1", "var"), ("dis_conv2d_layer_2", "b"), ("dis_conv2d_layer_2", "W")]
    assert names[-4:] == [("dis_dense_layer_6", "W"), ("dis_dense_layer_6", "b"), ("dis_output_layer_7", "W"), ("dis_output_layer_7", "b")]
    # dense W is 'f' order in the flattened vector
    l = d.layer("dis_dense_layer_6"); l.params["W"] = np.arange(1152 * 1024, dtype=np.float64).reshape(1152, 1024)
    flat = d.params_flat(); off = 4 + 1664 + 204928
    assert flat[off + 1] == l.params["W"][1, 0]
    d.set_params_flat(flat); assert np.array_equal(d.layer("dis_dense_layer_6").params["W"], l.params["W"])
    out = d.output(np.random.default_rng(0).standard_normal((3, 784))); assert out.shape == (3, 1)
    assert g.output(np.random.default_rng(0).standard_normal((3, 2))).shape == (3, 1, 28, 28)          # J:225
    G = o.dcgan_generator(); D = o.dcgan_discriminator()
    assert (G.num_params(), D.num_params()) == (3578627, 2767425)


def test_reference_iteration_replay_runs_and_aliased_step_tracks_it():
    """J:408-510 replayed literally (three graphs, two averaged workers) on a small batch."""
    dis = o.reference_discriminator(); gen = o.reference_generator(); gan, ng = o.reference_gan()
    # gen and gan start from the same generator weights, gan_dis from dis (the reference only syncs after step 1)
    for k, l in enumerate(gen.layers):
        if l.has_params:
            for p, _, _ in l.param_specs():
                gan.layers[k].params[p] = l.params[p].copy()
    rng = np.random.default_rng(0)
    x = np.round(rng.uniform(0, 1, (8, 784)), 2)
    z_d = rng.uniform(-1, 1, (8, 2)); z_g = rng.uniform(-1, 1, (8, 2))
    y_r = 1 + 0.05 * rng.standard_normal((8, 1)); y_f = 0.05 * rng.standard_normal((8, 1)); y_g = np.ones((8, 1))
    r = o.gan_iteration_reference(dis, gen, gan, ng, x, z_d, z_g, y_r, y_f, y_g)
    assert all(np.isfinite(r[k]) for k in ("score_d_real", "score_d_fake", "score_gan"))
    # the lr-0 "frozen" D inside gan still decays by l2*W during gan.fit (SURVEY.md 3.4 step 5) ...
    np.testing.assert_allclose(gan.layers[ng + 2].params["W"], dis.layers[2].params["W"] * (1 - 1e-4), rtol=1e-12)
    # ... and after the gan -> gen copies (J:474-510) the generator graphs agree
    np.testing.assert_array_equal(gen.layers[1].params["W"], gan.layers[1].params["W"])


def test_parameter_averaging_equals_gradient_averaging_for_sgd():
    """averagingFrequency=1 + linear updater: mean of worker params == one step on the mean gradient
    (upstream TestCompareParameterAveragingSparkVsSingleMachine; Python/gan.ipynb:182-186)."""
    def mk():
        return o.Net([o.Dense(4, 3, "tanh", updater=o.Sgd(0.1), name="a"), o.Output(3, 1, updater=o.Sgd(0.1), name="o")], seed=5)
    rng = np.random.default_rng(0)
    xs = [rng.standard_normal((6, 4)) for _ in range(2)]; ys = [rng.uniform(0, 1, (6, 1)) for _ in range(2)]
    master = mk(); ws = [mk(), mk()]
    for w, x, y in zip(ws, xs, ys):
        w.fit(x, y)
    o.parameter_average(ws, master)
    single = mk()
    g = []
    for x, y in zip(xs, ys):
        single.compute_gradient_and_score(x, y); g.append({(li, p): l.grads[p].copy() for li, l in enumerate(single.layers) for p in l.grads})
    single.apply_update(12, grads={k: g[0][k] + g[1][k] for k in g[0]})
    np.testing.assert_allclose(master.params_flat(), single.params_flat(), rtol=1e-12, atol=1e-14)


def test_transfer_learning_head_frozen_trunk_and_softmax_mcxent():
    """J:337-364 / J:512-545: frozen discriminator trunk (test-mode BN, no gradient, no update, no l2) + BN(1024) + softmax-10 MCXENT head."""
    dis = o.reference_discriminator()
    cv = o.reference_computer_vision(dis)
    assert cv.num_params() == 1388293 - 1025 + 4 * 1024 + 1024 * 10 + 10
    rng = np.random.default_rng(0)
    x = np.round(rng.uniform(0, 1, (6, 784)), 2); y = np.eye(10)[rng.integers(0, 10, 6)]
    # softmax + MCXENT gradient is p - y; cross-check with torch
    head = cv.layers[-1]
    z = rng.standard_normal((6, 10)); zt = torch.tensor(z, requires_grad=True)
    F.cross_entropy(zt, torch.tensor(y), reduction="sum").backward()
    s, g = o.mcxent_softmax_score_and_grad(z, y)
    np.testing.assert_allclose(g, zt.grad.numpy(), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(s, float(F.cross_entropy(torch.tensor(z), torch.tensor(y), reduction="sum")), rtol=1e-10)
    # finite differences on the trainable head only
    table = cv.param_table(); p0 = cv.params_flat().copy()
    cv.compute_gradient_and_score(x, y); g = cv.grads_flat() / 6
    off = 0; idx = []
    for li, name, p, shape, _ in table:
        k = int(np.prod(shape))
        if name in ("dis_batch", "dis_output_layer_7") and p not in ("mean", "var"):
            idx += list(range(off, off + min(k, 12)))
        off += k
    for i in idx:
        pp = p0.copy(); pp[i] += 1e-6; cv.set_params_flat(pp); sp = cv.compute_gradient_and_score(x, y)
        pm = p0.copy(); pm[i] -= 1e-6; cv.set_params_flat(pm); sm = cv.compute_gradient_and_score(x, y)
        num = (sp - sm) / 2e-6; l2 = 1e-4 * p0[i] if table and i >= len(p0) - 10250 and i < len(p0) - 10 else 0.0
        ana = g[i] + l2
        assert abs(num - ana) < 1e-8 or abs(num - ana) / (abs(num) + abs(ana)) < 1e-3, (i, num, ana)
    cv.set_params_flat(p0)
    # fit: only the new layers move; the trunk is bit-for-bit unchanged (not even l2-decayed, unlike an lr-0 layer)
    cv.fit(x, y); p1 = cv.params_flat()
    names = [(n, p) for li, n, p, sh, _ in table for _ in range(int(np.prod(sh)))]
    changed = {names[i][0] for i in np.flatnonzero(p0 != p1)}
    assert changed == {"dis_batch", "dis_output_layer_7"}
    assert np.allclose(cv.output(x).sum(1), 1.0)


def test_torch_cpu_step_matches_numpy_oracle():
    """oracle/torch_cpu.py (the CPU arm bench.py times) is the same step as dl4j_oracle.gan_step: fp64, two iterations, DCGAN with
    BatchNorm + LeakyReLU + transposed convs, Adam -- losses and every parameter to round-off; and the MLP-GAN (dense path)."""
    import copy
    import torch
    from oracle import torch_cpu as tc
    q = o.Quirks(xent_clip_eps=0.0)
    cases = [(o.dcgan_generator(16, 12, 8, 3, dtype=np.float64, quirks=q), o.dcgan_discriminator(16, 8, 3, dtype=np.float64, quirks=q), o.synthetic_batch(8, 16, 3, 12, seed=3)),
             (o.mlp_generator(10, 32, 24, dtype=np.float64, quirks=q), o.mlp_discriminator(24, 32, dtype=np.float64, quirks=q), None)]
    rng = np.random.default_rng(3)
    for G, D, data in cases:
        for net in (G, D):
            for l in net.layers:
                if l.has_params:
                    for p in l.params:
                        l.params[p] = l.params[p] * (1 + 0.2 * rng.random(l.params[p].shape)) if p == "var" else l.params[p] + 0.1 * rng.standard_normal(l.params[p].shape)
        if data is None:
            n = 16
            data = (rng.standard_normal((n, 24)), rng.uniform(-1, 1, (n, 10)), rng.uniform(-1, 1, (n, 10)),
                    1 + 0.05 * rng.standard_normal((n, 1)), 0.05 * rng.standard_normal((n, 1)), np.ones((n, 1)))
        data = [np.asarray(a, np.float64) for a in data]
        G2, D2 = copy.deepcopy(G), copy.deepcopy(D)
        t = tc.TorchCpuGan(G2, D2, dtype=torch.float64)
        for _ in range(2):
            r, r2 = o.gan_step(G, D, *data), t.step(*data)
            for k in ("loss_d_real", "loss_d_fake", "loss_g"):
                assert abs(r[k] - r2[k]) < 1e-10 * max(1.0, abs(r[k])), (k, r[k], r2[k])
            assert np.abs(r["x_fake"] - r2["x_fake"].reshape(r["x_fake"].shape)).max() < 1e-10
        t.G.export(); t.D.export()
        assert np.abs(G.params_flat() - G2.params_flat()).max() < 1e-9
        assert np.abs(D.params_flat() - D2.params_flat()).max() < 1e-9


def test_c_reference_matches_numpy_oracle():
    """oracle/cpu_ref.c -- the C + OpenMP restatement of DL4J's nd4j-native algorithm (im2col + SGEMM + separate passes, NCHW fp32) that
    bench.py times as the CPU arm (SURVEY.md 8d(i), P:104-108) -- computes the same adversarial step as dl4j_oracle.gan_step: three
    iterations of the DCGAN (transposed convs, BatchNorm, LeakyReLU / ReLU / tanh, Adam) and of the MLP-GAN, fp32 against the fp64 oracle.
    It also pins the golden step fixture (tests/golden/gan_step_dcgan16.npz losses) through the oracle it is compared with."""
    from oracle import cpu_ref
    from gan_deeplearning4j_b200 import models as m
    q = o.Quirks(xent_clip_eps=0.0)
    rng = np.random.default_rng(5)
    dc = o.synthetic_batch(8, 16, 3, 12, seed=3)
    n = 16
    mlp = (rng.standard_normal((n, 24)), rng.uniform(-1, 1, (n, 10)), rng.uniform(-1, 1, (n, 10)), 1 + 0.05 * rng.standard_normal((n, 1)), 0.05 * rng.standard_normal((n, 1)), np.ones((n, 1)))
    cases = [(o.dcgan_generator(16, 12, 8, 3, quirks=q), o.dcgan_discriminator(16, 8, 3, quirks=q), m.dcgan_generator(16, 12, 8, 3), m.dcgan_discriminator(16, 8, 3), 12, (3, 16, 16), dc),
             (o.mlp_generator(10, 32, 24, quirks=q), o.mlp_discriminator(24, 32, quirks=q), m.mlp_generator(10, 32, 24), m.mlp_discriminator(24, 32), 10, (24,), mlp)]
    for G, D, gs, ds, z, shape, data in cases:
        randomize(G, rng); randomize(D, rng)
        data = [np.asarray(a, np.float64) for a in data]
        c = cpu_ref.CpuRefGan(gs, ds, z, shape, data[0].shape[0])
        assert c.num_params(0) == G.num_params() and c.num_params(1) == D.num_params()
        c.set_params(0, G.params_flat()); c.set_params(1, D.params_flat())
        for _ in range(3):
            r, rc = o.gan_step(G, D, *data), c.step(*data)
            for k in ("loss_d_real", "loss_d_fake", "loss_g"):
                assert abs(r[k] - rc[k]) < 2e-6 * max(1.0, abs(r[k])), (k, r[k], rc[k])
            for net, ref in ((0, G), (1, D)):
                assert np.abs(c.get_params(net) - ref.params_flat()).max() < 5e-6 * np.abs(ref.params_flat()).max()
        c.close()


def test_golden_vectors_pin_the_oracle():
    """tests/golden/*.npz (made by tests/golden/make_golden.py) are fixed bytes: the oracle must keep reproducing them."""
    import importlib.util
    import os
    here = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    spec = importlib.util.spec_from_file_location("make_golden", os.path.join(here, "make_golden.py")); mg = importlib.util.module_from_spec(spec); spec.loader.exec_module(mg)
    for fname, fresh in (("gan_step_dcgan16.npz", mg.gan_step_vectors()), ("layer_cases.npz", mg.layer_vectors())):
        stored = np.load(os.path.join(here, fname))
        assert set(stored.files) == set(fresh), fname
        for k in stored.files:
            np.testing.assert_allclose(fresh[k], stored[k], rtol=1e-9, atol=1e-12, err_msg=f"{fname}:{k}")


@pytest.mark.parametrize("C", [1, 3, 4])
def test_pixel_shuffle_packing_reproduces_the_transposed_conv(C):
    """tests/helpers.pack_deconv_ps (the reference for the packed operand the BF16 updater writes), used as a 3x3 convolution over the 2x2
    output blocks, is the 4x4 stride-2 pad-1 Deconvolution2D forward of the oracle: out[2Y+py, 2X+px, c] = sum over (dyr, dxc, o) of
    P[py,px,c][dyr,dxc][o] * x[Y+dyr, X+dxc, o], with x zero outside the map."""
    rng = np.random.default_rng(C)
    n, O, H, W = 2, 6, 5, 7
    lay = o.Deconv2D(O, C, (4, 4), (2, 2), (1, 1), has_bias=False); lay.init(rng, np.float64)
    x = rng.standard_normal((n, O, H, W))
    ref = lay.forward(x, True)                                                  # [n, C, 2H, 2W]
    P = pack_deconv_ps(lay.params["W"].transpose(0, 2, 3, 1)).reshape(2, 2, 4, 3, 3, O)      # internal [O][4][4][C]
    xp = np.pad(x.transpose(0, 2, 3, 1), ((0, 0), (1, 1), (1, 1), (0, 0)))        # NHWC, one zero row / column each side
    got = np.zeros((n, H, 2, W, 2, 4))
    for dyr in (-1, 0, 1):
        for dxc in (-1, 0, 1):
            win = xp[:, 1 + dyr:1 + dyr + H, 1 + dxc:1 + dxc + W, :]            # x[Y+dyr, X+dxc]
            got += np.einsum("nyxo,pqco->nypxqc", win, P[:, :, :, dyr + 1, dxc + 1, :])
    assert not got[..., C:].any()                                               # padded channels stay empty
    got = got[..., :C].reshape(n, 2 * H, 2 * W, C).transpose(0, 3, 1, 2)
    np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-12)
