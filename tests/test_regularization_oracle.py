"""The oracle's regularization (l1, l2, l1Bias and l2Bias; b2g_regularization in include/b200gan.h): hand-computed one-element updates for
every updater kind and every sign of theta, the term apply_update adds against finite differences and float64 torch.autograd of the score's
terms, BatchNorm and frozen layers, which take none, and l2-only nets, which train exactly as specs without the other coefficients."""
import copy
import math

import numpy as np
import pytest
import torch

from gan_deeplearning4j_b200 import models as m
from oracle import dl4j_oracle as o

KINDS = ("sgd", "rmsprop", "adam", "noop") + o.EXT_UPDATERS
REG = {"l1": 0.03, "l2": 0.2, "l1_bias": 0.05, "l2_bias": 0.4}
UPD = {"sgd": m.sgd(0.1), "rmsprop": m.rmsprop(0.1, 0.9, 1e-8), "adam": m.adam(0.1, 0.9, 0.999, 1e-8), "noop": m.noop(),
       "nesterovs": m.nesterovs(0.1, 0.9), "adagrad": m.adagrad(0.1, 1e-6), "adamax": m.adamax(0.1, 0.9, 0.999), "nadam": m.nadam(0.1, 0.9, 0.999, 1e-8),
       "amsgrad": m.amsgrad(0.1, 0.9, 0.999, 1e-8), "adadelta": m.adadelta(0.95, 1e-6)}


def first_step(kind, g):
    """The first update u of each kind from fresh state (t = 1), from the formulas at b2g_updater."""
    u = UPD[kind]
    lr = u.get("lr", 0.0)
    if kind == "sgd":
        return lr * g
    if kind == "noop":
        return g
    if kind == "rmsprop":
        s = u["rms_decay"] * u["eps"] + (1 - u["rms_decay"]) * g * g
        return lr * g / (math.sqrt(s) + u["eps"])
    if kind in ("adam", "amsgrad"):
        b1, b2 = u["beta1"], u["beta2"]
        return lr * math.sqrt(1 - b2) / (1 - b1) * (1 - b1) * g / (math.sqrt((1 - b2) * g * g) + u["eps"])
    if kind == "nesterovs":
        return (1 + u["momentum"]) * lr * g
    if kind == "adagrad":
        return lr * g / (math.sqrt(u["eps"] + g * g) + u["eps"])
    if kind == "adamax":
        return lr / (1 - u["beta1"]) * (1 - u["beta1"]) * g / (abs(g) + 1e-32)
    if kind == "nadam":
        b1, b2 = u["beta1"], u["beta2"]
        mom = (1 - b1) * g
        return lr / (1 - b1) * (b1 * mom + (1 - b1) * g) / (math.sqrt((1 - b2) * g * g) + u["eps"])
    assert kind == "adadelta"
    return math.sqrt(u["eps"]) / math.sqrt((1 - u["rho"]) * g * g + u["eps"]) * g


def one_element_net(kind, reg):
    return o.net_from_specs([{"type": "output", "name": "out", "n_in": 1, "n_out": 1, "updater": copy.deepcopy(UPD[kind]), **reg}], (1,))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("theta", [0.7, -0.7, 0.0])
def test_one_element_update_by_hand(kind, theta):
    net = one_element_net(kind, REG)
    l = net.layers[0]
    beta = -theta / 2
    l.params["W"] = np.array([[theta]]); l.params["b"] = np.array([beta])
    gw, gb = 0.3, -0.2
    net.apply_update(1, grads={(0, "W"): np.array([[gw]]), (0, "b"): np.array([gb])})
    sign = lambda v: (v > 0) - (v < 0)
    want_w = theta - (first_step(kind, gw) + REG["l2"] * theta + REG["l1"] * sign(theta))
    want_b = beta - (first_step(kind, gb) + REG["l2_bias"] * beta + REG["l1_bias"] * sign(beta))
    assert l.params["W"][0, 0] == pytest.approx(want_w, rel=1e-12, abs=1e-15)
    assert l.params["b"][0] == pytest.approx(want_b, rel=1e-12, abs=1e-15)


def test_negative_zero_has_sign_zero():
    net = one_element_net("sgd", {"l1": 0.5, "l1_bias": 0.5})
    l = net.layers[0]
    l.params["W"] = np.array([[-0.0]]); l.params["b"] = np.array([0.0])
    net.apply_update(1, grads={(0, "W"): np.zeros((1, 1)), (0, "b"): np.zeros(1)})
    assert l.params["W"][0, 0] == 0 and l.params["b"][0] == 0


SPECS = [{"type": "conv2d", "name": "c1", "n_out": 4, "kernel": (3, 3), "stride": (2, 2), "padding": (1, 1), "activation": "tanh"},
         {"type": "batchnorm", "name": "bn", **REG},
         {"type": "deconv2d", "name": "dc", "n_out": 3, "kernel": (2, 2), "stride": (2, 2)},
         {"type": "cnn_to_ff", "name": "flat"},
         {"type": "dense", "name": "fc", "n_out": 5, "activation": "tanh"},
         {"type": "output", "name": "out", "n_out": 1}]


def reg_net(frozen_first=False):
    specs = copy.deepcopy(SPECS)
    for s in specs:
        if s["type"] in ("conv2d", "deconv2d", "dense", "output"):
            s.update(REG, updater=m.sgd(0.1))
    specs[0]["frozen"] = frozen_first
    net = o.net_from_specs(specs, (2, 6, 6), seed=4)
    rng = np.random.default_rng(1)
    for l in net.layers:
        for p, shape, _ in l.param_specs():
            v = rng.standard_normal(shape) * 0.3
            l.params[p] = v + 0.05 * np.sign(v)           # away from 0, where |theta| is differentiable
    return net


def reg_score(net):
    return net.calc_l1() + net.calc_l2()


def live_gemm(net):
    return [(li, l) for li, l in enumerate(net.layers) if l.has_params and l.l2_names() and not getattr(l, "frozen", False)]


def test_added_term_is_the_gradient_of_the_score_terms():
    net = reg_net()
    plain = copy.deepcopy(net)
    plain.layer_regularization = {}
    for l in plain.layers:
        l.l2 = 0.0
    grads = {(li, p): np.zeros(shape) for li, l in enumerate(net.layers) for p, shape, _ in l.param_specs()}
    net.apply_update(1, grads=copy.deepcopy(grads)); plain.apply_update(1, grads=copy.deepcopy(grads))
    fresh = reg_net()
    h = 1e-6
    for li, l in live_gemm(fresh):
        for p in ("W", "b"):
            term = (plain.layers[li].params[p] - net.layers[li].params[p]).ravel()
            fd = np.empty_like(term)
            for j in range(term.size):
                v = fresh.layers[li].params[p].reshape(-1)
                x0 = v[j]
                v[j] = x0 + h; up = reg_score(fresh)
                v[j] = x0 - h; dn = reg_score(fresh)
                v[j] = x0
                fd[j] = (up - dn) / (2 * h)
            np.testing.assert_allclose(term, fd, rtol=1e-6, atol=1e-9, err_msg=f"{l.name}.{p}")


def test_score_terms_against_torch_autograd():
    net = reg_net()
    l1 = l2 = 0.0
    for li, l in live_gemm(net):
        for p in ("W", "b"):
            t = torch.tensor(net.layers[li].params[p], dtype=torch.float64, requires_grad=True)
            c1, c2 = net.reg_coefs(l, p)
            a, q = c1 * t.abs().sum(), 0.5 * c2 * (t * t).sum()
            (a + q).backward()
            l1, l2 = l1 + a.item(), l2 + q.item()
            want = t.grad.numpy()
            copy_net = copy.deepcopy(net)
            copy_net.apply_update(1, grads={(i, pn): np.zeros(s) for i, ll in enumerate(net.layers) for pn, s, _ in ll.param_specs()})
            got = net.layers[li].params[p] - copy_net.layers[li].params[p]
            np.testing.assert_allclose(got, want, rtol=1e-12, err_msg=f"{l.name}.{p}")
    assert net.calc_l1() == pytest.approx(l1, rel=1e-12) and net.calc_l2() == pytest.approx(l2, rel=1e-12)
    assert net.l2_score() == net.calc_l2() + net.calc_l1()


def test_batchnorm_and_frozen_layers_take_no_term():
    net = reg_net()
    bn = net.layer("bn")
    assert all(net.reg_coefs(bn, p) == (0.0, 0.0) for p, _, _ in bn.param_specs())
    before = {p: v.copy() for p, v in bn.params.items()}
    zeros = {(li, p): np.zeros(s) for li, l in enumerate(net.layers) for p, s, _ in l.param_specs()}
    net.apply_update(1, grads=copy.deepcopy(zeros))
    assert all(np.array_equal(bn.params[p], before[p]) for p in ("gamma", "beta"))
    frozen = reg_net(frozen_first=True)
    c1 = frozen.layer("c1")
    only_c1 = REG["l1"] * np.abs(c1.params["W"]).sum() + REG["l1_bias"] * np.abs(c1.params["b"]).sum()
    assert frozen.calc_l1() == pytest.approx(reg_net().calc_l1() - only_c1, rel=1e-12)
    w0 = c1.params["W"].copy()
    frozen.apply_update(1, grads=copy.deepcopy(zeros))
    assert np.array_equal(c1.params["W"], w0)


def test_l2_only_nets_keep_their_update_and_score():
    """With l1 = l1Bias = l2Bias = 0 the update and the score are the l2-only ones: W -= lr g + l2 W, b -= lr g, score term 0.5 l2 ||W||^2."""
    net = reg_net()
    net.layer_regularization = {}
    want = sum(0.5 * l.l2 * float((l.params["W"] ** 2).sum()) for _, l in live_gemm(net))
    assert net.l2_score() == want and net.calc_l1() == 0.0
    fc = net.layer("fc")
    w, bb = fc.params["W"].copy(), fc.params["b"].copy()
    g = {(li, p): np.full(s, 0.25) for li, l in enumerate(net.layers) for p, s, _ in l.param_specs()}
    net.apply_update(1, grads=g)
    assert np.array_equal(fc.params["W"], w - (0.1 * 0.25 + REG["l2"] * w)) and np.array_equal(fc.params["b"], bb - 0.1 * 0.25)


def test_l2_only_specs_train_bit_for_bit_as_the_oracle():
    """Zero l1, l1Bias and l2Bias train exactly as specs that leave them out."""
    specs = copy.deepcopy(SPECS)
    for s in specs:
        if s["type"] in ("conv2d", "deconv2d", "dense", "output"):
            s.update(l2=0.2, updater=m.adam(0.01), constraints=[m.max_norm(0.5, ())])
    specs[1].pop("l1")
    zeros = [dict(s, l1=0.0, l1_bias=0.0, l2_bias=0.0) if s["type"] in ("conv2d", "deconv2d", "dense", "output") else s for s in specs]
    a, c = o.net_from_specs(zeros, (2, 6, 6), seed=4, grad_clip=0.5), o.net_from_specs(specs, (2, 6, 6), seed=4, grad_clip=0.5)
    assert np.array_equal(a.params_flat(), c.params_flat()) and a.layer_constraints == c.layer_constraints
    rng = np.random.default_rng(2)
    for _ in range(3):
        x, y = rng.uniform(-1, 1, (4, 2, 6, 6)), rng.uniform(0, 1, (4, 1))
        assert a.fit(x, y) == c.fit(x, y)
        assert np.array_equal(a.params_flat(), c.params_flat())
