"""CPU checks of the oracle's updaters: hand-computed answers over three steps for every new kind, float64 agreement with torch.optim where
the two forms are the same update, the spec builder's existing kinds against a hand-built net (alone and with gradient normalization and
schedules), the quirk flags, mixed-kind nets and parameter averaging of the new state."""
import copy
import math

import numpy as np
import pytest
import torch

from helpers import randomize
from gan_deeplearning4j_b200 import models as m
from oracle import dl4j_oracle as o

G3 = (0.5, -1.0, 2.0)          # the gradient after the division by the minibatch, three steps

# (W, state slots...) after each step from W = 1 with DL4J's default hyperparameters, worked by hand:
#   Nesterovs(0.1, 0.9):  v = -0.05, u = 1.9*0.05 = 0.095;  v = -0.045 + 0.1 = 0.055, u = -0.045 - 0.1045;  v = 0.0495 - 0.2, u = 0.0495 + 0.28595
#   AdaGrad(0.1, 1e-6):   h = 1e-6 + 0.25, u = 0.05 / (sqrt(h) + 1e-6); ...
#   AdaMax:               m = 0.05, u_inf = 0.5, u = 1e-3/0.1 * 0.05/0.5 = 1e-3; m = -0.055, u_inf = 1, u = 1e-3/0.19 * -0.055; ...
#   AdaDelta(0.95, 1e-6): msg = 0.05*0.25, u = sqrt(1e-6)/sqrt(0.0125 + 1e-6) * 0.5, msdx = 0.05*u^2; ...
KNOWN = {
    "nesterovs": [(0.905, -0.05), (1.0545, 0.055), (0.71905, -0.1505)],
    "adagrad": [(0.900000399998, 0.250001), (0.989443003321, 1.250001), (0.902155893635, 5.250001)],
    "adamax": [(0.999, 0.05, 0.5), (0.999289473684, -0.055, 1.0), (0.999011798407, 0.1505, 2.0)],
    "nadam": [(0.939916762457, 0.05, 0.00025), (0.962174237554, -0.055, 0.00124975), (0.945088220549, 0.1505, 0.00524850025)],
    "amsgrad": [(0.999000000632, 0.05, 0.00025, 0.00025), (0.999366104056, -0.055, 0.00124975, 0.00124975),
                (0.998946448495, 0.1505, 0.00524850025, 0.00524850025)],
    "adadelta": [(0.99552804292, 0.0125, 9.99920006399e-07), (1.00121323572, 0.061875, 2.56599486263e-06),
                 (0.993788976787, 0.25878125, 5.19367615192e-06)],
}
BUILDERS = {"nesterovs": m.nesterovs, "adagrad": m.adagrad, "adamax": m.adamax, "nadam": m.nadam, "amsgrad": m.amsgrad, "adadelta": m.adadelta}


def _scalar_net(upd, quirks=o.DEFAULT_QUIRKS, **kw):
    net = o.net_from_specs([{"type": "dense", "name": "d", "n_out": 1, "has_bias": False, "updater": upd}], (1,), quirks=quirks, **kw)
    net.layers[0].params["W"] = np.ones((1, 1))
    return net


def _step(net, g, mb=2):
    net.apply_update(mb, grads={(0, "W"): np.full((1, 1), g * mb)})


@pytest.mark.parametrize("kind", o.EXT_UPDATERS)
def test_known_answers_over_three_steps(kind):
    net = _scalar_net(BUILDERS[kind]())
    for it, (g, want) in enumerate(zip(G3, KNOWN[kind])):
        _step(net, g)
        got = (float(net.layers[0].params["W"][0, 0]),) + tuple(float(s[0, 0]) for s in net.state[(0, "W")])
        assert len(got) == len(want) == 1 + o.N_STATE[kind]
        assert np.allclose(got, want, rtol=1e-10, atol=0), (kind, it, got, want)
    assert net.iteration == 3


def _torch_run(opt_fn, g_seq, p0):
    p = torch.tensor(p0, dtype=torch.float64, requires_grad=True)
    opt = opt_fn([p])
    for g in g_seq:
        p.grad = torch.tensor(g, dtype=torch.float64)
        opt.step()
    return p.detach().numpy()


def _ref_run(u, g_seq, p0):
    p, st = np.array(p0, np.float64), o.init_state(u, np.shape(p0))
    for t, g in enumerate(g_seq, 1):
        p = p - o.update(u, st, np.asarray(g, np.float64), t)
    return p


@pytest.mark.parametrize("case", ["nesterovs", "adagrad", "adadelta"])
def test_float64_agreement_with_torch_optim(case):
    """SGD(momentum, nesterov=True) is Nesterovs rewritten in its buffer b = -v/lr (the same update at a constant lr); Adagrad with the history
    starting at eps and AdaDelta with lr 1 are the same formulas."""
    rng = np.random.default_rng(7)
    g_seq, p0 = [rng.standard_normal(13) for _ in range(6)], rng.standard_normal(13)
    if case == "nesterovs":
        u, fn = o.updater_cfg(m.nesterovs(0.05, 0.8)), lambda ps: torch.optim.SGD(ps, lr=0.05, momentum=0.8, nesterov=True)
    elif case == "adagrad":
        u, fn = o.updater_cfg(m.adagrad(0.1, 1e-6)), lambda ps: torch.optim.Adagrad(ps, lr=0.1, initial_accumulator_value=1e-6, eps=1e-6)
    else:
        u, fn = o.updater_cfg(m.adadelta(0.9, 1e-6)), lambda ps: torch.optim.Adadelta(ps, lr=1.0, rho=0.9, eps=1e-6)
    got, want = _ref_run(u, g_seq, p0), _torch_run(fn, g_seq, p0)
    assert np.allclose(got, want, rtol=1e-12, atol=1e-14), (case, np.abs(got - want).max())


def _old_specs(lr):
    return [{"type": "dense", "name": "d1", "n_out": 16, "activation": "tanh", "updater": m.adam(lr), "l2": 1e-3},
            {"type": "batchnorm", "name": "bn", "updater": m.rmsprop(1e-2, 0.9, 1e-8)},
            {"type": "dense", "name": "d2", "n_out": 8, "activation": "lrelu", "alpha": 0.2, "updater": m.sgd(0.05)},
            {"type": "dense", "name": "d3", "n_out": 8, "activation": "tanh", "updater": m.noop()},
            {"type": "output", "name": "out", "n_out": 1, "updater": m.adam(2e-3)}]


def _fit(net, steps, seed=3, shape=(6,)):
    rng = np.random.default_rng(seed)
    for _ in range(steps):
        net.fit(rng.uniform(-1, 1, (5,) + shape), rng.uniform(0, 1, (5, 1)))
    return net


def _same(a, b):
    assert a.iteration == b.iteration
    assert np.array_equal(a.params_flat(), b.params_flat())
    assert a.state.keys() == b.state.keys()
    for k in a.state:
        assert all(np.array_equal(x, y) for x, y in zip(a.state[k], b.state[k])), k


@pytest.mark.parametrize("stack", ["plain", "gradnorm+schedule"])
def test_existing_kinds_are_bit_identical_through_the_wrapper(stack):
    """The spec builder's nets of the existing kinds against the same net built by hand ("plain") and against schedules and a normalization
    mode set through the Net's methods."""
    sched = m.exponential_schedule(1e-2, 0.9)
    specs = _old_specs(sched if stack != "plain" else 1e-2)
    rng = np.random.default_rng(1)
    if stack == "plain":
        a = o.Net([o.Dense(6, 16, "tanh", updater=o.Adam(1e-2), l2=1e-3, name="d1"), o.BatchNorm(16, updater=o.RmsProp(1e-2, 0.9, 1e-8), name="bn"),
                   o.Dense(16, 8, "lrelu", 0.2, updater=o.Sgd(0.05), name="d2"), o.Dense(8, 8, "tanh", updater=o.UpdaterCfg("noop"), name="d3"),
                   o.Output(8, 1, updater=o.Adam(2e-3), name="out")], seed=4, grad_clip=0.5)
        b = o.net_from_specs(specs, (6,), seed=4, grad_clip=0.5)
    else:
        a = o.net_from_specs(_old_specs(o.value(sched, 0)), (6,), seed=4)
        a.set_lr_schedule(sched, "d1")
        b = o.net_from_specs(specs, (6,), seed=4)
        for net in (a, b):
            net.set_gradient_normalization("clip_l2_per_layer", 0.3)
    randomize(a, rng); b.set_params_flat(a.params_flat())
    _same(_fit(a, 4), _fit(b, 4))


def _mixed_specs():
    return [{"type": "dense", "name": "d1", "n_out": 16, "activation": "tanh", "updater": m.amsgrad(1e-2), "l2": 1e-3},
            {"type": "batchnorm", "name": "bn", "updater": m.adagrad(0.05)},
            {"type": "dense", "name": "d2", "n_out": 8, "activation": "lrelu", "alpha": 0.2, "updater": m.sgd(0.05)},
            {"type": "dense", "name": "d3", "n_out": 8, "activation": "tanh", "updater": m.adadelta()},
            {"type": "output", "name": "out", "n_out": 1, "updater": m.adam(2e-3)}]


def test_mixed_net_updates_each_layer_by_its_own_kind():
    """One update with fixed gradients: the Sgd / Adam layers move exactly as in a net whose other layers use NoOp, the new kinds as
    update() says, the BatchNorm mean/var through NoOp, and the iteration advances once."""
    specs = _mixed_specs()
    rng = np.random.default_rng(2)
    a = o.net_from_specs(specs, (6,), seed=4, grad_clip=0.7)
    randomize(a, rng)
    plain_specs = [dict(s, updater=m.noop()) if s["updater"]["kind"] in o.EXT_UPDATERS else s for s in specs]
    b = o.net_from_specs(plain_specs, (6,), seed=4, grad_clip=0.7); b.set_params_flat(a.params_flat())
    grads = {(li, p): 3 * rng.standard_normal(sh) for li, l in enumerate(a.layers) for p, sh, _ in l.param_specs()}
    before = {k: a.layers[k[0]].params[k[1]].copy() for k in grads}
    a.apply_update(4, grads=copy.deepcopy(grads)); b.apply_update(4, grads=copy.deepcopy(grads))
    assert a.iteration == b.iteration == 1
    for (li, p), g in grads.items():
        l = a.layers[li]
        if l.updater.kind not in o.EXT_UPDATERS:
            assert np.array_equal(l.params[p], b.layers[li].params[p]), (li, p)
            continue
        gd = g if p in l.noop_names() else g / 4
        gd = np.clip(gd, -0.7, 0.7)
        if p in l.noop_names():
            want = before[(li, p)] - gd
            assert (li, p) not in a.state
        else:
            upd = o.update(l.updater, o.init_state(l.updater, g.shape), gd, 1)
            want = before[(li, p)] - (upd + (l.l2 * before[(li, p)] if l.l2 and p in l.l2_names() else 0))
        assert np.allclose(l.params[p], want, rtol=1e-14, atol=1e-15), (li, p)


def test_schedules_and_gradient_normalization_reach_the_new_kinds():
    sched = m.step_schedule(0.1, 0.5, 1)
    specs = [{"type": "dense", "name": "d", "n_out": 3, "has_bias": False, "updater": m.nesterovs(sched, 0.9)}]
    net = o.net_from_specs(specs, (2,), seed=1)
    net.set_gradient_normalization("renormalize_l2_per_layer", 1.0)
    w = net.layers[0].params["W"].copy()
    v = np.zeros_like(w)
    rng = np.random.default_rng(5)
    for t in range(1, 4):
        g = rng.standard_normal(w.shape)
        net.apply_update(2, grads={(0, "W"): g.copy()})
        gn = (g / 2) * float(np.float32(1.0 / math.sqrt(float(((g / 2) ** 2).sum()))))     # the multiplier is rounded to fp32 once
        lr = float(np.float32(0.1 * 0.5 ** (t - 1)))          # a schedule value is rounded to fp32 once
        vp = v.copy(); v = 0.9 * v - lr * gn; w = w - (0.9 * vp - 1.9 * v)
        assert np.allclose(net.layers[0].params["W"], w, rtol=1e-13, atol=1e-15), t
        assert np.allclose(net.state[(0, "W")][0], v, rtol=1e-13, atol=1e-15), t


def test_parameter_average_averages_the_new_state():
    specs = _mixed_specs()
    nets = [_fit(o.net_from_specs(specs, (6,), seed=4), 2, seed=s) for s in (1, 2)]
    want = {k: [(x + y) / 2 for x, y in zip(nets[0].state[k], nets[1].state[k])] for k in nets[0].state}
    assert len(nets[0].state[(0, "W")]) == 3            # AMSGrad's three slots are all there
    into = copy.deepcopy(nets[0])
    o.parameter_average(nets, into)
    for k, v in want.items():
        assert all(np.array_equal(a, b) for a, b in zip(into.state[k], v)), k


def test_each_quirk_flag_changes_what_it_should():
    g = np.array([0.3, -2.0, 0.0])
    def run(kind, q, hp, steps=2):
        u = o.updater_cfg(BUILDERS[kind](**hp))
        st = o.init_state(u, g.shape, q=q)
        init = [s.copy() for s in st]
        us = [o.update(u, st, g, t, q) for t in range(1, steps + 1)]
        return init, us, st
    base = o.DEFAULT_QUIRKS
    flags = {"adagrad_history_init_eps": ("adagrad", {}), "adamax_floor_no_eps": ("adamax", {"eps": 0.1}),
             "nadam_v_uncorrected": ("nadam", {})}
    for flag, (kind, hp) in flags.items():
        q = o.Quirks(**{flag: not getattr(base, flag)})
        for other in o.EXT_UPDATERS:                          # the flag leaves every other kind alone, bit for bit
            if other != kind:
                a, b = run(other, base, {}), run(other, q, {})
                assert all(np.array_equal(x, y) for x, y in zip(a[1], b[1])), (flag, other)
        (i0, u0, s0), (i1, u1, s1) = run(kind, base, hp), run(kind, q, hp)
        assert not np.allclose(u0[-1][:2], u1[-1][:2], rtol=1e-6), flag
        if flag == "adagrad_history_init_eps":
            assert np.all(i0[0] == 1e-6) and np.all(i1[0] == 0)
        if flag == "adamax_floor_no_eps":
            assert s0[1][2] == 0.999 * 1e-32 + 1e-32 and s1[1][2] == 0.0           # the floor is stored back
            assert u0[-1][2] == 0.0 == u1[-1][2]
            assert np.allclose(u1[0][:2], 1e-3 / 0.1 * 0.1 * g[:2] / (np.abs(g[:2]) + 0.1))
        if flag == "nadam_v_uncorrected":
            assert np.allclose(u1[0][:2] / u0[0][:2], math.sqrt(1 - 0.999), rtol=1e-5)
