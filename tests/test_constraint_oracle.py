"""The oracle's weight constraints against hand-computed answers and an independent float64 torch restatement, their place in fit and the
GAN step and their resolution against the library's; the emulation of the device's summation order (ew_ref) against float64 sums.  CPU only."""
import copy

import numpy as np
import pytest
import torch

import ew_ref as er
from gan_deeplearning4j_b200 import engine as e
from gan_deeplearning4j_b200 import models as m
from oracle import dl4j_oracle as o

EPS = 1e-6


def test_max_norm_known_answers():
    """Dense W [nIn = 2, nOut = 3], norm per output unit (dims {0}): columns of norm 5 (above 2), 1 (below: shrinks by 1/(1+eps)) and 2
    (at the bound: 2/(2+eps))."""
    w = np.array([[3.0, 1.0, 0.0], [4.0, 0.0, 2.0]])
    got = o.apply_constraint(w, m.max_norm(2.0, (0,)))
    want = w * np.float32(np.array([2 / (5 + EPS), 1 / (1 + EPS), 2 / (2 + EPS)]))
    np.testing.assert_array_equal(got, want)
    assert got[1, 1] == 0.0 and got[0, 1] < 1.0


def test_min_max_norm_rates():
    w = np.array([[3.0, 0.3], [4.0, 0.4]])            # column norms 5 and 0.5, bounds [1, 2]
    full = o.apply_constraint(w, m.min_max_norm(1.0, 2.0, (0,)))
    np.testing.assert_array_equal(full, w * np.float32(np.array([2 / (5 + EPS), 1 / (0.5 + EPS)])))
    half = o.apply_constraint(w, m.min_max_norm(1.0, 2.0, (0,), rate=0.5))
    np.testing.assert_array_equal(half, w * np.float32(np.array([(0.5 * 2 + 0.5 * 5) / (5 + EPS), (0.5 * 1 + 0.5 * 0.5) / (0.5 + EPS)])))


def test_unit_norm_and_the_all_zero_group():
    w = np.array([[3.0, 0.0], [4.0, 0.0]])
    got = o.apply_constraint(w, m.unit_norm((0,)))
    np.testing.assert_array_equal(got[:, 0], np.array([3.0, 4.0]) * np.float32(1 / 5))
    np.testing.assert_array_equal(got[:, 1], [0.0, 0.0])               # the documented deviation: DL4J's 0/0
    nan = o.apply_constraint(w, m.unit_norm((0,)), o.Quirks(unit_norm_zero_group_unchanged=False))
    assert np.isnan(nan[:, 1]).all()
    z = o.apply_constraint(np.zeros((2, 2)), m.max_norm(1.0, (0,)))             # MaxNorm of a zero group: 0 * 0 / eps
    np.testing.assert_array_equal(z, 0.0)


def test_non_negative_keeps_negative_zero_and_nan():
    w = np.array([-1.5, -0.0, 0.0, 2.0, np.nan, -1e-30], np.float32)
    got = o.apply_constraint(w, m.non_negative())
    assert np.signbit(got[1]) and got[1] == 0.0 and np.isnan(got[4])
    np.testing.assert_array_equal(got[[0, 2, 3, 5]], [0.0, 0.0, 2.0, 0.0])
    assert not np.signbit(got[0])


CASES = [("conv", (7, 5, 3, 3), d) for d in ((1, 2, 3), (0,), (2, 3), (), (0, 3), (0, 1))] + [("conv", (6, 4, 4, 4), (0, 2, 3)), ("conv", (40, 24, 4, 4), (0, 2, 3))] + \
        [("dense", (37, 11), d) for d in ((0,), (1,))] + [("vector", (9,), d) for d in ((0,), (1,))]


def _torch_ref(w, c):
    t = torch.from_numpy(np.asarray(w, np.float64))
    if t.ndim == 1:
        t = t.reshape(1, -1)
    dims = tuple(c["dims"]) or tuple(range(t.ndim))
    norm = torch.linalg.vector_norm(t, dim=dims, keepdim=True)
    if c["constraint"] == "max_norm":
        mult = torch.clamp(norm, 0, c["max"]) / (norm + EPS)
    elif c["constraint"] == "min_max_norm":
        mult = (c["rate"] * torch.clamp(norm, c["min"], c["max"]) + (1 - c["rate"]) * norm) / (norm + EPS)
    else:
        mult = torch.where(norm == 0, torch.ones_like(norm), 1 / norm)
    return (t * mult).reshape(np.shape(w)).numpy()


@pytest.mark.parametrize("kind,shape,dims", CASES)
def test_restatement_agrees_with_torch_and_device_order(kind, shape, dims):
    rng = np.random.default_rng(len(shape) + sum(dims))
    w = rng.standard_normal(shape).astype(np.float32)
    s, _ = er.group_sums(kind, w, dims)
    norms = np.sqrt(s)
    lo, mid, hi = np.quantile(norms, [0.25, 0.5, 0.75])
    for c in (m.max_norm(mid, dims), m.min_max_norm(lo, hi, dims), m.min_max_norm(lo, hi, dims, rate=0.5), m.unit_norm(dims)):
        ours = o.apply_constraint(w.astype(np.float64), c)
        np.testing.assert_allclose(ours, _torch_ref(w, c), rtol=2e-7, atol=1e-12)
        np.testing.assert_allclose(er.device_apply(kind, w, c), ours, rtol=2e-7, atol=1e-12)
    # the device's order sums the same squares: float64 sums agree to rounding
    x = w.astype(np.float64).reshape((1,) + shape if kind == "vector" else shape)
    ref = np.sort(((x ** 2).sum(axis=tuple(dims) or None)).ravel())
    np.testing.assert_allclose(np.sort(s), ref, rtol=1e-13)


def test_plan_of_the_patterns_that_matter():
    assert er.plan("conv", (7, 3, 3, 5), (1, 2, 3)) == [7, 45, 1, 1, 1]      # conv W per output unit: contiguous groups
    assert er.plan("conv", (6, 4, 4, 3), (0, 2, 3)) == [1, 96, 1, 1, 3]      # deconv W per output unit: the innermost axis kept, strided
    assert er.plan("conv", (7, 3, 3, 5), (2, 3)) == [7, 9, 1, 1, 5]
    assert er.plan("conv", (7, 3, 3, 5), (0,)) == [1, 7, 1, 1, 45]
    assert er.plan("conv", (7, 3, 3, 5), (0, 3)) == [1, 7, 3, 3, 5]
    assert er.plan("conv", (7, 3, 3, 5), (0, 1)) == [1, 7, 9, 5, 1]
    assert er.plan("dense", (11, 1, 1, 37), (1,)) == [1, 11, 1, 1, 37]
    assert er.plan("dense", (11, 1, 1, 37), (0,)) == [11, 37, 1, 1, 1]       # dense W per output unit
    assert er.plan("vector", (1, 1, 1, 9), (0,)) == [9, 1, 1, 1, 1]          # each element its own group


def _mlp(frozen=False, constraints=None):
    specs = [{"type": "dense", "name": "a", "n_in": 3, "n_out": 4, "activation": "tanh", "updater": m.sgd(0.5), "frozen": frozen},
             {"type": "output", "name": "out", "n_in": 4, "n_out": 1, "updater": m.sgd(0.5)}]
    return specs, o.net_from_specs(specs, (3,), seed=3, constraints=constraints)


def test_fit_updates_then_constrains_and_frozen_layers_stay():
    rng = np.random.default_rng(0)
    x, y = rng.uniform(-1, 1, (5, 3)), rng.uniform(0, 1, (5, 1))
    cons = [m.max_norm(0.1, (0,))]
    _, plain = _mlp()
    plain.fit(x, y)
    _, net = _mlp(constraints=cons)
    net.fit(x, y)
    for l, p in zip(net.layers, plain.layers):
        np.testing.assert_array_equal(l.params["W"], o.apply_constraint(p.params["W"], cons[0]))
        np.testing.assert_array_equal(l.params["b"], p.params["b"])
    _, fnet = _mlp(frozen=True, constraints=cons)
    w0 = fnet.layers[0].params["W"].copy()
    assert "a" not in fnet.layer_constraints                               # a FrozenLayer has nothing to constrain
    fnet.fit(x, y); fnet.apply_constraints()
    np.testing.assert_array_equal(fnet.layers[0].params["W"], w0)


def test_gan_step_constrains_d_after_its_update_and_g_after_its_own():
    gs = m.dcgan_generator(16, 12, 8, 3, lr=2e-3)
    ds = m.dcgan_discriminator(16, 8, 3, lr=2e-3, loss="wasserstein", out_activation="identity")
    G, D = o.net_from_specs(gs, (12,), seed=1), o.net_from_specs(ds, (3, 16, 16), seed=2)
    data = [a.astype(np.float64) for a in o.synthetic_batch(4, 16, 3, 12, seed=3)][:3]
    labels = [np.ones((4, 1)), -np.ones((4, 1)), np.ones((4, 1))]
    Gp, Dp = copy.deepcopy(G), copy.deepcopy(D)
    o.gan_step(Gp, Dp, *data, *labels)
    dcons, gcons = [m.max_norm(0.05, (1, 2, 3))], [m.max_norm(0.05, (0, 2, 3))]
    Gc, Dc = o.net_from_specs(gs, (12,), seed=1, constraints=gcons), o.net_from_specs(ds, (3, 16, 16), seed=2, constraints=dcons)
    # D: the same D update as without constraints, then the constraint (the G step restores D's parameters after its backward)
    o.gan_step(Gc, Dc, *data, *labels)
    for lc, lp in zip(Dc.layers, Dp.layers):
        if getattr(lc, "params", None) and "W" in lc.params:
            np.testing.assert_array_equal(lc.params["W"], o.apply_constraint(lp.params["W"], dcons[0]))
            assert np.sqrt((lc.params["W"] ** 2).sum(axis=(1, 2, 3))).max() <= 0.05 + 1e-12
    for l in Gc.layers:
        if getattr(l, "params", None) and "W" in l.params:
            assert np.sqrt((l.params["W"] ** 2).sum(axis=(0, 2, 3))).max() <= 0.05 + 1e-12


GLOBAL_RULE_SPECS = [{"type": "dense", "name": "a", "n_in": 3, "n_out": 4, "constraints": [m.max_norm(2.0, (0,))]},
                     {"type": "batchnorm", "name": "bn", "constraints": [m.non_negative(on="bias")]},
                     {"type": "output", "name": "out", "n_in": 4, "n_out": 1}]


def test_global_constraints_fill_layers_whose_own_reach_nothing():
    """DL4J's builder gives the global lists to a layer whose own resolved constraints are empty: a BatchNorm with only constrainBias (no bias)
    takes the global constrainAllParameters; a dense layer with its own weight constraint keeps it."""
    glob = [m.unit_norm((1,), on="all")]
    net = o.net_from_specs(GLOBAL_RULE_SPECS, (3,), seed=1, constraints=glob)
    assert net.layer_constraints["a"] == {"W": [GLOBAL_RULE_SPECS[0]["constraints"][0]]}
    assert net.layer_constraints["bn"] == {p: glob for p in ("gamma", "beta", "mean", "var")}
    assert net.layer_constraints["out"] == {"b": glob, "W": glob}
    net.set_constraints([m.max_norm(1.0, (0,))], "a")                      # one layer's list replaced, the others kept
    assert net.layer_constraints["a"] == {"W": [m.max_norm(1.0, (0,))]} and net.layer_constraints["out"] == {"b": glob, "W": glob}
    net.set_constraints(None)
    assert net.layer_constraints == {}


def test_oracle_resolves_constraints_as_the_library_does():
    """Every spec table the constraint tests build, with its own constraints or with every layer given one constraint of each target or a
    mixed list, with and without biases, frozen and live: the oracle's constraints of each layer equal engine.resolve_constraints of its
    spec, and the global list reaches an unconstrained net's layers as each layer's own list does."""
    from test_gpu_constraints import BIG, ODD, _wgan_specs
    wg, wd = _wgan_specs([m.max_norm(0.5, (1, 2, 3))], [m.max_norm(0.8, (0, 2, 3))])
    tables = [(ODD, (5, 6, 6)), (BIG, (1024,)), (_mlp()[0], (3,)), (_mlp(frozen=True)[0], (3,)), (GLOBAL_RULE_SPECS, (3,)), (wg, (12,)),
              (wd, (3, 16, 16)), (m.dcgan_generator(16, 12, 8, 3), (12,)), (m.dcgan_discriminator(16, 8, 3), (3, 16, 16)),
              (m.dcgan_generator(32, 16, 64, 3), (16,)), (m.dcgan_discriminator(32, 64, 3), (3, 32, 32))]
    mixed = [m.non_negative(on="bias"), m.max_norm(1.0, (1,)), m.unit_norm((0,), on="all"), m.min_max_norm(0.5, 2.0, ())]
    lists = [None] + [[m.max_norm(1.0, (1,), on=on)] for on in o.CONSTRAINT_ON] + [mixed]       # None: the specs' own
    variants = [lambda i, sp: sp, lambda i, sp: dict(sp, has_bias=False) if sp["type"] in ("conv2d", "deconv2d", "dense") else sp,
                lambda i, sp: dict(sp, frozen=i % 2 == 0)]
    for specs, shape in tables:
        for lst in lists:
            for variant in variants:
                own = [variant(i, sp if lst is None else dict(sp, constraints=lst)) for i, sp in enumerate(specs)]
                net = o.net_from_specs(own, shape)
                for sp in own:
                    assert net.layer_constraints.get(sp["name"], {}) == e.resolve_constraints(sp), (sp["name"], lst)
                if lst is not None:
                    plain = [{k: v for k, v in sp.items() if k != "constraints"} for sp in own]
                    assert o.net_from_specs(plain, shape, constraints=lst).layer_constraints == net.layer_constraints
