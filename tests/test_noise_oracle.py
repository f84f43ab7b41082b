"""GaussianDropout, GaussianNoise, AlphaDropout and SpatialDropout on the CPU: the restatement's known answers and statistics, the layers'
gradients by finite differences, and the host-side plumbing (kind numbers, specs, models, checkpoints, exported symbols).  No GPU needed."""
import math
import os
import re
import subprocess

import numpy as np
import pytest

from helpers import ROOT, randomize
from oracle import dl4j_oracle as o


@pytest.mark.parametrize("xe,xo,want", [
    (0x80000000, 0x00000000, (1.177409921268428, 0.0)),            # u = 1/2 + 2^-24, v = 0: (sqrt(-2 ln u), 0)
    (0x80000000, 0x40000000, (0.0, 1.177409921268428)),            # v = 1/4: cos(pi/2) = 0, sin = 1
    (0x00000000, 0x80000000, (-5.768107546403532, 0.0)),           # u = 2^-24, the largest |z|: sqrt(48 ln 2); v = 1/2: cos(pi) = -1
    (0xFFFFFFFF, 0x00000000, (0.00034526698814612303, 0.0)),       # u = 1 - 2^-24, the smallest r
], ids=["half", "quarter_turn", "tail", "center"])
def test_box_muller_known_answers(xe, xo, want):
    ze, zo = o.box_muller(np.array([xe]), np.array([xo]))
    assert abs(ze[0] - want[0]) < 1e-12 and abs(zo[0] - want[1]) < 1e-12
    assert abs(-5.768107546403532) == pytest.approx(o.Z_MAX, rel=1e-15)


def test_normals_follow_the_pairing_and_nchw_order():
    """Element e takes z[e & 3] of counter e >> 2: pair (x0, x1) gives z0, z1 and pair (x2, x3) z2, z3; NCHW result of the NHWC order."""
    seed, rank, layer, pass_ = 5, 1, 3, 9
    z = o.dropout_normals(seed, rank, layer, pass_, 2, 3, 5, 7)
    assert z.shape == (2, 7, 3, 5)
    e = ((1 * 3 + 2) * 5 + 4) * 7 + 6             # (row 1, c 6, y 2, x 4)
    w = [int(v) for v in o.philox4x32_10((e >> 2, pass_, 0, layer | rank << 16), (seed, 0))]
    pair = (e & 3) >> 1
    ze, zo = o.box_muller(np.array([w[2 * pair]]), np.array([w[2 * pair + 1]]))
    assert z[1, 6, 2, 4] == (zo if e & 1 else ze)[0]
    assert np.array_equal(o.dropout_normals(seed, rank, layer, pass_, 1, 3, 5, 7, row0=1), z[1:])
    assert np.abs(z).max() <= o.Z_MAX


@pytest.mark.parametrize("p,a,b", [(0.5, 0.8864048946659319, 0.7791939305180315), (0.9, 0.9212845161497115, 0.16197097005757016)])
def test_alpha_dropout_coefficients(p, a, b):
    """a = 1 / sqrt(p + a'^2 p (1 - p)) and b = -a (1 - p) a' with a' = -1.0507009873554805 * 1.6732632423543772 = -1.7580993408473766, the
    hand values at the decimal p; the layer takes p as fp32 (0.9 -> 0.899999976), hence the 1e-6 relative tolerance."""
    ga, gb, gap = o.alpha_coefficients(p)
    assert gap == np.float32(-1.7580993408473766)
    assert abs(ga - a) <= 1e-6 * a and abs(gb - b) <= 1e-6 * b


def _layer(kind, value, layer=2, seed=11):
    l = o.Dropout(value, "n", index=layer, state=o.DropoutState(seed), kind=kind)
    l.last = True
    return l


def test_alpha_dropout_keeps_mean_zero_and_variance_one():
    n = 10 ** 6
    x = np.random.default_rng(0).standard_normal((1000, 1000))
    for p in (0.5, 0.9):
        y = _layer("alpha_dropout", p).forward(x, True)
        m4 = np.mean((y - y.mean()) ** 4)
        assert abs(y.mean()) < 5 / math.sqrt(n), (p, y.mean())
        assert abs(y.var() - 1) < 5 * math.sqrt((m4 - 1) / n), (p, y.var())


def test_gaussian_dropout_mean_and_variance():
    n, x0 = 10 ** 6, 1.5
    for rate in (0.2, 0.5):
        y = _layer("gaussian_dropout", rate).forward(np.full((1000, 1000), x0), True)
        var = x0 * x0 * rate / (1 - rate)
        assert abs(y.mean() - x0) < 5 * math.sqrt(var / n), rate
        assert abs(y.var() - var) < 5 * var * math.sqrt(2 / n) * 1.05, (rate, y.var(), var)     # the truncation at 5.8 sigma is far below this


def test_gaussian_noise_adds_sigma_z():
    x = np.random.default_rng(1).standard_normal((4, 3, 5, 6))
    l = _layer("gaussian_noise", 0.25)
    y = l.forward(x, True)
    z = o.dropout_normals(11, 0, 2, 0, 4, 5, 6, 3)
    assert np.allclose(y, x + np.float32(0.25) * z, rtol=0, atol=1e-15)
    assert l.state.pass_ == 1 and np.array_equal(l.backward(x), x)


def test_spatial_dropout_zeroes_whole_maps():
    x = np.random.default_rng(2).uniform(0.5, 1.5, (16, 8, 5, 3))
    l = _layer("spatial_dropout", 0.5)
    y = l.forward(x, True)
    keep = o.spatial_mask(11, 0, 2, 0, 16, 8, 0.5)
    assert 0 < keep.sum() < keep.size
    for r in range(16):
        for c in range(8):
            assert (y[r, c] != 0).all() == keep[r, c] and (y[r, c] == 0).all() == (not keep[r, c])
    assert np.allclose(y[keep], 2 * x[keep])
    # draw index j = row * C + c: word j & 3 of counter j >> 2
    j = 5 * 8 + 3
    w = o.philox4x32_10((j >> 2, 0, 0, 2), (11, 0))
    assert keep[5, 3] == (int(w[j & 3]) < int(math.floor(0.5 * 2 ** 32)))


def test_identity_cases_draw_nothing():
    x = np.ones((2, 3))
    for kind, v in (("alpha_dropout", 1.0), ("spatial_dropout", 1.0), ("gaussian_dropout", 0.0), ("gaussian_noise", 0.0)):
        l = _layer(kind, v)
        assert not l.active() and l.forward(x, True) is x and l.state.pass_ == 0
    l = _layer("gaussian_noise", 0.5)
    assert l.forward(x, False) is x
    l.frozen = True
    assert not l.active()


def _chain(kind, value, first):
    """conv -> lrelu -> [noise] -> conv -> BN -> tanh -> cnn_to_ff -> dense -> [noise] -> output, or the noise as entry 0."""
    noise = lambda name: {"type": "dropout", "name": name, "kind": kind, o.VALUE_KEY[kind]: value}
    dense_noise = [] if kind == "spatial_dropout" else [noise("n2")]
    return (([noise("n0")] if first else []) +
            [{"type": "conv2d", "name": "c1", "n_out": 4, "kernel": (3, 3), "stride": (2, 2), "padding": (1, 1)},
             {"type": "activation", "name": "a1", "activation": "lrelu", "alpha": 0.2}] + ([] if first else [noise("n1")]) +
            [{"type": "conv2d", "name": "c2", "n_out": 5, "kernel": (3, 3), "padding": (1, 1), "has_bias": False},
             {"type": "batchnorm", "name": "bn"}, {"type": "activation", "name": "a2", "activation": "tanh"},
             {"type": "cnn_to_ff", "name": "flat"}, {"type": "dense", "name": "d", "n_out": 6, "activation": "tanh"}] + dense_noise +
            [{"type": "output", "name": "out", "n_out": 1}])


@pytest.mark.parametrize("first", [False, True], ids=["hidden", "entry0"])
@pytest.mark.parametrize("kind,value", [("gaussian_noise", 0.3), ("gaussian_dropout", 0.4), ("alpha_dropout", 0.7), ("spatial_dropout", 0.6)])
def test_finite_differences_with_fixed_draws(kind, value, first):
    """Central differences of the score against the gradient with every draw fixed (an explicit pass): GradientCheckUtil's eps 1e-6,
    max relative error 1e-3 and min absolute error 1e-8, over 30 parameters."""
    rng = np.random.default_rng(7)
    specs = _chain(kind, value, first)
    net = o.net_from_specs(specs, (2, 6, 6), mask_seed=3, seed=3); randomize(net, rng)
    drops = [l for l in net.layers if isinstance(l, o.Dropout)]
    assert drops and all(l.kind == kind for l in drops) and drops[-1].last
    x = rng.uniform(-1, 1, (4, 2, 6, 6)); y = rng.uniform(0, 1, (4, 1))
    net.compute_gradient_and_score(x, y, pass_=2)
    g = net.grads_flat().copy(); theta = net.params_flat().copy()

    def score(t):
        net.set_params_flat(t)
        return net.compute_gradient_and_score(x, y, pass_=2) * x.shape[0]      # gradients are minibatch sums

    for i in rng.choice(theta.size, 30, replace=False):
        tp, tm = theta.copy(), theta.copy(); tp[i] += 1e-6; tm[i] -= 1e-6
        fd = (score(tp) - score(tm)) / 2e-6
        err = abs(fd - g[i]) / max(abs(fd), abs(g[i]), 1e-300)
        assert err < 1e-3 or abs(fd - g[i]) < 1e-8, (kind, i, fd, g[i])
    net.set_params_flat(theta)
    assert net.dropout.pass_ == 0


def test_kind_numbers_agree_across_header_python_and_java():
    from gan_deeplearning4j_b200 import engine
    with open(os.path.join(ROOT, "include", "b200gan.h")) as f:
        h = f.read()
    body = re.search(r"typedef enum \{([^}]*)\} b2g_dropout_kind;", h).group(1)
    codes = {k: int(v) for k, v in re.findall(r"B2G_DROPOUT(?:_(\w+))? = (\d+)", body)}
    assert codes == {"": 0, "GAUSSIAN_DROPOUT": 1, "GAUSSIAN_NOISE": 2, "ALPHA": 3, "SPATIAL": 4}
    names = {"": "dropout", "GAUSSIAN_DROPOUT": "gaussian_dropout", "GAUSSIAN_NOISE": "gaussian_noise", "ALPHA": "alpha_dropout", "SPATIAL": "spatial_dropout"}
    assert {names[k]: v for k, v in codes.items()} == {k: c for k, (c, _) in engine.DROPOUT_KINDS.items()}
    jdir = os.path.join(ROOT, "java", "src", "main", "java", "org", "deeplearning4j", "nn", "conf", "dropout")
    java = {}
    for cls in ("Dropout", "GaussianDropout", "GaussianNoise", "AlphaDropout", "SpatialDropout"):
        with open(os.path.join(jdir, cls + ".java")) as f:
            java[cls] = int(re.search(r"int kind\(\) \{ return (\d+); \}", f.read()).group(1))
    assert java == {"Dropout": 0, "GaussianDropout": 1, "GaussianNoise": 2, "AlphaDropout": 3, "SpatialDropout": 4}


def test_new_symbols_are_exported_and_bound():
    lib = os.path.join(ROOT, "gan_deeplearning4j_b200", "lib", "libb200gan.so")
    if not os.path.exists(lib):
        pytest.skip("library not built")
    out = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True).stdout
    assert re.search(r"\bb2g_test_dropout_kind\b", out)
    from gan_deeplearning4j_b200 import _lib
    assert "b2g_test_dropout_kind" in _lib.PROTOTYPES


def test_specs_models_and_checkpoint_round_trip(tmp_path):
    from gan_deeplearning4j_b200 import engine, models as m, serializer
    cases = [(m.gaussian_noise(0.1, "a"), 2, 0.1), (m.gaussian_dropout(0.5, "b"), 1, 0.5), (m.alpha_dropout(0.9, "c"), 3, 0.9),
             (m.spatial_dropout(0.8, "d"), 4, 0.8), ({"type": "dropout", "name": "e", "p": 0.25}, 0, 0.25)]
    for spec, code, v in cases:
        d = engine.layer_desc(spec)
        assert d.type == 11 and d.act == code and d.act_alpha == np.float32(v), spec
    with pytest.raises(ValueError):
        engine.layer_desc({"type": "dropout", "kind": "weight_noise", "p": 0.5})
    # instance noise: a GaussianNoise on the input, the rest of the specs unchanged; default None leaves the specs as they were
    for build, shape in ((m.dcgan_discriminator, (3, 64, 64)), (m.mlp_discriminator, (256,))):
        plain, noisy = build(), build(instance_noise=0.1)
        assert build(instance_noise=None) == plain and noisy[1:] == plain and noisy[0] == m.gaussian_noise(0.1, "dis_instance_noise")
        assert m.forward_macs(noisy, shape) == m.forward_macs(plain, shape)
    specs = [c[0] for c in cases[:2]] + [{"type": "dense", "name": "x", "n_out": 3}]
    path = str(tmp_path / "ck.zip")
    serializer.write_model(path, specs, (4,), np.arange(4, dtype=np.float32), None, {"dropout_pass": 5})
    back = serializer.read_model(path)
    assert back["specs"] == specs


def test_net_from_specs_agrees_with_the_library_specs():
    from gan_deeplearning4j_b200 import engine, models as m
    specs = m.dcgan_discriminator(16, 8, 3, instance_noise=0.1)
    specs = specs[:3] + [m.alpha_dropout(0.9, "ad"), m.spatial_dropout(0.7, "sd")] + specs[3:6] + [m.gaussian_dropout(0.3, "gd")] + specs[6:]
    net = o.net_from_specs(specs, (3, 16, 16))
    off = len(net.layers) - len(specs)
    for i, s in enumerate(specs):
        if s["type"] != "dropout":
            continue
        l, d = net.layers[off + i], engine.layer_desc(s)
        assert isinstance(l, o.Dropout) and l.index == i
        assert engine.DROPOUT_KINDS[l.kind][0] == d.act and np.float32(l.value) == np.float32(d.act_alpha)
    assert [l.last for l in net.layers if isinstance(l, o.Dropout)] == [False, False, False, True]


def test_schedule_values_at_chosen_iterations_and_epochs():
    """A scheduled layer's value: the schedule's fp32 value at the owning net's iteration (before the update's increment) or epoch, clamped
    into the kind's range; without a schedule, the constant."""
    from gan_deeplearning4j_b200 import models as m
    l = _layer("gaussian_noise", 0.5)
    l.schedule = m.exponential_schedule(0.5, 0.9)
    for it in (0, 1, 7, 100):
        assert l.value_at(it, 0) == np.float32(0.5 * 0.9 ** it) and l.active()
    l.schedule = m.step_schedule(0.4, 0.5, 2, type="epoch")
    for ep, want in ((0, 0.4), (1, 0.4), (2, 0.2), (5, 0.1)):
        assert l.value_at(1000, ep) == np.float32(want)
    # clamping: rate to [0, 1 - 2^-24], p to [2^-32, 1], stddev to >= 0
    assert o.clamp_value("gaussian_dropout", 2.0) == np.float32(1 - 2.0 ** -24) and o.clamp_value("gaussian_dropout", -1) == 0
    assert o.clamp_value("alpha_dropout", 0.0) == np.float32(2.0 ** -32) and o.clamp_value("spatial_dropout", 3.0) == 1
    assert o.clamp_value("gaussian_noise", -0.5) == 0 and o.clamp_value("dropout", 0.25) == np.float32(0.25)
    # a scheduled value of 0 still draws: the layer is stochastic whatever its value
    l = _layer("gaussian_noise", 0.0)
    assert not l.active()
    l.schedule = m.map_schedule({0: 0.0})
    assert l.active() and l.value_at(0, 0) == 0


def test_gan_step_reads_g_counters_in_the_generator_pass():
    """The D step's pass reads D's counters, the generator step's pass through D G's (which lag D's by the D update)."""
    from gan_deeplearning4j_b200 import models as m
    n, z, hid, d = 8, 6, 16, 10
    gs = m.mlp_generator(z, hid, d, lr=1e-2)
    ds = m.mlp_discriminator(d, hid, lr=1e-2, instance_noise=m.exponential_schedule(0.4, 0.5))
    rng = np.random.default_rng(3)
    G = o.net_from_specs(gs, (z,), seed=1); D = o.net_from_specs(ds, (d,), seed=2)
    randomize(G, rng); randomize(D, rng)
    seen = []
    l = next(x for x in D.layers if isinstance(x, o.Dropout))
    orig = l.value_at
    l.value_at = lambda it, ep: (seen.append(orig(it, ep)), seen[-1])[1]
    data = [rng.uniform(-1, 1, (n, d)), rng.uniform(-1, 1, (n, z)), rng.uniform(-1, 1, (n, z)), np.ones((n, 1)), np.zeros((n, 1)), np.ones((n, 1))]
    for _ in range(2):
        o.gan_step(G, D, *data)
    # per step: the real and fake minibatches at D's counters, then the generator pass at G's (D's counter has already moved: 0.2, 0.1)
    assert seen == [np.float32(0.4)] * 3 + [np.float32(0.2)] * 3
    assert D.dropout_value("dis_instance_noise") == np.float32(0.1)


def test_schedule_symbols_are_exported_and_bound_and_specs_carry_schedules():
    from gan_deeplearning4j_b200 import _lib, engine, models as m
    lib = os.path.join(ROOT, "gan_deeplearning4j_b200", "lib", "libb200gan.so")
    if os.path.exists(lib):
        out = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True).stdout
        for sym in ("b2g_net_set_dropout_schedule", "b2g_net_get_dropout_value", "Java_org_deeplearning4j_b200_Native_netSetDropoutSchedule",
                    "Java_org_deeplearning4j_b200_Native_netGetDropoutValue"):
            assert re.search(r"\b%s\b" % sym, out), sym
    for sym in ("b2g_net_set_dropout_schedule", "b2g_net_get_dropout_value"):
        assert sym in _lib.PROTOTYPES
    with open(os.path.join(ROOT, "java", "src", "main", "java", "org", "deeplearning4j", "b200", "Native.java")) as f:
        java = f.read()
    assert "netSetDropoutSchedule" in java and "netGetDropoutValue" in java
    sched = m.exponential_schedule(0.3, 0.99)
    spec = m.gaussian_noise(sched, "n")
    assert spec["stddev"] == sched and engine.layer_desc(spec).act_alpha == np.float32(0.3)
    assert m.dcgan_discriminator(16, 8, 3, instance_noise=sched)[0] == spec | {"name": "dis_instance_noise"}
