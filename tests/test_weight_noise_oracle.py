"""Weight noise (DropConnect, WeightNoise; b2g_weight_noise in include/b200gan.h) in the oracle's restatement: known answers,
the draws' statistics, straight-through gradients by finite differences with W' fixed, the pass counter shared with DropoutLayers, and the
host-side plumbing (kind numbers, specs, models, checkpoints, exported symbols).  No GPU needed."""
import copy
import os
import re
import subprocess

import numpy as np
import pytest

from helpers import randomize
from oracle import dl4j_oracle as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DC = {"weight_noise": "drop_connect", "p": 0.75, "apply_to_bias": False}


def _dense(n_in=6, n_out=5, wn=DC, seed=0):
    l = o.Dense(n_in, n_out, name="d")
    l.init(np.random.default_rng(seed), np.float64)
    l.params["b"] = np.arange(n_out, dtype=np.float64) / 10
    net = o.Net([l], mask_seed=9)
    net.set_weight_noise(wn)
    return net, l


def test_drop_connect_known_answer():
    """W' = keep ? W : +0 with keep = x[j & 3] < floor(p 2^32) of counter {j >> 2, P, L}, j the internal index; not rescaled by 1 / p; b' only
    with apply_to_bias, from j = 4 ceil(n_W / 4) on."""
    net, l = _dense()
    w_int = o.internal_w(l.params["W"]).astype(np.float32)
    words = o.philox_words(9, 0, 40, *o.dropout_counter(0, 0, 0))
    thr = int(np.float32(0.75) * 2.0 ** 32)
    want = np.array([w if words[j] < thr else 0.0 for j, w in enumerate(w_int)], np.float32)
    got, b = o.noisy_operands(l, DC, 0, 9, 0, 0)
    assert np.array_equal(got, want) and b is None
    assert np.array_equal(o.internal_w(o.dl4j_w(got, l.params["W"].shape)), got)
    wn = dict(DC, apply_to_bias=True)
    _, b = o.noisy_operands(l, wn, 0, 9, 0, 0)
    bw = l.params["b"].astype(np.float32)
    assert np.array_equal(b, np.where(words[32:37] < thr, bw, np.float32(0)))        # j0 = 4 * ceil(30 / 4) = 32
    inv = o.Quirks(dropconnect_inverted=True)
    got_inv, _ = o.noisy_operands(l, DC, 0, 9, 0, 0, q=inv)
    assert np.array_equal(got_inv[want != 0], want[want != 0] / np.float32(0.75))


def test_weight_noise_known_answers():
    """NORMAL n = std z + mean with z of the Box-Muller pairs; UNIFORM n = fmaf(upper - lower, (x >> 8) 2^-24, lower); additive or multiplicative."""
    _, l = _dense()
    w = o.internal_w(l.params["W"]).astype(np.float32)
    words = o.philox_words(9, 0, 32, *o.dropout_counter(0, 3, 5)).reshape(-1, 4)
    z = np.empty(words.shape)
    z[:, 0], z[:, 1] = o.box_muller(words[:, 0], words[:, 1])
    z[:, 2], z[:, 3] = o.box_muller(words[:, 2], words[:, 3])
    wn = {"weight_noise": "weight_noise", "distribution": {"distribution": "normal", "mean": 0.5, "std": 0.01}, "additive": True}
    got, _ = o.noisy_operands(l, wn, 3, 9, 0, 5)
    assert np.array_equal(got, (w + (0.01 * z.ravel()[:30] + 0.5).astype(np.float32)).astype(np.float32))
    wn = {"weight_noise": "weight_noise", "distribution": {"distribution": "uniform", "lower": 0.9, "upper": 1.1}, "additive": False}
    got, _ = o.noisy_operands(l, wn, 3, 9, 0, 5)
    u = (words.ravel()[:30] >> np.uint64(8)).astype(np.float64) / 2 ** 24
    n = (float(np.float32(1.1) - np.float32(0.9)) * u + float(np.float32(0.9))).astype(np.float32)
    assert np.array_equal(got, w * n) and np.all((n >= np.float32(0.9)) & (n <= np.float32(1.1)))


def test_drop_connect_keep_fraction_is_the_counters():
    """Over 10^6 draws the kept count is exactly the number of words below the threshold, and within 5 sigma of p n."""
    n, p = 1 << 20, 0.9
    keep = o.weight_noise_draw(DC, n, 0, 7, 0, 2, 11, p)
    words = o.philox_words(7, 0, n, *o.dropout_counter(0, 2, 11))
    assert keep.sum() == (words < np.uint64(int(np.float32(p) * 2.0 ** 32))).sum()
    assert abs(keep.sum() - p * n) < 5 * np.sqrt(n * p * (1 - p))
    assert o.weight_noise_draw(DC, 8, 0, 7, 0, 2, 11, 1.0).all()


@pytest.mark.parametrize("dist", ["normal", "uniform"])
def test_noise_moments(dist):
    """Mean and variance of 10^6 draws within 5 sigma of the distribution's (the normal is truncated at |z| <= 5.8, far beyond 5 sigma)."""
    n = 1 << 20
    if dist == "normal":
        d, mean, var = {"distribution": "normal", "mean": 0.25, "std": 2.0}, 0.25, 4.0
    else:
        d, mean, var = {"distribution": "uniform", "lower": -1.0, "upper": 3.0}, 1.0, 16.0 / 12
    x = o.weight_noise_draw({"weight_noise": "weight_noise", "distribution": d}, n, 0, 666, 0, 1, 4).astype(np.float64)
    assert abs(x.mean() - mean) < 5 * np.sqrt(var / n)
    fourth = 3 * var ** 2 if dist == "normal" else 9.0 / 5 * var ** 2
    assert abs(x.var() - var) < 5 * np.sqrt((fourth - var ** 2) / n)
    if dist == "uniform":
        assert x.min() >= -1 and x.max() < 3


def _chain(wn, dropout=False):
    """conv (bias) -> lrelu -> [dropout] -> conv (no bias) -> BN -> tanh -> cnn_to_ff -> dense -> output, every GEMM layer noisy."""
    d = [{"type": "dropout", "name": "drop", "p": 0.8}] if dropout else []
    return ([{"type": "conv2d", "name": "c1", "n_out": 4, "kernel": (3, 3), "stride": (2, 2), "padding": (1, 1), "weight_noise": wn},
             {"type": "activation", "name": "a1", "activation": "lrelu", "alpha": 0.2}] + d +
            [{"type": "conv2d", "name": "c2", "n_out": 5, "kernel": (3, 3), "padding": (1, 1), "has_bias": False, "weight_noise": wn},
             {"type": "batchnorm", "name": "bn"}, {"type": "activation", "name": "a2", "activation": "tanh"},
             {"type": "cnn_to_ff", "name": "flat"}, {"type": "dense", "name": "d", "n_out": 6, "activation": "tanh", "weight_noise": wn},
             {"type": "output", "name": "out", "n_out": 1, "weight_noise": wn}])


WNS = [dict(DC, apply_to_bias=True),
       {"weight_noise": "weight_noise", "distribution": {"distribution": "normal", "mean": 0.0, "std": 0.05}, "apply_to_bias": True, "additive": True},
       {"weight_noise": "weight_noise", "distribution": {"distribution": "uniform", "lower": 0.8, "upper": 1.2}, "apply_to_bias": False, "additive": False}]


@pytest.mark.parametrize("wn", WNS, ids=["dropconnect", "normal", "uniform"])
def test_straight_through_gradients_by_finite_differences(wn):
    """With W' fixed, the noisy net's input gradient and weight gradients are those of the clean net holding W' (straight through: dW is
    taken w.r.t. W' and applied to W); central differences of that net's score w.r.t. W' and x agree at GradientCheckUtil's eps 1e-6, max
    relative error 1e-3 and min absolute error 1e-8."""
    rng = np.random.default_rng(7)
    specs = _chain(wn)
    net = o.net_from_specs(specs, (2, 6, 6), mask_seed=3, seed=3); randomize(net, rng)
    x = rng.uniform(-1, 1, (4, 2, 6, 6)); y = rng.uniform(0, 1, (4, 1))
    theta = net.params_flat().copy()
    net.compute_gradient_and_score(x, y)
    assert net.dropout.pass_ == 1
    g = net.grads_flat().copy()
    # the clean net holding the pass's W' and b'
    plain = o.net_from_specs([{k: v for k, v in s.items() if k != "weight_noise"} for s in specs], (2, 6, 6), seed=3)
    plain.set_params_flat(theta)
    off = len(net.layers) - len(specs)
    for i, s in enumerate(specs):
        l = net.layers[off + i]
        if l.noisy is not None:
            for k, v in l.noisy.items():
                plain.layers[off + i].params[k] = v.copy()
    assert not np.array_equal(plain.params_flat(), theta)
    assert np.array_equal(net.params_flat(), theta)                     # the clean parameters are untouched
    _, _, _, ex = plain.compute_gradient_and_score(x, y, collect=True)
    _, _, _, ex_noisy = net.compute_gradient_and_score(x, y, collect=True, pass_=0)
    ex = np.asarray(ex).reshape(x.shape)
    assert np.allclose(np.asarray(ex_noisy).reshape(x.shape), ex, rtol=0, atol=1e-15)
    net.compute_gradient_and_score(x, y, pass_=0)
    assert np.allclose(net.grads_flat(), plain.grads_flat(), rtol=0, atol=1e-15)
    assert np.allclose(g, plain.grads_flat(), rtol=0, atol=1e-15)
    wprime = plain.params_flat().copy()

    def score(t, xx=x):
        plain.set_params_flat(t)
        return plain.compute_gradient_and_score(xx, y) * x.shape[0]       # gradients are minibatch sums

    for i in rng.choice(wprime.size, 30, replace=False):
        tp, tm = wprime.copy(), wprime.copy(); tp[i] += 1e-6; tm[i] -= 1e-6
        fd = (score(tp) - score(tm)) / 2e-6
        err = abs(fd - g[i]) / max(abs(fd), abs(g[i]), 1e-300)
        assert err < 1e-3 or abs(fd - g[i]) < 1e-8, (i, fd, g[i])
    for _ in range(10):
        idx = tuple(rng.integers(0, s) for s in x.shape)
        xp, xm = x.copy(), x.copy(); xp[idx] += 1e-6; xm[idx] -= 1e-6
        fd = (score(wprime, xp) - score(wprime, xm)) / 2e-6
        got = ex[idx]
        assert abs(fd - got) / max(abs(fd), abs(got), 1e-300) < 1e-3 or abs(fd - got) < 1e-8, (idx, fd, got)


def test_inference_and_frozen_layers_draw_nothing():
    net, l = _dense()
    x = np.ones((2, 6))
    y0 = net.output(x)
    assert net.dropout.pass_ == 0 and l.noisy is None
    clean = copy.deepcopy(net)
    clean.set_weight_noise(None)
    assert np.array_equal(y0, clean.forward(x, False))
    net.forward(x, True)
    assert net.dropout.pass_ == 1 and l.noisy is not None
    net.output(x)
    assert l.noisy is None
    l.frozen = True
    net.forward(x, True)
    assert net.dropout.pass_ == 1
    l.frozen = False
    net.set_weight_noise(dict(DC, p=1.0))
    net.forward(x, True)
    assert net.dropout.pass_ == 1 and not o.weight_noise_active(l)
    sched = {"schedule": "map", "values": [(0, 1.0)], "type": "iteration"}
    net.set_weight_noise(dict(DC, p=sched))
    net.forward(x, True)
    assert net.dropout.pass_ == 2 and o.weight_noise_active(l)             # a scheduled DropConnect draws whatever its value


def test_adding_weight_noise_leaves_dropout_masks_unchanged():
    """The draw reads P at the top of the pass and leaves advancing it to the last DropoutLayer: a dropout net's masks and counter are the
    same with and without weight noise."""
    rng = np.random.default_rng(2)
    plain_specs = [{k: v for k, v in s.items() if k != "weight_noise"} for s in _chain(DC, dropout=True)]
    a = o.net_from_specs(plain_specs, (2, 6, 6), mask_seed=4, seed=3); randomize(a, rng)
    b = o.net_from_specs(_chain(DC, dropout=True), (2, 6, 6), mask_seed=4, seed=3); b.set_params_flat(a.params_flat())
    x = rng.uniform(-1, 1, (3, 2, 6, 6))
    da = next(l for l in a.layers if isinstance(l, o.Dropout)); db = next(l for l in b.layers if isinstance(l, o.Dropout))
    for step in range(3):
        a.forward(x, True); b.forward(x, True)
        assert np.array_equal(da._m, db._m) and a.dropout.pass_ == b.dropout.pass_ == step + 1
    # each pass drew with the pass's P: the W' of the last pass is that of P = 2
    c1 = next(l for l in b.layers if l.name == "c1")
    w, _ = o.noisy_operands(c1, DC, 0, 4, 0, 2, dtype=np.float64)
    assert np.array_equal(c1.noisy["W"], o.dl4j_w(w, c1.params["W"].shape))


def test_gan_step_pass_bookkeeping():
    """A GAN step with weight noise on D only: the real and fake minibatches share the W' of pass P, the generator pass through D draws with
    P + 1, and D's counter ends at P + 2; G's own weight noise counts G's passes."""
    from gan_deeplearning4j_b200 import models as m
    n, z, hid, d = 4, 6, 16, 10
    gs = [dict(s, weight_noise=m.weight_noise(m.normal(0, 0.01))) for s in m.mlp_generator(z, hid, d, lr=1e-2)]
    ds = m.mlp_discriminator(d, hid, lr=1e-2, drop_connect=0.9)
    rng = np.random.default_rng(3)
    G = o.net_from_specs(gs, (z,), seed=1); D = o.net_from_specs(ds, (d,), seed=2)
    randomize(G, rng); randomize(D, rng)
    seen = []
    orig = o.noisy_operands
    l0 = D.layers[-3]

    def spy(layer, wn, index, seed, rank, pass_, *a, **k):
        if layer is l0:
            seen.append(pass_)
        return orig(layer, wn, index, seed, rank, pass_, *a, **k)
    o.noisy_operands = spy
    try:
        data = [rng.uniform(-1, 1, (n, d)), rng.uniform(-1, 1, (n, z)), rng.uniform(-1, 1, (n, z)), np.ones((n, 1)), np.zeros((n, 1)), np.ones((n, 1))]
        for _ in range(2):
            o.gan_step(G, D, *data)
    finally:
        o.noisy_operands = orig
    assert seen == [0, 0, 1, 2, 2, 3] and D.dropout.pass_ == 4
    assert G.dropout.pass_ == 2                                   # one train-mode pass of G per step (x_fake is an inference pass)


def test_gan_step_reads_g_counters_for_a_scheduled_drop_connect():
    from gan_deeplearning4j_b200 import models as m
    n, z, hid, d = 4, 6, 16, 10
    gs = m.mlp_generator(z, hid, d, lr=1e-2)
    ds = m.mlp_discriminator(d, hid, lr=1e-2, drop_connect=m.exponential_schedule(0.8, 0.5))
    rng = np.random.default_rng(3)
    G = o.net_from_specs(gs, (z,), seed=1); D = o.net_from_specs(ds, (d,), seed=2)
    seen = []
    orig = o.drop_connect_p
    o.drop_connect_p = lambda wn, c=(0, 0): (seen.append(orig(wn, c)), seen[-1])[1]
    try:
        data = [rng.uniform(-1, 1, (n, d)), rng.uniform(-1, 1, (n, z)), rng.uniform(-1, 1, (n, z)), np.ones((n, 1)), np.zeros((n, 1)), np.ones((n, 1))]
        for _ in range(2):
            o.gan_step(G, D, *data)
    finally:
        o.drop_connect_p = orig
    # three noisy layers per pass; per step the real and fake passes at D's counters, then the generator pass at G's, which lag D's by the
    # D update (at D's the first step's generator pass would read 0.4)
    assert seen[::3] == [np.float32(0.8)] * 3 + [np.float32(0.4)] * 3


def test_kind_numbers_agree_across_header_python_and_java():
    from gan_deeplearning4j_b200 import engine
    with open(os.path.join(ROOT, "include", "b200gan.h")) as f:
        h = f.read()
    body = re.search(r"typedef enum \{([^}]*)\} b2g_weight_noise_kind;", h).group(1)
    codes = dict(re.findall(r"B2G_WEIGHT_NOISE_(\w+) = (\d+)", body))
    assert codes == {"NONE": "0", "DROPCONNECT": "1", "WEIGHTNOISE": "2"}
    assert engine.WEIGHT_NOISE_KINDS == {"drop_connect": 1, "weight_noise": 2}
    body = re.search(r"typedef enum \{([^}]*)\} b2g_distribution_kind;", h).group(1)
    assert dict(re.findall(r"B2G_DIST_(\w+) = (\d+)", body)) == {"NORMAL": "0", "UNIFORM": "1"}
    assert {k: v[0] for k, v in engine.DISTRIBUTIONS.items()} == {"normal": 0, "uniform": 1}
    jdir = os.path.join(ROOT, "java", "src", "main", "java", "org", "deeplearning4j", "nn", "conf")
    java = {}
    for cls in ("DropConnect", "WeightNoise"):
        with open(os.path.join(jdir, "weightnoise", cls + ".java")) as f:
            java[cls] = int(re.search(r"int kind\(\) \{ return (\d+); \}", f.read()).group(1))
    assert java == {"DropConnect": 1, "WeightNoise": 2}
    for cls, code in (("NormalDistribution", 0), ("UniformDistribution", 1)):
        with open(os.path.join(jdir, "distribution", cls + ".java")) as f:
            assert int(re.search(r"int kind\(\) \{ return (\d+); \}", f.read()).group(1)) == code


def test_symbols_are_exported_and_bound():
    from gan_deeplearning4j_b200 import _lib
    for sym in ("b2g_net_set_weight_noise", "b2g_test_net_noisy_operand"):
        assert sym in _lib.PROTOTYPES
    with open(os.path.join(ROOT, "java", "src", "main", "java", "org", "deeplearning4j", "b200", "Native.java")) as f:
        assert "netSetWeightNoise" in f.read()
    lib = os.path.join(ROOT, "gan_deeplearning4j_b200", "lib", "libb200gan.so")
    if not os.path.exists(lib):
        pytest.skip("library not built")
    out = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True).stdout
    for sym in ("b2g_net_set_weight_noise", "b2g_test_net_noisy_operand", "Java_org_deeplearning4j_b200_Native_netSetWeightNoise"):
        assert re.search(r"\b%s\b" % sym, out), sym


def test_specs_models_and_checkpoint_round_trip(tmp_path):
    from gan_deeplearning4j_b200 import engine, models as m, serializer
    assert m.drop_connect(0.9) == {"weight_noise": "drop_connect", "p": 0.9, "apply_to_bias": False}
    wn = m.weight_noise(m.uniform(-0.1, 0.1), apply_to_bias=True, additive=False)
    s, _ = engine.weight_noise_struct(wn)
    assert (s.kind, s.apply_to_bias, s.dist, s.a, s.b, s.additive) == (2, 1, 1, np.float32(-0.1), np.float32(0.1), 0)
    s, keep = engine.weight_noise_struct(m.drop_connect(m.step_schedule(0.9, 0.5, 10), apply_to_biases=True))
    assert s.kind == 1 and s.apply_to_bias == 1 and s.p == np.float32(0.9) and s.p_schedule.contents.kind == 4 and keep
    assert engine.weight_noise_struct(None)[0].kind == 0
    for bad in ({"weight_noise": "gaussian"}, {"weight_noise": "weight_noise", "distribution": {"distribution": "binomial"}}):
        with pytest.raises(ValueError):
            engine.weight_noise_struct(bad)
    # drop_connect on the discriminators: every GEMM layer gets it, nothing else changes; the default leaves the specs as they were
    for build in (m.dcgan_discriminator, m.mlp_discriminator):
        plain, noisy = build(), build(drop_connect=0.9)
        assert build(drop_connect=None) == plain and len(noisy) == len(plain)
        for a, b in zip(plain, noisy):
            assert b == (dict(a, weight_noise=m.drop_connect(0.9)) if a["type"] in engine.GEMM_TYPES else a)
    specs = m.mlp_discriminator(8, 4, drop_connect=0.5)
    path = str(tmp_path / "ck.zip")
    serializer.write_model(path, specs, (8,), np.arange(4, dtype=np.float32), None, {"dropout_pass": 3})
    assert serializer.read_model(path)["specs"] == specs
