"""Weight initialization (b2g_net_init_weights; b2g_weight_init in include/b200gan.h) on the GPU against the oracle's restatement: every
scheme and distribution drawn on conv, deconv, dense and output layers in both precisions (bit for bit, the normal families within the fp32
Box-Muller tolerance), the bf16 operands, what a call leaves alone, what a failed call leaves alone, determinism, and DCGAN training from
Normal(0, 0.02) weights, eager and graph-replayed."""
import copy
import ctypes as C

import numpy as np
import pytest

from helpers import b200, check_weight_operands, gan_step_parity
from oracle import dl4j_oracle as o

pytestmark = pytest.mark.gpu
_ = b200

SEED = 4321
# conv 3x3 s1 p1 (64 -> 128), conv 4x4 s2 p1, deconv 4x4 s2 p1 onto 3 channels (the packed pixel-shuffle operand in BF16 nets), dense, output
IMAGE_SPECS = [{"type": "conv2d", "name": "c1", "n_in": 64, "n_out": 128, "kernel": (3, 3), "stride": (1, 1), "padding": (1, 1), "activation": "relu"},
               {"type": "conv2d", "name": "c2", "n_in": 128, "n_out": 64, "kernel": (4, 4), "stride": (2, 2), "padding": (1, 1), "activation": "relu"},
               {"type": "deconv2d", "name": "dc", "n_in": 64, "n_out": 3, "kernel": (4, 4), "stride": (2, 2), "padding": (1, 1), "activation": "tanh"},
               {"type": "cnn_to_ff", "name": "flat"},
               {"type": "dense", "name": "d", "n_in": 192, "n_out": 16, "activation": "tanh"},
               {"type": "output", "name": "out", "n_in": 16, "n_out": 1}]
IMAGE_IN = (64, 8, 8)
# the DCGAN generator's first layer (a transposed conv of a 1x1 map, computed as a 1x1 problem) and the discriminator's whole-input conv
HEAD_SPECS = [{"type": "ff_to_cnn", "name": "ff", "to": (1, 1, 16)},
              {"type": "deconv2d", "name": "g1", "n_in": 16, "n_out": 64, "kernel": (4, 4), "stride": (1, 1), "padding": (0, 0), "has_bias": False},
              {"type": "activation", "name": "a1", "activation": "relu"},
              {"type": "conv2d", "name": "dlast", "n_in": 64, "n_out": 1, "kernel": (4, 4), "stride": (1, 1), "padding": (0, 0)},
              {"type": "loss", "name": "loss"}]
HEAD_IN = (16,)
SQUARE_SPECS = [{"type": "dense", "name": "d1", "n_in": 16, "n_out": 16, "activation": "tanh"},
                {"type": "dense", "name": "d2", "n_in": 16, "n_out": 16, "activation": "tanh"},
                {"type": "output", "name": "out", "n_in": 16, "n_out": 1}]
SQUARE_IN = (16,)

DISTS = {"normal": {"distribution": "normal", "mean": 0.01, "std": 0.02},
         "uniform": {"distribution": "uniform", "lower": -0.3, "upper": 0.2},
         "truncated_normal": {"distribution": "truncated_normal", "mean": -0.05, "std": 0.1},
         "log_normal": {"distribution": "log_normal", "mean": -2.0, "std": 0.5},
         "binomial": {"distribution": "binomial", "n_trials": 5, "p": 0.25},
         "constant": {"distribution": "constant", "value": -0.125}}
CASES = [(s, {"weight_init": s, "bias_init": 0.0625}) for s in o.SCHEMES if s not in ("distribution", "identity")] + \
        [("dist_" + k, {"weight_init": "distribution", "distribution": d, "bias_init": -0.5}) for k, d in DISTS.items()]


def _gemm(specs):
    return [(i, s) for i, s in enumerate(specs) if s["type"] in ("conv2d", "deconv2d", "dense", "output")]


def layer_of(spec):
    """The oracle layer of a GEMM spec (n_in given): what fans() and the W shape come from."""
    k, s, p = spec.get("kernel", (1, 1)), spec.get("stride", (1, 1)), spec.get("padding", (0, 0))
    if spec["type"] == "conv2d":
        return o.Conv2D(spec["n_in"], spec["n_out"], tuple(k), tuple(s), tuple(p))
    if spec["type"] == "deconv2d":
        return o.Deconv2D(spec["n_in"], spec["n_out"], tuple(k), tuple(s), tuple(p))
    return o.Dense(spec["n_in"], spec["n_out"])


def _check_layer(net, spec, li, wi, what):
    """get_param("W") against the restatement (bit for bit; normal families within 8 fp32 ulps of |std z| <= 6 std plus the rounding of the
    result; log-normal relative to its value), and every bias element equal to bias_init."""
    layer = layer_of(spec)
    want = o.weights(wi, layer, SEED, li)
    got = net.get_param(spec["name"], "W", want.size)
    kind, a, b = o.resolve(wi, layer)
    if kind in ("normal", "truncated_normal"):
        tol = 8 * np.spacing(np.float32(6 * float(b))) + 2 * np.spacing(np.abs(want))
        assert np.all(np.abs(got - want) <= tol), (what, spec["name"], np.max(np.abs(got - want)))
    elif kind == "log_normal":
        tol = np.abs(want) * (8 * np.spacing(np.float32(abs(float(a)) + 6 * float(b))) + 4 * 2.0 ** -24)
        assert np.all(np.abs(got - want) <= tol), (what, spec["name"], np.max(np.abs(got - want) / np.abs(want)))
    else:
        assert np.array_equal(got, want), (what, spec["name"], np.sum(got != want))
    if spec.get("has_bias", True):
        assert np.all(net.get_param(spec["name"], "b", spec["n_out"]) == np.float32(wi["bias_init"])), (what, spec["name"], "b")


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("name,wi", CASES, ids=[c[0] for c in CASES])
def test_every_scheme_draws_the_restatement(b200, prec, name, wi):
    """Net(weight_init=...) on every GEMM layer of the image chain and of the generator-head / whole-input-conv chain: W as restated, b =
    bias_init; in BF16 nets the bf16 copies and the packed pixel-shuffle operand are the rounded master."""
    b, ctx = b200
    precision = b.BF16 if prec == "bf16" else b.FP32
    packed = 0
    for specs, shape in ((IMAGE_SPECS, IMAGE_IN), (HEAD_SPECS, HEAD_IN)):
        net = b.Net(ctx, specs, shape, max_batch=4, precision=precision, seed=SEED, weight_init=wi)
        for li, s in _gemm(specs):
            _check_layer(net, s, li, wi, (prec, name))
            assert net.specs[li]["weight_init"] == wi
        if precision == b.BF16:
            packed += check_weight_operands(b, net, specs, f"{name} {prec}")
        net.close()
    assert packed == (1 if prec == "bf16" else 0)


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_identity_on_a_square_dense_layer(b200, prec):
    """IDENTITY on the square dense layers only (a per-layer setting), with the other layers keeping b2g_net_create's draw."""
    b, ctx = b200
    precision = b.BF16 if prec == "bf16" else b.FP32
    plain = b.Net(ctx, SQUARE_SPECS, SQUARE_IN, max_batch=4, precision=precision, seed=SEED)
    specs = copy.deepcopy(SQUARE_SPECS)
    for s in specs[:2]:
        s["weight_init"] = {"weight_init": "identity", "bias_init": 0.5}
    net = b.Net(ctx, specs, SQUARE_IN, max_batch=4, precision=precision, seed=SEED)
    for li, s in _gemm(specs)[:2]:
        _check_layer(net, s, li, s["weight_init"], prec)
    assert np.array_equal(net.get_param("out", "W", 16), plain.get_param("out", "W", 16))
    if precision == b.BF16:
        check_weight_operands(b, net, specs, "identity")
    net.close(); plain.close()


def _state(net):
    return net.params(), net.updater_state(), net.iteration(), net.dropout_pass(), net.epoch()


def _trained_net(b, ctx, precision=None):
    """The image chain with Adam, after two fits and an epoch count, so that the updater state and counters are not at their defaults."""
    precision = b.FP32 if precision is None else precision
    specs = [dict(s, updater={"kind": "adam", "lr": 1e-3, "beta1": 0.9, "beta2": 0.999, "eps": 1e-8}) if "n_out" in s else s for s in IMAGE_SPECS]
    specs.insert(2, {"type": "batchnorm", "name": "bn", "updater": {"kind": "adam", "lr": 1e-3, "beta1": 0.9, "beta2": 0.999, "eps": 1e-8}})
    net = b.Net(ctx, specs, IMAGE_IN, max_batch=4, precision=precision, seed=SEED)
    rng = np.random.default_rng(1)
    x, y = rng.uniform(-1, 1, (4,) + IMAGE_IN), rng.uniform(0, 1, (4, 1))
    net.fit(x, y); net.fit(x, y); net.set_epoch(3)
    return net, specs


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_a_named_call_changes_only_its_layer(b200, prec):
    """init_weights on one layer rewrites its W and b; every other parameter (BatchNorm included), the updater state, the iteration counter,
    the dropout pass counter and the epoch stay bit-identical."""
    b, ctx = b200
    net, specs = _trained_net(b, ctx, b.BF16 if prec == "bf16" else b.FP32)
    p0, st0, it0, pass0, ep0 = _state(net)
    wi = {"weight_init": "relu_uniform", "bias_init": 0.25}
    net.init_weights(wi, "c2")
    p1, st1, it1, pass1, ep1 = _state(net)
    li = next(i for i, s in enumerate(specs) if s.get("name") == "c2")
    _check_layer(net, specs[li], li, wi, "named")
    off = 0
    changed = np.zeros(p0.size, bool)
    for s in specs:       # flattened [b | W] per conv layer, in spec order
        if "n_out" not in s or s["type"] == "batchnorm":
            off += 4 * 64 if s["type"] == "batchnorm" else 0
            continue
        k = s.get("kernel", (1, 1)); n = s["n_in"] * s["n_out"] * k[0] * k[1] + (s["n_out"] if s.get("has_bias", True) else 0)
        if s["name"] == "c2":
            changed[off:off + n] = True
        off += n
    assert off == p0.size
    assert np.array_equal(p1[~changed], p0[~changed]) and not np.array_equal(p1[changed], p0[changed])
    assert np.array_equal(st1, st0) and (it1, pass1, ep1) == (it0, pass0, ep0)
    assert net.specs[li]["weight_init"] == wi and "weight_init" not in net.specs[0]
    if prec == "bf16":
        check_weight_operands(b, net, specs, "named call")
    net.close()


def test_failed_calls_change_nothing(b200):
    """Every refused call returns its code and leaves the whole net bit-identical; IDENTITY on all layers fails on the first conv before
    the square-free dense layers are touched."""
    b, ctx = b200
    net, specs = _trained_net(b, ctx)
    before = _state(net)

    def call(layer, scheme, dist=0, a=0.0, bb=0.0, bias=0.0):
        s = b.engine._lib.WeightInit(scheme, dist, a, bb, bias)
        return net.lib.b2g_net_init_weights(net.h, None if layer is None else layer.encode(), C.byref(s))

    cases = [(-1, ("c1", 21)), (-1, ("c1", -1)), (-1, ("c1", 0, 7)), (-1, ("c1", 0, -1)),
             (-1, ("c1", 0, 0, 0.0, -0.5)), (-1, ("c1", 0, 1, 0.5, 0.25)), (-1, ("c1", 0, 4, 2.5, 0.5)), (-1, ("c1", 0, 4, 70000.0, 0.5)),
             (-1, ("c1", 0, 4, 3.0, 1.5)), (-1, ("c1", 0, 0, float("nan"), 1.0)), (-1, ("c1", 7, 0, 0.0, 0.0, float("inf"))),
             (-1, ("nope", 7)), (-1, ("bn", 7)), (-1, ("flat", 7)),
             (-2, ("c1", 13)), (-2, ("dc", 13)), (-2, ("d", 13)), (-2, (None, 13)),
             (-6, ("c1", 0, 6, 1.0, 0.0)), (-6, (None, 0, 6, 1.0, 0.0))]
    for code, args in cases:
        assert call(*args) == code, args
        after = _state(net)
        for u, v in zip(before, after):
            assert np.array_equal(u, v), args
    with pytest.raises(ValueError):
        net.init_weights({"weight_init": "identity"}, "c1")
    with pytest.raises(ValueError):
        net.init_weights({"weight_init": "distribution", "distribution": {"distribution": "orthogonal", "gain": 1.0}})
    assert all(np.array_equal(u, v) for u, v in zip(before, _state(net)))
    net.close()


def test_draws_are_deterministic(b200):
    """The same seed gives the same bits in a second net; FP32 and BF16 nets and any max_batch get the same fp32 master; another seed or
    another layer index gives other bits."""
    b, ctx = b200
    wi = {"weight_init": "var_scaling_normal_fan_avg"}
    nets = [b.Net(ctx, SQUARE_SPECS, SQUARE_IN, max_batch=mb, precision=p, seed=SEED, weight_init=wi)
            for mb, p in ((4, b.FP32), (4, b.FP32), (64, b.FP32), (4, b.BF16))]
    ref = nets[0].params()
    for n in nets[1:]:
        assert np.array_equal(n.params(), ref)
    other = b.Net(ctx, SQUARE_SPECS, SQUARE_IN, max_batch=4, seed=SEED + 1, weight_init=wi)
    w = lambda n, name: n.get_param(name, "W", 256)
    assert not np.array_equal(w(other, "d1"), w(nets[0], "d1"))
    assert not np.array_equal(w(nets[0], "d1"), w(nets[0], "d2"))        # same shape and scheme, layer index 0 vs 1
    for n in nets + [other]:
        n.close()


def _dcgan_specs(lr=2e-3):
    from gan_deeplearning4j_b200 import models as m
    gs, ds = m.dcgan_generator(16, 12, 8, 3, lr=lr), m.dcgan_discriminator(16, 8, 3, lr=lr)
    # n_in on every GEMM layer, as the oracle's layers need it
    for specs, c0 in ((gs, 12), (ds, 3)):
        c = c0
        for s in specs:
            if s["type"] in ("conv2d", "deconv2d"):
                s.setdefault("n_in", c); c = s["n_out"]
    return gs, ds


def test_dcgan_from_normal_002_trains_like_the_oracle(b200):
    """A DCGAN pair initialized with DISTRIBUTION(Normal(0, 0.02)) on every GEMM layer: the oracle, started from those parameters, agrees
    with the library's adversarial step (helpers.gan_step_parity: eager and graph-replayed, losses and parameters over 3 steps)."""
    b, ctx = b200
    from gan_deeplearning4j_b200 import models as m
    gs, ds = _dcgan_specs()
    wi = m.weight_init("distribution", m.normal(0, 0.02))
    bG = b.Net(ctx, gs, (12,), max_batch=8, seed=11, weight_init=wi)
    bD = b.Net(ctx, ds, (3, 16, 16), max_batch=16, bn_groups=2, seed=12, weight_init=wi)
    G, D = o.net_from_specs(gs, (12,), seed=1), o.net_from_specs(ds, (3, 16, 16), seed=2)
    G.set_params_flat(bG.params().astype(np.float64)); D.set_params_flat(bD.params().astype(np.float64))
    w = bD.get_param("dis_conv_1", "W", 3 * 8 * 16)
    assert abs(float(np.std(w)) - 0.02) < 0.005 and np.all(bD.get_param("dis_conv_1", "b", 8) == 0)
    bG.close(); bD.close()
    data = [a.astype(np.float64) for a in o.synthetic_batch(8, 16, 3, 12, seed=3)]
    gan_step_parity(b, ctx, gs, ds, G, D, data, data[3:], 2e-3, "normal(0, 0.02) init")


def test_a_captured_gan_step_reads_the_new_weights(b200):
    """A CUDA-graph GAN step captured before init_weights replays on the new weights at its next step: its losses and parameters equal an
    eager step's after the same call, bit for bit, and differ from a run without the call."""
    b, ctx = b200
    from gan_deeplearning4j_b200 import models as m
    gs, ds = _dcgan_specs()
    data = o.synthetic_batch(8, 16, 3, 12, seed=3)
    runs = {}
    for graph, reinit in ((True, True), (False, True), (True, False)):
        bG = b.Net(ctx, gs, (12,), max_batch=8, seed=11)
        bD = b.Net(ctx, ds, (3, 16, 16), max_batch=16, bn_groups=2, seed=12)
        gan = b.Gan(bG, bD, use_cuda_graph=graph)
        gan.step(*data)
        if reinit:
            bG.init_weights(m.weight_init("distribution", m.normal(0, 0.02)))
            bD.init_weights(m.weight_init("xavier_uniform", bias_init=0.01))
        losses = gan.step(*data)
        runs[(graph, reinit)] = (np.array(losses), bG.params(), bD.params())
        gan.close(); bG.close(); bD.close()
    for u, v in zip(runs[(True, True)], runs[(False, True)]):
        assert np.array_equal(u, v)
    assert not np.array_equal(runs[(True, True)][0], runs[(True, False)][0])
