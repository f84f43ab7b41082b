"""Weight initialization (b2g_weight_init in include/b200gan.h) in the oracle's restatement: known answers worked by hand
from Philox words, the fan table, the statistics of every scheme and distribution over 10^6 draws, and the separation of the init streams
from the DropoutLayer and weight-noise streams.  No GPU needed."""
import math

import numpy as np
import pytest

from oracle import dl4j_oracle as o

SEED = 1234


def _word(seed, layer, j, k=0):
    """Philox word of view index j in round k, straight from the generator: word j & 3 of ctr {j >> 2, k, 0, L | 2^31}."""
    w = o.philox4x32_10((j >> 2, k, 0, layer | 0x80000000), (seed & 0xFFFFFFFF, seed >> 32))
    return int(w[j & 3])


def _z(seed, layer, j, k=0):
    """Box-Muller by hand: u from the even word of j's pair, v from the odd one; the even element takes r cos, the odd r sin."""
    e = j & ~1
    xe, xo = _word(seed, layer, e, k), _word(seed, layer, e + 1, k)
    u = ((xe >> 9) + 0.5) * 2.0 ** -23
    v = (xo >> 8) * 2.0 ** -24
    r = math.sqrt(-2.0 * math.log(u))
    return r * (math.cos(2 * math.pi * v) if j == e else math.sin(2 * math.pi * v))


def test_known_answers_per_family():
    """A few elements of each draw kind worked by hand from the Philox words, against the restatement's vectorised draw."""
    L, n = 3, 23
    for j in (0, 5, 6, 22):
        z = _z(SEED, L, j)
        assert np.float32(o.weight_init_draw("normal", np.float32(0.5), np.float32(0.02), n, SEED, L)[j]) == np.float32(np.float64(np.float32(0.02)) * z + 0.5)
        assert o.weight_init_draw("log_normal", np.float32(0), np.float32(0.5), n, SEED, L)[j] == np.float32(math.exp(float(np.float32(0.5 * z))))
        u = (_word(SEED, L, j) >> 8) * 2.0 ** -24
        assert o.weight_init_draw("uniform", np.float32(-0.25), np.float32(0.75), n, SEED, L)[j] == np.float32(-0.25 + u)
        thr = math.floor(float(np.float32(0.3)) * 2.0 ** 32)
        assert o.weight_init_draw("binomial", 7, np.float32(0.3), n, SEED, L)[j] == sum(_word(SEED, L, j, t) < thr for t in range(7))
        k = next((k for k in range(16) if abs(_z(SEED, L, j, k)) <= 2), None)
        zt = _z(SEED, L, j, k) if k is not None else min(max(_z(SEED, L, j, 15), -2.0), 2.0)
        assert o.weight_init_draw("truncated_normal", np.float32(0), np.float32(0.1), n, SEED, L)[j] == np.float32(np.float64(np.float32(0.1)) * zt)
    assert np.all(o.weight_init_draw("constant", np.float32(0.125), np.float32(0), n, SEED, L) == np.float32(0.125))
    eye = o.weight_init_draw("identity", 0, 0, 16, SEED, L, n_in=4).reshape(4, 4)
    assert np.array_equal(eye, np.eye(4, dtype=np.float32))
    # seed 0 is 666, and the layer index and the seed both change the words
    assert np.array_equal(o.weight_init_words(0, 1, 8, 0), o.weight_init_words(666, 1, 8, 0))
    assert not np.array_equal(o.weight_init_words(SEED, 1, 8, 0), o.weight_init_words(SEED, 2, 8, 0))
    assert not np.array_equal(o.weight_init_words(SEED, 1, 8, 0), o.weight_init_words(SEED + 1, 1, 8, 0))


def test_truncated_normal_redraws_and_clamps():
    """Elements whose round-0 z is beyond 2 take a later round's; none is ever beyond 2, and the rounds used are the first that qualify."""
    n = 4000
    z0 = o.weight_init_normals(SEED, 0, n, 0)
    zt = o.truncated_z(SEED, 0, n)
    assert np.all(np.abs(zt) <= 2)
    inside = np.abs(z0) <= 2
    assert np.array_equal(zt[inside], z0[inside]) and (~inside).sum() > 50
    z1 = o.weight_init_normals(SEED, 0, n, 1)
    second = ~inside & (np.abs(z1) <= 2)
    assert np.array_equal(zt[second], z1[second])


@pytest.mark.parametrize("case", ["conv_s1", "conv_s2", "deconv", "g_first_deconv", "whole_input_conv", "dense"])
def test_fan_table(case):
    """fanIn = nIn kH kW, fanOut = nOut kH kW / (sH sW) for conv and deconv, whatever geometry the engine runs them with; nIn, nOut for dense;
    XAVIER_LEGACY takes nIn + nOut for all of them."""
    layer, want = {
        "conv_s1": (o.Conv2D(64, 128, (3, 3), (1, 1), (1, 1)), (576, 1152)),
        "conv_s2": (o.Conv2D(64, 128, (4, 4), (2, 2), (1, 1)), (1024, 512)),
        "deconv": (o.Deconv2D(128, 3, (4, 4), (2, 2), (1, 1)), (2048, 12)),
        "g_first_deconv": (o.Deconv2D(100, 512, (4, 4), (1, 1), (0, 0)), (1600, 8192)),
        "whole_input_conv": (o.Conv2D(512, 1, (4, 4), (1, 1), (0, 0)), (8192, 16)),
        "dense": (o.Dense(784, 256), (784, 256)),
    }[case]
    assert tuple(float(v) for v in layer.fans()) == want
    fi, fo = want
    kind, a, b = o.resolve({"weight_init": "xavier"}, layer)
    assert (kind, a, b) == ("normal", 0, np.float32(math.sqrt(2.0 / (fi + fo))))
    assert o.resolve({"weight_init": "var_scaling_normal_fan_out"}, layer)[2] == np.float32(math.sqrt(1.0 / fo))
    assert o.resolve({"weight_init": "relu_uniform"}, layer)[1:] == (-np.float32(math.sqrt(6.0 / fi)), np.float32(math.sqrt(6.0 / fi)))
    assert o.resolve({"weight_init": "xavier_legacy"}, layer)[2] == np.float32(1.0 / math.sqrt(layer.n_in + layer.n_out))


def expected_moments(kind, a, b):
    """(mean, variance) of the draw kind with fp32 parameters a, b: the normal's; the uniform's; the truncated normal's; the log-normal's;
    the binomial's n p, n p (1 - p); a constant's."""
    a, b = float(a), float(b)
    if kind == "normal":
        return a, b * b
    if kind == "uniform":
        return (a + b) / 2, (b - a) ** 2 / 12
    if kind == "truncated_normal":
        t = o.DEFAULT_QUIRKS.truncation_sigmas
        phi = math.exp(-t * t / 2) / math.sqrt(2 * math.pi)
        mass = math.erf(t / math.sqrt(2))
        return a, b * b * (1 - 2 * t * phi / mass)
    if kind == "log_normal":
        return math.exp(a + b * b / 2), (math.exp(b * b) - 1) * math.exp(2 * a + b * b)
    if kind == "binomial":
        return a * b, a * b * (1 - b)
    return a, 0.0


def _check_moments(x, mean, var, what):
    x = np.asarray(x, np.float64)
    n = x.size
    m, v = x.mean(), x.var()
    m4 = np.mean((x - m) ** 4)
    se_m, se_v = math.sqrt(max(var, 1e-300) / n), math.sqrt(max(m4 - v * v, 1e-300) / n)
    assert abs(m - mean) <= 5 * se_m, (what, m, mean, se_m)
    assert abs(v - var) <= 5 * se_v, (what, v, var, se_v)


N_DRAWS = 10 ** 6
LAYER = o.Conv2D(64, 128, (3, 3), (1, 1), (1, 1))


@pytest.mark.parametrize("scheme", [s for s in o.SCHEMES if s not in ("distribution", "identity")])
def test_scheme_moments(scheme):
    """10^6 draws of each scheme's resolved distribution on a 3x3 conv (fanIn 576, fanOut 1152): mean and variance within 5 standard errors;
    truncated normals within +-2 std, uniforms within their bounds; ZERO and ONES exact."""
    kind, a, b = o.resolve({"weight_init": scheme}, LAYER)
    x = o.weight_init_draw(kind, a, b, N_DRAWS, SEED, 7)
    if kind == "constant":
        assert np.all(x == a) and a in (0, 1)
        return
    _check_moments(x, *expected_moments(kind, a, b), scheme)
    if kind == "uniform":
        assert x.min() >= a and x.max() < b
    if kind == "truncated_normal":
        assert np.all(np.abs(x) <= 2 * b)


@pytest.mark.parametrize("dist", [{"distribution": "normal", "mean": 0.1, "std": 0.02},
                                  {"distribution": "uniform", "lower": -0.3, "upper": 0.5},
                                  {"distribution": "truncated_normal", "mean": -0.2, "std": 0.5},
                                  {"distribution": "log_normal", "mean": 0.0, "std": 0.5},
                                  {"distribution": "binomial", "n_trials": 10, "p": 0.3},
                                  {"distribution": "constant", "value": 0.75}], ids=lambda d: d["distribution"])
def test_distribution_moments(dist):
    """DISTRIBUTION with each distribution: 10^6 draws within 5 standard errors of the mean and variance (binomial: n p, n p (1 - p));
    the truncated normal within mean +- 2 std, the uniform within its bounds, the binomial whole numbers in [0, n]."""
    kind, a, b = o.resolve({"weight_init": "distribution", "distribution": dist}, LAYER)
    x = o.weight_init_draw(kind, a, b, N_DRAWS, SEED, 2)
    if kind == "constant":
        assert np.all(x == np.float32(0.75))
        return
    _check_moments(x, *expected_moments(kind, a, b), kind)
    if kind == "truncated_normal":
        assert np.all(np.abs(x.astype(np.float64) - a) <= 2 * float(b) * (1 + 1e-6))
    if kind == "uniform":
        assert x.min() >= a and x.max() < b
    if kind == "binomial":
        assert np.all(x == np.round(x)) and x.min() >= 0 and x.max() <= 10


def test_streams_never_meet_dropout_or_weight_noise_draws():
    """For the same seed S and layer L, every DropoutLayer and weight-noise draw uses counter word 3 = L | r << 16 with r < 2^15 (below 2^31),
    every init draw L | 2^31: no (counter, key) is shared.  The words of the two streams differ where their other counter words coincide."""
    for L in (0, 1, 7, 255):
        drop_tags = {L | (r << 16) for r in (0, 1, 2, 2 ** 15 - 1)}
        assert max(drop_tags) < 2 ** 31 and (L | o.WEIGHT_INIT_TAG) not in drop_tags and (L | o.WEIGHT_INIT_TAG) >= 2 ** 31
    # init round k = pass P's low word with P < 2^32: counter words 0-2 coincide, word 3 does not, so the draws differ
    init = o.weight_init_words(SEED, 3, 64, 0)
    drop = o.philox_words(SEED, 0, 64, *o.dropout_counter(0, 3, 0))
    assert not np.array_equal(init, drop) and np.mean(init == drop) < 0.1


def test_init_layer_writes_the_view_order():
    """init_layer puts view index j at the element b2g_net_get_param returns j-th: the oracle's flattened parameters of the layer are the
    drawn W (bias first for conv), and the bias is bias_init."""
    conv = o.Conv2D(3, 4, (3, 3), (1, 1), (1, 1))
    dense = o.Dense(5, 6)
    for layer in (conv, dense):
        layer.init(np.random.default_rng(0), np.float32)
        wi = {"weight_init": "uniform", "bias_init": 0.25}
        o.init_layer(layer, wi, SEED, 4)
        flat = np.concatenate([layer.params[p].ravel(order=ordr.upper()) for p, _, ordr in layer.param_specs()])
        w = o.weights(wi, layer, SEED, 4)
        assert np.array_equal(flat[-w.size:] if isinstance(layer, o.Conv2D) else flat[:w.size], w)
        assert np.all(layer.params["b"] == np.float32(0.25))
