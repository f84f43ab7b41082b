"""Weight initialization (b2g_weight_init in include/b200gan.h: DL4J's WeightInit, Distribution and biasInit) restated on top of the DL4J
oracle: each scheme's distribution from the layer's fans (the oracle layers' fans()), and the library's draws from Philox4x32-10 exactly.

The draw: S = the net's seed (0: 666), L = the layer's index in the desc array, j = the element's index in DL4J's view order of W (what
b2g_net_get_param returns).  Round k of element j uses word x[j & 3] of Philox4x32-10(ctr = {j >> 2, k, 0, L | 0x80000000}, key = {lo32(S),
hi32(S)}).  NORMAL: fmaf(std, z, mean), z of the Box-Muller pairs (x0, x1), (x2, x3) of round 0 (noise_ref.box_muller, float64 here; the
device's is fp32, so normal draws agree within its tolerance).  UNIFORM: fmaf(upper - lower, (x >> 8) 2^-24, lower).  TRUNCATED_NORMAL: z
of the first round k < 16 with |z| <= 2, else round 15's z clamped.  LOG_NORMAL: exp of the NORMAL value.  BINOMIAL: the count over rounds
t < nTrials of x_t < floor(p 2^32).  CONSTANT, ZERO, ONES, IDENTITY: no draw.

DL4J 1.0.0-beta3, recalled; parity unpinned like the rest of the DL4J semantics.  The points of medium confidence are WeightInitQuirks fields."""
import math
from dataclasses import dataclass

import numpy as np

from oracle import dl4j_oracle as o
import noise_ref as nr


@dataclass(frozen=True)
class WeightInitQuirks:
    # LECUN_UNIFORM's bound 3 / sqrt(fanIn), recalled from WeightInitUtil (other libraries use sqrt(3 / fanIn)); medium confidence
    lecun_uniform_three_over_sqrt: bool = True
    # VAR_SCALING_UNIFORM_FAN_{IN,OUT,AVG} bounds 3 / sqrt(fan), recalled the same way (not sqrt(3 / fan)); medium confidence
    var_scaling_uniform_three_over_sqrt: bool = True
    # XAVIER_LEGACY's std 1 / sqrt(shape[0] + shape[1]), i.e. 1 / sqrt(nIn + nOut) for conv, deconv and dense W alike; medium confidence
    xavier_legacy_shape01: bool = True
    # TruncatedNormalDistribution and VAR_SCALING_NORMAL_*: values beyond this many std are redrawn; recalled as 2, medium confidence
    truncation_sigmas: float = 2.0
    # NORMAL is N(0, 1 / sqrt(fanIn)), not unit variance; recalled, medium confidence
    normal_scaled_by_fan_in: bool = True


WQ = WeightInitQuirks()
SCHEMES = ("distribution", "zero", "ones", "sigmoid_uniform", "normal", "lecun_normal", "uniform", "xavier", "xavier_uniform", "xavier_fan_in",
           "xavier_legacy", "relu", "relu_uniform", "identity", "lecun_uniform", "var_scaling_normal_fan_in", "var_scaling_normal_fan_out",
           "var_scaling_normal_fan_avg", "var_scaling_uniform_fan_in", "var_scaling_uniform_fan_out", "var_scaling_uniform_fan_avg")
DISTRIBUTIONS = ("normal", "uniform", "truncated_normal", "log_normal", "binomial", "constant", "orthogonal")
TAG = 0x80000000
ROUNDS = 16


def fans(layer):
    """(fanIn, fanOut) of an oracle layer: conv and deconv nIn kH kW and nOut kH kW / (sH sW), dense nIn and nOut."""
    if isinstance(layer, (o.Conv2D, o.Deconv2D)):
        return layer.fans()
    return layer.n_in, layer.n_out


def layer_of(spec):
    """The oracle layer of a GEMM spec (n_in given): what fans() and the W shape come from."""
    k, s, p = spec.get("kernel", (1, 1)), spec.get("stride", (1, 1)), spec.get("padding", (0, 0))
    if spec["type"] == "conv2d":
        return o.Conv2D(spec["n_in"], spec["n_out"], tuple(k), tuple(s), tuple(p))
    if spec["type"] == "deconv2d":
        return o.Deconv2D(spec["n_in"], spec["n_out"], tuple(k), tuple(s), tuple(p))
    return o.Dense(spec["n_in"], spec["n_out"])


def w_size(layer) -> int:
    k = getattr(layer, "k", (1, 1))
    return layer.n_in * layer.n_out * k[0] * k[1]


def resolve(wi, layer, q: WeightInitQuirks = WQ):
    """What the scheme draws on the layer: (kind, a, b) with kind a distribution name or "identity"; a, b fp32, each computed in double and
    rounded once (binomial: (nTrials, p))."""
    scheme = wi["weight_init"]
    fi, fo = (float(v) for v in fans(layer))
    N = lambda sd: ("normal", np.float32(0), np.float32(sd))
    U = lambda r: ("uniform", -np.float32(r), np.float32(r))
    T = lambda sd: ("truncated_normal", np.float32(0), np.float32(sd))
    u3 = lambda fan: 3.0 / math.sqrt(fan) if q.var_scaling_uniform_three_over_sqrt else math.sqrt(3.0 / fan)
    if scheme == "distribution":
        d = wi["distribution"]
        kind = d["distribution"]
        if kind in ("normal", "truncated_normal", "log_normal"):
            return kind, np.float32(d["mean"]), np.float32(d["std"])
        if kind == "uniform":
            return kind, np.float32(d["lower"]), np.float32(d["upper"])
        if kind == "binomial":
            return kind, int(d["n_trials"]), np.float32(d["p"])
        if kind == "constant":
            return kind, np.float32(d["value"]), np.float32(0)
        raise ValueError(kind)
    table = {
        "zero": lambda: ("constant", np.float32(0), np.float32(0)),
        "ones": lambda: ("constant", np.float32(1), np.float32(0)),
        "sigmoid_uniform": lambda: U(4.0 * math.sqrt(6.0 / (fi + fo))),
        "normal": lambda: N(1.0 / math.sqrt(fi) if q.normal_scaled_by_fan_in else 1.0),
        "lecun_normal": lambda: N(1.0 / math.sqrt(fi)),
        "uniform": lambda: U(1.0 / math.sqrt(fi)),
        "xavier": lambda: N(math.sqrt(2.0 / (fi + fo))),
        "xavier_uniform": lambda: U(math.sqrt(6.0) / math.sqrt(fi + fo)),
        "xavier_fan_in": lambda: N(1.0 / math.sqrt(fi)),
        "xavier_legacy": lambda: N(1.0 / math.sqrt(layer.n_in + layer.n_out) if q.xavier_legacy_shape01 else 1.0 / math.sqrt(fi + fo)),
        "relu": lambda: N(math.sqrt(2.0 / fi)),
        "relu_uniform": lambda: U(math.sqrt(6.0 / fi)),
        "identity": lambda: ("identity", np.float32(0), np.float32(0)),
        "lecun_uniform": lambda: U(3.0 / math.sqrt(fi) if q.lecun_uniform_three_over_sqrt else math.sqrt(3.0 / fi)),
        "var_scaling_normal_fan_in": lambda: T(math.sqrt(1.0 / fi)),
        "var_scaling_normal_fan_out": lambda: T(math.sqrt(1.0 / fo)),
        "var_scaling_normal_fan_avg": lambda: T(math.sqrt(2.0 / (fi + fo))),
        "var_scaling_uniform_fan_in": lambda: U(u3(fi)),
        "var_scaling_uniform_fan_out": lambda: U(u3(fo)),
        "var_scaling_uniform_fan_avg": lambda: U(u3((fi + fo) / 2.0)),
    }
    return table[scheme]()


def words(seed, layer_index, n, k):
    """Round k's Philox word of every view index j < n (uint64 holding uint32)."""
    seed = int(seed) or 666
    g = np.arange((n + 3) // 4, dtype=np.uint64)
    w = np.stack(o.philox4x32_10((g, int(k), 0, int(layer_index) | TAG), (seed & 0xFFFFFFFF, seed >> 32)), -1).ravel()
    return w[:n]


def normals(seed, layer_index, n, k=0):
    """Round k's float64 Box-Muller normal of every view index j < n: pair (x0, x1) -> z0, z1, pair (x2, x3) -> z2, z3."""
    w4 = words(seed, layer_index, 4 * ((n + 3) // 4), k).reshape(-1, 4)        # a tail element's pair partner exists past n
    z = np.empty(w4.shape)
    z[:, 0], z[:, 1] = nr.box_muller(w4[:, 0], w4[:, 1])
    z[:, 2], z[:, 3] = nr.box_muller(w4[:, 2], w4[:, 3])
    return z.ravel()[:n]


def truncated_z(seed, layer_index, n, q: WeightInitQuirks = WQ):
    """The z of the first round k < 16 with |z| <= the truncation, else round 15's z clamped."""
    lim = q.truncation_sigmas
    z = np.zeros(n)
    todo = np.ones(n, bool)
    for k in range(ROUNDS):
        t = normals(seed, layer_index, n, k)
        hit = todo & (np.abs(t) <= lim)
        z[hit] = t[hit]
        todo &= ~hit
        if k == ROUNDS - 1:
            z[todo] = np.clip(t[todo], -lim, lim)
        if not todo.any():
            break
    return z


def fmaf(a, b, c):
    """fp32 fmaf(a, b, c) for fp32 a, c and float64 b: exact in double where a * b fits (uniform draws), one rounding to fp32."""
    return (np.float64(np.float32(a)) * np.asarray(b, np.float64) + np.float64(np.float32(c))).astype(np.float32)


def draw(kind, a, b, n, seed, layer_index, n_in=None, q: WeightInitQuirks = WQ):
    """n fp32 values in view order.  identity: n_in = nIn of the square dense W (view index j = o nIn + i)."""
    if kind == "normal":
        return fmaf(b, normals(seed, layer_index, n), a)
    if kind == "log_normal":
        return np.exp(fmaf(b, normals(seed, layer_index, n), a).astype(np.float64)).astype(np.float32)
    if kind == "truncated_normal":
        return fmaf(b, truncated_z(seed, layer_index, n, q), a)
    if kind == "uniform":
        u = (words(seed, layer_index, n, 0) >> np.uint64(8)).astype(np.float64) * 2.0 ** -24
        return fmaf(np.float32(b) - np.float32(a), u, a)
    if kind == "binomial":
        thr = np.uint64(math.floor(float(np.float32(b)) * 2.0 ** 32))
        c = np.zeros(n, np.int64)
        for t in range(int(a)):
            c += words(seed, layer_index, n, t) < thr
        return c.astype(np.float32)
    if kind == "constant":
        return np.full(n, np.float32(a), np.float32)
    if kind == "identity":
        j = np.arange(n)
        return (j // n_in == j % n_in).astype(np.float32)
    raise ValueError(kind)


def weights(wi, layer, seed, layer_index, q: WeightInitQuirks = WQ):
    """W of the layer in DL4J's flattened view order (b2g_net_get_param's), fp32."""
    kind, a, b = resolve(wi, layer, q)
    if kind == "identity" and (not isinstance(layer, o.Dense) or layer.n_in != layer.n_out):
        raise ValueError("IDENTITY needs a square dense W")
    return draw(kind, a, b, w_size(layer), seed, layer_index, layer.n_in, q)


def init_layer(layer, wi, seed, layer_index, q: WeightInitQuirks = WQ):
    """The oracle layer's W and b (if it has one) as b2g_net_init_weights leaves them, in the layer's dtype."""
    flat = weights(wi, layer, seed, layer_index, q)
    W = layer.params["W"]
    order = "F" if isinstance(layer, o.Dense) else "C"
    layer.params["W"] = flat.astype(W.dtype).reshape(W.shape, order=order)
    if "b" in layer.params:
        layer.params["b"] = np.full(layer.params["b"].shape, np.float32(wi.get("bias_init", 0.0)), layer.params["b"].dtype)
    return layer


def expected_moments(kind, a, b):
    """(mean, variance) of the draw kind with fp32 parameters a, b: the normal's; the uniform's; the 2-sigma truncated normal's; the
    log-normal's; the binomial's n p, n p (1 - p); a constant's."""
    a, b = float(a), float(b)
    if kind == "normal":
        return a, b * b
    if kind == "uniform":
        return (a + b) / 2, (b - a) ** 2 / 12
    if kind == "truncated_normal":
        t = WQ.truncation_sigmas
        phi = math.exp(-t * t / 2) / math.sqrt(2 * math.pi)
        mass = math.erf(t / math.sqrt(2))
        return a, b * b * (1 - 2 * t * phi / mass)
    if kind == "log_normal":
        return math.exp(a + b * b / 2), (math.exp(b * b) - 1) * math.exp(2 * a + b * b)
    if kind == "binomial":
        return a * b, a * b * (1 - b)
    return a, 0.0
