"""Host-side mirror of the C-ABI objects: Context (b2g_ctx), Net (b2g_net ~ ComputationGraph), Gan (b2g_gan).

Layer specs are plain dicts (see models.py); `layer_desc` turns one into the C struct the Java facade's layer
builders fill (ConvolutionLayer.Builder(kH,kW).stride().padding().nIn().nOut() ... J:135-140).
All tensors cross as NumPy fp32 arrays in DL4J layouts (NCHW / [N,F]; parameters in flattened-view order).
"""
from __future__ import annotations

import copy
import ctypes as C
import math
from typing import Dict, List, Optional, Sequence

import numpy as np

from . import _lib
from ._lib import GanConfig, LayerDesc, LrSchedule, NetConfig, check

LAYER_TYPES = {"conv2d": 0, "deconv2d": 1, "batchnorm": 2, "dense": 3, "activation": 4, "maxpool": 5, "upsample2d": 6,
               "output": 7, "loss": 8, "ff_to_cnn": 9, "cnn_to_ff": 10, "dropout": 11, "subsampling": 12, "global_pooling": 13,
               "cnn_loss": 14, "elementwise": 15, "merge": 16, "prelu": 17}
# ElementWiseVertex.Op -> b2g_elementwise_op, carried in b2g_layer_desc.act of "elementwise" specs (semantics in include/b200gan.h)
ELEMENTWISE_OPS = {"add": 0, "subtract": 1, "product": 2, "average": 3, "max": 4}
VERTEX_TYPES = ("elementwise", "merge")
# org.deeplearning4j.nn.conf.layers.PoolingType -> b2g_pooling, carried in b2g_layer_desc.act of "subsampling" (avg / sum / pnorm; max is the
# "maxpool" layer) and "global_pooling" (all four) specs; PNORM's p in act_alpha (formulas at b2g_pooling in include/b200gan.h)
POOLINGS = {"max": 0, "avg": 1, "sum": 2, "pnorm": 3}
GLOBAL_PNORM_DEFAULT = 2             # GlobalPoolingLayer.Builder().pnorm default
# org.nd4j.linalg.activations.Activation -> b2g_activation (codes 5-16: formulas at b2g_activation in include/b200gan.h)
ACTS = {"identity": 0, "tanh": 1, "sigmoid": 2, "relu": 3, "lrelu": 4, "elu": 5, "selu": 6, "softplus": 7, "softsign": 8, "hardtanh": 9,
        "hardsigmoid": 10, "relu6": 11, "swish": 12, "cube": 13, "rationaltanh": 14, "rectifiedtanh": 15, "thresholdedrelu": 16}
# the spec's "alpha" when it has none: LeakyReLU's alpha 0.01, ELU's alpha and ThresholdedReLU's theta 1.0 (DL4J's defaults)
ACT_ALPHA_DEFAULTS = {"elu": 1.0, "thresholdedrelu": 1.0}
# LossFunctions.LossFunction -> b2g_loss.  XENT / MCXENT imply their sigmoid / softmax; the others apply the spec's "activation" (b2g_loss)
LOSSES = {"xent": 0, "mcxent": 1, "mse": 2, "l1": 3, "l2": 4, "mae": 5, "hinge": 6, "squared_hinge": 7, "wasserstein": 8}
UPDATERS = {"sgd": 0, "rmsprop": 1, "adam": 2, "noop": 3, "nesterovs": 4, "adagrad": 5, "adamax": 6, "nadam": 7, "amsgrad": 8, "adadelta": 9}
# updaters without a learning rate: their layers take no schedule and have no getLearningRate
NO_LR_UPDATERS = ("noop", "adadelta")
# DL4J GradientNormalization -> b2g_gradient_normalization (DL4J's ordinals).  ClipElementWiseAbsoluteValue is the `grad_clip` argument of Net.
GRADIENT_NORMALIZATIONS = {"none": 0, "renormalize_l2_per_layer": 1, "renormalize_l2_per_param_type": 2, "clip_l2_per_layer": 4,
                           "clip_l2_per_param_type": 5}
# DL4J ISchedule -> b2g_schedule_kind / b2g_schedule_type (models.py builds the dicts: exponential_schedule, ..., map_schedule)
SCHEDULE_KINDS = {"exponential": 1, "inverse": 2, "sigmoid": 3, "step": 4, "map": 5}
SCHEDULE_TYPES = {"iteration": 0, "epoch": 1}
FP32, BF16 = 0, 1


def is_schedule(lr) -> bool:
    return isinstance(lr, dict)


def schedule_value(sched: Dict, i) -> float:
    """ISchedule.valueAt in double at counter value i (the arithmetic of b2g_lr_schedule in include/b200gan.h; the device rounds it to fp32)."""
    k, i = sched["schedule"], float(i)
    if k == "exponential":
        return sched["initial"] * math.pow(sched["gamma"], i)
    if k == "inverse":
        return sched["initial"] / math.pow(1.0 + sched["gamma"] * i, sched["power"])
    if k == "sigmoid":
        return sched["initial"] / (1.0 + math.exp(-sched["gamma"] * (i - sched["step"])))
    if k == "step":
        return sched["initial"] * math.pow(sched["decay_rate"], math.floor(i / sched["step"]))
    if k == "map":
        below = [(int(key), float(v)) for key, v in sched["values"] if int(key) <= i]
        return max(below)[1] if below else 0.0          # no key <= i: the engine rejects such a map (it must hold key 0)
    raise ValueError(f"unknown learning-rate schedule {k!r}")


def constant_lr(lr) -> float:
    """The float b2g_layer_desc.lr carries for an updater's lr: the number itself, or a schedule's value at 0 (what the Java facade's
    updaters write for new Adam(ISchedule): schedule.valueAt(0, 0)).  The engine returns to it when the layer's schedule is cleared."""
    return float(lr) if not is_schedule(lr) else float(schedule_value(lr, 0))


def schedule_struct(sched: Optional[Dict]):
    """A schedule dict (models.py) -> (b2g_lr_schedule, arrays it points into).  None -> kind NONE."""
    s = LrSchedule()
    if sched is None:
        return s, ()
    if sched.get("schedule") not in SCHEDULE_KINDS:
        raise ValueError(f"unknown learning-rate schedule {sched.get('schedule')!r}; one of {sorted(SCHEDULE_KINDS)} (PolySchedule is not supported)")
    if sched.get("type", "iteration") not in SCHEDULE_TYPES:
        raise ValueError(f"unknown schedule type {sched.get('type')!r}; one of {sorted(SCHEDULE_TYPES)}")
    s.kind, s.type = SCHEDULE_KINDS[sched["schedule"]], SCHEDULE_TYPES[sched.get("type", "iteration")]
    s.initial, s.gamma, s.power = sched.get("initial", 0.0), sched.get("gamma", 0.0), sched.get("power", 0.0)
    s.step, s.decay_rate = sched.get("step", 0.0), sched.get("decay_rate", 0.0)
    keep = ()
    if sched["schedule"] == "map":
        pairs = [(int(k), float(v)) for k, v in sched["values"]]
        keys = np.array([k for k, _ in pairs], np.int32); vals = np.array([v for _, v in pairs], np.float64)
        s.n_map = len(pairs)
        s.map_keys = keys.ctypes.data_as(C.POINTER(C.c_int32)); s.map_values = vals.ctypes.data_as(C.POINTER(C.c_double))
        keep = (keys, vals)
    return s, keep


# PReLULayer (B2G_LAYER_PRELU in include/b200gan.h): DL4J's 1-based sharedAxes (1 = C, 2 = H, 3 = W) -> the bit mask b2g_layer_desc.act carries
def prelu_shared_mask(spec: Dict) -> int:
    """The shared-axes bit mask of a "prelu" spec; ValueError for an axis outside 1-3 (the engine refuses a bit outside the input's rank)."""
    axes = [int(a) for a in spec.get("shared_axes", ())]
    if any(a not in (1, 2, 3) for a in axes):
        raise ValueError(f"prelu layer {spec.get('name', '')!r}: shared axes {axes}; DL4J's axes are 1 (C), 2 (H) and 3 (W)")
    return sum(1 << (a - 1) for a in set(axes))


def prelu_groups(rows: int, row_elems: int) -> int:
    """The row groups of a PReLU backward over `rows` rows of `row_elems` elements (the summation order at B2G_LAYER_PRELU in
    include/b200gan.h): each writes one fp32 slope partial per row element."""
    bx = -(-row_elems // 2048)
    g0 = max(1, min(rows, 64, max(1, 1024 // bx)))
    rpg = -(-rows // g0)
    return -(-rows // rpg)


# a PReLU layer's slopes take ZERO, ONES and DISTRIBUTION (the other schemes need fans it does not have)
PRELU_WEIGHT_INITS = ("zero", "ones", "distribution")


def layer_has_lr(spec: Dict) -> bool:
    """A layer whose updater has a learning rate: it has parameters, is not frozen and its updater is neither NoOp nor AdaDelta.  A spec
    without an updater is Sgd with lr 0 (layer_desc), so it has one.  The engine applies the same rule (engine.cu layer_has_lr)."""
    u = spec.get("updater") or {"kind": "sgd"}
    return spec["type"] in ("conv2d", "deconv2d", "dense", "output", "batchnorm", "prelu") and not spec.get("frozen", False) and u["kind"] not in NO_LR_UPDATERS


def follow_lr_schedule(specs: List[Dict], constant: List[float], schedule: Optional[Dict], layer: Optional[str] = None):
    """Writes what b2g_net_set_lr_schedule(layer, schedule) did into the layer specs a checkpoint saves: the schedule, or (schedule None) the
    layer's creation-time constant lr constant[i] the engine returns to.  layer None: every layer with a learning rate; a name: the first layer
    of that name, as the engine looks it up."""
    for i, sp in enumerate(specs):
        if layer is not None and sp.get("name") != layer:
            continue
        if layer_has_lr(sp):
            if not sp.get("updater"):
                sp["updater"] = {"kind": "sgd", "lr": 0.0}
            sp["updater"]["lr"] = copy.deepcopy(schedule) if schedule is not None else constant[i]
        if layer is not None:
            break


# org.deeplearning4j.nn.conf.constraint.* -> b2g_constraint_kind (models.py builds the dicts: max_norm, min_max_norm, unit_norm, non_negative)
CONSTRAINT_KINDS = {"max_norm": 0, "min_max_norm": 1, "unit_norm": 2, "non_negative": 3}
CONSTRAINT_ON = ("all", "weights", "bias")      # also the order a layer's lists apply in: constrainAllParameters, Weights, Bias
GEMM_TYPES = ("conv2d", "deconv2d", "dense", "output")
# the layers whose W takes l1 / l2: the GEMM layers and PReLU's slopes
REG_TYPES = GEMM_TYPES + ("prelu",)


def constraint_params(spec: Dict, on: str) -> List[str]:
    """The parameters a constraint with target `on` applies to on a layer of this spec (DL4J initializeConstraints): "weights" is W of a
    conv2d / deconv2d / dense / output layer (nothing on BatchNorm, whose weight keys are empty); "bias" is b where the layer has one; "all"
    is every parameter, BatchNorm's gamma, beta, mean and var included.  Layers without parameters and FrozenLayers get nothing."""
    if on not in CONSTRAINT_ON:
        raise ValueError(f"constraint target {on!r}; one of {list(CONSTRAINT_ON)}")
    t, bias = spec["type"], spec.get("has_bias", True)
    if spec.get("frozen", False):
        return []
    if t in GEMM_TYPES:
        return {"weights": ["W"], "bias": ["b"] if bias else [], "all": (["b", "W"] if bias else ["W"])}[on]
    if t == "batchnorm":
        return ["gamma", "beta", "mean", "var"] if on == "all" else []
    return []


def constraint_struct(c: Dict):
    """A constraint dict (models.py) -> b2g_constraint."""
    if c.get("constraint") not in CONSTRAINT_KINDS:
        raise ValueError(f"unknown constraint {c.get('constraint')!r}; one of {sorted(CONSTRAINT_KINDS)}")
    s = _lib.Constraint()
    s.kind = CONSTRAINT_KINDS[c["constraint"]]
    s.dims_mask = sum(1 << int(d) for d in set(c.get("dims", ())))
    s.max_norm, s.min_norm, s.rate = c.get("max", 0.0), c.get("min", 0.0), c.get("rate", 1.0)
    return s


def resolve_constraints(spec: Dict) -> Dict[str, List[Dict]]:
    """A layer spec's "constraints" as parameter name -> the ordered list each tensor runs: all-parameter constraints, then weight, then bias
    constraints, each in the order given."""
    out: Dict[str, List[Dict]] = {}
    for c in spec.get("constraints", ()):
        constraint_params(spec, c.get("on", "weights"))          # rejects an unknown target
    for on in CONSTRAINT_ON:
        for c in spec.get("constraints", ()):
            if c.get("on", "weights") == on:
                for p in constraint_params(spec, on):
                    out.setdefault(p, []).append(c)
    return out


# Regularization of a GEMM layer spec (b2g_regularization in include/b200gan.h): "l1" and "l2" on W, "l1_bias" and "l2_bias" on b, applied
# after the updater and added to the score.  "l2" travels in b2g_layer_desc; a spec with any of the other three gets them all set at creation.
REGULARIZATION_KEYS = ("l1", "l2", "l1_bias", "l2_bias")


def check_regularization(values: Dict, where: str = "regularization") -> Dict[str, float]:
    """The coefficients of a regularization dict, each a finite number >= 0 as b2g_net_set_regularization requires (DL4J ignores a value
    <= 0; refusing negatives is a deliberate deviation).  ValueError for an unknown key or a bad value."""
    unknown = set(values) - set(REGULARIZATION_KEYS)
    if unknown:
        raise ValueError(f"{where}: unknown key(s) {sorted(unknown)}; one of {list(REGULARIZATION_KEYS)}")
    out = {}
    for k, v in values.items():
        f = np.float32(v)
        if not (np.isfinite(f) and f >= 0):
            raise ValueError(f"{where}: {k} = {v!r} must be finite and >= 0")
        out[k] = float(v)
    return out


def spec_regularization(spec: Dict) -> Dict[str, float]:
    """The four coefficients a GEMM layer spec carries (a missing key is 0)."""
    return {k: float(spec.get(k, 0.0)) for k in REGULARIZATION_KEYS}


def resolve_regularization(specs: List[Dict], regularization: Optional[Dict] = None) -> List[Dict]:
    """Fills in the global builder's coefficients (regularization, may be None) in place: every non-frozen conv, deconv, dense, output and
    prelu spec takes each key it does not set itself, as DL4J's builder fills in a layer's NaN fields.  Then checks each such spec's "l1",
    "l1_bias" and "l2_bias" ("l2" is the desc's, as before).  Returns specs."""
    if regularization is not None:
        glob = check_regularization(regularization)
        for sp in specs:
            if sp["type"] in REG_TYPES and not sp.get("frozen", False):
                for k, v in glob.items():
                    sp.setdefault(k, v)
    for sp in specs:
        if sp["type"] in REG_TYPES:
            check_regularization({k: sp[k] for k in REGULARIZATION_KEYS if k in sp and k != "l2"}, f"layer {sp.get('name', '')!r}")
    return specs


def regularization_struct(values: Dict) -> "_lib.Regularization":
    r = _lib.Regularization()
    for k in REGULARIZATION_KEYS:
        setattr(r, k, float(values.get(k, 0.0)))
    return r


def _fp(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _f32(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float32)


def resolve_vertices(specs: Sequence[Dict]) -> List[Optional[tuple]]:
    """Each vertex spec's ("inputs": [name, name]) as (j, order): j the index of the skip source, order 0 when the inputs are (spine, j) and 1
    when they are (j, spine); None for the other specs.  The spine is the previous spec.  ValueError for a graph that is not spine plus skip:
    a vertex without exactly two inputs, neither of them the previous spec, a name that is not an earlier spec or names several, the net input
    as an input, or a loss-bearing source."""
    out: List[Optional[tuple]] = []
    for i, sp in enumerate(specs):
        if sp["type"] not in VERTEX_TYPES:
            out.append(None)
            continue
        name, inputs = sp.get("name", ""), list(sp.get("inputs", ()))
        if len(inputs) != 2:
            raise ValueError(f"vertex {name!r}: needs exactly two inputs, got {inputs}")
        if i == 0:
            raise ValueError(f"vertex {name!r}: the net input cannot be a vertex input")
        if sp["type"] == "elementwise" and sp.get("op") not in ELEMENTWISE_OPS:
            raise ValueError(f"vertex {name!r}: unknown op {sp.get('op')!r}; one of {sorted(ELEMENTWISE_OPS)}")
        earlier = [s.get("name", "") for s in specs[:i]]
        spine = earlier[-1]
        if inputs[0] == spine:
            order, other = 0, inputs[1]
        elif inputs[1] == spine:
            order, other = 1, inputs[0]
        else:
            raise ValueError(f"vertex {name!r}: one input must be the previous layer {spine!r} (spine plus skip), got {inputs}")
        hits = [j for j, nm in enumerate(earlier) if nm == other]
        if len(hits) != 1:
            raise ValueError(f"vertex {name!r}: input {other!r} names {len(hits)} earlier layers (needs exactly one)")
        if specs[hits[0]]["type"] in ("loss", "cnn_loss", "output"):
            raise ValueError(f"vertex {name!r}: input {other!r} is a loss-bearing layer")
        out.append((hits[0], order))
    return out


# IDropout of a "dropout" spec (b2g_dropout_kind in include/b200gan.h): kind -> (code, the key of its value).  No "kind": Dropout(p).
DROPOUT_KINDS = {"dropout": (0, "p"), "gaussian_dropout": (1, "rate"), "gaussian_noise": (2, "stddev"), "alpha_dropout": (3, "p"),
                 "spatial_dropout": (4, "p")}


def dropout_kind_value(spec: Dict):
    """(b2g_dropout_kind code, value) of a "dropout" spec; the value is the retain probability p, the rate or the stddev: a number, or a
    schedule dict (new GaussianNoise(ISchedule)) whose value at 0 the desc carries, as for a scheduled lr; the schedule is set after creation."""
    kind = spec.get("kind", "dropout")
    if kind not in DROPOUT_KINDS:
        raise ValueError(f"dropout layer {spec.get('name', '')!r}: unknown kind {kind!r}; one of {sorted(DROPOUT_KINDS)}")
    code, key = DROPOUT_KINDS[kind]
    return code, constant_lr(spec[key])


def dropout_value_key(spec: Dict) -> str:
    return DROPOUT_KINDS[spec.get("kind", "dropout")][1]


# Weight noise of a GEMM layer spec's "weight_noise" (b2g_weight_noise in include/b200gan.h; models.drop_connect / models.weight_noise)
WEIGHT_NOISE_KINDS = {"drop_connect": 1, "weight_noise": 2}
DISTRIBUTIONS = {"normal": (0, "mean", "std"), "uniform": (1, "lower", "upper")}


def weight_noise_struct(wn: Optional[Dict]):
    """A weight-noise dict (models.py) -> (b2g_weight_noise, what it points into).  None -> kind NONE."""
    s = _lib.WeightNoise()
    if wn is None:
        return s, ()
    kind = wn.get("weight_noise")
    if kind not in WEIGHT_NOISE_KINDS:
        raise ValueError(f"unknown weight noise {kind!r}; one of {sorted(WEIGHT_NOISE_KINDS)}")
    s.kind, s.apply_to_bias = WEIGHT_NOISE_KINDS[kind], int(bool(wn.get("apply_to_bias", False)))
    keep = ()
    if kind == "drop_connect":
        s.p = constant_lr(wn["p"])
        if is_schedule(wn["p"]):
            sched, arrays = schedule_struct(wn["p"])
            s.p_schedule = C.pointer(sched)
            keep = (sched, arrays)
    else:
        dist = wn["distribution"]
        if dist.get("distribution") not in DISTRIBUTIONS:
            raise ValueError(f"unknown distribution {dist.get('distribution')!r}; one of {sorted(DISTRIBUTIONS)}")
        code, ka, kb = DISTRIBUTIONS[dist["distribution"]]
        s.dist, s.a, s.b = code, float(dist[ka]), float(dist[kb])
        s.additive = int(bool(wn.get("additive", True)))
    return s, keep


# Weight initialization of a GEMM layer spec's "weight_init" (b2g_weight_init in include/b200gan.h; models.weight_init): DL4J's WeightInit
# ordinals, and every b2g_distribution_kind with its two parameter keys (ORTHOGONAL is refused)
WEIGHT_INIT_SCHEMES = {"distribution": 0, "zero": 1, "ones": 2, "sigmoid_uniform": 3, "normal": 4, "lecun_normal": 5, "uniform": 6, "xavier": 7,
                       "xavier_uniform": 8, "xavier_fan_in": 9, "xavier_legacy": 10, "relu": 11, "relu_uniform": 12, "identity": 13,
                       "lecun_uniform": 14, "var_scaling_normal_fan_in": 15, "var_scaling_normal_fan_out": 16, "var_scaling_normal_fan_avg": 17,
                       "var_scaling_uniform_fan_in": 18, "var_scaling_uniform_fan_out": 19, "var_scaling_uniform_fan_avg": 20}
INIT_DISTRIBUTIONS = {"normal": (0, "mean", "std"), "uniform": (1, "lower", "upper"), "truncated_normal": (2, "mean", "std"),
                      "log_normal": (3, "mean", "std"), "binomial": (4, "n_trials", "p"), "constant": (5, "value", None),
                      "orthogonal": (6, "gain", None)}


def weight_init_struct(wi: Dict, spec: Optional[Dict] = None):
    """A weight-init dict (models.weight_init) -> b2g_weight_init, with ValueError for whatever b2g_net_init_weights refuses: an unknown
    scheme or distribution, OrthogonalDistribution, DISTRIBUTION without a distribution or with a non-finite or out-of-range parameter, a
    non-finite bias_init; with the layer's spec also IDENTITY on a convolution or on a dense layer whose given nIn != nOut."""
    scheme = wi.get("weight_init")
    if scheme not in WEIGHT_INIT_SCHEMES:
        raise ValueError(f"unknown weight init {scheme!r}; one of {sorted(WEIGHT_INIT_SCHEMES)}")
    s = _lib.WeightInit()
    s.scheme, s.bias_init = WEIGHT_INIT_SCHEMES[scheme], float(wi.get("bias_init", 0.0))
    if not np.isfinite(np.float32(s.bias_init)):
        raise ValueError(f"bias_init {wi.get('bias_init')!r} is not finite")
    if scheme == "distribution":
        dist = wi.get("distribution") or {}
        kind = dist.get("distribution")
        if kind not in INIT_DISTRIBUTIONS:
            raise ValueError(f"weight init 'distribution' needs a distribution; got {kind!r}, one of {sorted(INIT_DISTRIBUTIONS)}")
        if kind == "orthogonal":
            raise ValueError("OrthogonalDistribution is not supported (it needs an SVD)")
        code, ka, kb = INIT_DISTRIBUTIONS[kind]
        s.dist, s.a, s.b = code, float(dist[ka]), float(dist[kb]) if kb else 0.0
        a, b = np.float32(s.a), np.float32(s.b)
        if not (np.isfinite(a) and np.isfinite(b)):
            raise ValueError(f"{kind} distribution parameters must be finite: {dist}")
        if kind in ("normal", "truncated_normal", "log_normal") and b < 0:
            raise ValueError(f"{kind} distribution std {dist['std']} < 0")
        if kind == "uniform" and b < a:
            raise ValueError(f"uniform distribution upper {dist['upper']} < lower {dist['lower']}")
        if kind == "binomial" and not (0 <= a <= 65536 and a == np.floor(a) and 0 <= b <= 1):
            raise ValueError(f"binomial distribution needs a whole n_trials in [0, 65536] and p in [0, 1]: {dist}")
    if spec is not None and spec["type"] == "prelu" and scheme not in PRELU_WEIGHT_INITS:
        raise ValueError(f"layer {spec.get('name', '')!r}: weight init {scheme!r} needs fans, which a PReLU's slopes do not have; one of {list(PRELU_WEIGHT_INITS)}")
    if scheme == "identity" and spec is not None:
        if spec["type"] not in ("dense", "output"):
            raise ValueError(f"layer {spec.get('name', '')!r}: weight init 'identity' needs a dense or output layer")
        if spec.get("n_in") and spec["n_in"] != spec.get("n_out"):
            raise ValueError(f"layer {spec.get('name', '')!r}: weight init 'identity' needs nIn == nOut, got {spec['n_in']} and {spec.get('n_out')}")
    return s


def layer_desc(spec: Dict, skip: Optional[tuple] = None) -> LayerDesc:
    """skip: the vertex's (j, order) from resolve_vertices."""
    d = LayerDesc()
    d.type = LAYER_TYPES[spec["type"]]
    d.name = spec.get("name", "").encode()[:63]
    d.n_in, d.n_out = spec.get("n_in", 0), spec.get("n_out", 0)
    k, s, p = spec.get("kernel", (1, 1)), spec.get("stride", (1, 1)), spec.get("padding", (0, 0))
    if spec["type"] == "upsample2d":
        k = (spec.get("size", 2), spec.get("size", 2))
    d.k_h, d.k_w, d.s_h, d.s_w, d.p_h, d.p_w = k[0], k[1], s[0], s[1], p[0], p[1]
    d.has_bias = 1 if spec.get("has_bias", True) else 0
    act = spec.get("activation", "identity")
    d.act = ACTS[act]
    d.act_alpha = spec.get("alpha", ACT_ALPHA_DEFAULTS.get(act, 0.01))
    if spec["type"] == "dropout":       # DropoutLayer.Builder(IDropout): the b2g_dropout_kind in act, its value in act_alpha
        d.act, d.act_alpha = dropout_kind_value(spec)
    if spec["type"] in ("subsampling", "global_pooling"):      # the pooling kind in act, PNORM's p in act_alpha (0 = none given: refused)
        d.act = POOLINGS[spec.get("pooling", "max")]
        d.act_alpha = float(spec.get("pnorm", GLOBAL_PNORM_DEFAULT if spec["type"] == "global_pooling" else 0))
    u = spec.get("updater") or {"kind": "sgd", "lr": 0.0}
    d.updater = UPDATERS[u["kind"]]
    d.lr = constant_lr(u.get("lr", 0.0))     # new Adam(ISchedule): the schedule itself is set after b2g_net_create
    if u["kind"] == "rmsprop":          # RmsProp(learningRate, rmsDecay, epsilon)
        d.beta1, d.beta2, d.eps = u.get("rms_decay", 0.95), 0.0, u.get("eps", 1e-8)
    elif u["kind"] == "nesterovs":      # Nesterovs(learningRate, momentum): momentum in beta1
        d.beta1, d.beta2, d.eps = u.get("momentum", 0.9), 0.0, 0.0
    elif u["kind"] == "adagrad":        # AdaGrad(learningRate, epsilon)
        d.beta1, d.beta2, d.eps = 0.0, 0.0, u.get("eps", 1e-6)
    elif u["kind"] == "adadelta":       # AdaDelta(rho, epsilon): rho in beta1, no learning rate
        d.lr, d.beta1, d.beta2, d.eps = 0.0, u.get("rho", 0.95), 0.0, u.get("eps", 1e-6)
    else:
        d.beta1, d.beta2, d.eps = u.get("beta1", 0.9), u.get("beta2", 0.999), u.get("eps", 1e-8)
    d.l2 = spec.get("l2", 0.0)
    d.bn_decay, d.bn_eps = spec.get("decay", 0.9), spec.get("eps", 1e-5)
    to = spec.get("to", (0, 0, 0))      # FeedForwardToCnnPreProcessor(h, w, c)
    d.pre_h, d.pre_w, d.pre_c = to
    d.loss = LOSSES[spec.get("loss", "xent")]
    d.frozen = 1 if spec.get("frozen", False) else 0
    if spec["type"] in VERTEX_TYPES:       # the op in act, the skip source and the input order in pre_h / pre_w
        d.act = ELEMENTWISE_OPS[spec["op"]] if spec["type"] == "elementwise" else 0
        d.pre_h, d.pre_w = skip
    if spec["type"] == "prelu":            # the shared-axes mask in act, inputShape [C, H, W] or [F] in pre_c, pre_h, pre_w (0: not given)
        d.act, d.act_alpha = prelu_shared_mask(spec), 0.0
        shape = [int(v) for v in spec.get("input_shape", ())]
        if len(shape) not in (0, 1, 3):
            raise ValueError(f"prelu layer {spec.get('name', '')!r}: input_shape {shape} is neither [C, H, W] nor [F]")
        d.pre_c, d.pre_h, d.pre_w = (shape + [0, 0, 0])[:3] if len(shape) != 3 else shape
    return d


class Context:
    """b2g_ctx: one CUDA device + stream.  Replaces Nd4j backend selection / CudaEnvironment setup (J:103-115)."""

    def __init__(self, device: int = 0):
        self.lib = _lib.load()
        h = C.c_void_p()
        check(self.lib.b2g_ctx_create(device, C.byref(h)))
        self.h = h
        self.world, self.rank = 1, 0

    def sync(self):
        check(self.lib.b2g_sync(self.h))

    def timer_start(self):
        check(self.lib.b2g_timer_start(self.h))

    def timer_stop_ms(self) -> float:
        v = C.c_float()
        check(self.lib.b2g_timer_stop_ms(self.h, C.byref(v)))
        return v.value

    def flush_l2(self):
        check(self.lib.b2g_flush_l2(self.h))

    def launch_count(self) -> int:
        v = C.c_uint64()
        check(self.lib.b2g_launch_count(self.h, C.byref(v)))
        return v.value

    def device_info(self):
        sm, mj, mn, mem = C.c_int32(), C.c_int32(), C.c_int32(), C.c_uint64()
        check(self.lib.b2g_device_info(self.h, C.byref(sm), C.byref(mj), C.byref(mn), C.byref(mem)))
        return dict(sm_count=sm.value, cc=(mj.value, mn.value), mem_bytes=mem.value)

    def comm_init(self, world: int, rank: int, unique_id: bytes):
        buf = C.create_string_buffer(unique_id, 128)
        check(self.lib.b2g_ctx_comm_init(self.h, world, rank, C.cast(buf, C.c_void_p)))
        self.world, self.rank = world, rank

    def allreduce_test(self, a: np.ndarray) -> np.ndarray:
        a = _f32(a).copy()
        check(self.lib.b2g_ctx_allreduce_test(self.h, _fp(a), a.size))
        return a

    def close(self):
        if self.h:
            self.lib.b2g_ctx_destroy(self.h)
            self.h = None


def comm_unique_id() -> bytes:
    buf = C.create_string_buffer(128)
    check(_lib.load().b2g_comm_unique_id(C.cast(buf, C.c_void_p)))
    return buf.raw


class Net:
    """b2g_net: a spine-plus-skip ComputationGraph (init / output / fit / getLayer(..).getParam/setParam; J:166-170,420-510)."""

    def __init__(self, ctx: Context, specs: Sequence[Dict], input_shape, max_batch: int, precision: int = FP32,
                 grad_clip: float = 0.0, xent_clip_eps: float = 1e-5, bn_groups: int = 1, seed: int = 666,
                 gradient_normalization: str = "none", gradient_normalization_threshold: float = 1.0,
                 constraints: Optional[Sequence[Dict]] = None, weight_noise: Optional[Dict] = None, weight_init: Optional[Dict] = None,
                 regularization: Optional[Dict] = None):
        """constraints: the global builder's constraints (models.max_norm, ...), for every layer whose own "constraints" reach none of its
        parameters (none given, or e.g. only bias constraints on a BatchNorm), as DL4J's builder fills them in; the specs the net keeps (and a
        checkpoint saves) carry them per layer.  weight_noise: the global builder's weightNoise (models.drop_connect / models.weight_noise) for
        every non-frozen conv, deconv, dense and output layer without a "weight_noise" of its own; the kept specs carry it per layer.
        weight_init: the global builder's weightInit / dist / biasInit (models.weight_init) for every conv, deconv, dense and output layer
        without a "weight_init" of its own, drawn right after creation; the kept specs carry it per layer.  Layers with neither keep
        b2g_net_create's Xavier draw.  regularization: the global builder's l1 / l2 / l1Bias / l2Bias ({"l1": .., "l2": .., "l1_bias": ..,
        "l2_bias": ..}): every non-frozen conv, deconv, dense and output layer takes each key its spec does not set, as DL4J's builder fills
        them in; the kept specs carry them per layer."""
        self.ctx, self.lib, self.specs = ctx, ctx.lib, copy.deepcopy(list(specs))
        resolve_regularization(self.specs, regularization)
        if weight_init is not None:
            for sp in self.specs:
                if sp["type"] in GEMM_TYPES and "weight_init" not in sp:
                    sp["weight_init"] = copy.deepcopy(weight_init)
        inits = [(sp["name"], weight_init_struct(sp["weight_init"], sp)) for sp in self.specs if sp["type"] in REG_TYPES and sp.get("weight_init") is not None]
        if constraints:
            for sp in self.specs:
                if sp["type"] in GEMM_TYPES + ("batchnorm",) and not resolve_constraints(sp):
                    sp["constraints"] = copy.deepcopy(list(constraints))
        if weight_noise is not None:
            for sp in self.specs:
                if sp["type"] in GEMM_TYPES and not sp.get("frozen", False) and "weight_noise" not in sp:
                    sp["weight_noise"] = copy.deepcopy(weight_noise)
        # each layer's b2g_layer_desc.lr: what the engine uses again when a schedule is cleared
        self.lr_constants = [constant_lr((sp.get("updater") or {}).get("lr", 0.0)) for sp in self.specs]
        c, h, w = input_shape if len(input_shape) == 3 else (input_shape[0], 1, 1)
        self.input_shape = tuple(input_shape)
        cfg = NetConfig(h, w, c, max_batch, precision, grad_clip, xent_clip_eps, bn_groups, seed)
        arr = (LayerDesc * len(specs))(*[layer_desc(s, v) for s, v in zip(self.specs, resolve_vertices(specs))])     # the kept specs: a global l2 included
        hnd = C.c_void_p()
        check(self.lib.b2g_net_create(ctx.h, C.byref(cfg), arr, len(specs), C.byref(hnd)))
        self.h = hnd
        self.max_batch, self.precision = max_batch, precision
        n = C.c_int64()
        check(self.lib.b2g_net_num_params(self.h, C.byref(n)))
        self.n_params = n.value
        check(self.lib.b2g_net_output_size(self.h, C.byref(n)))
        self.out_elems = n.value
        try:
            for name, s in inits:         # Layer.Builder.weightInit / dist / biasInit, at init()
                check(self.lib.b2g_net_init_weights(self.h, name.encode(), C.byref(s)))
            for sp in self.specs:         # Layer.Builder.l1 / l1Bias / l2Bias (l2 alone travels in the desc)
                r = spec_regularization(sp)
                if sp["type"] in REG_TYPES and (r["l1"] or r["l1_bias"] or r["l2_bias"]):
                    check(self.lib.b2g_net_set_regularization(self.h, sp["name"].encode(), C.byref(regularization_struct(r))))
            if gradient_normalization != "none":
                self.set_gradient_normalization(gradient_normalization, gradient_normalization_threshold)
            for sp in self.specs:         # an updater constructed with an ISchedule: new Adam(new StepSchedule(...))
                lr = (sp.get("updater") or {}).get("lr", 0.0)
                if is_schedule(lr) and layer_has_lr(sp):
                    self.set_lr_schedule(lr, sp["name"])
            for sp in self.specs:
                if sp.get("constraints"):
                    self._push_constraints(sp, {})
            self.dropout_constants = {sp["name"]: dropout_kind_value(sp)[1] for sp in self.specs if sp["type"] == "dropout" and sp.get("name")}
            for sp in self.specs:         # new GaussianNoise(ISchedule) and the other IDropout schedule constructors
                if sp["type"] == "dropout" and is_schedule(sp[dropout_value_key(sp)]):
                    self.set_dropout_schedule(sp[dropout_value_key(sp)], sp["name"])
            for sp in self.specs:         # Layer.Builder.weightNoise
                if sp.get("weight_noise") is not None:
                    self.set_weight_noise(sp["weight_noise"], sp["name"])
            for sp in self.specs[:-1]:
                if sp.get("loss_weights") is not None:
                    raise ValueError(f"layer {sp.get('name')!r}: loss_weights belong to the net's last (loss) layer")
            if self.specs and self.specs[-1].get("loss_weights") is not None:     # new LossMCXENT(weights), ...
                self.set_loss_weights(self.specs[-1]["loss_weights"])
        except Exception:
            self.close()
            raise

    # --- parameters (DL4J flattened-view order) ---
    def num_params(self) -> int:
        return self.n_params

    def set_param(self, layer: str, name: str, value):
        v = _f32(value).ravel()
        check(self.lib.b2g_net_set_param(self.h, layer.encode(), name.encode(), _fp(v), v.size))

    def get_param(self, layer: str, name: str, size: int) -> np.ndarray:
        out = np.empty(size, np.float32)
        check(self.lib.b2g_net_get_param(self.h, layer.encode(), name.encode(), _fp(out), size))
        return out

    def params(self) -> np.ndarray:
        out = np.empty(self.n_params, np.float32)
        check(self.lib.b2g_net_get_params(self.h, _fp(out), out.size))
        return out

    def set_params(self, flat):
        v = _f32(flat).ravel()
        check(self.lib.b2g_net_set_params(self.h, _fp(v), v.size))

    def gradients(self) -> np.ndarray:
        out = np.empty(self.n_params, np.float32)
        check(self.lib.b2g_net_get_gradients(self.h, _fp(out), out.size))
        return out

    def updater_state_size(self) -> int:
        """Elements of the updater state: 2 x numParams ([state0 | state1]), 3 x numParams on a net with an AMSGrad layer (| state2)."""
        n = C.c_int64()
        check(self.lib.b2g_net_updater_state_size(self.h, C.byref(n)))
        return n.value

    def updater_state(self) -> np.ndarray:
        out = np.empty(self.updater_state_size(), np.float32)
        check(self.lib.b2g_net_get_updater_state(self.h, _fp(out), out.size))
        return out

    def set_updater_state(self, st):
        v = _f32(st).ravel()
        check(self.lib.b2g_net_set_updater_state(self.h, _fp(v), v.size))

    # --- checkpoint / resume (ModelSerializer.writeModel, J:606-618; serializer.py) ---
    def save(self, path, save_updater: bool = True):
        from . import serializer
        serializer.save_net(self, path, self.specs, self.input_shape, save_updater,
                            {"precision": "bf16" if self.precision == BF16 else "fp32", "max_batch": self.max_batch, "iteration": self.iteration(),
                             "dropout_pass": self.dropout_pass(), "epoch": self.epoch()})

    def restore(self, path, load_updater: bool = True):
        """Loads parameters (and updater state) of a checkpoint written by save() into this net (same architecture)."""
        from . import serializer
        return serializer.restore_into(self, path, load_updater)

    # --- execution ---
    def output(self, x, train: bool = False) -> np.ndarray:
        x = _f32(x)
        out = np.empty((x.shape[0], self.out_elems), np.float32)
        check(self.lib.b2g_net_output(self.h, _fp(x), x.shape[0], int(train), _fp(out)))
        return out

    def layer_output_size(self, layer: int) -> int:
        n = C.c_int64()
        check(self.lib.b2g_net_layer_output_size(self.h, layer, C.byref(n)))
        return n.value

    def activation(self, layer: int, batch: int) -> np.ndarray:
        out = np.empty((batch, self.layer_output_size(layer)), np.float32)
        check(self.lib.b2g_net_get_activation(self.h, layer, batch, _fp(out)))
        return out

    def _mask(self, mask, batch: int):
        """A labels mask as (contiguous fp32, width): [batch] or [batch, 1] per example, [batch, nOut] per output, NCHW [batch, 1 or C, H, W]
        on a CnnLossLayer; the width is its second dimension, and the mask holds exactly what the engine reads for it."""
        m = _f32(mask)
        width = m.shape[1] if m.ndim >= 2 else 1
        cols = C.c_int32()
        check(self.lib.b2g_net_loss_columns(self.h, C.byref(cols)))
        per = self.out_elems // max(1, cols.value) * width
        if m.shape[0] != batch or m.size != batch * per:
            raise ValueError(f"labels mask of shape {m.shape}: {batch} examples of {self.out_elems // max(1, cols.value)} values per column of "
                             f"its width {width} (1 or {cols.value})")
        return m, width

    def compute_gradient_and_score(self, x, y, mask=None) -> float:
        """mask: DataSet's labels mask (semantics at b2g_loss in include/b200gan.h), or None."""
        x, y = _f32(x), _f32(y)
        s = C.c_float()
        if mask is None:
            check(self.lib.b2g_net_compute_gradient_and_score(self.h, _fp(x), _fp(y), x.shape[0], C.byref(s)))
        else:
            m, width = self._mask(mask, x.shape[0])
            check(self.lib.b2g_net_compute_gradient_and_score_masked(self.h, _fp(x), _fp(y), x.shape[0], C.byref(s), _fp(m), width))
        return s.value

    def fit(self, x, y, mask=None) -> float:
        """mask: DataSet's labels mask (semantics at b2g_loss in include/b200gan.h), or None."""
        x, y = _f32(x), _f32(y)
        s = C.c_float()
        if mask is None:
            check(self.lib.b2g_net_fit(self.h, _fp(x), _fp(y), x.shape[0], C.byref(s)))
        else:
            m, width = self._mask(mask, x.shape[0])
            check(self.lib.b2g_net_fit_masked(self.h, _fp(x), _fp(y), x.shape[0], C.byref(s), _fp(m), width))
        return s.value

    def set_loss_weights(self, weights, layer: Optional[str] = None):
        """The per-output weights of the net's loss layer (new LossMCXENT(weights), new LossBinaryXENT(weights), new LossMSE(weights), ...):
        nOut (C on a CnnLossLayer) finite floats, None clears.  The kept specs (and so checkpoints) carry them."""
        name = layer.encode() if layer is not None else None
        if weights is None:
            check(self.lib.b2g_net_set_loss_weights(self.h, name, None, 0))
            self.specs[-1].pop("loss_weights", None)
            return
        w = _f32(weights).ravel()
        check(self.lib.b2g_net_set_loss_weights(self.h, name, _fp(w), w.size))
        self.specs[-1]["loss_weights"] = [float(v) for v in w]

    def set_gradient_normalization(self, mode: str, threshold: float = 1.0):
        """DL4J's GradientNormalization for every layer of the net, applied from the next update on: "none", "renormalize_l2_per_layer",
        "renormalize_l2_per_param_type", "clip_l2_per_layer" or "clip_l2_per_param_type" (the clip modes need a finite threshold > 0; the
        renormalize modes ignore it).  ClipElementWiseAbsoluteValue is `grad_clip` at construction, and excludes the L2 modes."""
        if mode not in GRADIENT_NORMALIZATIONS:
            raise ValueError(f"unknown gradient normalization {mode!r}; one of {sorted(GRADIENT_NORMALIZATIONS)} (element-wise clipping is grad_clip)")
        check(self.lib.b2g_net_set_gradient_normalization(self.h, GRADIENT_NORMALIZATIONS[mode], float(threshold)))

    def set_lr_schedule(self, schedule: Optional[Dict], layer: Optional[str] = None):
        """ComputationGraph.setLearningRate(ISchedule) (layer None: every layer whose updater has a learning rate) or setLearningRate(layer,
        ISchedule); schedule None = back to the layer's constant lr from creation (b2g_layer_desc.lr).  Applied from the next update on; the
        specs a checkpoint writes follow (follow_lr_schedule)."""
        s, _arrays = schedule_struct(schedule)       # _arrays: the MAP entries s points into, alive for the call
        check(self.lib.b2g_net_set_lr_schedule(self.h, None if layer is None else layer.encode(), C.byref(s)))
        follow_lr_schedule(self.specs, self.lr_constants, schedule, layer)

    def _push_constraints(self, spec: Dict, before: Dict[str, List[Dict]]):
        now = resolve_constraints(spec)
        for p in sorted(set(now) | set(before)):
            lst = now.get(p, [])
            arr = (_lib.Constraint * max(1, len(lst)))(*[constraint_struct(c) for c in lst])
            check(self.lib.b2g_net_set_constraints(self.h, spec["name"].encode(), p.encode(), arr, len(lst)))

    def set_constraints(self, constraints: Optional[Sequence[Dict]], layer: Optional[str] = None):
        """Replaces the "constraints" of one layer's spec (layer None: of every layer with parameters), as Layer.Builder.constrainWeights /
        constrainBias / constrainAllParameters would have set them; None or [] removes them.  Applied from the next update on (a captured GAN
        step is re-captured); the specs a checkpoint writes follow."""
        for sp in self.specs:
            if (layer is not None and sp.get("name") != layer) or sp["type"] not in GEMM_TYPES + ("batchnorm",):
                continue
            before = resolve_constraints(sp)
            new = dict(sp, constraints=copy.deepcopy(list(constraints or [])))
            resolve_constraints(new)                    # validates before anything changes
            sp["constraints"] = new["constraints"]
            if not sp["constraints"]:
                del sp["constraints"]
            self._push_constraints(sp, before)
            if layer is not None:
                break

    def apply_constraints(self):
        """Model.applyConstraints: every constraint of the net once, now (the updates apply them by themselves)."""
        check(self.lib.b2g_net_apply_constraints(self.h))

    def set_dropout_schedule(self, schedule: Optional[Dict], layer: Optional[str] = None):
        """An ISchedule in place of a DropoutLayer's value (p, rate or stddev; b2g_net_set_dropout_schedule): layer None = every non-frozen
        DropoutLayer; schedule None = back to the value from creation.  The specs a checkpoint writes follow."""
        s, _arrays = schedule_struct(schedule)
        check(self.lib.b2g_net_set_dropout_schedule(self.h, None if layer is None else layer.encode(), C.byref(s)))
        for sp in self.specs:
            if sp["type"] != "dropout" or (layer is None and sp.get("frozen", False)) or (layer is not None and sp.get("name") != layer):
                continue
            sp[dropout_value_key(sp)] = copy.deepcopy(schedule) if schedule is not None else self.dropout_constants[sp["name"]]
            if layer is not None:
                break

    def set_weight_noise(self, weight_noise: Optional[Dict], layer: Optional[str] = None):
        """DropConnect or WeightNoise on a layer's weights (b2g_net_set_weight_noise; models.drop_connect / models.weight_noise): layer None =
        every non-frozen conv, deconv, dense and output layer; None clears it.  Drawn anew in every train-mode pass from the next one on; the
        specs a checkpoint writes follow."""
        s, _keep = weight_noise_struct(weight_noise)
        check(self.lib.b2g_net_set_weight_noise(self.h, None if layer is None else layer.encode(), C.byref(s)))
        for sp in self.specs:
            if sp["type"] not in GEMM_TYPES or (layer is None and sp.get("frozen", False)) or (layer is not None and sp.get("name") != layer):
                continue
            sp.pop("weight_noise", None)
            if weight_noise is not None:
                sp["weight_noise"] = copy.deepcopy(weight_noise)
            if layer is not None:
                break

    def init_weights(self, weight_init: Dict, layer: Optional[str] = None):
        """Redraws W and sets b = bias_init now (b2g_net_init_weights; models.weight_init): layer None = every conv, deconv, dense and output
        layer; a named prelu layer takes "zero", "ones" and "distribution" for its slopes.  Nothing else changes.  The specs a checkpoint
        writes follow."""
        targets = [sp for sp in self.specs if (sp["type"] in GEMM_TYPES or (layer is not None and sp["type"] == "prelu")) and (layer is None or sp.get("name") == layer)]
        if layer is not None:
            targets = targets[:1]
        s = weight_init_struct(weight_init)
        for sp in targets:
            weight_init_struct(weight_init, sp)          # the IDENTITY shape checks, before anything changes
        check(self.lib.b2g_net_init_weights(self.h, None if layer is None else layer.encode(), C.byref(s)))
        for sp in targets:
            sp["weight_init"] = copy.deepcopy(weight_init)

    def set_regularization(self, l1: float = 0.0, l2: float = 0.0, l1_bias: float = 0.0, l2_bias: float = 0.0, layer: Optional[str] = None):
        """l1 / l2 on W and l1Bias / l2Bias on b (b2g_net_set_regularization): layer None = every non-frozen conv, deconv, dense, output and
        prelu layer (a prelu layer's W is its slopes; it has no b).  Replaces all four coefficients (the spec's "l2" too), from the next update
        and score on.  The specs a checkpoint writes follow: a coefficient of 0 leaves no key."""
        r = check_regularization({"l1": l1, "l2": l2, "l1_bias": l1_bias, "l2_bias": l2_bias})
        check(self.lib.b2g_net_set_regularization(self.h, None if layer is None else layer.encode(), C.byref(regularization_struct(r))))
        for sp in self.specs:
            if sp["type"] not in REG_TYPES or (layer is None and sp.get("frozen", False)) or (layer is not None and sp.get("name") != layer):
                continue
            for k, v in r.items():
                if v:
                    sp[k] = v
                else:
                    sp.pop(k, None)
            if layer is not None:
                break

    def get_regularization(self, layer: str) -> Dict[str, float]:
        """The four coefficients of a conv, deconv, dense, output or prelu layer, as the engine holds them (fp32)."""
        r = _lib.Regularization()
        check(self.lib.b2g_net_get_regularization(self.h, layer.encode(), C.byref(r)))
        return {k: getattr(r, k) for k in REGULARIZATION_KEYS}

    def calc_regularization(self):
        """(calcL1(true), calcL2(true)): the score's L1 and L2 terms over the current parameters, in double (b2g_net_calc_regularization)."""
        l1, l2 = C.c_double(), C.c_double()
        check(self.lib.b2g_net_calc_regularization(self.h, C.byref(l1), C.byref(l2)))
        return l1.value, l2.value

    def noisy_operand(self, layer: int, which: int, size: int) -> np.ndarray:
        """What the latest train-mode pass of a weight-noise layer drew (b2g_test_net_noisy_operand): which 0 = W' in the internal order, 1 = the
        packed pixel-shuffle W' (BF16), 2 = b'."""
        out = np.empty(size, np.float32)
        check(self.lib.b2g_test_net_noisy_operand(self.h, layer, which, _fp(out), size))
        return out

    def dropout_value(self, layer: str) -> float:
        """The value (p, rate or stddev) the DropoutLayer's next train-mode forward uses, evaluated and clamped on the device."""
        v = C.c_float()
        check(self.lib.b2g_net_get_dropout_value(self.h, layer.encode(), C.byref(v)))
        return v.value

    def learning_rate(self, layer: str) -> float:
        """ComputationGraph.getLearningRate(layer): the fp32 learning rate the layer's next update uses (before Adam's bias correction),
        evaluated on the device."""
        v = C.c_float()
        check(self.lib.b2g_net_get_learning_rate(self.h, layer.encode(), C.byref(v)))
        return v.value

    def epoch(self) -> int:
        """The epoch count EPOCH schedules read (ComputationGraph.getEpochCount); part of a checkpoint."""
        v = C.c_int64()
        check(self.lib.b2g_net_get_epoch(self.h, C.byref(v)))
        return v.value

    def set_epoch(self, epoch: int):
        check(self.lib.b2g_net_set_epoch(self.h, int(epoch)))

    def set_grad_allreduce(self, enabled: bool):
        """False = the reference's parameter-averaging mode: fit() updates locally, average_parameters() synchronises."""
        check(self.lib.b2g_net_set_grad_allreduce(self.h, int(enabled)))

    def set_sync_bn(self, enabled: bool):
        """Cross-replica BatchNorm statistics (SURVEY.md 8e): W ranks x N/W then equals 1 rank x N."""
        check(self.lib.b2g_net_set_sync_bn(self.h, int(enabled)))

    def set_grad_payload_bf16(self, enabled: bool):
        check(self.lib.b2g_net_set_grad_payload_bf16(self.h, int(enabled)))

    def enable_p2p_allreduce(self) -> bool:
        """COLLECTIVE (every rank, nets in the same order): gradient all-reduce as one kernel over NVLink peer memory (CUDA IPC) instead of
        ncclAllReduce; returns whether every rank could map its peers (otherwise all ranks stay on NCCL)."""
        out = C.c_int32(0)
        check(self.lib.b2g_net_enable_p2p_allreduce(self.h, C.byref(out)))
        return bool(out.value)

    def average_parameters(self):
        """ParameterAveragingTrainingMaster: params and updater state <- mean over ranks (J:325-330)."""
        check(self.lib.b2g_net_average_parameters(self.h))

    def iteration(self) -> int:
        """The updater's iteration counter (Adam's t - 1); part of a checkpoint."""
        v = C.c_int64()
        check(self.lib.b2g_net_get_iteration(self.h, C.byref(v)))
        return v.value

    def set_iteration(self, it: int):
        check(self.lib.b2g_net_set_iteration(self.h, int(it)))

    def dropout_pass(self) -> int:
        """The dropout pass counter P: train-mode forwards that applied a DropoutLayer mask; part of a checkpoint."""
        v = C.c_int64()
        check(self.lib.b2g_net_get_dropout_pass(self.h, C.byref(v)))
        return v.value

    def set_dropout_pass(self, p: int):
        check(self.lib.b2g_net_set_dropout_pass(self.h, int(p)))

    def simt_gemm_calls(self) -> int:
        """BF16 nets: GEMM-shaped operations that ran on the SIMT kernels instead of the tensor-core kernels since creation."""
        v = C.c_uint64()
        check(self.lib.b2g_net_simt_gemm_calls(self.h, C.byref(v)))
        return v.value

    def time_hbm_kernels(self, rows: int, channels: int, iters: int = 10):
        """(updater, BatchNorm apply, BatchNorm backward apply) ms per launch, each after an L2 flush.  Perturbs the parameters: bench only."""
        ms = np.zeros(3, np.float32)
        check(self.lib.b2g_test_hbm_kernels(self.h, rows, channels, iters, _fp(ms)))
        return [float(v) for v in ms]

    def weight_operand(self, layer: int, which: int, size: int) -> np.ndarray:
        """BF16 nets: the bf16 copy of layer `layer`'s W that the next forward reads (which = 0, internal [A][taps][B] order, `size` = W's
        element count), or the packed pixel-shuffle operand [(py,px,c)][(dyr,dxc)][O] of the <= 4-channel transposed conv (which = 1,
        `size` = 144 * O), widened to fp32."""
        out = np.empty(size, np.float32)
        check(self.lib.b2g_test_net_shadow(self.h, layer, which, _fp(out), out.size))
        return out

    def input_gradient(self, batch: int) -> np.ndarray:
        out = np.empty((batch, int(np.prod(self.input_shape))), np.float32)
        check(self.lib.b2g_net_get_input_gradient(self.h, batch, _fp(out)))
        return out

    def close(self):
        if self.h:
            self.lib.b2g_net_destroy(self.h)
            self.h = None


class Gan:
    """b2g_gan: the adversarial iteration J:408-471 with dis/gan/gen sharing storage."""

    def __init__(self, gen: Net, dis: Net, fake_bn_train: bool = False, use_cuda_graph: bool = True):
        self.gen, self.dis, self.lib = gen, dis, gen.lib
        cfg = GanConfig(int(fake_bn_train), int(use_cuda_graph))
        h = C.c_void_p()
        check(self.lib.b2g_gan_create(gen.h, dis.h, C.byref(cfg), C.byref(h)))
        self.h = h

    def _args(self, x_real, z_d, z_g, y_real, y_fake, y_gen):
        """fp32 arrays; each label vector becomes [N, out_elems] of the discriminator (NCHW for a CnnLossLayer patch map): per-image labels
        ([N] or [N, 1]) are broadcast over the map."""
        x = _f32(x_real)
        n, oe = x.shape[0], self.dis.out_elems
        ys = []
        for name, y in (("y_real", y_real), ("y_fake", y_fake), ("y_gen", y_gen)):
            y = _f32(y).reshape(n, -1)
            if y.shape[1] == 1 and oe > 1:
                y = np.ascontiguousarray(np.broadcast_to(y, (n, oe)))
            if y.shape[1] != oe:
                raise ValueError(f"{name}: {y.shape[1]} labels per example; the discriminator has {oe} outputs per example (or pass one per image)")
            ys.append(y)
        return [x, _f32(z_d), _f32(z_g)] + ys

    def step(self, x_real, z_d, z_g, y_real, y_fake, y_gen):
        a = self._args(x_real, z_d, z_g, y_real, y_fake, y_gen)
        losses = np.zeros(3, np.float32)
        check(self.lib.b2g_gan_step(self.h, *[_fp(v) for v in a], a[0].shape[0], _fp(losses)))
        return losses

    def step_ptr(self, ptrs, batch: int, losses: np.ndarray):
        """Raw-pointer variant for pinned host buffers (bench e2e): ptrs = 6 integer addresses."""
        args = [C.cast(C.c_void_p(p), C.POINTER(C.c_float)) for p in ptrs]
        check(self.lib.b2g_gan_step(self.h, *args, batch, _fp(losses)))

    def upload(self, x_real, z_d, z_g, y_real, y_fake, y_gen):
        a = self._args(x_real, z_d, z_g, y_real, y_fake, y_gen)
        check(self.lib.b2g_gan_upload(self.h, *[_fp(v) for v in a], a[0].shape[0]))
        self.gen.ctx.sync()

    def set_label_masks(self, m_real, m_fake, m_gen):
        """Labels masks of the discriminator's loss for every later step (b2g_gan_set_label_masks): [batch, 1] per example, or NCHW
        [batch, 1 or C, H, W] on a CnnLossLayer discriminator.  All three None clears."""
        if m_real is None and m_fake is None and m_gen is None:
            check(self.lib.b2g_gan_set_label_masks(self.h, None, None, None, 0, 0))
            return
        ms = [_f32(m) for m in (m_real, m_fake, m_gen)]
        batch = ms[0].shape[0]
        width = self.dis._mask(ms[0], batch)[1]
        for m in ms[1:]:
            if m.shape != ms[0].shape:
                raise ValueError(f"labels masks of shapes {[v.shape for v in ms]}")
        check(self.lib.b2g_gan_set_label_masks(self.h, *[_fp(m) for m in ms], width, batch))

    def step_resident(self, batch: int):
        check(self.lib.b2g_gan_step_resident(self.h, batch))

    def losses(self) -> np.ndarray:
        out = np.zeros(3, np.float32)
        check(self.lib.b2g_gan_read_losses(self.h, _fp(out)))
        return out

    def last_step_ms(self) -> float:
        v = C.c_float()
        check(self.lib.b2g_gan_last_step_ms(self.h, C.byref(v)))
        return v.value

    def close(self):
        if self.h:
            self.lib.b2g_gan_destroy(self.h)
            self.h = None


def test_conv(ctx: Context, kind: int, impl: int, precision: int, geom: Dict[str, int], a, b, out_size: int, iters: int = 1):
    """Kernel-level hook: kind 0 fprop / 1 dgrad / 2 wgrad; impl 0 SIMT / 1 tensor-core. Returns (out, ms_per_iter)."""
    g = _lib.ConvGeom(**geom)
    a, b = _f32(a).ravel(), _f32(b).ravel()
    out = np.empty(out_size, np.float32)
    ms = C.c_float()
    check(ctx.lib.b2g_test_conv(ctx.h, kind, impl, precision, C.byref(g), _fp(a), _fp(b), _fp(out), iters, C.byref(ms)))
    return out, ms.value


EPI_PLAIN, EPI_STATS, EPI_BNBWD, EPI_ACTBWD = 0, 1, 2, 3


def test_conv_ex(ctx: Context, kind: int, geom: Dict[str, int], a, b, out_size: int, *, epi: int = 0, act: str = "identity", alpha: float = 0.0,
                 bias=None, scale=None, groups: int = 1, aux=None, aux2=None, iters: int = 1, impl: int = 1, bn: int = 0, max_ctas: int = 0,
                 poison: bool = False, w_mn: bool = False, per_tap: bool = False, info: Optional[dict] = None, defer: bool = False, db=None,
                 precision: int = BF16, param_offset: int = 0, splits: int = 0):
    """Tensor-core fprop (kind 0) / dgrad (kind 1) with the epilogue the training step uses (impl 3, kind 1: the pixel-shuffle deconv, b = the
    [O][4][4][C] weight).  bn forces the 64- / 128-column tile, max_ctas caps the persistent grid (0: production choice for both); poison
    fills the output with NaN before every launch; w_mn (kind 0, 1x1): b is the [C][O] dense weight; per_tap keeps a 4x4 s2 p1 shape on
    one activation box per tap instead of the slabs two taps share.  info, if given, receives "slab": whether the launch used the slabs, and
    "splits": the split-K count of a SIMT / skinny-layer / dense kernel or of a tensor-core weight gradient.
    The tensor-core skinny-layer conv (impl 3, kind 0) takes bias and act / alpha, and max_ctas as its CTA target (tiles per CTA =
    ceil(tiles / max_ctas)).
    Weight gradients (kind 2, impl 1 / 3): defer queues the split-K sum and runs it as the backward pass's one reduce-list launch; db (impl 3,
    a float32 array of O elements) receives the bias gradient the edge kernel computes beside dw; splits forces the split count (impl 1:
    the grid's split dimension, trailing splits may be empty; impl 3: the CTA target, tiles per CTA = ceil(tiles / splits)); poison fills
    dw, db and the partials with NaN before every launch; param_offset puts dw and db that many elements past an aligned address.
    The SIMT (impl 0), skinny-layer (impl 2) and dense (impl 4) kernels run in either precision with the bias / scale / activation their
    production wrapper takes; param_offset puts their fp32 weight operand (FP32) or weight gradient that many elements past an aligned address.
    Returns (out, stats or None, kernel name, ms)."""
    g = _lib.ConvGeom(**geom)
    a, b = _f32(a).ravel(), _f32(b).ravel()
    out = np.empty(out_size, np.float32)
    oc = geom["o"] if kind == 0 else geom["c"]
    o = _lib.TestConvOpts()
    o.epi, o.act, o.alpha, o.groups = epi, ACTS[act], alpha, groups
    o.bn, o.max_ctas, o.poison, o.w_mn, o.per_tap, o.defer = bn, max_ctas, int(poison), int(w_mn), int(per_tap), int(defer)
    o.param_offset, o.splits = param_offset, splits
    if db is not None:
        assert db.dtype == np.float32 and db.flags.c_contiguous
        o.db = _fp(db)
    keep = []
    for name, v in (("bias", bias), ("scale", scale), ("aux", aux), ("aux2", aux2)):
        if v is not None:
            arr = _f32(v).ravel(); keep.append(arr); setattr(o, name, _fp(arr))
    stats = None
    if epi in (EPI_STATS, EPI_BNBWD):
        stats = np.zeros((groups, 2, oc), np.float64); o.stats = stats.ctypes.data_as(C.POINTER(C.c_double))
    ms = C.c_float()
    check(ctx.lib.b2g_test_conv_ex(ctx.h, kind, impl, precision, C.byref(g), _fp(a), _fp(b), _fp(out), iters, C.byref(ms), C.byref(o)))
    if info is not None:
        info["slab"], info["splits"] = bool(o.slab), o.splits
    return out, stats, o.kernel.decode(), ms.value


def test_bn(ctx: Context, precision: int, path: int, x, eps_out, gamma, beta, run_mean, run_var, *, act: str = "identity", alpha: float = 0.0,
            eps: float = 1e-5, decay: float = 0.9, g_gamma=None, g_beta=None, want_param_grads: bool = True, replicas: int | None = None):
    """One BatchNorm(+activation) forward and backward through the training-step kernels (b2g_test_bn).  x, eps_out: [groups, rows, C].
    Returns a dict with y, eps_in ([groups, rows, C]), g_gamma, g_beta (accumulated into the given initial values), g_mean, g_var ([C]) and
    mean, invstd ([groups, C]).
    replicas=R: cross-replica BatchNorm as R data-parallel ranks run it (b2g_test_bn_ex; BF16, path 1 or 2).  x, eps_out: [R, groups, rows, C],
    replica r's rows at [r]; every result gains a leading replica axis (g_gamma, g_beta, g_mean, g_var [R, C]; mean, invstd [R, groups, C])."""
    x, e = _f32(x), _f32(eps_out)
    par = [_f32(v).ravel() for v in (gamma, beta, run_mean, run_var)]
    if replicas is not None:
        R, groups, rows, ch = x.shape
        if R != replicas or precision != BF16:
            raise ValueError(f"replicas={replicas}: x must be [replicas, groups, rows, C] ({x.shape}) and the precision BF16")
        o = _lib.TestBnOpts(path, replicas, groups, rows, ch, ACTS[act], alpha, eps, decay, int(want_param_grads))
        g0 = [_f32(np.zeros(ch) if v is None else v).ravel() for v in (g_gamma, g_beta)]
        r = {k: np.empty(x.shape, np.float32) for k in ("y", "eps_in")}
        r.update({k: np.empty((R, ch), np.float32) for k in ("g_gamma", "g_beta", "g_mean", "g_var")})
        r.update({k: np.empty((R, groups, ch), np.float32) for k in ("mean", "invstd")})
        check(ctx.lib.b2g_test_bn_ex(ctx.h, C.byref(o), _fp(x), _fp(e), *[_fp(v) for v in par + g0],
                                     *[_fp(r[k]) for k in ("y", "eps_in", "g_gamma", "g_beta", "g_mean", "g_var", "mean", "invstd")]))
        return r
    groups, rows, ch = x.shape
    r = {k: np.empty(x.shape, np.float32) for k in ("y", "eps_in")}
    r["g_gamma"] = _f32(np.zeros(ch) if g_gamma is None else g_gamma).copy()
    r["g_beta"] = _f32(np.zeros(ch) if g_beta is None else g_beta).copy()
    r.update({k: np.empty(ch, np.float32) for k in ("g_mean", "g_var")})
    r.update({k: np.empty((groups, ch), np.float32) for k in ("mean", "invstd")})
    check(ctx.lib.b2g_test_bn(ctx.h, precision, path, groups, rows, ch, _fp(x), _fp(e), *[_fp(v) for v in par], ACTS[act], alpha, eps, decay,
                              int(want_param_grads), *[_fp(r[k]) for k in ("y", "eps_in", "g_gamma", "g_beta", "g_mean", "g_var", "mean", "invstd")]))
    return r


def test_dropout_kind(ctx: Context, precision: int, kind: str, x, dy, value: float, *, seed: int = 666, layer: int = 0, rank: int = 0, pass_: int = 0):
    """One DropoutLayer forward and backward of an IDropout kind (a DROPOUT_KINDS name) and its value (b2g_test_dropout_kind); as test_dropout."""
    x, e = _f32(x), _f32(dy)
    rows = x.shape[0]
    h, w, c = (x.shape[1:] if x.ndim == 4 else (1, 1, int(np.prod(x.shape[1:]))))
    y, dx = np.empty_like(x), np.empty_like(x)
    check(ctx.lib.b2g_test_dropout_kind(ctx.h, precision, DROPOUT_KINDS[kind][0], seed, layer, rank, pass_, rows, h, w, c, value, _fp(x), _fp(e), _fp(y), _fp(dx)))
    return y, dx


def test_dropout(ctx: Context, precision: int, x, dy, p: float, *, seed: int = 666, layer: int = 0, rank: int = 0, pass_: int = 0):
    """One DropoutLayer forward and backward through the training-step kernels (b2g_test_dropout).  x, dy: [rows, H, W, C] in the engine's NHWC
    order (or [rows, F]).  Returns (y, dx) in the same shape."""
    x, e = _f32(x), _f32(dy)
    rows = x.shape[0]
    h, w, c = (x.shape[1:] if x.ndim == 4 else (1, 1, int(np.prod(x.shape[1:]))))
    y, dx = np.empty_like(x), np.empty_like(x)
    check(ctx.lib.b2g_test_dropout(ctx.h, precision, seed, layer, rank, pass_, rows, h, w, c, p, _fp(x), _fp(e), _fp(y), _fp(dx)))
    return y, dx


EW_OPS = {"reduce_splits": 0, "reduce_multi": 1, "colsum": 2, "xent": 3, "softmax_xent": 4, "act_fwd": 5, "act_bwd": 6, "maxpool": 7,
          "upsample": 8, "sumsq": 9, "loss": 10, "act_ext_fwd": 11, "act_ext_bwd": 12,
          "cnn_xent": 13, "cnn_softmax_xent": 14, "vertex_fwd": 15, "vertex_bwd": 16, "merge_fwd": 17, "merge_bwd": 18, "skip_add": 19,
          "prelu_fwd": 20, "prelu_bwd": 21, "nchw_to_nhwc": 22, "nhwc_to_nchw": 23, "permute": 24, "cast_bf16": 25}


def test_ew(ctx: Context, precision: int, op: str, in0, in1=None, out_sizes=(0, 0, 0), *, act: str = "identity", jobs=None, segments=None,
            loss: str = "xent", **opts):
    """One reduction / loss / element-wise kernel through its production wrapper (b2g_test_ew; operands per op in include/b200gan.h).
    vertex_fwd / vertex_bwd: act is an ELEMENTWISE_OPS name and groups the input order.
    act_ext_fwd / act_ext_bwd (act: a name of codes 5-16): in0 = z, in1 = eps_out, out0 = f(z) / eps_out * f'(z).
    prelu_fwd / prelu_bwd: in0 = x then alpha, in1 = dy; shared = the shared-axes bit mask (1 = C, 2 = H, 4 = W), the map in N, H, W, C;
    out0 = y / dx, out1 = dalpha (0: not asked for).
    out_sizes: element counts of out0..out2 (0: not asked for).  opts: the b2g_test_ew_opts sizes and switches (n, rows, cols, groups, splits,
    stride, N, H, W, C, KH, KW, SH, SW, alpha, clip_eps, offset, in_place, accumulate, poison).  jobs (reduce_multi): dicts of n, splits,
    stride, src_off, dst_off.  segments (sumsq): (offsets, lengths, coefficients).  loss (op "loss"): a LOSSES name of codes 2-8.
    Returns ([out0, out1, out2] with None where not asked for, {"kernel": names, "sumsq": float, "wide": [per job]})."""
    o = _lib.TestEwOpts()
    o.op, o.act, o.loss = EW_OPS[op], ELEMENTWISE_OPS[act] if op in ("vertex_fwd", "vertex_bwd") else ACTS[act], LOSSES[loss]
    if op in ("prelu_fwd", "prelu_bwd"):
        o.act = int(opts.pop("shared", 0))
    for k, v in opts.items():
        setattr(o, k, int(v) if isinstance(v, bool) else v)
    keep = []
    if jobs is not None:
        arr = (_lib.EwReduceJob * len(jobs))(*[_lib.EwReduceJob(j["n"], j["stride"], j["src_off"], j["dst_off"], j["splits"], 0) for j in jobs])
        o.n_jobs, o.jobs = len(jobs), arr
        keep.append(arr)
    if segments is not None:
        so, sl, sc = (np.ascontiguousarray(segments[0], np.int64), np.ascontiguousarray(segments[1], np.int64), _f32(segments[2]))
        keep += [so, sl, sc]
        o.n_seg = len(so)
        o.seg_off, o.seg_len, o.seg_coef = so.ctypes.data_as(C.POINTER(C.c_int64)), sl.ctypes.data_as(C.POINTER(C.c_int64)), _fp(sc)
    ins = [None if v is None else _f32(v).ravel() for v in (in0, in1)]
    outs = [np.empty(k, np.float32) if k else None for k in out_sizes]
    ptr = lambda a: None if a is None else _fp(a)
    check(ctx.lib.b2g_test_ew(ctx.h, precision, C.byref(o), *[ptr(a) for a in ins], *[ptr(a) for a in outs]))
    info = {"kernel": o.kernel.decode(), "sumsq": o.sumsq, "wide": [o.jobs[i].wide for i in range(o.n_jobs)] if jobs is not None else []}
    return outs, info


LOSS_TEST_KERNELS = {"xent": 0, "softmax_xent": 1, "codes": 2, "cnn_xent": 3, "cnn_softmax_xent": 4}


def test_loss(ctx: Context, precision: int, kernel: str, z, y, w=None, mask=None, *, rows: int, cols: int, groups: int = 1, loss: str = "mse",
              act: str = "identity", alpha: float = 0.0, clip_eps: float = 0.0, offset: int = 0, poison: bool = False):
    """A weighted / masked loss kernel through its production wrapper (b2g_test_loss; operands in include/b200gan.h).  mask: [groups * rows,
    width].  Returns (dz, loss_sums, kernel name)."""
    o = _lib.TestLossOpts()
    o.kernel, o.rows, o.cols, o.groups, o.loss, o.act = LOSS_TEST_KERNELS[kernel], rows, cols, groups, LOSSES[loss], ACTS[act]
    o.alpha, o.clip_eps, o.offset, o.poison = alpha, clip_eps, offset, int(poison)
    zz, yy = _f32(z).ravel(), _f32(y).ravel()
    ww = None if w is None else _f32(w).ravel()
    mm = None if mask is None else _f32(mask)
    if mm is not None:
        o.mask_width = mm.shape[1] if mm.ndim > 1 else 1
        mm = mm.ravel()
    dz, ls = np.empty(zz.size, np.float32), np.empty(groups, np.float32)
    ptr = lambda a: None if a is None else _fp(a)
    check(ctx.lib.b2g_test_loss(ctx.h, precision, C.byref(o), _fp(zz), _fp(yy), ptr(ww), ptr(mm), _fp(dz), _fp(ls)))
    return dz, ls, o.kernel_name.decode()


POOL_TEST_OPS = {"pool2d": 0, "global_pool": 1}


def test_pool(ctx: Context, precision: int, op: str, in0, in1, out_sizes=(0, 0, 0), *, pooling: str = "max", pnorm: float = 2.0, **opts):
    """One pooling layer's forward and backward kernels through their production wrappers (b2g_test_pool; operands in include/b200gan.h).
    op "pool2d" (pooling avg / sum / pnorm) or "global_pool" (any POOLINGS name); opts: N, H, W, C, KH, KW, SH, SW, PH, PW, offset, poison.
    Returns ([out0, out1, out2] with None where not asked for, {"kernel": "forward,backward", "splits": int})."""
    o = _lib.TestPoolOpts()
    o.op, o.pool, o.pnorm = POOL_TEST_OPS[op], POOLINGS[pooling], float(pnorm)
    for k, v in opts.items():
        setattr(o, k, int(v))
    ins = [_f32(v).ravel() for v in (in0, in1)]
    outs = [np.empty(k, np.float32) if k else None for k in out_sizes]
    ptr = lambda a: None if a is None else _fp(a)
    check(ctx.lib.b2g_test_pool(ctx.h, precision, C.byref(o), *[ptr(a) for a in ins], *[ptr(a) for a in outs]))
    return outs, {"kernel": o.kernel.decode(), "splits": o.splits}
