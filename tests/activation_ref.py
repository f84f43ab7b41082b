"""Test-only float64 restatement of DL4J's activations of b2g_activation codes 5-16 (ELU, SELU, Softplus, Softsign, HardTanh, HardSigmoid, ReLU6,
Swish, Cube, RationalTanh, RectifiedTanh, ThresholdedReLU) on top of the DL4J oracle (oracle/dl4j_oracle.py) without changing it.

Semantics recalled from DL4J 1.0.0-beta3 org.nd4j.linalg.activations.impl.* (PARITY UNPINNED, like the rest of the oracle; the library's statement
is include/b200gan.h, b2g_activation).  f'(z) is taken from the pre-activation z, as IActivation.backprop(in, epsilon) takes it.  The recalls of
medium confidence are ActQuirks flags; the engine implements the defaults.

The oracle's layers call dl4j_oracle.act_forward / act_backward by name, and loss_ref's losses call loss_ref.score_and_grad.  enable() wraps those
three module functions so that the new names reach this module; every other name goes to the original function, bit for bit.  It runs on
import and is idempotent.  `oracle_from_specs` fills the per-kind default of "alpha" (ELU's alpha and ThresholdedReLU's theta: 1.0) the way
engine.layer_desc does, then builds the oracle net through loss_ref."""
from __future__ import annotations

import dataclasses

import numpy as np

import loss_ref as lr
from oracle import dl4j_oracle as o

KINDS = ("elu", "selu", "softplus", "softsign", "hardtanh", "hardsigmoid", "relu6", "swish", "cube", "rationaltanh", "rectifiedtanh",
         "thresholdedrelu")
CODES = {k: 5 + i for i, k in enumerate(KINDS)}
ALPHA_DEFAULTS = {"elu": 1.0, "thresholdedrelu": 1.0}
SELU_LAMBDA, SELU_ALPHA = 1.0507009873554805, 1.6732632423543772
RT_A, RT_C = 1.7159, 1.41645


@dataclasses.dataclass
class ActQuirks:
    hardtanh_closed: bool = True           # [recall, medium] HardTanh' = 1 on the CLOSED interval [-1, 1]
    hardsigmoid_closed: bool = True        # [recall, medium] HardSigmoid' = 0.2 on the CLOSED interval [-2.5, 2.5]
    relu6_open: bool = True                # [recall, medium] ReLU6' = 1 on the OPEN interval (0, 6)
    thresholded_relu_in_beta3: bool = True  # [recall, medium] ActivationThresholdedReLU exists in 1.0.0-beta3 (False: the name is refused)


DEFAULT_ACT_QUIRKS = ActQuirks()
_quirks = DEFAULT_ACT_QUIRKS


def _sigmoid(z):
    return o._sigmoid(np.asarray(z, np.float64))


def _check(name, q):
    if name not in KINDS:
        raise ValueError(name)
    if name == "thresholdedrelu" and not q.thresholded_relu_in_beta3:
        raise ValueError("ThresholdedReLU is not part of DL4J 1.0.0-beta3 under ActQuirks.thresholded_relu_in_beta3 = False")


def forward(name: str, z, alpha: float = None, q: ActQuirks = None) -> np.ndarray:
    """f(z) in float64 (alpha None: the kind's default)."""
    q = q or _quirks
    _check(name, q)
    z = np.asarray(z, np.float64)
    a = ALPHA_DEFAULTS.get(name, 0.0) if alpha is None else float(alpha)
    if name == "elu":
        return np.where(z >= 0, z, a * np.expm1(np.minimum(z, 0)))
    if name == "selu":
        return SELU_LAMBDA * np.where(z > 0, z, SELU_ALPHA * np.expm1(np.minimum(z, 0)))
    if name == "softplus":
        return np.maximum(z, 0) + np.log1p(np.exp(-np.abs(z)))
    if name == "softsign":
        return z / (1 + np.abs(z))
    if name == "hardtanh":
        return np.clip(z, -1.0, 1.0)
    if name == "hardsigmoid":
        return np.clip(0.2 * z + 0.5, 0.0, 1.0)
    if name == "relu6":
        return np.clip(z, 0.0, 6.0)
    if name == "swish":
        return z * _sigmoid(z)
    if name == "cube":
        return z ** 3
    if name == "rationaltanh":
        y = 2.0 * z / 3.0
        A = 1 + np.abs(y) + y * y + RT_C * y ** 4
        return RT_A * np.sign(y) * (1 - 1 / A)
    if name == "rectifiedtanh":
        return np.maximum(0.0, np.tanh(z))
    return np.where(z > a, z, 0.0)          # thresholdedrelu


def derivative(name: str, z, alpha: float = None, q: ActQuirks = None) -> np.ndarray:
    """f'(z) in float64."""
    q = q or _quirks
    _check(name, q)
    z = np.asarray(z, np.float64)
    a = ALPHA_DEFAULTS.get(name, 0.0) if alpha is None else float(alpha)
    if name == "elu":
        return np.where(z >= 0, 1.0, a * np.exp(np.minimum(z, 0)))
    if name == "selu":
        return np.where(z > 0, SELU_LAMBDA, SELU_LAMBDA * SELU_ALPHA * np.exp(np.minimum(z, 0)))
    if name == "softplus":
        return _sigmoid(z)
    if name == "softsign":
        return 1 / (1 + np.abs(z)) ** 2
    if name == "hardtanh":
        inside = (z >= -1) & (z <= 1) if q.hardtanh_closed else (z > -1) & (z < 1)
        return np.where(inside, 1.0, 0.0)
    if name == "hardsigmoid":
        inside = (z >= -2.5) & (z <= 2.5) if q.hardsigmoid_closed else (z > -2.5) & (z < 2.5)
        return np.where(inside, 0.2, 0.0)
    if name == "relu6":
        inside = (z > 0) & (z < 6) if q.relu6_open else (z >= 0) & (z <= 6)
        return np.where(inside, 1.0, 0.0)
    if name == "swish":
        s = _sigmoid(z)
        return s * (1 + z * (1 - s))
    if name == "cube":
        return 3 * z * z
    if name == "rationaltanh":
        y = 2.0 * z / 3.0
        A = 1 + np.abs(y) + y * y + RT_C * y ** 4
        return RT_A * (2.0 / 3.0) * (1 + np.sign(y) * (2 * y + 4 * RT_C * y ** 3)) / (A * A)
    if name == "rectifiedtanh":
        t = np.tanh(z)
        return np.where(z > 0, 1 - t * t, 0.0)
    return np.where(z > a, 1.0, 0.0)        # thresholdedrelu


# ------------------------------------------------------------------ wiring into the oracle -------------------
_orig = {}


def _act_forward(name, z, alpha=0.01):
    return forward(name, z, alpha) if name in KINDS else _orig["fwd"](name, z, alpha)


def _act_backward(name, z, eps, alpha=0.01):
    return eps * derivative(name, z, alpha) if name in KINDS else _orig["bwd"](name, z, eps, alpha)


def _score_and_grad(loss, act, alpha, z, y, q=lr.DEFAULT_LOSS_QUIRKS):
    """A loss of codes 2-8 on a = f(z) of a new kind: the loss on a with the identity, then dL/dz = dL/da * f'(z)."""
    if act not in KINDS:
        return _orig["loss"](loss, act, alpha, z, y, q)
    s, g = _orig["loss"](loss, "identity", 0.0, forward(act, z, alpha), y, q)
    return s, g * derivative(act, z, alpha)


def enable(quirks: ActQuirks = DEFAULT_ACT_QUIRKS):
    """Routes the new names through this module in the oracle and loss_ref (idempotent); quirks applies to every later call."""
    global _quirks
    _quirks = quirks
    if not _orig:
        _orig.update(fwd=o.act_forward, bwd=o.act_backward, loss=lr.score_and_grad)
        o.act_forward, o.act_backward, lr.score_and_grad = _act_forward, _act_backward, _score_and_grad


enable()


def with_alpha_defaults(specs):
    """The specs with "alpha" filled where engine.layer_desc fills it for a new kind (ELU / ThresholdedReLU: 1.0)."""
    out = []
    for s in specs:
        s = dict(s)
        if s.get("activation") in ALPHA_DEFAULTS and "alpha" not in s:
            s["alpha"] = ALPHA_DEFAULTS[s["activation"]]
        out.append(s)
    return out


def oracle_from_specs(specs, input_shape, **kw):
    """loss_ref.oracle_from_specs on the specs with the per-kind alpha defaults."""
    return lr.oracle_from_specs(with_alpha_defaults(specs), input_shape, **kw)
