"""Test-only NumPy restatement of DL4J's regression and margin losses (LossMSE, LossL1, LossL2, LossMAE, LossHinge, LossSquaredHinge,
LossWasserstein) on top of the DL4J oracle (oracle/dl4j_oracle.py) without changing it.

Semantics recalled from DL4J 1.0.0-beta3 org.nd4j.linalg.lossfunctions.impl.* (PARITY UNPINNED, like the rest of the oracle; the library's
statement is include/b200gan.h, b2g_loss).  Each is ILossFunction.computeGradient(labels, preOutput, activationFn): a = act(z),
dL/dz = dL/da * act'(a) with the derivative taken from the output a, per-example scores summed over the nOut outputs:
  mse            sum (a-y)^2 / nOut          2(a-y) / nOut
  l1             sum |a-y|                   sign(a-y)              (sign(0) = 0)
  l2             sum (a-y)^2                 2(a-y)
  mae            sum |a-y| / nOut            sign(a-y) / nOut
  hinge          sum max(0, 1 - y a)         -y where 1 - y a > 0 (strictly), else 0
  squared_hinge  sum max(0, 1 - y a)^2       -2y max(0, 1 - y a)
  wasserstein    sum y a / nOut              y / nOut               (the / nOut: LossQuirks.wasserstein_per_output)

`Output` and `LossLayer` subclass the oracle's layers with a (loss, activation) pair, so the oracle's Net.compute_gradient_and_score, fit and
gan_step run on them unchanged.  `oracle_from_specs` builds an oracle Net from layer specs (updater_ref's builder) and gives its last layer the
spec's loss when it is one of LOSSES."""
from __future__ import annotations

import dataclasses

import numpy as np

import updater_ref as ur
from oracle import dl4j_oracle as o

LOSSES = ("mse", "l1", "l2", "mae", "hinge", "squared_hinge", "wasserstein")
CODES = {"mse": 2, "l1": 3, "l2": 4, "mae": 5, "hinge": 6, "squared_hinge": 7, "wasserstein": 8}


@dataclasses.dataclass
class LossQuirks:
    wasserstein_per_output: bool = True     # [recall, medium confidence] LossWasserstein divides score and gradient by nOut (moot at nOut = 1)


DEFAULT_LOSS_QUIRKS = LossQuirks()


def act_grad_from_out(act: str, a: np.ndarray, alpha: float = 0.01) -> np.ndarray:
    """f'(z) from the output a = f(z), as the library's act_grad_from_out takes it (LeakyReLU: sign(a) = sign(z) for alpha > 0)."""
    if act == "identity":
        return np.ones_like(a)
    if act == "tanh":
        return 1 - a * a
    if act == "sigmoid":
        return a * (1 - a)
    if act == "relu":
        return (a > 0).astype(a.dtype)
    if act == "lrelu":
        return np.where(a > 0, 1.0, alpha).astype(a.dtype)
    raise ValueError(act)


def per_output(loss: str, q: LossQuirks = DEFAULT_LOSS_QUIRKS) -> bool:
    """Whether the loss divides its score and gradient by nOut."""
    return loss in ("mse", "mae") or (loss == "wasserstein" and q.wasserstein_per_output)


def score_and_grad(loss: str, act: str, alpha: float, z: np.ndarray, y: np.ndarray, q: LossQuirks = DEFAULT_LOSS_QUIRKS):
    """z, y: [N, nOut].  Returns (sum over the N examples of the per-example scores, dL/dz [N, nOut])."""
    a = o.act_forward(act, z, alpha)
    e, m = a - y, 1 - y * a
    if loss in ("mse", "l2"):
        s, g = (e * e).sum(), 2 * e
    elif loss in ("l1", "mae"):
        s, g = np.abs(e).sum(), np.sign(e)
    elif loss == "hinge":
        s, g = np.maximum(m, 0).sum(), np.where(m > 0, -y, 0.0)
    elif loss == "squared_hinge":
        s, g = (np.maximum(m, 0) ** 2).sum(), -2 * y * np.maximum(m, 0)
    elif loss == "wasserstein":
        s, g = (y * a).sum(), y * np.ones_like(a)
    else:
        raise ValueError(loss)
    if per_output(loss, q):
        n = z.shape[1]
        s, g = s / n, g / n
    return float(s), g * act_grad_from_out(act, a, alpha)


class Output(o.Output):
    """OutputLayer.Builder(loss).activation(act).nOut(n): Dense + one of LOSSES on act(z)."""

    def __init__(self, n_in, n_out, loss, act="identity", alpha=0.01, updater=None, l2=0.0, name="", quirks=o.DEFAULT_QUIRKS,
                 loss_quirks: LossQuirks = DEFAULT_LOSS_QUIRKS):
        super().__init__(n_in, n_out, updater, l2, name, quirks)
        self.loss, self.loss_act, self.loss_alpha, self.lq = loss, act, alpha, loss_quirks

    def forward(self, x, train):
        z = o.Dense.forward(self, x, train)          # the identity Dense: z; the loss applies the activation
        return o.act_forward(self.loss_act, z, self.loss_alpha)

    def score_and_eps(self, y):
        return score_and_grad(self.loss, self.loss_act, self.loss_alpha, self._z, y, self.lq)


class LossLayer(o.LossLayer):
    """LossLayer.Builder(loss).activation(act): one of LOSSES on act of the incoming pre-activations, no parameters."""

    def __init__(self, loss, act="identity", alpha=0.01, name="", quirks=o.DEFAULT_QUIRKS, loss_quirks: LossQuirks = DEFAULT_LOSS_QUIRKS):
        super().__init__(name, quirks)
        self.loss, self.loss_act, self.loss_alpha, self.lq = loss, act, alpha, loss_quirks

    def forward(self, x, train):
        self._z = x
        return o.act_forward(self.loss_act, x, self.loss_alpha)

    def score_and_eps(self, y):
        z = self._z
        s, g = score_and_grad(self.loss, self.loss_act, self.loss_alpha, z.reshape(y.shape), y, self.lq)
        return s, g.reshape(z.shape)


def with_loss(layer, spec, loss_quirks: LossQuirks = DEFAULT_LOSS_QUIRKS):
    """The oracle's Output / LossLayer `layer` (parameters, updater and all) as this module's layer with the spec's loss and activation."""
    cls = Output if isinstance(layer, o.Output) else LossLayer
    new = cls.__new__(cls)
    new.__dict__.update(layer.__dict__)
    new.loss, new.loss_act, new.loss_alpha, new.lq = spec["loss"], spec.get("activation", "identity"), spec.get("alpha", 0.01), loss_quirks
    return new


def oracle_from_specs(specs, input_shape, loss_quirks: LossQuirks = DEFAULT_LOSS_QUIRKS, **kw):
    """updater_ref.oracle_from_specs, with the last layer carrying the spec's loss when that is one of LOSSES."""
    net = ur.oracle_from_specs(specs, input_shape, **kw)
    if specs[-1].get("loss") in LOSSES:
        net.layers[-1] = with_loss(net.layers[-1], specs[-1], loss_quirks)
    return net
