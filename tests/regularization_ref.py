"""Regularization (b2g_regularization in include/b200gan.h: DL4J's l1, l2, l1Bias and l2Bias) on top of the DL4J oracle.

The oracle restates l2 on W: `apply_update` adds l2 * W after the updater, and `l2_score` is sum 0.5 * l2 * ||W||^2.  RegNet adds the other
three coefficients, resolved per parameter as beta3's getL1ByParam / getL2ByParam do: a conv, deconv, dense or output layer's W takes l1
(and the oracle's own l2), its b takes l1Bias and l2Bias.  BatchNorm parameters and FrozenLayers take nothing.
  update:  u = updater(g) + l2 * theta + l1 * sign(theta),  sign(+-0) = 0;  theta -= u;  then the constraints
  score:   sum(loss) / mb + calc_l2() + calc_l1()
A layer's coefficients are its attributes l1, l1_bias, l2_bias (0 when missing) beside the oracle's l2.

DL4J 1.0.0-beta3, recalled; parity unpinned like the rest of the DL4J semantics.  The point of medium confidence is a RegQuirks field."""
import inspect
from dataclasses import dataclass

import numpy as np

from oracle import dl4j_oracle as o


@dataclass(frozen=True)
class RegQuirks:
    # beta3's BatchNormalization.getL1ByParam / getL2ByParam return 0 for gamma, beta, mean and var
    batchnorm_unregularized: bool = True


RQ = RegQuirks()
GEMM = (o.Conv2D, o.Deconv2D, o.Dense)          # Output and OutputSoftmax are Dense


def reg_coefs(layer, pname):
    """(l1, l2) of one parameter: W takes the layer's l1 / l2, b of a layer with a W its l1_bias / l2_bias; everything else (0, 0)."""
    if isinstance(layer, o.BatchNorm) and not RQ.batchnorm_unregularized:
        raise NotImplementedError("only beta3's unregularized BatchNorm is restated")
    if not isinstance(layer, GEMM):
        return 0.0, 0.0
    if pname == "W":
        return float(getattr(layer, "l1", 0.0)), float(layer.l2)
    if pname == "b":
        return float(getattr(layer, "l1_bias", 0.0)), float(getattr(layer, "l2_bias", 0.0))
    return 0.0, 0.0


def set_coefs(layer, l1=0.0, l2=0.0, l1_bias=0.0, l2_bias=0.0):
    layer.l1, layer.l2, layer.l1_bias, layer.l2_bias = l1, l2, l1_bias, l2_bias


class RegNet(o.Net):
    """o.Net with l1 on W and l1_bias / l2_bias on b."""

    def _live(self):
        return [(li, l) for li, l in enumerate(self.layers) if l.has_params and not getattr(l, "frozen", False)]

    def _reg_sum(self, which, norm):
        s = 0.0
        for _, l in self._live():
            for p, _, _ in l.param_specs():
                c = reg_coefs(l, p)[which]
                if c:
                    s += norm(c, l.params[p].astype(np.float64))
        return s

    def calc_l2(self) -> float:
        """ComputationGraph.calcL2(true): sum of 0.5 * l2 * ||W||^2 + 0.5 * l2_bias * ||b||^2 over the live layers, in parameter order (the
        oracle's l2_score when only l2 is set)."""
        return self._reg_sum(1, lambda c, v: 0.5 * c * float((v ** 2).sum()))

    def calc_l1(self) -> float:
        """ComputationGraph.calcL1(true): sum of l1 * ||W||_1 + l1_bias * ||b||_1 over the live layers."""
        return self._reg_sum(0, lambda c, v: c * float(np.abs(v).sum()))

    def l2_score(self):
        """The score's whole regularization term; compute_gradient_and_score and gan_step read it under this name."""
        return self.calc_l2() + self.calc_l1()

    def apply_update(self, mb, grads=None, frozen_from=None):
        """The oracle's update (which adds l2 * W), less the terms it does not restate, each from theta before the update; the constraints
        run last, on the result."""
        extra = {}
        for li, l in self._live():
            for p, _, _ in l.param_specs():
                c1, c2 = reg_coefs(l, p)
                c2 = 0.0 if p == "W" else c2          # the oracle adds l2 * W itself
                if c1 or c2:
                    v = l.params[p]
                    extra[(li, p)] = (c2 * v if c2 else 0.0) + (c1 * np.sign(v) if c1 else 0.0)
        constraints, self.layer_constraints = self.layer_constraints, {}
        try:
            super().apply_update(mb, grads, frozen_from)
        finally:
            self.layer_constraints = constraints
        for (li, p), t in extra.items():
            l = self.layers[li]
            l.params[p] = (l.params[p] - t).astype(self.dtype)
        if self.layer_constraints:
            self.apply_constraints()


def net_from_specs(specs, input_shape, **kw):
    """o.net_from_specs as a RegNet: the same layers, parameters, schedules and constraints, with each GEMM spec's "l1", "l1_bias" and
    "l2_bias" on its layer (the oracle reads "l2" itself)."""
    base = o.net_from_specs(specs, input_shape, **kw)
    a = inspect.signature(o.net_from_specs).bind(specs, input_shape, **kw)
    a.apply_defaults()
    a = a.arguments
    net = RegNet(base.layers, seed=a["seed"], dtype=a["dtype"], grad_clip=a["grad_clip"], quirks=a["quirks"], mask_seed=a["mask_seed"],
                 rank=a["rank"])                  # the same seed draws the same initial parameters again
    net.schedules, net.layer_constraints = base.schedules, base.layer_constraints
    off = len(net.layers) - len(specs)            # the convolutionalFlat reshape net_from_specs may prepend
    for s, l in zip(specs, net.layers[off:]):
        if isinstance(l, GEMM):
            l.l1, l.l1_bias, l.l2_bias = (float(s.get(k, 0.0)) for k in ("l1", "l1_bias", "l2_bias"))
    return net
