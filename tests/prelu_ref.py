"""PReLULayer (B2G_LAYER_PRELU in include/b200gan.h) on top of the DL4J oracle and the regularization restatement (regularization_ref).

  forward   y = x < 0 ? alpha * x : x
  backward  dx = x < 0 ? alpha * eps : eps;  dalpha = sum over the minibatch and the shared axes of (x < 0 ? x * eps : 0), not divided by it
alpha ("W") has DL4J's weight shape: the layer's input shape ([C, H, W] or [F]) with every shared axis (DL4J's 1-based sharedAxes) of extent 1,
so in the oracle's NCHW layout it broadcasts over the minibatch and the shared axes as it is.  A FrozenLayer PReLU is the same function in both
modes and passes an input gradient, so PReLUNet's backward does not stop at one (the oracle stops at any other frozen layer).
PReLUNet is a RegNet: l1 and l2 reach alpha as they reach a GEMM layer's W (update and score); alpha has no bias.

DL4J 1.0.0-beta3, recalled; parity unpinned like the rest of the DL4J semantics.  The points of medium confidence are PReLUQuirks fields."""
import inspect
from dataclasses import dataclass

import numpy as np

from oracle import dl4j_oracle as o
import regularization_ref as rr


@dataclass(frozen=True)
class PReLUQuirks:
    # beta3's PReLULayer.Builder sets weightInit(ZERO) itself: alpha starts at 0 (a new PReLU is a ReLU) and the global weightInit is not
    # inherited
    alpha_init_zero: bool = True
    # "W" is a weight parameter: the layer's l1 / l2 (and the global builder's) regularize alpha
    alpha_regularized: bool = True
    # libnd4j prelu compares x < 0: x = +-0 is not negative (dy passes, no slope term)
    zero_is_negative: bool = False


PQ = PReLUQuirks()


class PReLU(o.Layer):
    """PReLULayer.Builder().inputShape(in_shape).sharedAxes(shared_axes): in_shape (C, H, W) or (F,), shared_axes DL4J's 1-based axes."""
    has_params = True

    def __init__(self, in_shape, shared_axes=(), updater=None, l2=0.0, name="", l1=0.0):
        self.in_shape = tuple(int(d) for d in in_shape)
        self.shared = tuple(sorted({int(a) for a in shared_axes}))
        if any(a < 1 or a > len(self.in_shape) for a in self.shared):
            raise ValueError(f"prelu {name!r}: shared axes {self.shared} outside the input's {len(self.in_shape)} dimension(s)")
        self.alpha_shape = tuple(1 if i + 1 in self.shared else d for i, d in enumerate(self.in_shape))
        self.updater, self.l2, self.l1, self.name = updater, l2, l1, name

    def param_specs(self):
        return [("W", self.alpha_shape, "c")]

    def l2_names(self):
        return ("W",) if PQ.alpha_regularized else ()

    def init(self, rng, dtype):
        super().init(rng, dtype)
        if not PQ.alpha_init_zero:
            raise NotImplementedError("only beta3's ZERO initial alpha is restated")
        self.params["W"] = np.zeros(self.alpha_shape, dtype)

    def _neg(self, x):
        return x <= 0 if PQ.zero_is_negative else x < 0

    def forward(self, x, train):
        self._x = x
        return np.where(self._neg(x), self.params["W"][None] * x, x)

    def backward(self, eps):
        x, neg = self._x, self._neg(self._x)
        if not getattr(self, "frozen", False):
            axes = (0,) + self.shared           # DL4J axis a is array axis a of the [N, ...] activation
            self.grads["W"] = np.where(neg, x * eps, 0.0).sum(axis=axes, keepdims=True).reshape(self.alpha_shape)
        return np.where(neg, self.params["W"][None] * eps, eps)


class PReLUNet(rr.RegNet):
    """RegNet with PReLU layers: their l1 / l2 in the update and the score, and a backward that passes through a frozen PReLU."""

    def _prelus(self):
        return [(li, l) for li, l in self._live() if isinstance(l, PReLU)]

    def calc_l2(self) -> float:
        return super().calc_l2() + sum(0.5 * l.l2 * float((l.params["W"].astype(np.float64) ** 2).sum()) for _, l in self._prelus()
                                       if l.l2 and PQ.alpha_regularized)

    def calc_l1(self) -> float:
        return super().calc_l1() + sum(l.l1 * float(np.abs(l.params["W"].astype(np.float64)).sum()) for _, l in self._prelus()
                                       if l.l1 and PQ.alpha_regularized)

    def apply_update(self, mb, grads=None, frozen_from=None):
        """RegNet's update (the oracle adds l2 * alpha through l2_names), then l1 * sign(alpha) from alpha before the update."""
        extra = {li: l.l1 * np.sign(l.params["W"]) for li, l in self._prelus() if l.l1 and PQ.alpha_regularized}
        super().apply_update(mb, grads, frozen_from)
        for li, t in extra.items():
            l = self.layers[li]
            l.params["W"] = (l.params["W"] - t).astype(self.dtype)

    def backward_from_prefix(self, eps, collect=False):
        hi = len(self.layers) - 1
        lo = max((i + 1 for i in range(hi) if getattr(self.layers[i], "frozen", False) and not isinstance(self.layers[i], PReLU)), default=0)
        return self._backward(eps, lo, hi, collect)


def net_from_specs(specs, input_shape, **kw):
    """rr.net_from_specs with "prelu" specs: each becomes a PReLU on the shape its input has (the same layers, initial parameters, schedules,
    constraints and coefficients otherwise), with the spec's "shared_axes", "updater", "l1", "l2" and "frozen"."""
    holders = [{"type": "activation", "activation": "identity", "name": s.get("name", ""), "updater": s.get("updater")} if s["type"] == "prelu" else s
               for s in specs]
    base = rr.net_from_specs(holders, input_shape, **kw)
    off = len(base.layers) - len(specs)            # the convolutionalFlat reshape net_from_specs may prepend
    _, acts = base.forward(np.zeros((1,) + tuple(input_shape)), train=False, collect=True)
    layers = list(base.layers)
    for i, s in enumerate(specs):
        if s["type"] != "prelu":
            continue
        in_shape = acts[off + i - 1].shape[1:] if off + i > 0 else tuple(input_shape)
        l = PReLU(in_shape, s.get("shared_axes", ()), o.updater_cfg(s.get("updater")), s.get("l2", 0.0), s.get("name", ""), s.get("l1", 0.0))
        if s.get("frozen", False):
            l.frozen = True
        layers[off + i] = l
    a = inspect.signature(o.net_from_specs).bind(specs, input_shape, **kw)
    a.apply_defaults()
    a = a.arguments
    net = PReLUNet(layers, seed=a["seed"], dtype=a["dtype"], grad_clip=a["grad_clip"], quirks=a["quirks"], mask_seed=a["mask_seed"],
                   rank=a["rank"])                  # PReLU draws nothing at init: the other layers get the same initial parameters
    net.schedules, net.layer_constraints = base.schedules, base.layer_constraints
    return net
