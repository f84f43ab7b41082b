"""Weight noise (b2g_weight_noise in include/b200gan.h: DL4J's DropConnect and WeightNoise) on top of the DL4J oracle, with the library's
draws restated exactly: a train-mode pass draws W' (and b') of every noisy layer once at its top, uses them in that layer's forward and input
gradient, and leaves the weight and bias gradients straight through.  The pass counter is the net's DropoutState, shared with its
DropoutLayers (tests/noise_ref.py): the draw advances it only when no DropoutLayer of the pass will.

DL4J 1.0.0-beta3, recalled; parity unpinned like the rest of the DL4J semantics.  The points of medium confidence are WeightNoiseQuirks fields."""
import math
from dataclasses import dataclass

import numpy as np

from oracle import dl4j_oracle as o
import noise_ref as nr


@dataclass(frozen=True)
class WeightNoiseQuirks:
    # DropConnect applies ND4J's DropOut op, not DropOutInverted: W' = keep ? W : 0, not rescaled by 1 / p
    dropconnect_inverted: bool = False
    # DL4J's `train && isWeight || (applyToBias && isBias)` also perturbs biases at inference; the library perturbs nothing there (a deviation)
    noise_on_bias_in_inference: bool = False


WQ = WeightNoiseQuirks()
GEMM = (o.Conv2D, o.Deconv2D, o.Dense)


def internal_w(layer, W):
    """W in the library's internal [A][taps][B] order, flattened: conv [nOut][kH*kW][nIn], transposed conv [nIn][kH*kW][nOut], dense [nOut][nIn]."""
    if isinstance(layer, o.Dense):
        return np.asarray(W).T.ravel()
    a, b = W.shape[0], W.shape[1]
    return np.asarray(W).reshape(a, b, -1).transpose(0, 2, 1).ravel()


def dl4j_w(layer, flat):
    """The inverse of internal_w: the internal order back to the layer's W shape."""
    W = layer.params["W"]
    if isinstance(layer, o.Dense):
        return np.asarray(flat).reshape(W.shape[1], W.shape[0]).T
    a, b = W.shape[0], W.shape[1]
    return np.asarray(flat).reshape(a, -1, b).transpose(0, 2, 1).reshape(W.shape)


def bias_j0(n_w: int) -> int:
    """Draw index of bias element 0: 4 * ceil(n_W / 4), so W and b never share a Philox counter."""
    return 4 * ((n_w + 3) // 4)


def drop_connect_p(wn, counters=(0, 0)) -> np.float32:
    """DropConnect's retain probability of a pass: the constant, or the schedule's fp32 value at the pass's (iteration, epoch) clamped to
    [2^-32, 1]."""
    p = wn["p"]
    if isinstance(p, dict):
        return nr.clamp_value("dropout", o.lr_at(p, *counters))
    return np.float32(p)


def draw(wn, n, j0, seed, rank, layer, pass_, p=None):
    """The draws of n elements with indices j0 .. j0 + n - 1 (j0 a multiple of 4): DropConnect's keep bits (bool), or WeightNoise's noise n in
    fp32: NORMAL fmaf(std, z, mean) with the Box-Muller z of noise_ref (float64 here), UNIFORM fmaf(upper - lower, (x >> 8) 2^-24, lower)."""
    assert j0 % 4 == 0
    g1 = ((j0 + n + 3) // 4) * 4
    words = nr.philox_words(seed, rank, layer, pass_, j0, g1)
    if wn["weight_noise"] == "drop_connect":
        p = np.float32(p)
        if p >= 1:
            return np.ones(n, bool)
        return words[:n] < np.uint64(math.floor(float(p) * 2.0 ** 32))
    d = wn["distribution"]
    if d["distribution"] == "normal":
        w4 = words.reshape(-1, 4)
        z = np.empty(w4.shape)
        z[:, 0], z[:, 1] = nr.box_muller(w4[:, 0], w4[:, 1])
        z[:, 2], z[:, 3] = nr.box_muller(w4[:, 2], w4[:, 3])
        return (np.float32(d["std"]) * z.ravel()[:n] + np.float32(d["mean"])).astype(np.float32)
    lo, hi = np.float32(d["lower"]), np.float32(d["upper"])
    u = (words[:n] >> np.uint64(8)).astype(np.float64) * 2.0 ** -24
    return (np.float64(np.float32(hi - lo)) * u + np.float64(lo)).astype(np.float32)


def apply(wn, w, d, p=None, q: WeightNoiseQuirks = WQ):
    """W' from the clean values w and the draws d, in w's dtype (float32: the library's fp32 operand, each result rounded once)."""
    t = w.dtype.type
    if wn["weight_noise"] == "drop_connect":
        kept = w / t(np.float32(p)) if q.dropconnect_inverted else w
        return np.where(d, kept, t(0))
    n = d.astype(w.dtype)
    return (w + n if wn.get("additive", True) else w * n).astype(w.dtype)


def noisy_operands(layer, wn, index, seed, rank, pass_, counters=(0, 0), dtype=np.float32, q: WeightNoiseQuirks = WQ):
    """(W' in the internal order, b' or None) of one layer for pass `pass_`, from its parameters taken as `dtype`."""
    p = drop_connect_p(wn, counters) if wn["weight_noise"] == "drop_connect" else None
    w = internal_w(layer, layer.params["W"]).astype(dtype)
    w_n = apply(wn, w, draw(wn, w.size, 0, seed, rank, index, pass_, p), p, q)
    b_n = None
    if wn.get("apply_to_bias", False) and getattr(layer, "has_bias", False):
        b = np.asarray(layer.params["b"]).astype(dtype)
        b_n = apply(wn, b, draw(wn, b.size, bias_j0(w.size), seed, rank, index, pass_, p), p, q)
    return w_n, b_n


def active(layer) -> bool:
    """A layer whose train-mode passes draw: it has weight noise, is not frozen, and is not a constant DropConnect(1)."""
    wn = getattr(layer, "wn", None)
    if wn is None or getattr(layer, "frozen", False):
        return False
    return wn["weight_noise"] != "drop_connect" or isinstance(wn["p"], dict) or np.float32(wn["p"]) < 1


class NoisyLayerMixin:
    """A GEMM layer whose forward and backward run on the W' (b') its net drew for the pass (wn_draw), with dW, db from x and dy as always."""

    def _run(self, fn, *args):
        if getattr(self, "_wn_live", None) is None:
            return fn(*args)
        clean = {k: self.params[k] for k in self._wn_live}
        self.params.update(self._wn_live)
        try:
            return fn(*args)
        finally:
            self.params.update(clean)

    def forward(self, x, train):
        if not train:
            self._wn_live = None
        return self._run(super().forward, x, train)

    def backward(self, eps):
        return self._run(super().backward, eps)


class WeightNoiseNet(o.Net):
    """An oracle Net whose train-mode forwards draw the weight noise of its noisy layers at the top of the pass."""

    def wn_counters(self):
        c = getattr(self.dropout, "counters", None)
        return c() if c is not None else (self.iteration, self.epoch)

    def wn_draw(self):
        noisy = [l for l in self.layers if active(l)]
        if not noisy:
            return
        pass_, _ = self.dropout.current()
        for l in noisy:
            w, b = noisy_operands(l, l.wn, l.wn_index, self.dropout.seed, self.dropout.rank, pass_, self.wn_counters(), self.dtype, l.wq)
            l._wn_live = {"W": dl4j_w(l, w)} | ({"b": b} if b is not None else {})
        if not any(isinstance(l, o.Dropout) and l.active() for l in self.layers):
            self.dropout.finish()

    def forward(self, x, train: bool, collect: bool = False):
        for l in self.layers:
            if isinstance(l, NoisyLayerMixin):
                l._wn_live = None
        if train:
            self.wn_draw()
        return super().forward(x, train, collect)

    def _has_active_dropout(self) -> bool:
        """Stochastic pass: a DropoutLayer or a noisy layer draws (o.gan_step then runs real | fake as one pass of P, the G step's D pass P + 1)."""
        return super()._has_active_dropout() or any(active(l) for l in self.layers)


_CLASSES = {}


def _noisy_class(cls):
    if cls not in _CLASSES:
        _CLASSES[cls] = type("Noisy" + cls.__name__, (NoisyLayerMixin, cls), {})
    return _CLASSES[cls]


def set_weight_noise(net, wn, layer=None, index=None, q: WeightNoiseQuirks = WQ):
    """The library Net's set_weight_noise on an oracle net: layer None = every non-frozen GEMM layer; wn None clears.  index: layer name ->
    the library's chain index (the Philox word L); default: the position among the net's layers."""
    if not isinstance(net, WeightNoiseNet):
        net.__class__ = WeightNoiseNet
    for i, l in enumerate(net.layers):
        if not isinstance(l, GEMM) or (layer is not None and l.name != layer) or (layer is None and getattr(l, "frozen", False)):
            continue
        if not isinstance(l, NoisyLayerMixin):
            l.__class__ = _noisy_class(type(l))
            l._wn_live = None
        l.wn, l.wq = wn, q
        l.wn_index = index[l.name] if index is not None else i
    return net


def attach(net, specs, off=None):
    """Puts each spec's "weight_noise" on its layer of `net` (built by o.net_from_specs or noise_ref.net_from_specs); the Philox word L is the
    spec's position.  Returns net."""
    if off is None:
        off = len(net.layers) - len(specs)
    index = {s["name"]: i for i, s in enumerate(specs)}
    if not isinstance(net, WeightNoiseNet):
        net.__class__ = WeightNoiseNet
    for s in specs:
        if s.get("weight_noise") is not None:
            set_weight_noise(net, s["weight_noise"], s["name"], index)
    if not hasattr(net.dropout, "counters"):
        net.dropout.counters = lambda: (net.iteration, net.epoch)
    return net


def net_from_specs(specs, input_shape, **kw):
    """noise_ref.net_from_specs (any dropout kind) with each spec's weight noise."""
    return attach(nr.net_from_specs([{k: v for k, v in s.items() if k != "weight_noise"} for s in specs], input_shape, **kw), specs)


def gan_step(G, D, *args, **kw):
    """o.gan_step through noise_ref.gan_step: D's scheduled values (DropConnect p included) at D's counters in the D step and at G's in the
    generator step's pass through D; D's real and fake minibatches share one draw (pass P), the generator pass draws with P + 1."""
    return nr.gan_step(G, D, *args, **kw)
