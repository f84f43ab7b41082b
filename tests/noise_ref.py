"""The other IDropout kinds of a DropoutLayer (b2g_dropout_kind in include/b200gan.h) on top of the DL4J oracle: GaussianDropout,
GaussianNoise, AlphaDropout and SpatialDropout with the library's draws restated exactly, as a Dropout layer the oracle's Net and gan_step
treat like its own (one pass counter, the last stochastic layer advances it).

DL4J 1.0.0-beta3, recalled; parity unpinned like the rest of the DL4J semantics.  The recalled constants are NoiseQuirks fields."""
import math
from dataclasses import dataclass

import numpy as np

from oracle import dl4j_oracle as o


@dataclass(frozen=True)
class NoiseQuirks:
    selu_alpha: float = 1.6732632423543772       # AlphaDropout's alpha' = -lambda * alpha (SELU's constants)
    selu_lambda: float = 1.0507009873554805
    # the library's Box-Muller: u = ((x_even >> 9) + 0.5) 2^-23 and v = (x_odd >> 8) 2^-24, so |z| <= sqrt(-2 ln 2^-24); DL4J draws its own
    u_shift: int = 9
    v_shift: int = 8


NQ = NoiseQuirks()
KINDS = ("dropout", "gaussian_dropout", "gaussian_noise", "alpha_dropout", "spatial_dropout")
VALUE_KEY = {"dropout": "p", "gaussian_dropout": "rate", "gaussian_noise": "stddev", "alpha_dropout": "p", "spatial_dropout": "p"}
Z_MAX = math.sqrt(-2.0 * math.log(2.0 ** -24))


def philox_words(seed, rank, layer, pass_, j0, j1):
    """The Philox4x32-10 word of each draw index j in [j0, j1) (uint32): word j & 3 of counter {j >> 2, lo32(P), hi32(P), L | r << 16}."""
    seed, pass_ = int(seed) or 666, int(pass_)
    g = np.arange(j0 >> 2, ((j1 - 1) >> 2) + 1, dtype=np.uint64)
    words = np.stack(o.philox4x32_10((g, pass_ & 0xFFFFFFFF, pass_ >> 32, int(layer) | (int(rank) << 16)), (seed & 0xFFFFFFFF, seed >> 32)), -1).ravel()
    return words[j0 - 4 * (j0 >> 2):][:j1 - j0]


def box_muller(x_even, x_odd, q: NoiseQuirks = NQ):
    """float64 normals (z_even, z_odd) of Philox word pairs, from the library's exact u and v."""
    u = ((np.asarray(x_even, np.uint64) >> np.uint64(q.u_shift)).astype(np.float64) + 0.5) * 2.0 ** -23
    v = (np.asarray(x_odd, np.uint64) >> np.uint64(q.v_shift)).astype(np.float64) * 2.0 ** -24
    r = np.sqrt(-2.0 * np.log(u))
    return r * np.cos(2 * np.pi * v), r * np.sin(2 * np.pi * v)


def dropout_normals(seed, rank, layer, pass_, rows, h, w, c, row0=0, q: NoiseQuirks = NQ):
    """The normal z of each element of rows [row0, row0 + rows) of pass `pass_`, in float64, NCHW [rows, c, h, w]: element e (its NHWC index in
    the pass) takes z[e & 3] of the four normals its counter e >> 2 gives, pair (x0, x1) -> z0, z1 and pair (x2, x3) -> z2, z3."""
    per = h * w * c
    e0, e1 = row0 * per, (row0 + rows) * per
    g0 = e0 >> 2
    words = philox_words(seed, rank, layer, pass_, 4 * g0, 4 * (((e1 - 1) >> 2) + 1)).reshape(-1, 4)
    z = np.empty(words.shape)
    z[:, 0], z[:, 1] = box_muller(words[:, 0], words[:, 1], q)
    z[:, 2], z[:, 3] = box_muller(words[:, 2], words[:, 3], q)
    return z.ravel()[e0 - 4 * g0:][:e1 - e0].reshape(rows, h, w, c).transpose(0, 3, 1, 2)


def spatial_mask(seed, rank, layer, pass_, rows, c, p, row0=0):
    """SpatialDropout's keep bit of each (row, channel) of rows [row0, row0 + rows), [rows, c]: draw index j = row * C + c."""
    p = np.float32(p)
    if p >= 1:
        return np.ones((rows, c), bool)
    words = philox_words(seed, rank, layer, pass_, row0 * c, (row0 + rows) * c)
    return (words < np.uint64(math.floor(float(p) * 2.0 ** 32))).reshape(rows, c)


def clamp_value(kind, v) -> np.float32:
    """A scheduled value clamped into its kind's range (the library's documented deviation): rate to [0, 1 - 2^-24], stddev to >= 0, p to
    [2^-32, 1]."""
    v = np.float32(v)
    if kind == "gaussian_dropout":
        return np.float32(min(max(v, np.float32(0)), np.float32(1 - 2.0 ** -24)))
    if kind == "gaussian_noise":
        return np.float32(max(v, np.float32(0)))
    return np.float32(min(max(v, np.float32(2.0 ** -32)), np.float32(1)))


def gaussian_sigma(rate) -> np.float32:
    """GaussianDropout's stddev sqrt(rate / (1 - rate)), in double from the fp32 rate, rounded to fp32 once."""
    r = float(np.float32(rate))
    return np.float32(math.sqrt(r / (1.0 - r)))


def alpha_coefficients(p, q: NoiseQuirks = NQ):
    """AlphaDropout's (a, b, alpha') for the fp32 retain probability p: alpha' = -lambda alpha, a = 1 / sqrt(p + alpha'^2 p (1 - p)),
    b = -a (1 - p) alpha', each in double and rounded to fp32 once."""
    p = float(np.float32(p))
    ap = -q.selu_lambda * q.selu_alpha
    a = 1.0 / math.sqrt(p + ap * ap * p * (1.0 - p))
    return np.float32(a), np.float32(-a * (1.0 - p) * ap), np.float32(ap)


class NoiseDropout(o.Dropout):
    """DropoutLayer.Builder(IDropout) of one of KINDS with its value (p, rate or stddev).  Train mode draws from the net's DropoutState as the
    oracle's Dropout does; the identity cases (p = 1, rate = 0, stddev = 0, frozen, inference) draw nothing and count no pass."""

    def __init__(self, kind, value, name="", index=0, state=None, frozen=False, q: NoiseQuirks = NQ, schedule=None):
        assert kind in KINDS, kind
        super().__init__(1.0, name, index, state, frozen)
        self.kind, self.value, self.nq, self.schedule = kind, float(np.float32(value)), q, schedule
        self._dm = None

    def active(self):
        if self.frozen:
            return False
        if self.schedule is not None:          # a scheduled layer is stochastic whatever its value
            return True
        return self.value > 0 if self.kind in ("gaussian_dropout", "gaussian_noise") else self.value < 1

    def current_value(self) -> float:
        """The value the next train-mode forward uses: the schedule's fp32 value at the counters of the pass, clamped into the kind's range,
        or the constant."""
        if self.schedule is None:
            return self.value
        it, ep = self.state.counters() if hasattr(self.state, "counters") else (0, 0)
        return float(clamp_value(self.kind, o.lr_at(self.schedule, it, ep)))

    def forward(self, x, train):
        self._m = self._dm = None
        if not train or not self.active():
            return x
        value = self.current_value()
        pass_, row0 = self.state.current()
        _, c, h, w = x.shape if x.ndim == 4 else (x.shape[0], x.shape[1], 1, 1)
        args = (self.state.seed, self.state.rank, self.index, pass_, x.shape[0])
        t = x.dtype.type
        if self.kind == "dropout":
            keep = o.dropout_mask(*args, h, w, c, value, row0).reshape(x.shape)
            self._m = keep * t(np.float32(1) / np.float32(value)); y = x * self._m
        elif self.kind in ("gaussian_noise", "gaussian_dropout"):
            z = dropout_normals(*args, h, w, c, row0, self.nq).reshape(x.shape)
            if self.kind == "gaussian_noise":
                y = x + t(np.float32(value)) * z
            else:
                self._m = 1 + t(gaussian_sigma(value)) * z; y = x * self._m
        elif self.kind == "alpha_dropout":
            keep = o.dropout_mask(*args, h, w, c, value, row0).reshape(x.shape)
            a, b, ap = (t(v) for v in alpha_coefficients(value, self.nq))
            self._m = keep * a; y = a * np.where(keep, x, ap) + b
        else:
            if x.ndim != 4 or h * w == 1:
                raise ValueError("SpatialDropout needs a [N, C, H, W] input")
            keep = spatial_mask(self.state.seed, self.state.rank, self.index, pass_, x.shape[0], c, value, row0)[:, :, None, None]
            self._m = np.broadcast_to(keep * t(np.float32(1) / np.float32(value)), x.shape); y = x * self._m
        if self.last:
            self.state.finish()
        return y


def plain_specs(specs):
    """The specs with every dropout kind other than Dropout(p) replaced by a Dropout(1) placeholder o.net_from_specs reads."""
    out = []
    for s in specs:
        if s["type"] == "dropout" and (s.get("kind", "dropout") != "dropout" or isinstance(s.get("p"), dict)):
            s = {k: v for k, v in s.items() if k not in ("kind", "rate", "stddev", "p")}
            s["p"] = 1.0
        out.append(s)
    return out


def attach(net, specs, off=None):
    """Puts a NoiseDropout at each dropout spec of `net` (built from plain_specs(specs)); off: the oracle's index of spec 0 (1 when it
    prepended its input reshape).  The mask index L stays the spec's position.  Returns net."""
    if off is None:
        off = len(net.layers) - len(specs)
    for i, s in enumerate(specs):
        if s["type"] == "dropout":
            old = net.layers[off + i]
            kind = s.get("kind", "dropout")
            v = s[VALUE_KEY[kind]]
            sched = v if isinstance(v, dict) else None
            l = NoiseDropout(kind, o.value(sched, 0) if sched else v, old.name, index=i, frozen=getattr(old, "frozen", False), schedule=sched)
            l.q = old.q
            net.layers[off + i] = l
    relink(net)
    net.dropout.counters = lambda: (net.iteration, net.epoch)
    return net


def relink(net):
    """The DropoutState links and the last-stochastic-layer flag, as o.Net sets them at construction."""
    drops = [l for l in net.layers if isinstance(l, o.Dropout)]
    for l in drops:
        l.state, l.last = net.dropout, False
    active = [l for l in drops if l.active()]
    if active:
        active[-1].last = True


def net_from_specs(specs, input_shape, **kw):
    """o.net_from_specs for specs with any dropout kind."""
    return attach(o.net_from_specs(plain_specs(specs), input_shape, **kw), specs)


def set_dropout_schedule(net, schedule, layer=None):
    """The library Net's set_dropout_schedule on an oracle net: layer None = every non-frozen DropoutLayer; schedule None = the constant."""
    for l in net.layers:
        if isinstance(l, NoiseDropout) and (l.name == layer if layer is not None else not l.frozen):
            l.schedule = schedule
    relink(net)


def dropout_value(net, layer) -> float:
    return next(l for l in net.layers if isinstance(l, NoiseDropout) and l.name == layer).current_value()


def gan_step(G, D, *args, **kw):
    """o.gan_step with D's scheduled DropoutLayers read at D's counters in the D step and at G's in the generator step's pass through D (the
    reference's stacked gan graph counts its own fits): D's iteration counter moves exactly once, at D's update, between the two."""
    it0 = D.iteration
    D.dropout.counters = lambda: (D.iteration, D.epoch) if D.iteration == it0 else (G.iteration, G.epoch)
    try:
        return o.gan_step(G, D, *args, **kw)
    finally:
        D.dropout.counters = lambda: (D.iteration, D.epoch)
