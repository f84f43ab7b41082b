"""Test-only float64 restatement of DL4J's average, sum and p-norm pooling (SubsamplingLayer AVG / SUM / PNORM with padding, GlobalPoolingLayer
MAX / AVG / SUM / PNORM) on top of the DL4J oracle (oracle/dl4j_oracle.py) without changing it.

Semantics recalled from DL4J 1.0.0-beta3 (PARITY UNPINNED, like the rest of the oracle; the library's statement is include/b200gan.h,
b2g_pooling).  Truncate geometry OH = (H + 2 ph - kh) / sh + 1; positions outside the input are zero padding.
  AVG    y = window sum / (kh*kw)                dx += eps / (kh*kw)
  SUM    y = window sum                          dx += eps
  PNORM  y = (sum |x|^p)^(1/p)                   dx += eps * sign(x)|x|^(p-1) / max(y^(p-1), 1e-8)
GlobalPoolingLayer pools over H x W to [mb, C]; MAX routes eps to the first maximum in row-major pixel order.  The recalls of medium confidence
are PoolQuirks flags; the engine implements the defaults.  The p-norm floor is SubsamplingLayer's eps; DL4J's GlobalPoolingLayer has no floor
(a zero map gives NaN there), so for global pooling the floor is a deliberate deviation of the library, kept here as the default.

`oracle_from_specs` builds an oracle Net from specs that may hold {"type": "subsampling"} / {"type": "global_pooling"} layers: it delegates to
activation_ref (losses, activations, updaters, dropout-free specs) with an identity stand-in for each pooling layer, then puts the pooling layers
in place and corrects the shapes the stand-ins hid from the builder."""
from __future__ import annotations

import dataclasses

import numpy as np

import activation_ref as ar
from oracle import dl4j_oracle as o

KINDS = ("max", "avg", "sum", "pnorm")
CODES = {k: i for i, k in enumerate(KINDS)}
PNORM_EPS = 1e-8


@dataclasses.dataclass
class PoolQuirks:
    avg_include_pad_in_divisor: bool = True   # [recall, medium] AVG divides by kh*kw, padding included (beta4 added the switch)
    pnorm_denominator_floor: bool = True      # [recall, medium] y^(p-1) floored at 1e-8 (SubsamplingLayer); global pooling: deliberate deviation
    global_max_first_tie: bool = True         # [recall, medium] global MAX routes eps to the FIRST maximum in row-major order (False: the last)


DEFAULT_POOL_QUIRKS = PoolQuirks()


def _den(y, p, q):
    d = y ** (p - 1)
    return np.maximum(d, PNORM_EPS) if q.pnorm_denominator_floor else d


def _num(x, p):
    return np.sign(x) * np.abs(x) ** (p - 1)


def pool2d_forward(kind, x, kernel, stride, padding, p=2, q: PoolQuirks = DEFAULT_POOL_QUIRKS):
    """x [N,C,H,W] float64 -> y [N,C,OH,OW]."""
    (kh, kw), (sh, sw), (ph, pw) = kernel, stride, padding
    cols = o.im2col(np.asarray(x, np.float64), kh, kw, sh, sw, ph, pw)          # [N,OH,OW,C,kh,kw], zero padded
    if kind == "avg":
        if q.avg_include_pad_in_divisor:
            div = kh * kw
        else:
            div = o.im2col(np.ones((1, 1) + x.shape[2:]), kh, kw, sh, sw, ph, pw).sum((-2, -1))[0, :, :, 0][None, :, :, None]
        y = cols.sum((-2, -1)) / div
    elif kind == "sum":
        y = cols.sum((-2, -1))
    elif kind == "pnorm":
        y = (np.abs(cols) ** p).sum((-2, -1)) ** (1.0 / p)
    else:
        raise ValueError(kind)
    return y.transpose(0, 3, 1, 2)


def pool2d_backward(kind, x, y, eps, kernel, stride, padding, p=2, q: PoolQuirks = DEFAULT_POOL_QUIRKS):
    """dL/dx [N,C,H,W] from eps = dL/dy [N,C,OH,OW] (y = the forward's output)."""
    (kh, kw), (sh, sw), (ph, pw) = kernel, stride, padding
    x = np.asarray(x, np.float64)
    e = np.asarray(eps, np.float64).transpose(0, 2, 3, 1)[..., None, None]      # [N,OH,OW,C,1,1]
    shape = e.shape[:4] + (kh, kw)
    if kind == "avg":
        if q.avg_include_pad_in_divisor:
            dcols = np.broadcast_to(e / (kh * kw), shape)
        else:
            cnt = o.im2col(np.ones((1, 1) + x.shape[2:]), kh, kw, sh, sw, ph, pw).sum((-2, -1))[0, :, :, 0][None, :, :, None, None, None]
            dcols = np.broadcast_to(e / cnt, shape)
    elif kind == "sum":
        dcols = np.broadcast_to(e, shape)
    elif kind == "pnorm":
        cols = o.im2col(x, kh, kw, sh, sw, ph, pw)
        yy = np.asarray(y, np.float64).transpose(0, 2, 3, 1)[..., None, None]
        dcols = e * _num(cols, p) / _den(yy, p, q)
    else:
        raise ValueError(kind)
    return o.col2im(np.ascontiguousarray(dcols), x.shape, kh, kw, sh, sw, ph, pw)


def global_forward(kind, x, p=2, q: PoolQuirks = DEFAULT_POOL_QUIRKS):
    """x [N,C,H,W] (or [N,C]) -> (y [N,C], MAX's row-major pixel index [N,C] or None)."""
    x = np.asarray(x, np.float64)
    f = x.reshape(x.shape[0], x.shape[1], -1)
    if kind == "max":
        idx = f.argmax(-1) if q.global_max_first_tie else f.shape[-1] - 1 - f[..., ::-1].argmax(-1)
        return np.take_along_axis(f, idx[..., None], -1)[..., 0], idx
    if kind == "avg":
        return f.mean(-1), None
    if kind == "sum":
        return f.sum(-1), None
    if kind == "pnorm":
        return (np.abs(f) ** p).sum(-1) ** (1.0 / p), None
    raise ValueError(kind)


def global_backward(kind, x, y, idx, eps, p=2, q: PoolQuirks = DEFAULT_POOL_QUIRKS):
    x = np.asarray(x, np.float64)
    f = x.reshape(x.shape[0], x.shape[1], -1)
    e = np.asarray(eps, np.float64)[..., None]
    if kind == "max":
        d = np.zeros_like(f)
        np.put_along_axis(d, idx[..., None], e, -1)
    elif kind == "avg":
        d = np.broadcast_to(e / f.shape[-1], f.shape)
    elif kind == "sum":
        d = np.broadcast_to(e, f.shape)
    elif kind == "pnorm":
        d = e * _num(f, p) / _den(np.asarray(y, np.float64)[..., None], p, q)
    else:
        raise ValueError(kind)
    return np.ascontiguousarray(d).reshape(x.shape)


class Subsampling(o.Layer):
    """SubsamplingLayer.Builder(PoolingType.AVG / SUM / PNORM).kernelSize().stride().padding().pnorm()."""

    def __init__(self, kind, kernel, stride=(1, 1), padding=(0, 0), p=2, name="", quirks: PoolQuirks = DEFAULT_POOL_QUIRKS):
        self.kind, self.k, self.s, self.pad, self.p, self.name, self.q = kind, tuple(kernel), tuple(stride), tuple(padding), p, name, quirks

    def init(self, rng, dtype):
        super().init(rng, dtype)

    def out_shape(self, s):
        n, c, h, w = s
        return (n, c, o.out_size(h, self.k[0], self.s[0], self.pad[0]), o.out_size(w, self.k[1], self.s[1], self.pad[1]))

    def forward(self, x, train):
        self._x = x
        self._y = pool2d_forward(self.kind, x, self.k, self.s, self.pad, self.p, self.q)
        return self._y

    def backward(self, eps):
        return pool2d_backward(self.kind, self._x, self._y, eps, self.k, self.s, self.pad, self.p, self.q)


class GlobalPooling(o.Layer):
    """GlobalPoolingLayer.Builder(PoolingType).pnorm(p): [N,C,H,W] -> [N,C]."""

    def __init__(self, kind="max", p=2, name="", quirks: PoolQuirks = DEFAULT_POOL_QUIRKS):
        self.kind, self.p, self.name, self.q = kind, p, name, quirks

    def init(self, rng, dtype):
        super().init(rng, dtype)

    def out_shape(self, s):
        return (s[0], s[1])

    def forward(self, x, train):
        self._x = x
        self._y, self._idx = global_forward(self.kind, x, self.p, self.q)
        return self._y

    def backward(self, eps):
        return global_backward(self.kind, self._x, self._y, self._idx, eps, self.p, self.q)


# ------------------------------------------------------------------ specs -> oracle net ----------------------------------------------------
def spec_shapes(specs, input_shape):
    """The input shape (C, H, W) of every spec, as the engine infers it (feed-forward: (F, 1, 1))."""
    c, h, w = input_shape if len(input_shape) == 3 else (input_shape[0], 1, 1)
    out = []
    for s in specs:
        out.append((c, h, w))
        t = s["type"]
        k, st, p = s.get("kernel", (1, 1)), s.get("stride", (1, 1)), s.get("padding", (0, 0))
        if t == "conv2d":
            c, h, w = s["n_out"], o.out_size(h, k[0], st[0], p[0]), o.out_size(w, k[1], st[1], p[1])
        elif t == "deconv2d":
            c, h, w = s["n_out"], st[0] * (h - 1) + k[0] - 2 * p[0], st[1] * (w - 1) + k[1] - 2 * p[1]
        elif t in ("dense", "output"):
            c, h, w = s["n_out"], 1, 1
        elif t in ("maxpool", "subsampling"):
            h, w = o.out_size(h, k[0], st[0], p[0] if t == "subsampling" else 0), o.out_size(w, k[1], st[1], p[1] if t == "subsampling" else 0)
        elif t == "upsample2d":
            h, w = h * s.get("size", 2), w * s.get("size", 2)
        elif t == "ff_to_cnn":
            h, w, c = s["to"]
        elif t in ("cnn_to_ff", "global_pooling"):
            c, h, w = (c * h * w if t == "cnn_to_ff" else c), 1, 1
    return out


def oracle_from_specs(specs, input_shape, quirks: PoolQuirks = DEFAULT_POOL_QUIRKS, **kw):
    """activation_ref.oracle_from_specs for specs that may hold subsampling / global_pooling layers (see the module docstring)."""
    shapes = spec_shapes(specs, input_shape)
    stand_in = []
    for s, (c, h, w) in zip(specs, shapes):
        if s["type"] in ("subsampling", "global_pooling"):
            stand_in.append({"type": "activation", "activation": "identity", "name": s.get("name", "")})
        elif s["type"] in ("conv2d", "deconv2d", "dense", "output") and not s.get("n_in"):
            stand_in.append(dict(s, n_in=c * h * w if s["type"] in ("dense", "output") else c))
        else:
            stand_in.append(s)
    net = ar.oracle_from_specs(stand_in, input_shape, **kw)
    shift = len(net.layers) - len(specs)
    for i, (s, (c, h, w)) in enumerate(zip(specs, shapes)):
        if s["type"] == "subsampling":
            layer = Subsampling(s["pooling"], s["kernel"], s.get("stride", (1, 1)), s.get("padding", (0, 0)), s.get("pnorm", 0), s.get("name", ""), quirks)
        elif s["type"] == "global_pooling":
            layer = GlobalPooling(s.get("pooling", "max"), s.get("pnorm", 2), s.get("name", ""), quirks)
        elif s["type"] == "cnn_to_ff":
            net.layers[i + shift].to_shape = (c * h * w,)          # the builder saw the stand-ins' unreduced shapes
            continue
        else:
            continue
        layer.init(None, net.dtype)
        if s.get("frozen", False):
            layer.frozen = True
        net.layers[i + shift] = layer
    return net
