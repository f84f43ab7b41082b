"""DL4J 1.0.0-beta3's ElementWiseVertex and MergeVertex restated in float64 on the unchanged oracle (semantics at b2g_elementwise_op in
include/b200gan.h), for spine-plus-skip graphs: entry i reads entry i-1's output, and a vertex also reads an earlier entry j's output.

The oracle's Net walks its layers as a chain, in forward (Net.forward) and in every backward (backward_from, backward_from_prefix and the
generator loop of gan_step).  The skip edges ride along that walk without changing it: a skip source remembers its output in the net's
GraphState when its forward runs, a vertex reads it there and leaves the skip input's share of its epsilon in the state's float64
accumulator of j (the first vertex the backward visits writes it, the later ones add), and the source adds that accumulator to the spine
epsilon when its own backward starts.  So all three backward walks are skip-aware, and a net without vertices computes what it always did."""
import numpy as np

from oracle import dl4j_oracle as o

import cnn_loss_ref


class GraphState:
    """The skip sources' forward outputs and gradient accumulators of one net (keyed by the oracle layer index)."""

    def __init__(self):
        self.outs, self.acc = {}, {}

    def add(self, j, g):
        self.acc[j] = self.acc[j] + g if j in self.acc else g


class SkipSource:
    """Mixed into a skip source's own layer class (source_class): remembers the output, adds the accumulated skip gradient in backward."""

    def forward(self, x, train):
        y = super().forward(x, train)
        self.gstate.outs[self.gidx] = y
        self.gstate.acc.pop(self.gidx, None)       # a new forward starts a new backward
        return y

    def backward(self, eps):
        a = self.gstate.acc.pop(self.gidx, None)
        if a is not None:
            eps = eps + a.reshape(eps.shape)
        return super().backward(eps)


_SOURCE_CLASSES = {}


def source_class(cls):
    if cls not in _SOURCE_CLASSES:
        _SOURCE_CLASSES[cls] = type("Skip" + cls.__name__, (SkipSource, cls), {})
    return _SOURCE_CLASSES[cls]


OPS = ("add", "subtract", "product", "average", "max")


def ew_forward(op, a, b):
    if op == "add":
        return a + b
    if op == "subtract":
        return a - b
    if op == "product":
        return a * b
    if op == "average":
        return (a + b) * 0.5
    return np.where(a >= b, a, b)           # a tie takes the first input


def ew_backward(op, e, a, b):
    """(dL/da, dL/db) of ew_forward; MAX sends e to the larger input, a tie to the first."""
    if op == "add":
        return e, e
    if op == "subtract":
        return e, -e
    if op == "product":
        return e * b, e * a
    if op == "average":
        return e * 0.5, e * 0.5
    first = a >= b
    return np.where(first, e, 0.0), np.where(first, 0.0, e)


class ElementWiseVertex(o.Layer):
    """new ElementWiseVertex(op) on (spine, skip) (order 0) or (skip, spine) (order 1); no parameters."""

    def __init__(self, op, src, order, gstate, name=""):
        assert op in OPS, op
        self.op, self.src, self.order, self.gstate, self.name = op, src, order, gstate, name

    def forward(self, x, train):
        s = self.gstate.outs[self.src]
        self._a, self._b = (x, s) if self.order == 0 else (s, x)
        return ew_forward(self.op, self._a, self._b)

    def backward(self, eps):
        da, db = ew_backward(self.op, eps, self._a, self._b)
        spine, skip = (da, db) if self.order == 0 else (db, da)
        self.gstate.add(self.src, skip)
        return spine


class MergeVertex(o.Layer):
    """new MergeVertex(): the inputs concatenated along dimension 1 in input order; no parameters."""

    def __init__(self, src, order, src_channels, gstate, name=""):
        self.src, self.order, self.src_c, self.gstate, self.name = src, order, src_channels, gstate, name

    def out_shape(self, s):
        return (s[0], s[1] + self.src_c) + tuple(s[2:])

    def forward(self, x, train):
        s = self.gstate.outs[self.src]
        self._cx = x.shape[1]
        return np.concatenate((x, s) if self.order == 0 else (s, x), axis=1)

    def backward(self, eps):
        cs = self._cx if self.order == 0 else self.src_c
        first, second = eps[:, :cs], eps[:, cs:]
        spine, skip = (first, second) if self.order == 0 else (second, first)
        self.gstate.add(self.src, np.ascontiguousarray(skip))
        return np.ascontiguousarray(spine)


def net_from_specs(specs, input_shape, *, dtype=np.float64, seed=1, quirks=o.DEFAULT_QUIRKS, grad_clip=0.0, flat_input=True, mask_seed=666,
                   rank=0) -> o.Net:
    """oracle.dl4j_oracle.net_from_specs (with cnn_loss_ref's CnnLossLayer) for specs that may hold "elementwise" / "merge" vertices, resolved
    as the library resolves them (engine.resolve_vertices).  Each other layer is built by the oracle's own builder from its spec alone.  The
    layer indices are the specs' (+ 1 with the convolutionalFlat reshape, as in the oracle)."""
    from gan_deeplearning4j_b200.engine import resolve_vertices
    skips = resolve_vertices(specs)
    gstate = GraphState()
    layers, shape, off = [], (1,) + tuple(input_shape), 0
    if len(input_shape) == 3 and flat_input:
        layers.append(o.Reshape(tuple(input_shape), name="in_reshape"))
        off = 1
    out_shapes, schedules = [], {}
    for i, s in enumerate(specs):
        if s["type"] == "elementwise":
            l = ElementWiseVertex(s["op"], skips[i][0] + off, skips[i][1], gstate, s.get("name", ""))
        elif s["type"] == "merge":
            j = skips[i][0]
            l = MergeVertex(j + off, skips[i][1], out_shapes[j][1], gstate, s.get("name", ""))
        else:
            l = cnn_loss_ref.net_from_specs([s], shape[1:], dtype=dtype, quirks=quirks, flat_input=False).layers[-1]
            if isinstance(l, o.Dropout):
                l.index = i             # the mask's layer index is the position in the specs, as the library and the oracle's builder count it
            lr = (s.get("updater") or {}).get("lr")
            if isinstance(lr, dict):
                schedules[s.get("name", "")] = lr
        layers.append(l)
        shape = l.out_shape(shape)
        out_shapes.append(shape)
    for i, sk in enumerate(skips):
        if sk is not None:
            src = layers[sk[0] + off]
            if not isinstance(src, SkipSource):
                src.__class__ = source_class(type(src))
                src.gstate, src.gidx = gstate, sk[0] + off
    net = o.Net(layers, seed=seed, dtype=dtype, grad_clip=grad_clip, quirks=quirks, mask_seed=mask_seed, rank=rank)
    for l in net.layers:
        if isinstance(l, cnn_loss_ref.CnnLossLayer):
            l.q = net.q
    for name, sched in schedules.items():
        net.set_lr_schedule(sched, name)
    return net
