"""Test-only NumPy restatement of the DropoutLayer, on top of the DL4J oracle (oracle/dl4j_oracle.py) without changing it.

Semantics recalled from DL4J 1.0.0-beta3 (PARITY UNPINNED, like the rest of the oracle): new DropoutLayer.Builder(p), p = the RETAIN
probability; training forward = inverted dropout y = x * m, m = 1/p with probability p else 0; backward dx = dy * m; inference and a
FrozenLayer are the identity.  ND4J's random stream cannot be restated, so the mask is the CUDA library's own definition (include/b200gan.h,
B2G_LAYER_DROPOUT), restated here exactly: parity with DL4J holds in distribution, with the library element for element.

A net's DropoutLayers share one `DropoutState` (seed, rank, pass counter P).  Like the library, the last masking DropoutLayer of a train-mode
forward advances P once it has drawn its mask; `DropoutState.queue` holds explicit (pass, first row) draws that replace the counter for the
next forwards without advancing it.  `gan_step` wraps the oracle's step so that D's real and fake minibatches are rows [0, N) and [N, 2N) of
pass P (the library runs them as one 2N-row pass) and the generator step's D pass is P + 1."""
from __future__ import annotations

import math

import numpy as np

from helpers import oracle_from_specs as _oracle_from_specs
from oracle import dl4j_oracle as o

_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """Philox4x32-10 (Random123 constants), vectorised: ctr = 4 arrays / ints of 32-bit words, key = 2.  Returns the 4 output words (uint32)."""
    c = [np.asarray(v, np.uint64) & _M32 for v in ctr]
    k0, k1 = (np.uint64(int(v) & 0xFFFFFFFF) for v in key)
    m0, m1, w0, w1, sh = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), np.uint64(0x9E3779B9), np.uint64(0xBB67AE85), np.uint64(32)
    for r in range(10):
        if r:
            k0, k1 = (k0 + w0) & _M32, (k1 + w1) & _M32
        p0, p1 = m0 * c[0], m1 * c[2]          # 32 x 32 -> 64-bit products, exact in uint64
        c = [(p1 >> sh) ^ c[1] ^ k0, p1 & _M32, (p0 >> sh) ^ c[3] ^ k1, p0 & _M32]
    return [v.astype(np.uint32) for v in c]


def dropout_mask(seed, rank, layer, pass_, rows, h, w, c, p, row0=0):
    """Keep mask of a DropoutLayer (True = kept) for rows [row0, row0 + rows) of pass `pass_`, returned NCHW [rows, c, h, w].  Element
    e = ((row*h + y)*w + x)*c + ch (NHWC index in the pass) keeps iff p >= 1 or Philox4x32-10(ctr = {e >> 2, lo32(P), hi32(P), layer | rank << 16},
    key = {lo32(S), hi32(S)})[e & 3] < floor(p * 2^32), with p taken as fp32 and S = seed (0 -> 666)."""
    p = np.float32(p)
    per = h * w * c
    e0, e1 = row0 * per, (row0 + rows) * per
    if p >= 1:
        keep = np.ones(e1 - e0, bool)
    else:
        seed, pass_ = int(seed) or 666, int(pass_)
        g = np.arange(e0 >> 2, ((e1 - 1) >> 2) + 1, dtype=np.uint64)
        words = np.stack(philox4x32_10((g, pass_ & 0xFFFFFFFF, pass_ >> 32, int(layer) | (int(rank) << 16)), (seed & 0xFFFFFFFF, seed >> 32)), -1).ravel()
        keep = words[e0 - 4 * (e0 >> 2):][:e1 - e0] < np.uint64(math.floor(float(p) * 2.0 ** 32))
    return keep.reshape(rows, h, w, c).transpose(0, 3, 1, 2)


class DropoutState:
    """The mask inputs a net's DropoutLayers share: seed (the library's b2g_net_config.seed), rank, pass counter P, explicit draws."""

    def __init__(self, seed=666, rank=0):
        self.seed, self.rank, self.pass_, self.queue = seed, rank, 0, []

    def current(self):
        return self.queue[0] if self.queue else (self.pass_, 0)

    def finish(self):          # end of a masking train-mode forward
        if self.queue:
            self.queue.pop(0)
        else:
            self.pass_ += 1


class Dropout(o.Layer):
    """DropoutLayer.Builder(p).  `index` = the layer's chain index in the CUDA library's layer array (the mask's L)."""

    def __init__(self, p, name="", index=0, state=None, frozen=False):
        self.p, self.name, self.index, self.state, self.frozen, self.last = float(np.float32(p)), name, index, state, frozen, False
        self._m = None

    def init(self, rng, dtype):
        super().init(rng, dtype)

    def active(self):
        return self.p < 1 and not self.frozen

    def forward(self, x, train):
        self._m = None
        if not train or self.p >= 1:
            return x
        pass_, row0 = self.state.current()
        _, c, h, w = x.shape if x.ndim == 4 else (x.shape[0], x.shape[1], 1, 1)
        keep = dropout_mask(self.state.seed, self.state.rank, self.index, pass_, x.shape[0], h, w, c, self.p, row0).reshape(x.shape)
        self._m = keep * x.dtype.type(np.float32(1) / np.float32(self.p))
        if self.last:
            self.state.finish()
        return x * self._m

    def backward(self, eps):
        return eps if self._m is None else eps * self._m


def oracle_from_specs(specs, input_shape, mask_seed=666, rank=0, **kw):
    """tests/helpers.oracle_from_specs for specs that may hold {"type": "dropout", "p": p} layers.  The net gets a `dropout` DropoutState;
    each DropoutLayer's chain index is its position in `specs` (the library's index, not the oracle's, which a prepended input reshape shifts)."""
    stand_in = [dict(type="activation", activation="identity", name=s.get("name", "")) if s["type"] == "dropout" else s for s in specs]
    net = _oracle_from_specs(stand_in, input_shape, **kw)
    shift = len(net.layers) - len(specs)
    net.dropout = DropoutState(mask_seed, rank)
    drops = []
    for i, s in enumerate(specs):
        if s["type"] == "dropout":
            d = Dropout(s["p"], s.get("name", ""), i, net.dropout, bool(s.get("frozen", False)))
            d.init(None, net.dtype)
            net.layers[i + shift] = d
            drops.append(d)
    active = [d for d in drops if d.active()]
    if active:
        active[-1].last = True
    return net


def has_active_dropout(net):
    return any(isinstance(l, Dropout) and l.active() for l in net.layers)


def compute_gradient_and_score(net, x, y, pass_, row0=0, collect=False):
    """net.compute_gradient_and_score with the masks of rows [row0, row0 + batch) of pass `pass_`; the pass counter is left alone."""
    if has_active_dropout(net):
        net.dropout.queue.append((pass_, row0))
    return net.compute_gradient_and_score(x, y, collect=collect)


def gan_step(G, D, x_real, z_d, z_g, y_real, y_fake, y_gen, fake_bn_train: bool = False):
    """oracle gan_step with D's DropoutLayers drawn as the library draws them: the real and fake minibatches are rows [0, N) and [N, 2N) of
    pass P, the generator step's D pass is P + 1 (and advances the counter to P + 2)."""
    st = getattr(D, "dropout", None)
    if st is not None and has_active_dropout(D):
        n = x_real.shape[0]
        P = st.pass_
        st.queue += [(P, 0), (P, n)]
        st.pass_ = P + 1
    return o.gan_step(G, D, x_real, z_d, z_g, y_real, y_fake, y_gen, fake_bn_train=fake_bn_train)
