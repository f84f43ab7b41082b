"""DL4J 1.0.0-beta3's CnnLossLayer restated in float64 on the unchanged oracle (semantics at B2G_LAYER_CNN_LOSS in include/b200gan.h): the
[N, C, H, W] map reshaped to [N*H*W, C] rows (reshape4dTo2d), the per-row losses of oracle.dl4j_oracle (xent_score_and_grad,
mcxent_softmax_score_and_grad, score_and_grad), the score summed over the rows.  The medium-confidence recall -- the score divided by the
minibatch, not by the pixel count -- sits behind CnnQuirks."""
import dataclasses
from typing import Optional

import numpy as np

from oracle import dl4j_oracle as o


@dataclasses.dataclass
class CnnQuirks:
    # CnnLossLayer.computeScore: score /= getInputMiniBatchSize() (True); False: the row mean over N*H*W (score and gradient / (H*W) more)
    cnn_loss_score_per_minibatch: bool = True


DEFAULT_CNN_QUIRKS = CnnQuirks()


def to_rows(a):
    """[N, C, H, W] -> [N*H*W, C] (pixel-major, channel-minor: the engine's NHWC buffer)."""
    n, c = a.shape[:2]
    return np.ascontiguousarray(np.moveaxis(a, 1, -1)).reshape(-1, c)


def from_rows(r, shape):
    n, c, h, w = shape
    return np.ascontiguousarray(r.reshape(n, h, w, c).transpose(0, 3, 1, 2))


def softmax_channels(z):
    e = np.exp(z - z.max(1, keepdims=True))
    return e / e.sum(1, keepdims=True)


class CnnLossLayer(o.LossLayer):
    """CnnLossLayer.Builder(loss).activation(act): no parameters; forward returns the activated map (sigmoid for XENT, the per-pixel
    softmax over the channels for MCXENT, act otherwise).  A LossLayer subclass, so the oracle's backward passes skip it as they skip LossLayer."""

    def __init__(self, name="", quirks: Optional[o.Quirks] = None, loss="xent", activation="identity", alpha=0.01,
                 cq: CnnQuirks = DEFAULT_CNN_QUIRKS):
        super().__init__(name, quirks, loss, activation, alpha)
        self.cq = cq
        if loss == "mcxent":
            self.loss_act = "softmax"

    def forward(self, x, train):
        x = np.asarray(x)
        if x.ndim == 2:                       # a feed-forward input is the 1x1 map
            x = x.reshape(x.shape + (1, 1))
        self._z = x
        if self.loss == "mcxent":
            return softmax_channels(x)
        return o._layer_act_forward(self.loss_act, x, self.loss_alpha, self.q)

    def score_and_eps(self, y):
        z = self._z
        y = np.asarray(y, z.dtype).reshape(z.shape)
        zr, yr = to_rows(z), to_rows(y)
        if self.loss == "xent":
            s, g = o.xent_score_and_grad(zr, yr, self.q.xent_clip_eps)
        elif self.loss == "mcxent":
            s, g = o.mcxent_softmax_score_and_grad(zr, yr)
        else:
            s, g = o.score_and_grad(self.loss, self.loss_act, self.loss_alpha, zr, yr, self.q)
        g = from_rows(g, z.shape)
        if not self.cq.cnn_loss_score_per_minibatch:
            hw = z.shape[2] * z.shape[3]
            s, g = s / hw, g / hw
        return float(s), g


def net_from_specs(specs, input_shape, cq: CnnQuirks = DEFAULT_CNN_QUIRKS, **kw):
    """oracle.dl4j_oracle.net_from_specs with "cnn_loss" specs: the net of the specs before a trailing cnn_loss, then the CnnLossLayer (it
    has no parameters, so the other layers' initialisation is that of the same specs without it)."""
    if not specs or specs[-1]["type"] != "cnn_loss":
        return o.net_from_specs(specs, input_shape, **kw)
    if any(s["type"] == "cnn_loss" for s in specs[:-1]):
        raise ValueError("a cnn_loss spec must be the last layer")
    net = o.net_from_specs(specs[:-1], input_shape, **kw)
    s = specs[-1]
    act = s.get("activation", "identity")
    layer = CnnLossLayer(s.get("name", ""), loss=s.get("loss", "xent"), activation=act, alpha=s.get("alpha", o.ACT_ALPHA_DEFAULTS.get(act, 0.01)), cq=cq)
    layer.q = net.q
    layer.init(None, net.dtype)
    net.layers.append(layer)
    return net
