"""Per-output loss weights and labels masks (semantics at b2g_loss in include/b200gan.h) on top of the unchanged DL4J oracle.

For row r (an example, or a pixel of a CnnLossLayer) and column j (an output, or a channel), weight w_j and mask m_rj:
  XENT, codes 2-8   score terms w_j m_rj l(a_rj, y_rj), dz_rj = w_j m_rj dz_rj
  MCXENT            score -m_r sum_j w_j y_rj log clamp(p_rj), dz_rj = m_r (p_rj sum_k w_k y_rk - w_j y_rj) (weighted), m_r (p_rj - y_rj)
The score stays the loss sum over the minibatch; MSE, MAE and Wasserstein still divide by nOut / C.  A mask is [N, 1] or [N, nOut] on
OUTPUT / LOSS layers and NCHW [N, 1, H, W] or [N, C, H, W] on a CnnLossLayer.

MaskNet is an oracle Net whose compute_gradient_and_score / fit take mask=, net_from_specs reads a loss spec's "loss_weights", and gan_step
takes the three masks of the adversarial step.  DL4J 1.0.0-beta3, recalled; parity unpinned like the rest of the DL4J semantics.  The points
of medium confidence are LossMaskQuirks fields."""
from dataclasses import dataclass

import numpy as np

from oracle import dl4j_oracle as o


@dataclass(frozen=True)
class LossMaskQuirks:
    # BaseOutputLayer.computeScore divides the masked sum by the minibatch, not by the number of unmasked entries
    score_per_minibatch: bool = True
    # LossMCXENT throws "Per output masking for MCXENT + softmax: not supported" for a mask wider than one column
    mcxent_per_output_mask_refused: bool = True
    # the losses without a weights constructor in beta3
    weightless_losses: tuple = ("hinge", "squared_hinge", "wasserstein")
    # the mask shapes a CnnLossLayer takes (NCHW): one value per pixel [N, 1, H, W], or one per output [N, C, H, W]
    cnn_mask_channels: tuple = ("one", "all")


MQ = LossMaskQuirks()


def _act_out(loss_act, alpha, z, q):
    return o.forward(loss_act, z, alpha, q) if loss_act in o.EXT_ACTS else o.act_forward(loss_act, z, alpha)


def _elem_scores(loss, act, alpha, z, y, q):
    """The per-element scores of codes 2-8 before the / nOut of the per-output losses (what score_and_grad sums)."""
    a = _act_out(act, alpha, z, q)
    e, m = a - y, 1 - y * a
    return {"mse": e * e, "l2": e * e, "l1": np.abs(e), "mae": np.abs(e), "hinge": np.maximum(m, 0),
            "squared_hinge": np.maximum(m, 0) ** 2, "wasserstein": y * a}[loss]


def check_weights(loss, weights, cols):
    if weights is None:
        return None
    w = np.asarray(weights, np.float64).ravel()
    if loss in MQ.weightless_losses:
        raise NotImplementedError(f"{loss} takes no per-output weights")
    if w.size != cols:
        raise ValueError(f"{w.size} loss weights for {cols} outputs")
    if not np.all(np.isfinite(w)):
        raise ValueError("loss weights must be finite")
    return w


def check_mask(loss, mask, rows, cols):
    """mask as rows: [rows, 1] or [rows, cols]."""
    if mask is None:
        return None
    m = np.asarray(mask, np.float64).reshape(rows, -1)
    if m.shape[1] not in (1, cols):
        raise ValueError(f"mask width {m.shape[1]}: 1 or {cols}")
    if m.shape[1] > 1 and loss == "mcxent" and MQ.mcxent_per_output_mask_refused:
        raise NotImplementedError("per-output masking for MCXENT + softmax is not supported")
    return m


def rows_score_and_grad(loss, act, alpha, z, y, w=None, m=None, q=o.DEFAULT_QUIRKS):
    """The weighted / masked loss on rows z, y [R, C] (w [C] or None, m [R, 1 | C] or None): (summed score, dL/dz [R, C])."""
    s = np.ones_like(z)
    if w is not None:
        s = s * w[None, :]
    if m is not None:
        s = s * m
    if loss == "mcxent":
        e = np.exp(z - z.max(1, keepdims=True))
        p = e / e.sum(1, keepdims=True)
        pc = np.clip(p, 1e-10, 1 - 1e-10)
        score = float(-((y * np.log(pc)) * s).sum())
        mr = m if m is not None else 1.0
        if w is not None:
            wy = w[None, :] * y
            g = mr * (p * wy.sum(1, keepdims=True) - wy)
        else:
            g = mr * (p - y)
        return score, g
    if loss == "xent":
        _, g = o.xent_score_and_grad(z, y, q.xent_clip_eps)
        clip = q.xent_clip_eps
        if clip > 0:
            pp = np.clip(o._sigmoid(z), clip, 1 - clip)
            l = -(y * np.log(pp) + (1 - y) * np.log(1 - pp))
        else:
            l = np.maximum(z, 0) + np.log1p(np.exp(-np.abs(z))) - y * z
        return float((l * s).sum()), g * s
    _, g = o.score_and_grad(loss, act, alpha, z, y, q)
    score = (_elem_scores(loss, act, alpha, z, y, q) * s).sum()
    if o.per_output(loss, q):
        score = score / z.shape[1]
    return float(score), g * s


def layer_score_and_eps(layer, y, w=None, mask=None):
    """The last layer's score_and_eps with weights w and a mask (None: that part absent), for Output, OutputSoftmax, LossLayer and
    CnnLossLayer."""
    z = layer._z
    if isinstance(layer, o.CnnLossLayer):
        n, c, h, wd = z.shape
        zr, yr = o.to_rows(z), o.to_rows(np.asarray(y, z.dtype).reshape(z.shape))
        if mask is not None:
            mk = np.asarray(mask, np.float64).reshape(n, -1, h, wd)
            if mk.shape[1] not in (1, c):
                raise ValueError(f"mask channels {mk.shape[1]}: 1 or {c}")
            mask = o.to_rows(mk)
        w, m = check_weights(layer.loss, w, c), check_mask(layer.loss, mask, zr.shape[0], c)
        s, g = rows_score_and_grad(layer.loss, layer.loss_act, layer.loss_alpha, zr, yr, w, m, layer.q)
        g = o.from_rows(g, z.shape)
        if not layer.q.cnn_loss_score_per_minibatch:
            s, g = s / (h * wd), g / (h * wd)
        return float(s), g
    loss = "mcxent" if isinstance(layer, o.OutputSoftmax) else layer.loss
    y = np.asarray(y, z.dtype)
    zr = z.reshape(y.shape)
    w, m = check_weights(loss, w, zr.shape[1]), check_mask(loss, mask, zr.shape[0], zr.shape[1])
    act, alpha = (None, None) if loss == "mcxent" else (layer.loss_act, layer.loss_alpha)
    s, g = rows_score_and_grad(loss, act, alpha, zr, y, w, m, layer.q)
    return s, g.reshape(z.shape)


class MaskNet(o.Net):
    """An oracle Net with the loss layer's weights (loss_weights) and a labels mask per pass: pass_masks holds what the next passes' losses
    take, in order (None: no mask)."""
    loss_weights = None
    pass_masks = ()
    in_gan_step = False

    def _loss_backward(self, y):
        """o.Net._loss_backward with the weighted / masked score_and_eps of the last layer."""
        last = self.layers[-1]
        m = self.pass_masks.pop(0) if self.pass_masks else None
        loss_sum, eps = layer_score_and_eps(last, np.asarray(y, self.dtype), self.loss_weights, m)
        if last.has_params:
            eps = last.backward(eps)
        return (loss_sum,) + self.backward_from_prefix(eps, collect=True)

    def compute_gradient_and_score(self, x, y, collect=False, pass_=None, row0=0, mask=None):
        if mask is not None and not MQ.score_per_minibatch:
            raise NotImplementedError("only the minibatch divisor is restated")
        if not self.in_gan_step:
            self.pass_masks = [mask]
        return super().compute_gradient_and_score(x, y, collect, pass_, row0)

    def fit(self, x, y, mask=None):
        score = self.compute_gradient_and_score(x, y, mask=mask)
        self.apply_update(x.shape[0])
        return score


def to_mask_net(net: o.Net, loss_weights=None) -> MaskNet:
    net.__class__ = MaskNet
    net.loss_weights = None if loss_weights is None else np.asarray(loss_weights, np.float64).ravel()
    return net


def net_from_specs(specs, input_shape, **kw) -> MaskNet:
    """o.net_from_specs, the last spec's "loss_weights" becoming the loss layer's weights (checked as the library checks them)."""
    for s in specs[:-1]:
        if s.get("loss_weights") is not None:
            raise ValueError("loss_weights belong to the net's last (loss) layer")
    base = [dict(s) for s in specs]
    w = base[-1].pop("loss_weights", None)
    net = to_mask_net(o.net_from_specs(base, input_shape, **kw))
    if w is not None:
        last = net.layers[-1]
        _, acts = net.forward(np.zeros((1,) + tuple(input_shape)), train=False, collect=True)
        cols = acts[-1].shape[1]                  # nOut, or the CnnLossLayer's channels
        net.loss_weights = check_weights("mcxent" if isinstance(last, o.OutputSoftmax) else last.loss, w, cols)
    return net


def gan_step(G, D: MaskNet, x_real, z_d, z_g, y_real, y_fake, y_gen, m_real=None, m_fake=None, m_gen=None, fake_bn_train=False):
    """o.gan_step with labels masks on the D update's real and fake halves and on the G update through D."""
    D.pass_masks, D.in_gan_step = [m_real, m_fake, m_gen], True
    try:
        return o.gan_step(G, D, x_real, z_d, z_g, y_real, y_fake, y_gen, fake_bn_train)
    finally:
        D.pass_masks, D.in_gan_step = [], False
