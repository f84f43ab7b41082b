"""Test-only NumPy restatement of DL4J's Nesterovs, AdaGrad, AdaMax, Nadam, AMSGrad and AdaDelta updaters, on top of the DL4J oracle
(oracle/dl4j_oracle.py) without changing it.

Semantics recalled from DL4J 1.0.0-beta3 org.nd4j.linalg.learning.*Updater (PARITY UNPINNED, like the rest of the oracle; the library's
statement is include/b200gan.h, b2g_updater).  They take the updater's place in  g /= mb -> [normalization] -> clip -> updater -> + l2*W ->
theta -= u,  with t = iteration + 1:
  nesterovs  vPrev = v;  v = mu*v - lr*g;  u = mu*vPrev - (1+mu)*v
  adagrad    h += g^2;  u = lr*g / (sqrt(h) + eps)                                   (h starts at eps)
  adamax     m = b1*m + (1-b1)*g;  u_inf = max(b2*u_inf, |g|) + 1e-32;  u = lr/(1-b1^t) * m / u_inf
  nadam      Adam's m, v;  u = lr * (b1*m + (1-b1)*g) / (1-b1^t) / (sqrt(v) + eps)
  amsgrad    Adam's m, v;  vhat = max(vhat, v);  u = lr*sqrt(1-b2^t)/(1-b1^t) * m / (sqrt(vhat) + eps)
  adadelta   msg = rho*msg + (1-rho)*g^2;  u = sqrt(msdx + eps)/sqrt(msg + eps) * g;  msdx = rho*msdx + (1-rho)*u^2   (no learning rate)
The state of a parameter lives in the oracle Net's own `state` dict, in the library's slot order (state0, state1, state2), so the oracle's
`parameter_average` averages it.

`enable(net, specs)` gives one oracle Net the updaters of the specs whose kind is one of these: it wraps the net's `apply_update`, updates those
layers itself and hands the other layers to the wrapped update, so the oracle's `fit` and `gan_step` pick them up unchanged.  Call it after
gradnorm_ref.enable (whose normalization it applies to its own layers too) and before schedule_ref.enable (whose lr it reads)."""
from __future__ import annotations

import dataclasses
import types

import numpy as np

import gradnorm_ref as gr
import schedule_ref as sr
from helpers import oracle_from_specs as _plain_oracle_from_specs
from oracle import dl4j_oracle as o

KINDS = ("nesterovs", "adagrad", "adamax", "nadam", "amsgrad", "adadelta")
N_STATE = {"nesterovs": 1, "adagrad": 1, "adamax": 2, "nadam": 2, "amsgrad": 3, "adadelta": 2}


@dataclasses.dataclass
class UpdaterQuirks:
    adagrad_history_init_eps: bool = True   # [recall, medium confidence] AdaGrad's history starts at eps (else at 0)
    adamax_floor_no_eps: bool = True        # [recall, medium confidence] AdaMax: u_inf gets + 1e-32 and the denominator has no eps (else u_inf + eps)
    nadam_v_uncorrected: bool = True        # [recall, medium confidence] Nadam divides by sqrt(v) + eps (else by sqrt(v / (1-b2^t)) + eps)


DEFAULT_UPDATER_QUIRKS = UpdaterQuirks()


def updater_cfg(u):
    """An updater spec dict (models.py) of one of KINDS -> the oracle's UpdaterCfg (momentum and rho in beta1, as in b2g_layer_desc)."""
    k = u["kind"]
    lr = 0.0 if k == "adadelta" else u.get("lr", 0.0)
    if k == "nesterovs":
        return o.UpdaterCfg(k, lr=lr, beta1=u.get("momentum", 0.9))
    if k == "adagrad":
        return o.UpdaterCfg(k, lr=lr, eps=u.get("eps", 1e-6))
    if k == "adadelta":
        return o.UpdaterCfg(k, lr=0.0, beta1=u.get("rho", 0.95), eps=u.get("eps", 1e-6))
    return o.UpdaterCfg(k, lr=lr, beta1=u.get("beta1", 0.9), beta2=u.get("beta2", 0.999), eps=u.get("eps", 1e-8))


def init_state(u: o.UpdaterCfg, shape, dtype=np.float64, q: UpdaterQuirks = DEFAULT_UPDATER_QUIRKS):
    """The initial state slots of one parameter tensor."""
    st = [np.zeros(shape, dtype) for _ in range(N_STATE[u.kind])]
    if u.kind == "adagrad" and q.adagrad_history_init_eps:
        st[0][...] = u.eps
    return st


def update(u: o.UpdaterCfg, st, g, t: int, q: UpdaterQuirks = DEFAULT_UPDATER_QUIRKS):
    """The updater step u(g) of one parameter tensor at t = iteration + 1; the state slots st are updated in place."""
    lr, b1, b2, eps = u.lr, u.beta1, u.beta2, u.eps
    if u.kind == "nesterovs":
        v = st[0]; v_prev = v.copy()
        v[...] = b1 * v - lr * g
        return b1 * v_prev - (1 + b1) * v
    if u.kind == "adagrad":
        h = st[0]
        h[...] = h + g * g
        return lr * g / (np.sqrt(h) + eps)
    if u.kind == "adamax":
        m, ui = st
        m[...] = b1 * m + (1 - b1) * g
        if q.adamax_floor_no_eps:
            ui[...] = np.maximum(b2 * ui, np.abs(g)) + 1e-32
            return lr / (1 - b1 ** t) * m / ui
        ui[...] = np.maximum(b2 * ui, np.abs(g))
        return lr / (1 - b1 ** t) * m / (ui + eps)
    if u.kind in ("nadam", "amsgrad"):
        m, v = st[0], st[1]
        m[...] = b1 * m + (1 - b1) * g
        v[...] = b2 * v + (1 - b2) * g * g
        if u.kind == "nadam":
            vv = v if q.nadam_v_uncorrected else v / (1 - b2 ** t)
            return lr * (b1 * m + (1 - b1) * g) / (1 - b1 ** t) / (np.sqrt(vv) + eps)
        vh = st[2]
        vh[...] = np.maximum(vh, v)
        return lr * np.sqrt(1 - b2 ** t) / (1 - b1 ** t) * m / (np.sqrt(vh) + eps)
    if u.kind == "adadelta":
        msg, msdx = st
        msg[...] = b1 * msg + (1 - b1) * g * g
        d = np.sqrt(msdx + eps) / np.sqrt(msg + eps) * g
        msdx[...] = b1 * msdx + (1 - b1) * d * d
        return d
    raise ValueError(u.kind)


def _ext_layers(net):
    return [li for li, l in enumerate(net.layers) if l.has_params and not getattr(l, "frozen", False) and l.updater is not None and l.updater.kind in KINDS]


def _apply_update(self, mb, grads=None, frozen_from=None):
    ext = _ext_layers(self)
    if not ext:
        return self.base_apply_update(mb, grads, frozen_from)
    t = self.iteration + 1
    if getattr(self, "grad_norm", "none") != "none":      # gradnorm_ref: the normalized gradients after /mb; the division is then exact
        g_all, _ = gr.normalize(self, gr.divided_grads(self, mb, grads), self.grad_norm, self.grad_norm_threshold, self.grad_norm_quirks)
        div = 1
    else:
        g_all, div = None, mb
    for li in ext:
        l = self.layers[li]
        for pname, _, _ in l.param_specs():
            noop = pname in l.noop_names()
            if g_all is not None:
                g = np.asarray(g_all[(li, pname)], self.dtype).copy()
            else:
                g = (grads[(li, pname)] if grads is not None else l.grads[pname]).astype(self.dtype).copy()
            if not (noop and self.q.bn_stats_minibatch_exempt):
                g = g / div
            if self.grad_clip > 0 and (not noop or self.q.bn_stats_clipped):
                g = np.clip(g, -self.grad_clip, self.grad_clip)
            upd = g if noop else update(l.updater, self.state[(li, pname)], g, t, self.updater_quirks)
            if l.l2 and pname in l.l2_names():
                upd = upd + l.l2 * l.params[pname]
            l.params[pname] = (l.params[pname] - upd).astype(self.dtype)
    # the other layers through the wrapped update, which skips frozen layers and increments the iteration
    held = {li: self.layers[li].__dict__.get("frozen", None) for li in ext}
    try:
        for li in ext:
            self.layers[li].frozen = True
        self.base_apply_update(mb, grads, frozen_from)
    finally:
        for li, f in held.items():
            if f is None:
                del self.layers[li].frozen
            else:
                self.layers[li].frozen = f


def enable(net, specs, quirks: UpdaterQuirks = DEFAULT_UPDATER_QUIRKS):
    """Gives the oracle Net `net` the updater of every spec (by layer name) whose kind is one of KINDS, with fresh state; returns net."""
    by_name = {l.name: (li, l) for li, l in enumerate(net.layers)}
    for s in specs:
        u = s.get("updater")
        if not u or u["kind"] not in KINDS or s.get("name") not in by_name:
            continue
        li, l = by_name[s["name"]]
        l.updater = updater_cfg(u)
        if s.get("frozen", False):
            continue
        for pname, shape, _ in l.param_specs():
            if pname not in l.noop_names():
                net.state[(li, pname)] = init_state(l.updater, shape, net.dtype, quirks)
    if not hasattr(net, "base_apply_update"):
        net.base_apply_update = net.apply_update
        net.apply_update = types.MethodType(_apply_update, net)
    net.updater_quirks = quirks
    return net


def oracle_from_specs(specs, input_shape, grad_norm=None, quirks: UpdaterQuirks = DEFAULT_UPDATER_QUIRKS, **kw):
    """helpers.oracle_from_specs for specs whose updaters may be any kind and whose lr may be a schedule; grad_norm = (mode, threshold) enables
    gradnorm_ref first.  The wrappers are stacked gradnorm -> updaters -> schedules."""
    net = _plain_oracle_from_specs(sr.constant_specs(specs), input_shape, **kw)
    if grad_norm is not None:
        gr.enable(net, *grad_norm)
    enable(net, specs, quirks)
    return sr.enable(net, sr.scheduled_layers(specs))
