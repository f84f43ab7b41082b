"""Test-only NumPy restatement of DL4J's L2 gradient normalization, on top of the DL4J oracle (oracle/dl4j_oracle.py) without changing it.

Semantics recalled from DL4J 1.0.0-beta3 BaseMultiLayerUpdater.preApply (PARITY UNPINNED, like the rest of the oracle; the library's statement
is include/b200gan.h, b2g_net_set_gradient_normalization).  One update becomes  g /= mb -> normalization -> updater -> + l2*W -> theta -= g:
  renormalize_l2_per_layer        g <- g / ||g_layer||  (a zero norm divides by `l2norm_zero_floor` instead; the threshold is ignored)
  renormalize_l2_per_param_type   the same per parameter tensor
  clip_l2_per_layer               g <- g * threshold / ||g_layer||  when ||g_layer|| > threshold
  clip_l2_per_param_type          the same per parameter tensor
A layer is one oracle layer with parameters that is not frozen; its BatchNorm mean/var pseudo-gradients (not divided by mb) are inside its norm
and scaled with it when `bn_stats_normalized` holds.  The multiplier is rounded to fp32 once, as the library does.

`enable(net, mode, threshold)` gives one oracle Net the mode: it replaces the net's `apply_update` by one that normalizes the gradients after
the division by mb and then runs the oracle's own `apply_update` with mb = 1 (an exact division), so `fit` and the oracle's `gan_step` pick the
mode up unchanged."""
from __future__ import annotations

import dataclasses
import math
import types

import numpy as np

from oracle import dl4j_oracle as o

MODES = ("none", "renormalize_l2_per_layer", "renormalize_l2_per_param_type", "clip_l2_per_layer", "clip_l2_per_param_type")


@dataclasses.dataclass
class GradNormQuirks:
    bn_stats_normalized: bool = True     # [recall, medium confidence] BatchNorm mean/var pseudo-gradients count in the layer's norm and are scaled
    l2norm_zero_floor: float = 1e-5      # [recall, medium confidence] Renormalize divides by this instead of a zero norm


DEFAULT_GN_QUIRKS = GradNormQuirks()


def multiplier(sumsq: float, mode: str, threshold: float, q: GradNormQuirks = DEFAULT_GN_QUIRKS) -> np.float32:
    """The fp32 multiplier of one norm group from its sum of squares."""
    norm = math.sqrt(sumsq)
    if mode.startswith("renormalize"):
        return np.float32(1.0 / (norm if norm != 0.0 else q.l2norm_zero_floor))
    thr = float(np.float32(threshold))
    return np.float32(thr / norm) if norm > thr else np.float32(1.0)


def divided_grads(net, mb, grads=None):
    """{(layer, param): g after the division by mb} for every layer the updater touches (BatchNorm mean/var are not divided)."""
    out = {}
    for li, l in enumerate(net.layers):
        if not l.has_params or getattr(l, "frozen", False):
            continue
        for p, _, _ in l.param_specs():
            g = np.asarray(grads[(li, p)] if grads is not None else l.grads[p], net.dtype)
            noop = p in l.noop_names()
            out[(li, p)] = g if (noop and net.q.bn_stats_minibatch_exempt) else g / mb
    return out


def norm_groups(net, g, mode, q: GradNormQuirks = DEFAULT_GN_QUIRKS):
    """The mode's norm groups over the divided gradients g: lists of (layer, param) keys, in parameter order."""
    groups = {}
    for (li, p) in g:
        l = net.layers[li]
        if p in l.noop_names() and not q.bn_stats_normalized:
            continue
        groups.setdefault(li if mode.endswith("per_layer") else (li, p), []).append((li, p))
    return list(groups.values())


def normalize(net, g, mode, threshold, q: GradNormQuirks = DEFAULT_GN_QUIRKS):
    """Applies the mode to the divided gradients g (a new dict); also returns the groups' norms."""
    out, norms = dict(g), []
    for keys in norm_groups(net, g, mode, q):
        ss = sum(float((np.asarray(g[k], np.float64) ** 2).sum()) for k in keys)
        norms.append(math.sqrt(ss))
        m = multiplier(ss, mode, threshold, q)
        for k in keys:
            out[k] = g[k] * float(m)
    return out, norms


def _apply_update(self, mb, grads=None, frozen_from=None):
    if self.grad_norm == "none":
        return o.Net.apply_update(self, mb, grads, frozen_from)
    assert self.grad_clip == 0, "DL4J allows one gradient normalization per layer"
    g, self.grad_norm_last_norms = normalize(self, divided_grads(self, mb, grads), self.grad_norm, self.grad_norm_threshold, self.grad_norm_quirks)
    return o.Net.apply_update(self, 1, grads=g)        # / 1 is exact: the division by mb is already in g


def enable(net, mode="none", threshold=1.0, quirks: GradNormQuirks = DEFAULT_GN_QUIRKS):
    """Gives the oracle Net `net` the gradient normalization `mode` (one of MODES); returns net."""
    assert mode in MODES, mode
    net.grad_norm, net.grad_norm_threshold, net.grad_norm_quirks, net.grad_norm_last_norms = mode, threshold, quirks, []
    net.apply_update = types.MethodType(_apply_update, net)
    return net
