"""DL4J's weight constraints (LayerConstraint: MaxNorm, MinMaxNorm, UnitNorm, NonNegative) restated on top of the DL4J oracle, and an exact
emulation of the library's summation order for bit-for-bit checks of the device kernels.  Semantics: b2g_constraint in include/b200gan.h.

``constrain(net, specs, global_constraints)`` gives an oracle Net the constraints of the layer specs, resolved to parameters by the library's
rule (engine.resolve_constraints), and makes its ``apply_update`` run them after every update, so ``fit``, ``gan_step``,
``gan_iteration_reference`` and parameter averaging's local fits pick them up.  Its recalls are ``ConstraintQuirks`` fields whose defaults the
library implements.
"""
from __future__ import annotations

import dataclasses
from typing import Dict, List, Optional, Sequence

import numpy as np

from oracle import dl4j_oracle as o


@dataclasses.dataclass
class ConstraintQuirks:
    constraint_eps: float = 1e-6             # BaseConstraint.DEFAULT_EPSILON
    unit_norm_zero_group_unchanged: bool = True   # UnitNorm leaves an all-zero group as it is (DL4J: 0/0 = NaN)


DEFAULT = ConstraintQuirks()
CHUNK, SCHUNK = 4096, 256          # kernels.h CON_CHUNK / CON_SCHUNK


def multiplier(c: Dict, norm, q: ConstraintQuirks = DEFAULT):
    """The fp32 multiplier of a group of L2 norm `norm` (float64 arrays), computed in double and rounded once."""
    norm = np.asarray(norm, np.float64)
    eps = q.constraint_eps
    k = c["constraint"]
    if k == "max_norm":
        m = np.minimum(norm, c["max"]) / (norm + eps)
    elif k == "min_max_norm":
        rate = c.get("rate", 1.0)
        m = (rate * np.minimum(np.maximum(norm, c["min"]), c["max"]) + (1.0 - rate) * norm) / (norm + eps)
    elif k == "unit_norm":
        with np.errstate(divide="ignore", invalid="ignore"):
            m = 1.0 / norm
        if q.unit_norm_zero_group_unchanged:
            m = np.where(norm == 0.0, 1.0, m)
    else:
        raise ValueError(k)
    return m.astype(np.float32)


def apply(w: np.ndarray, c: Dict, q: ConstraintQuirks = DEFAULT) -> np.ndarray:
    """One constraint on one parameter in its DL4J shape ([n] vectors as [1, n]; float64 or float32), the norm over c["dims"] (() = all) taken in float64."""
    dt = w.dtype
    if c["constraint"] == "non_negative":
        return np.where(w < 0, np.zeros((), dt), w)
    if w.ndim == 1:                    # b, gamma, beta, mean, var: DL4J's [1, n]
        return apply(w.reshape(1, -1), c, q).reshape(w.shape)
    dims = tuple(sorted(set(c.get("dims", ())))) or tuple(range(w.ndim))
    norm = np.sqrt((w.astype(np.float64) ** 2).sum(axis=dims, keepdims=True))
    return (w * multiplier(c, norm, q).astype(dt)).astype(dt)


def apply_constraints(net: o.Net, q: Optional[ConstraintQuirks] = None):
    """Model.applyConstraints: every live (not frozen) layer's tensors, each through its list in order."""
    q = q or getattr(net, "constraint_quirks", DEFAULT)
    for l in net.layers:
        if not l.has_params or getattr(l, "frozen", False):
            continue
        for p, lst in net.constraints.get(l.name, {}).items():
            for c in lst:
                l.params[p] = apply(l.params[p], c, q)


class _Constrained:
    def apply_update(self, *a, **k):
        super().apply_update(*a, **k)
        apply_constraints(self)


def constrain(net: o.Net, specs: Sequence[Dict], global_constraints: Optional[Sequence[Dict]] = None, q: ConstraintQuirks = DEFAULT) -> o.Net:
    """net (built from specs) with the specs' constraints, or the global ones on a layer whose own reach none of its parameters, after every
    update."""
    from gan_deeplearning4j_b200.engine import GEMM_TYPES, resolve_constraints
    net.constraints = {}
    for sp in specs:
        if global_constraints and sp["type"] in GEMM_TYPES + ("batchnorm",) and not resolve_constraints(sp):
            sp = dict(sp, constraints=list(global_constraints))
        r = resolve_constraints(sp)
        if r:
            net.constraints[sp["name"]] = r
    net.constraint_quirks = q
    if not isinstance(net, _Constrained):
        net.__class__ = type("Constrained" + type(net).__name__, (_Constrained, type(net)), {})
    return net


# ------------------------------------------------------------------ the device's summation order ---------------------------------------
def internal(kind: str, w: np.ndarray) -> np.ndarray:
    """A DL4J-shaped parameter as the engine's [A][kH][kW][B] array: conv / deconv W [a, b, kh, kw] -> [a][kh][kw][b]; dense W [nIn, nOut] ->
    [nOut][1][1][nIn]; a vector [n] -> [1][1][1][n]."""
    if kind == "conv":
        return w.transpose(0, 2, 3, 1)
    if kind == "dense":
        return w.T.reshape(w.shape[1], 1, 1, w.shape[0])
    return w.reshape(1, 1, 1, -1)


def from_internal(kind: str, x: np.ndarray, shape) -> np.ndarray:
    if kind == "conv":
        return x.transpose(0, 3, 1, 2)
    if kind == "dense":
        return x.reshape(shape[1], shape[0]).T
    return x.reshape(shape)


DIM_AXIS = {"conv": (0, 3, 1, 2), "dense": (3, 0), "vector": (0, 3)}     # DL4J dimension -> internal axis


def plan(kind: str, internal_shape, dims) -> List[int]:
    """[K0, R0, K1, R1, K2]: the runs of kept / reduced internal axes, size-1 axes dropped; a kept innermost run after a reduced one is K2
    (engine.cu net_build_constraints)."""
    rank = len(DIM_AXIS[kind])
    red = [False] * 4
    for d in range(rank):
        if not dims or d in dims:
            red[DIM_AXIS[kind][d]] = True
    runs = []
    for x in range(4):
        if internal_shape[x] == 1:
            continue
        f = int(red[x])
        if runs and runs[-1][0] == f:
            runs[-1][1] *= internal_shape[x]
        else:
            runs.append([f, internal_shape[x]])
    slot = [1] * 5
    if len(runs) >= 2 and runs[-1][0] == 0:       # a kept innermost run after a reduced one: strided groups
        slot[4] = runs.pop()[1]
    si = -1
    for f, n in runs:
        si = f if si < 0 else si + 1
        slot[si] = n
    return slot


def _butterfly(v):
    """One warp's xor butterfly over the last axis (32 lanes): lane 0's result."""
    lanes = np.arange(32)
    for o_ in (16, 8, 4, 2, 1):
        v = v + v[..., lanes ^ o_]
    return v[..., 0]


def group_sums(kind: str, w: np.ndarray, dims):
    """Each group's sum of squares in the device's order (kernels_constraint.cu), and the [G, R] view of the internal tensor it used."""
    x = internal(kind, np.asarray(w, np.float32))
    K0, R0, K1, R1, K2 = plan(kind, x.shape, tuple(dims))
    g = np.ascontiguousarray(x).reshape(K0, R0, K1, R1, K2).transpose(0, 2, 4, 1, 3).reshape(K0 * K1 * K2, R0 * R1)
    sq = g.astype(np.float64) ** 2
    G, R = sq.shape
    total = np.zeros(G)
    if K2 == 1:
        for c0 in range(0, R, CHUNK):
            blk = np.zeros((G, CHUNK)); blk[:, :min(CHUNK, R - c0)] = sq[:, c0:c0 + CHUNK]
            acc = np.zeros((G, 256))
            for qq in range(CHUNK // 256):
                acc = acc + blk[:, qq * 256:(qq + 1) * 256]
            warps = _butterfly(acc.reshape(G, 8, 32))
            t = np.zeros(G)
            for wi in range(8):
                t = t + warps[:, wi]
            total = total + t
    else:
        for c0 in range(0, R, SCHUNK):
            blk = np.zeros((G, SCHUNK)); blk[:, :min(SCHUNK, R - c0)] = sq[:, c0:c0 + SCHUNK]
            rows = blk.reshape(G, SCHUNK // 8, 8)
            acc = np.zeros((G, 8))
            for i in range(SCHUNK // 8):
                acc = acc + rows[:, i, :]
            t = np.zeros(G)
            for wi in range(8):
                t = t + acc[:, wi]
            total = total + t
    return total, (K0, R0, K1, R1, K2)


def device_apply(kind: str, w: np.ndarray, c: Dict) -> np.ndarray:
    """What the device makes of the fp32 DL4J-shaped parameter w under constraint c, bit for bit."""
    w = np.asarray(w, np.float32)
    if c["constraint"] == "non_negative":
        return np.where(w < 0, np.float32(0), w)
    s, (K0, R0, K1, R1, K2) = group_sums(kind, w, c.get("dims", ()))
    norm = np.sqrt(s)
    if c["constraint"] == "min_max_norm":       # the kernel rounds each product and the sum (no fused multiply-add)
        rate = c.get("rate", 1.0)
        m = ((rate * np.minimum(np.maximum(norm, c["min"]), c["max"])) + ((1.0 - rate) * norm)) / (norm + DEFAULT.constraint_eps)
        m = m.astype(np.float32)
    else:
        m = multiplier(c, norm)
    x = internal(kind, w)
    v = np.ascontiguousarray(x).reshape(K0, R0, K1, R1, K2) * m.reshape(K0, 1, K1, 1, K2)
    return from_internal(kind, v.astype(np.float32).reshape(x.shape), w.shape)
