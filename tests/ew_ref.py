"""References for the reduction, loss and element-wise kernels of the training step (tests/test_gpu_ew_kernels.py) and for the weight
constraints' kernels (tests/test_gpu_constraints.py).

The split-K reductions are restated as exact emulations of their documented summation orders in float32 NumPy: every addition is one IEEE
fp32 addition in the kernel's order, so a kernel that keeps its order matches them bit for bit.  The constraints' group norms are emulated
the same way in float64, the kernels' accumulator type.  Losses, pooling, upsampling and the constraints' multipliers reuse the oracle
(oracle/dl4j_oracle.py); the activations are restated in float64 from the values the kernel stored, as the backward pass evaluates them.
"""
import numpy as np

from oracle import dl4j_oracle as o

F32 = np.float32


# ---------------------------------------------------------------- split-K reductions (kernels_ew.cu) ----------------------------------------
def reduce_narrow(src, init=None):
    """reduce_splits_kernel and reduce_multi_kernel's thread-per-output mode: a = (init or 0); a += src[k] for k = 0..S-1.  src: [S, n]."""
    src = np.asarray(src, F32)
    a = np.zeros(src.shape[1], F32) if init is None else np.array(init, F32)
    for k in range(src.shape[0]):
        a = a + src[k]
    return a


def warp_lanes(src):
    """The 32 lane sums of the warp-per-output mode before the shuffle tree: lane l sums splits l, l+32, ... in order, from 0.  -> [32, n]"""
    src = np.asarray(src, F32)
    lanes = np.zeros((32, src.shape[1]), F32)
    for k in range(src.shape[0]):
        lanes[k % 32] = lanes[k % 32] + src[k]
    return lanes


def xor_tree(lanes):
    """__shfl_xor_sync butterfly with m = 16, 8, 4, 2, 1: every lane adds its partner's value; lane 0's result.  lanes: [32, ...], any dtype"""
    v = np.asarray(lanes)
    idx = np.arange(32)
    for m in (16, 8, 4, 2, 1):
        v = v + v[idx ^ m]
    return v[0]


def reduce_wide(src, init=None):
    """reduce_splits_wide_kernel (and the list's warp-per-output mode with init None): (init or 0) + xor_tree(warp_lanes(src))."""
    t = xor_tree(warp_lanes(src))
    return (np.zeros_like(t) if init is None else np.asarray(init, F32)) + t


def splits_view(buf, off, splits, stride, n):
    """[splits, n] view of the partials at buf[off + s*stride + i]"""
    return np.stack([np.asarray(buf, F32)[off + s * stride: off + s * stride + n] for s in range(splits)])


def reduce_multi(buf, jobs, wide):
    """reduce_multi_kernel over a job list in one buffer: each job's destination = its partials summed in the order of its mode (wide[j]
    as the list reports it: warp per output, else thread per output).  Other elements are unchanged."""
    out = np.array(buf, F32)
    for j, w in zip(jobs, wide):
        part = splits_view(buf, j["src_off"], j["splits"], j["stride"], j["n"])
        out[j["dst_off"]: j["dst_off"] + j["n"]] = reduce_wide(part) if w else reduce_narrow(part)
    return out


# ---------------------------------------------------------------- weight constraints (kernels_constraint.cu) --------------------------------
CHUNK, SCHUNK = 4096, 256          # kernels.h CON_CHUNK / CON_SCHUNK
DIM_AXIS = {"conv": (0, 3, 1, 2), "dense": (3, 0), "vector": (0, 3)}     # DL4J dimension -> internal axis


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


def plan(kind: str, internal_shape, dims):
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


def constraint_path(kind: str, shape, dims) -> str:
    """The kernel path of a norm constraint over dims on a parameter of DL4J shape `shape`: "one-pass" (the innermost stored axis reduced,
    groups of at most CHUNK elements) or "two-launch"."""
    K0, R0, K1, R1, K2 = plan(kind, internal(kind, np.empty(shape, F32)).shape, tuple(dims))
    return "one-pass" if K2 == 1 and R0 * R1 <= CHUNK else "two-launch"


def group_sums(kind: str, w: np.ndarray, dims):
    """Each group's sum of squares in the device's order (kernels_constraint.cu), and the plan of the internal tensor it used."""
    x = internal(kind, np.asarray(w, F32))
    K0, R0, K1, R1, K2 = plan(kind, x.shape, tuple(dims))
    g = np.ascontiguousarray(x).reshape(K0, R0, K1, R1, K2).transpose(0, 2, 4, 1, 3).reshape(K0 * K1 * K2, R0 * R1)
    sq = g.astype(np.float64) ** 2
    G, R = sq.shape
    size, width = (CHUNK, 256) if K2 == 1 else (SCHUNK, 8)     # a chunk's j's; the running sums: 256 threads, or 8 warps (a lane per group)
    total = np.zeros(G)
    for c0 in range(0, R, size):
        blk = np.zeros((G, size)); blk[:, :min(size, R - c0)] = sq[:, c0:c0 + size]
        acc = np.zeros((G, width))
        for i in range(size // width):
            acc = acc + blk[:, i * width:(i + 1) * width]
        warps = xor_tree(np.moveaxis(acc.reshape(G, 8, 32), -1, 0)) if K2 == 1 else acc      # [G, 8]: each warp's sum
        t = np.zeros(G)
        for wi in range(8):
            t = t + warps[:, wi]
        total = total + t
    return total, (K0, R0, K1, R1, K2)


def device_apply(kind: str, w: np.ndarray, c) -> np.ndarray:
    """What the device makes of the fp32 DL4J-shaped parameter w under constraint c, bit for bit: the oracle's multiplier of each group's
    norm (NumPy rounds each product and sum, as the kernel does: no fused multiply-add) times each element, rounded to fp32."""
    w = np.asarray(w, F32)
    if c["constraint"] == "non_negative":
        return np.where(w < 0, F32(0), w)
    s, (K0, R0, K1, R1, K2) = group_sums(kind, w, c.get("dims", ()))
    m = o.constraint_multiplier(c, np.sqrt(s))
    x = internal(kind, w)
    v = np.ascontiguousarray(x).reshape(K0, R0, K1, R1, K2) * m.reshape(K0, 1, K1, 1, K2)
    return from_internal(kind, v.astype(F32).reshape(x.shape), w.shape)


# ---------------------------------------------------------------- activations (common.cuh act_fwd / act_grad_from_out) ----------------------
def act_fwd(x, act, alpha=0.0):
    x = np.asarray(x, np.float64)
    if act == "tanh":
        return np.tanh(x)
    if act == "sigmoid":
        e = np.exp(-np.abs(x))                             # 1 / (1 + e^-x) without overflow or cancellation
        return np.where(x >= 0, 1.0 / (1.0 + e), e / (1.0 + e))
    if act == "relu":
        return np.maximum(x, 0.0)
    if act == "lrelu":
        return np.where(x > 0, x, alpha * x)
    return x


def act_grad_from_out(a, act, alpha=0.0):
    """f'(z) from the stored output a = f(z): tanh 1 - a^2, sigmoid a (1 - a), relu / leaky relu from the sign of a (a == 0 takes the
    negative side), identity 1."""
    a = np.asarray(a, np.float64)
    if act == "tanh":
        return 1.0 - a * a
    if act == "sigmoid":
        return a * (1.0 - a)
    if act == "relu":
        return np.where(a > 0, 1.0, 0.0)
    if act == "lrelu":
        return np.where(a > 0, 1.0, alpha)
    return np.ones_like(a)


# ---------------------------------------------------------------- losses: the oracle ---------------------------------------------------------
def xent(z, y, clip_eps):
    """LossBinaryXENT + sigmoid per group: z, y [groups, rows] -> (loss sum per group [groups], dz [groups, rows]) in float64."""
    z = np.asarray(z, np.float64); y = np.asarray(y, np.float64)
    with np.errstate(over="ignore"):
        res = [o.xent_score_and_grad(z[g], y[g], clip_eps) for g in range(z.shape[0])]
    return np.array([r[0] for r in res]), np.stack([r[1] for r in res])


def mcxent(z, y):
    """LossMCXENT + softmax: (loss sum, dz = p - y, p) in float64."""
    z = np.asarray(z, np.float64); y = np.asarray(y, np.float64)
    loss, dz = o.mcxent_softmax_score_and_grad(z, y)
    return loss, dz, dz + y


# ---------------------------------------------------------------- pooling / upsampling: the oracle (NHWC in and out) -------------------------
def maxpool(x_nhwc, eps_nhwc, k, s):
    """SubsamplingLayer(MAX), truncate mode, first max in row-major window order wins.  -> (y, argmax r*KW+q, eps_in), all NHWC."""
    layer = o.MaxPool(k, s)
    layer.init(np.random.default_rng(0), np.float64)
    y = layer.forward(np.asarray(x_nhwc, np.float64).transpose(0, 3, 1, 2), True)
    arg = layer._arg                                                 # [N, OH, OW, C]
    ei = layer.backward(np.asarray(eps_nhwc, np.float64).transpose(0, 3, 1, 2))
    return y.transpose(0, 2, 3, 1), arg, ei.transpose(0, 2, 3, 1)


def upsample(x_nhwc, eps_nhwc, f):
    layer = o.Upsample2D(f)
    layer.init(np.random.default_rng(0), np.float64)
    y = layer.forward(np.asarray(x_nhwc, np.float64).transpose(0, 3, 1, 2), True)
    ei = layer.backward(np.asarray(eps_nhwc, np.float64).transpose(0, 3, 1, 2))
    return y.transpose(0, 2, 3, 1), ei.transpose(0, 2, 3, 1)
