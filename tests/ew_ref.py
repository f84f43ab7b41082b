"""References for the reduction, loss and element-wise kernels of the training step (tests/test_gpu_ew_kernels.py).

The split-K reductions are restated as exact emulations of their documented summation orders in float32 NumPy: every addition is one IEEE
fp32 addition in the kernel's order, so a kernel that keeps its order matches them bit for bit.  Losses, pooling and upsampling reuse the
oracle (oracle/dl4j_oracle.py); the activations are restated in float64 from the values the kernel stored, as the backward pass evaluates them.
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
    """__shfl_xor_sync butterfly with m = 16, 8, 4, 2, 1: every lane adds its partner's value; lane 0's result.  lanes: [32, n]"""
    v = np.asarray(lanes, F32)
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
