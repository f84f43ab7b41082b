"""Float64 references of the tensor-core GEMMs, NHWC, fast enough for whole batches at the benchmark shapes.

Each convolution is a loop over the filter taps; a tap is one float64 matmul of a strided view of the zero-padded input (forward) or a
scatter-add into the padded input gradient (its adjoint).  ConvolutionMode.Truncate output sizes, as oracle/dl4j_oracle.py Conv2D.
tests/test_conv_ref.py pins these functions to the oracle.
"""
import numpy as np


def _pair(v):
    return (v, v) if np.isscalar(v) else tuple(v)


def out_size(n, k, s, p):
    return (n - k + 2 * p) // s + 1


def conv2d(x, w, stride=1, pad=0):
    """x [N, H, W, C], w [O, KH, KW, C] -> y [N, OH, OW, O] = cross-correlation of the zero-padded x."""
    x = np.asarray(x, np.float64); w = np.asarray(w, np.float64)
    (sh, sw), (ph, pw) = _pair(stride), _pair(pad)
    n, h, wd, c = x.shape
    o, kh, kw, c2 = w.shape
    assert c == c2, (x.shape, w.shape)
    oh, ow = out_size(h, kh, sh, ph), out_size(wd, kw, sw, pw)
    xp = np.pad(x, ((0, 0), (ph, ph), (pw, pw), (0, 0)))
    y = np.zeros((n, oh, ow, o))
    for i in range(kh):
        for j in range(kw):
            y += xp[:, i:i + sh * (oh - 1) + 1:sh, j:j + sw * (ow - 1) + 1:sw, :] @ w[:, i, j, :].T
    return y


def conv2d_input_grad(dy, w, hw, stride=1, pad=0):
    """Adjoint of conv2d in x: dy [N, OH, OW, O], w [O, KH, KW, C], hw = (H, W) of x -> dx [N, H, W, C] (= the transposed-conv forward)."""
    dy = np.asarray(dy, np.float64); w = np.asarray(w, np.float64)
    (sh, sw), (ph, pw) = _pair(stride), _pair(pad)
    n, oh, ow, o = dy.shape
    o2, kh, kw, c = w.shape
    assert o == o2, (dy.shape, w.shape)
    h, wd = hw
    assert (oh, ow) == (out_size(h, kh, sh, ph), out_size(wd, kw, sw, pw)), (dy.shape, hw)
    # rows / columns past the last window (Truncate) receive nothing: the padded buffer covers both them and every window
    xp = np.zeros((n, max(h + 2 * ph, sh * (oh - 1) + kh), max(wd + 2 * pw, sw * (ow - 1) + kw), c))
    for i in range(kh):
        for j in range(kw):
            xp[:, i:i + sh * (oh - 1) + 1:sh, j:j + sw * (ow - 1) + 1:sw, :] += dy @ w[:, i, j, :]
    return xp[:, ph:ph + h, pw:pw + wd, :]


def conv2d_weight_grad(x, dy, kh, kw, stride=1, pad=0):
    """Adjoint of conv2d in w: x [N, H, W, C], dy [N, OH, OW, O] -> dw [O, KH, KW, C] = sum over (n, oy, ox) of dy times the input pixel each
    tap reads (zero in the padding; rows / columns past the last window are read by no tap)."""
    x = np.asarray(x, np.float64); dy = np.asarray(dy, np.float64)
    (sh, sw), (ph, pw) = _pair(stride), _pair(pad)
    n, h, wd, c = x.shape
    n2, oh, ow, o = dy.shape
    assert n == n2 and (oh, ow) == (out_size(h, kh, sh, ph), out_size(wd, kw, sw, pw)), (x.shape, dy.shape)
    xp = np.zeros((n, max(h + 2 * ph, sh * (oh - 1) + kh), max(wd + 2 * pw, sw * (ow - 1) + kw), c))
    xp[:, ph:ph + h, pw:pw + wd, :] = x
    dw = np.zeros((o, kh, kw, c))
    d2 = dy.reshape(-1, o)
    for i in range(kh):
        for j in range(kw):
            dw[:, i, j, :] = d2.T @ xp[:, i:i + sh * (oh - 1) + 1:sh, j:j + sw * (ow - 1) + 1:sw, :].reshape(-1, c)
    return dw


def dense(x, w, w_mn=False):
    """x [N, C] -> [N, O]; w is [O][C] (a 1x1 conv's weight), or [C][O] when w_mn (a dense layer's [nOut][nIn] weight as the operand of its
    input gradient: C = nOut, O = nIn)."""
    x = np.asarray(x, np.float64); w = np.asarray(w, np.float64)
    return x @ (w if w_mn else w.T)
