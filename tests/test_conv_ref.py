"""CPU: the float64 NHWC references of tests/conv_ref.py against the oracle's ConvolutionLayer (oracle/dl4j_oracle.py Conv2D), and the
pixel-shuffle operand packing (helpers.pack_deconv_ps) against the transposed conv it stands for."""
import numpy as np
import pytest

import conv_ref
from helpers import pack_deconv_ps
from oracle import dl4j_oracle as o

# n, h, w, c, o, k, s, p
CASES = [
    (2, 8, 8, 3, 5, 4, 2, 1),        # the DCGAN 4x4 s2 p1
    (2, 9, 7, 4, 6, 5, 2, 2),        # 5x5 s2 p2 on a non-square image
    (2, 8, 12, 3, 4, 5, 2, 2),
    (3, 7, 9, 5, 6, 5, 2, 0),        # Truncate: the last input row / column is in no window
    (1, 6, 10, 2, 3, 3, 1, 1),
    (2, 8, 6, 3, 4, 2, 2, 0),
    (4, 1, 1, 7, 5, 1, 1, 0),        # dense as a 1x1 conv
]


@pytest.mark.parametrize("case", CASES, ids=[f"n{c[0]}_{c[1]}x{c[2]}_c{c[3]}_o{c[4]}_k{c[5]}s{c[6]}p{c[7]}" for c in CASES])
def test_conv_reference_matches_oracle_conv2d(case):
    n, h, w, c, oc, k, s, p = case
    rng = np.random.default_rng(7)
    x = rng.standard_normal((n, h, w, c)); wt = rng.standard_normal((oc, k, k, c))
    lay = o.Conv2D(c, oc, (k, k), (s, s), (p, p), has_bias=False); lay.init(np.random.default_rng(0), np.float64)
    lay.params["W"] = wt.transpose(0, 3, 1, 2).copy()
    y = lay.forward(x.transpose(0, 3, 1, 2), True).transpose(0, 2, 3, 1)
    got = conv_ref.conv2d(x, wt, s, p)
    assert got.shape == y.shape
    np.testing.assert_allclose(got, y, rtol=1e-12, atol=1e-12)
    dy = rng.standard_normal(y.shape)
    dx = lay.backward(dy.transpose(0, 3, 1, 2)).transpose(0, 2, 3, 1)
    got = conv_ref.conv2d_input_grad(dy, wt, (h, w), s, p)
    assert got.shape == dx.shape
    np.testing.assert_allclose(got, dx, rtol=1e-12, atol=1e-12)


def test_dense_reference_both_weight_layouts():
    rng = np.random.default_rng(8)
    x = rng.standard_normal((6, 5)); w = rng.standard_normal((3, 5))
    ref = np.array([[sum(x[i, j] * w[q, j] for j in range(5)) for q in range(3)] for i in range(6)])
    np.testing.assert_allclose(conv_ref.dense(x, w), ref, rtol=1e-12)
    np.testing.assert_allclose(conv_ref.dense(x, np.ascontiguousarray(w.T), w_mn=True), ref, rtol=1e-12)
    np.testing.assert_allclose(conv_ref.dense(x, w), conv_ref.conv2d(x[:, None, None, :], w[:, None, None, :])[:, 0, 0, :], rtol=1e-12)


@pytest.mark.parametrize("c", [1, 3, 4])
@pytest.mark.parametrize("hw", [(4, 4), (3, 5)], ids=["square", "non-square"])
def test_pixel_shuffle_packing_is_the_transposed_conv(c, hw):
    """The pixel-shuffle kernel's operand: a 3x3 s1 p1 conv of dy with pack_deconv_ps(w) as a [16][3][3][O] weight gives, per dy pixel
    (Y, X), the 2x2 output block (py, px, c4); scattered to (2Y + py, 2X + px, c) it is the 4x4 s2 p1 transposed conv, and the padded
    channels c >= C are zero."""
    oh, ow = hw
    rng = np.random.default_rng(9 + c)
    nimg, O = 2, 6
    w = rng.standard_normal((O, 4, 4, c)); dy = rng.standard_normal((nimg, oh, ow, O))
    blocks = conv_ref.conv2d(dy, pack_deconv_ps(w).reshape(16, 3, 3, O), 1, 1).reshape(nimg, oh, ow, 2, 2, 4)
    assert not blocks[..., c:].any()
    dx = blocks[..., :c].transpose(0, 1, 3, 2, 4, 5).reshape(nimg, 2 * oh, 2 * ow, c)
    np.testing.assert_allclose(dx, conv_ref.conv2d_input_grad(dy, w, (2 * oh, 2 * ow), 2, 1), rtol=1e-12, atol=1e-12)
