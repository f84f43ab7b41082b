"""The oracle's L2 gradient normalization against hand-computed answers on tiny layers, and the plumbing of the mode
names through the C header, the ctypes binding, the Java enum and the JNI shim.  CPU only."""
import copy
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from oracle import dl4j_oracle as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _dense(l2=0.0, lr=1.0):
    """Dense(2 -> 1) with SGD: theta' = theta - lr * g_normalized (- l2 * W); W and b start at zero unless set."""
    net = o.Net([o.Dense(2, 1, updater=o.Sgd(lr), l2=l2, name="d")], seed=1)
    net.layers[0].params["W"][...] = 0.0
    net.layers[0].params["b"][...] = 0.0
    return net


def _update(net, mode, threshold, grads, mb, **q):
    net.q = o.Quirks(**q)
    net.set_gradient_normalization(mode, threshold)
    net.apply_update(mb, grads=grads)
    return net


# mb = 2; summed gradients W = (6, 8), b = 24  ->  after / mb: W = (3, 4) (norm 5), b = 12 (norm 12); the layer's norm is 13
G = {(0, "W"): np.array([[6.0], [8.0]]), (0, "b"): np.array([24.0])}


@pytest.mark.parametrize("mode,thr,w,b", [
    ("renormalize_l2_per_layer", 123.0, (3 / 13, 4 / 13), 12 / 13),      # the threshold is ignored
    ("renormalize_l2_per_param_type", 123.0, (0.6, 0.8), 1.0),            # per tensor: differs from per layer
    ("clip_l2_per_layer", 26.0, (3, 4), 12),                              # threshold above the norm: unchanged
    ("clip_l2_per_layer", 13.0, (3, 4), 12),                              # exactly equal: not scaled
    ("clip_l2_per_layer", 6.5, (1.5, 2), 6),                              # below: scaled by 6.5 / 13
    ("clip_l2_per_param_type", 6.0, (3, 4), 6),                           # W (5) keeps, b (12) is scaled to norm 6
    ("clip_l2_per_param_type", 2.5, (1.5, 2), 2.5),                       # both scaled
    ("none", 1.0, (3, 4), 12),
])
def test_known_answers_dense(mode, thr, w, b):
    net = _update(_dense(), mode, thr, G, 2)
    np.testing.assert_allclose(-net.layers[0].params["W"].ravel(), w, rtol=1e-6)
    np.testing.assert_allclose(-net.layers[0].params["b"], [b], rtol=1e-6)


def test_multiplier_is_rounded_to_fp32_once():
    net = _update(_dense(), "renormalize_l2_per_layer", 1.0, G, 2)
    m = np.float32(1.0 / 13.0)
    assert -net.layers[0].params["W"][1, 0] == 4.0 * float(m)
    assert o.multiplier(169.0, "clip_l2_per_layer", 13.0) == 1.0 and o.multiplier(169.0 * 1.01, "clip_l2_per_layer", 13.0) < 1.0
    assert o.multiplier(169.0 * 1.01, "clip_l2_per_layer", 13.0) == np.float32(13.0 / np.sqrt(169.0 * 1.01))


def test_zero_gradient_under_renormalize_moves_only_by_l2():
    for mode in ("renormalize_l2_per_layer", "renormalize_l2_per_param_type"):
        net = _dense(l2=0.1, lr=0.5)
        net.layers[0].params["W"][...] = [[2.0], [-4.0]]
        net.layers[0].params["b"][...] = [3.0]
        zero = {(0, "W"): np.zeros((2, 1)), (0, "b"): np.zeros(1)}
        _update(net, mode, 1.0, zero, 8)
        assert net.grad_norm_last_norms and all(n == 0.0 for n in net.grad_norm_last_norms)
        assert np.all(np.isfinite(net.layers[0].params["W"]))
        np.testing.assert_array_equal(net.layers[0].params["W"].ravel(), [2.0 * 0.9, -4.0 * 0.9])     # W - l2 * W, no gradient part
        np.testing.assert_array_equal(net.layers[0].params["b"], [3.0])                               # no l2 on b
    assert o.multiplier(0.0, "renormalize_l2_per_layer", 1.0) == np.float32(1e5)


def _bn_net():
    net = o.Net([o.BatchNorm(2, updater=o.Sgd(1.0), name="bn")], seed=1)
    return net


# mb = 4; gamma summed gradient (4, 0) -> (1, 0) after / mb; beta 0; the mean pseudo-gradient (2, 0) is NOT divided by mb; var 0
BN_G = {(0, "gamma"): np.array([4.0, 0.0]), (0, "beta"): np.zeros(2), (0, "mean"): np.array([2.0, 0.0]), (0, "var"): np.zeros(2)}


def test_batchnorm_stats_inside_the_layer_norm():
    """bn_stats_normalized: ||g_layer|| = sqrt(1^2 + 2^2) (2, not 2/4: mean/var skip the division), and mean/var are scaled with the layer."""
    net = _update(_bn_net(), "renormalize_l2_per_layer", 1.0, BN_G, 4)
    m = float(np.float32(1 / np.sqrt(5.0)))
    np.testing.assert_allclose(net.layers[0].params["gamma"], [1 - m, 1], rtol=1e-7)
    np.testing.assert_allclose(net.layers[0].params["mean"], [-2 * m, 0], rtol=1e-7)
    np.testing.assert_allclose(net.layers[0].params["var"], [1, 1])
    np.testing.assert_allclose(net.grad_norm_last_norms, [np.sqrt(5.0)])


def test_batchnorm_stats_outside_the_layer_norm():
    """bn_stats_normalized off: the norm is gamma/beta's alone (1) and the mean/var pseudo-gradients pass unscaled (and undivided)."""
    net = _update(_bn_net(), "renormalize_l2_per_layer", 1.0, BN_G, 4, bn_stats_normalized=False)
    np.testing.assert_allclose(net.layers[0].params["gamma"], [0, 1], atol=1e-12)
    np.testing.assert_allclose(net.layers[0].params["mean"], [-2, 0])
    np.testing.assert_allclose(net.grad_norm_last_norms, [1.0])


def test_batchnorm_per_param_type():
    net = _update(_bn_net(), "clip_l2_per_param_type", 0.5, BN_G, 4)
    np.testing.assert_allclose(net.layers[0].params["gamma"], [0.5, 1])          # norm 1 > 0.5
    np.testing.assert_allclose(net.layers[0].params["mean"], [-0.5, 0])          # norm 2 > 0.5
    np.testing.assert_allclose(sorted(net.grad_norm_last_norms), [0, 0, 1, 2])


def test_frozen_layers_are_left_out_and_gan_step_picks_the_mode_up():
    """A two-layer net through fit: the oracle's fit and gan_step call apply_update, so the mode needs no other hook; frozen layers have no
    group."""
    rng = np.random.default_rng(0)
    base = o.Net([o.Dense(3, 4, "tanh", updater=o.Sgd(0.1), name="a"), o.Output(4, 1, updater=o.Sgd(0.1), name="out")], seed=3)
    x, y = rng.uniform(-1, 1, (5, 3)), rng.uniform(0, 1, (5, 1))
    plain, normed = copy.deepcopy(base), copy.deepcopy(base)
    normed.set_gradient_normalization("renormalize_l2_per_layer")
    plain.fit(x, y); normed.fit(x, y)
    assert len(normed.grad_norm_last_norms) == 2
    d_plain = base.params_flat() - plain.params_flat()
    d_norm = base.params_flat() - normed.params_flat()
    # each layer's step is its plain step divided by that layer's norm: unit norm per layer over lr
    for sl in (slice(0, 16), slice(16, 21)):
        np.testing.assert_allclose(np.linalg.norm(d_norm[sl]), 0.1, rtol=1e-6)
        np.testing.assert_allclose(d_norm[sl] / np.linalg.norm(d_norm[sl]), d_plain[sl] / np.linalg.norm(d_plain[sl]), rtol=1e-9)
    frozen = copy.deepcopy(base)
    frozen.set_gradient_normalization("renormalize_l2_per_layer")
    frozen.layers[0].frozen = True
    frozen.compute_gradient_and_score(x, y)
    frozen.apply_update(5)
    assert len(frozen.grad_norm_last_norms) == 1


def _header_gn_values():
    src = open(os.path.join(ROOT, "include", "b200gan.h")).read()
    body = re.search(r"typedef enum \{([^}]*)\} b2g_gradient_normalization;", src).group(1)
    return {k: int(v) for k, v in re.findall(r"B2G_GN_(\w+) = (\d+)", body)}


def test_mode_names_match_header_java_and_python():
    from gan_deeplearning4j_b200.engine import GRADIENT_NORMALIZATIONS
    h = _header_gn_values()
    assert h == {"NONE": 0, "RENORM_L2_LAYER": 1, "RENORM_L2_PARAM": 2, "CLIP_ELEMENTWISE": 3, "CLIP_L2_LAYER": 4, "CLIP_L2_PARAM": 5}
    assert GRADIENT_NORMALIZATIONS == {"none": 0, "renormalize_l2_per_layer": 1, "renormalize_l2_per_param_type": 2, "clip_l2_per_layer": 4,
                                       "clip_l2_per_param_type": 5}
    assert set(GRADIENT_NORMALIZATIONS) == set(o.GRAD_NORMS)
    java = open(os.path.join(ROOT, "java/src/main/java/org/deeplearning4j/nn/conf/GradientNormalization.java")).read()
    names = re.search(r"enum GradientNormalization \{\s*([^;}]*)", java).group(1).replace(" ", "").replace("\n", "").split(",")
    assert names == ["None", "RenormalizeL2PerLayer", "RenormalizeL2PerParamType", "ClipElementWiseAbsoluteValue", "ClipL2PerLayer", "ClipL2PerParamType"]


@pytest.fixture(scope="module")
def lib():
    import gan_deeplearning4j_b200 as b
    if not os.path.exists(b.LIB_PATH):
        sys.path.insert(0, ROOT)
        import __graft_entry__
        __graft_entry__.build()
    return b.load()


def test_entry_point_and_jni_symbol_exported(lib):
    assert hasattr(lib, "b2g_net_set_gradient_normalization")
    out = subprocess.run(["nm", "-D", "--defined-only", os.path.join(ROOT, "gan_deeplearning4j_b200", "lib", "libb200gan.so")], capture_output=True, text=True).stdout
    assert "Java_org_deeplearning4j_b200_Native_netSetGradientNormalization" in out
    native = open(os.path.join(ROOT, "java/src/main/java/org/deeplearning4j/b200/Native.java")).read()
    assert "public static native int netSetGradientNormalization(long net, int mode, float threshold);" in native
