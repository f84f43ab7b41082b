"""DL4J's PReLULayer on the device: the forward and backward kernels bit for bit against a CPU emulation of the documented order (every mask,
both paths, FP32 and BF16, ragged shapes, poisoned outputs); FP32 fit against the oracle's restatement on MLP and conv + BatchNorm
nets with several updaters, l1 / l2 and a schedule, frozen PReLUs, parameter round trips and the engine's refusals; BF16 nets; the GAN step
against the oracle (graph replay == eager), D's slopes untouched by the G step, a generator ending in a PReLU, and the launch count."""
import copy
import ctypes

import numpy as np
import pytest

from gan_deeplearning4j_b200 import _lib, engine, models as m
from helpers import (b200, bf16_round, check_weight_operands, compare_params_and_state, gan_step_parity, launches_per_step,  # noqa: F401
                     pclose, push_params, randomize, rel_err)
from oracle import dl4j_oracle as o

pytestmark = pytest.mark.gpu
TOL = 1e-3


# ------------------------------------------------------------------ CPU emulation of the kernels (include/b200gan.h, B2G_LAYER_PRELU) --------
def _index(H, W, C, mask):
    """(k, s, K, S) per row element j = (h*W + w)*C + c."""
    j = np.arange(H * W * C)
    c, pix = j % C, j // C
    h, w = pix // W, pix % W
    cs, hs, ws = mask & 1, mask & 2, mask & 4
    aH, aW, sH, sW = (1 if hs else H), (1 if ws else W), (H if hs else 1), (W if ws else 1)
    k = ((np.where(cs, 0, c)) * aH + np.where(hs, 0, h)) * aW + np.where(ws, 0, w)
    s = ((np.where(cs, c, 0)) * sH + np.where(hs, h, 0)) * sW + np.where(ws, w, 0)
    K = (1 if cs else C) * aH * aW
    return k, s, K, H * W * C // K


def _groups(R, M):
    bx = (M + 2047) // 2048
    g0 = max(1, min(R, max(1, min(64, 1024 // bx))))
    rpg = -(-R // g0)
    return -(-R // rpg), rpg


def emulate(x, alpha, dy, H, W, C, mask, bf16):
    """(y, dx, dalpha) as the kernels compute them; x, dy [R][H*W*C] NHWC fp32 (already rounded to bf16 in a BF16 run)."""
    R, M = x.shape
    k, s, K, S = _index(H, W, C, mask)
    a = alpha.astype(np.float32)[k][None]
    neg = x < 0
    rnd = bf16_round if bf16 else (lambda v: v)
    y = rnd(np.where(neg, a * x, x).astype(np.float32))
    dx = rnd(np.where(neg, a * dy, dy).astype(np.float32))
    term = np.where(neg, x * dy, np.float32(0)).astype(np.float32)
    G, rpg = _groups(R, M)
    part = np.zeros((G * S, K), np.float32)
    for g in range(G):
        acc = np.zeros(M, np.float32)
        for r in range(g * rpg, min(R, (g + 1) * rpg)):
            acc = acc + term[r]
        part[g * S + s, k] = acc
    T = G * S
    if T >= 64 and K <= 65536:        # the reduce list's warp-per-output job
        lanes = np.zeros((32, K), np.float32)
        for t in range(T):
            lanes[t % 32] = lanes[t % 32] + part[t]
        for msk in (16, 8, 4, 2, 1):
            lanes = lanes + lanes[np.arange(32) ^ msk]
        da = lanes[0]
    else:
        da = np.zeros(K, np.float32)
        for t in range(T):
            da = da + part[t]
    return y, dx, da


def _run(b, ctx, prec, x, alpha, dy, N, H, W, C, mask, offset, **kw):
    n = N * H * W * C
    (y, _, _), fi = b.test_ew(ctx, prec, "prelu_fwd", np.concatenate([x.ravel(), alpha]), None, (n, 0, 0), shared=mask, N=N, H=H, W=W, C=C,
                               offset=offset, poison=True)
    (dx, da, _), bi = b.test_ew(ctx, prec, "prelu_bwd", np.concatenate([x.ravel(), alpha]), dy, (n, alpha.size, 0), shared=mask, N=N, H=H, W=W,
                                C=C, offset=offset, poison=True)
    return y, dx, da, fi["kernel"], bi["kernel"]


SHAPES = [(5, 3, 4, 8), (71, 4, 4, 16), (3, 5, 3, 5), (9, 1, 1, 37), (6, 1, 1, 64)]


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("shape", SHAPES)
def test_kernels_bit_for_bit(b200, prec, shape):
    b, ctx = b200
    p = b.FP32 if prec == "fp32" else b.BF16
    N, H, W, C = shape
    masks = range(8) if H * W > 1 else (0, 1)
    rng = np.random.default_rng(N * 1000 + C)
    for mask in masks:
        k, s, K, S = _index(H, W, C, mask)
        x = rng.uniform(-1, 1, (N, H * W * C)).astype(np.float32)
        x.ravel()[::7] = 0.0; x.ravel()[3::11] = -0.0; x.ravel()[5] = np.nan
        dy = rng.standard_normal((N, H * W * C)).astype(np.float32)
        alpha = rng.uniform(-0.5, 0.8, K).astype(np.float32)
        xs, dys = (x, dy) if p == b.FP32 else (bf16_round(x), bf16_round(dy))
        want = emulate(xs, alpha, dys, H, W, C, mask, p == b.BF16)
        V = 4 if p == b.FP32 else 8
        for offset in (0, 1):
            y, dx, da, fk, bk = _run(b, ctx, p, x, alpha, dy, N, H, W, C, mask, offset)
            path = "vec" if offset == 0 and (H * W * C) % V == 0 else "scalar"
            assert fk == f"prelu_fwd_kernel<{path}>" and bk == f"prelu_bwd_kernel<{path}>,reduce_multi_kernel", (fk, bk)
            np.testing.assert_array_equal(y, want[0].ravel(), err_msg=f"y {shape} mask {mask} offset {offset}")
            np.testing.assert_array_equal(dx, want[1].ravel(), err_msg=f"dx {shape} mask {mask} offset {offset}")
            np.testing.assert_array_equal(da, want[2], err_msg=f"dalpha {shape} mask {mask} offset {offset}")
            assert np.signbit(y.reshape(x.shape)[x == 0]).tolist() == np.signbit(xs[x == 0]).tolist()


def test_backward_without_slope_gradient_or_dx(b200):
    b, ctx = b200
    N, H, W, C, mask = 7, 4, 4, 8, 6
    rng = np.random.default_rng(2)
    x, dy = rng.uniform(-1, 1, (N, H * W * C)).astype(np.float32), rng.standard_normal((N, H * W * C)).astype(np.float32)
    alpha = rng.uniform(0, 0.5, C).astype(np.float32)
    _, dx_want, _ = emulate(x, alpha, dy, H, W, C, mask, False)
    (dx, _, _), info = b.test_ew(ctx, b.FP32, "prelu_bwd", np.concatenate([x.ravel(), alpha]), dy, (x.size, 0, 0), shared=mask, N=N, H=H, W=W, C=C)
    np.testing.assert_array_equal(dx, dx_want.ravel())
    assert info["kernel"] == "prelu_bwd_kernel<vec>"        # no slope gradient: no reduce launch


# ------------------------------------------------------------------ nets against the oracle ----------------------------------------------
REG = {"l1": 2e-3, "l2": 1e-2}


def _upd(kind):
    return {"sgd": m.sgd(0.05), "adam": m.adam(2e-3), "nesterovs": m.nesterovs(0.02), "rmsprop": m.rmsprop(2e-3, 0.95, 1e-8), "amsgrad": m.amsgrad(2e-3)}[kind]


def _bound(kind):
    step = {"nesterovs": 0.02, "amsgrad": 2e-3, "adam": 2e-3, "rmsprop": 2e-3 / np.sqrt(0.05), "sgd": 0.0}[kind]
    return 2 * step + 2 * REG["l1"]


def _specs(net, kind, reg=True):
    u = lambda: _upd(kind)
    pre = lambda axes, name, **kw: dict(m.prelu(axes, name), updater=u(), **(REG if reg else {}), **kw)
    if net == "mlp":
        return [{"type": "dense", "name": "d1", "n_out": 32, "updater": u()}, pre((), "p1"),
                {"type": "dense", "name": "d2", "n_out": 16, "activation": "tanh", "updater": u()}, pre((1,), "p2", input_shape=(16,)),
                {"type": "output", "name": "out", "n_out": 1, "updater": u()}], (24,)
    return [{"type": "conv2d", "name": "c1", "n_out": 8, "kernel": (3, 3), "stride": (2, 2), "padding": (1, 1), "updater": u()}, pre((), "p1"),
            {"type": "conv2d", "name": "c2", "n_out": 12, "kernel": (3, 3), "stride": (1, 1), "padding": (1, 1), "has_bias": False, "updater": u()},
            {"type": "batchnorm", "name": "bn2", "updater": u()}, pre((2, 3), "p2", input_shape=(12, 4, 4)), {"type": "cnn_to_ff", "name": "flat"},
            {"type": "dense", "name": "fc", "n_out": 10, "activation": "tanh", "updater": u()}, {"type": "output", "name": "out", "n_out": 1, "updater": u()}], (3, 8, 8)


def _oracle(specs, shape, seed):
    rng = np.random.default_rng(seed)
    onet = o.net_from_specs(specs, shape, seed=2)
    randomize(onet, rng)
    for l in onet.layers:
        if isinstance(l, o.PReLU):
            l.params["W"] = rng.uniform(-0.3, 0.6, l.alpha_shape)
    return onet, rng


def _fit_and_compare(b, ctx, specs, shape, steps=3, seed=11, precision=None, **kw):
    onet, rng = _oracle(specs, shape, seed)
    bnet = b.Net(ctx, specs, shape, max_batch=6, precision=b.FP32 if precision is None else precision, **kw)
    push_params(onet, bnet)
    bounds = {s["name"]: _bound(s["updater"]["kind"]) for s in specs if s.get("updater")}
    for it in range(steps):
        x, y = rng.uniform(-1, 1, (6,) + shape), rng.uniform(0, 1, (6, 1))
        so, sb = onet.fit(x, y), bnet.fit(x, y)
        if precision is None:
            assert abs(so - sb) < TOL * max(1.0, abs(so)), (it, so, sb)
            compare_params_and_state(onet, bnet, it, TOL, bounds)
    return onet, bnet


@pytest.mark.parametrize("kind", ["sgd", "adam", "nesterovs", "rmsprop", "amsgrad"])
@pytest.mark.parametrize("net", ["mlp", "convbn"])
def test_fp32_fit_matches_oracle(b200, net, kind):
    b, ctx = b200
    specs, shape = _specs(net, kind)
    onet, bnet = _fit_and_compare(b, ctx, specs, shape)
    l1, l2 = bnet.calc_regularization()
    assert abs(l1 - onet.calc_l1()) < 1e-4 * onet.calc_l1() and abs(l2 - onet.calc_l2()) < 1e-4 * onet.calc_l2()
    assert bnet.get_regularization("p1") == pytest.approx({"l1": 2e-3, "l2": 1e-2, "l1_bias": 0.0, "l2_bias": 0.0})
    bnet.close()


def test_fp32_fit_with_schedule_and_gradient_normalization(b200):
    b, ctx = b200
    specs, shape = _specs("convbn", "adam")
    for s in specs:
        if s.get("updater"):
            s["updater"]["lr"] = m.exponential_schedule(2e-3, 0.8)
    onet, bnet = _fit_and_compare(b, ctx, specs, shape)
    assert bnet.learning_rate("p2") == onet.learning_rate("p2")
    bnet.close()
    specs, shape = _specs("mlp", "adam")
    onet, rng = _oracle(specs, shape, 4)
    onet.set_gradient_normalization("clip_l2_per_layer", 0.05)
    bnet = b.Net(ctx, specs, shape, max_batch=6, precision=b.FP32, gradient_normalization="clip_l2_per_layer", gradient_normalization_threshold=0.05)
    push_params(onet, bnet)
    for it in range(3):
        x, y = rng.uniform(-1, 1, (6,) + shape), rng.uniform(0, 1, (6, 1))
        onet.fit(x, y); bnet.fit(x, y)
        compare_params_and_state(onet, bnet, it, TOL, {s["name"]: _bound("adam") for s in specs})
    bnet.close()


@pytest.mark.parametrize("trainable_below", [False, True])
def test_frozen_prelu_under_a_trainable_head(b200, trainable_below):
    b, ctx = b200
    u = lambda: m.adam(2e-3)
    specs = [dict({"type": "dense", "name": "d1", "n_out": 16, "updater": u()}, **({} if trainable_below else {"frozen": True})),
             dict(m.prelu((), "p1"), updater=u(), frozen=True),
             {"type": "dense", "name": "d2", "n_out": 8, "activation": "tanh", "updater": u()}, {"type": "output", "name": "out", "n_out": 1, "updater": u()}]
    onet, bnet = _fit_and_compare(b, ctx, specs, (12,))
    a = onet.layer("p1").params["W"].astype(np.float32)
    np.testing.assert_array_equal(bnet.get_param("p1", "W", a.size), a.ravel())       # never updated
    bnet.close()


def test_param_round_trips_in_dl4j_order(b200):
    b, ctx = b200
    specs, shape = _specs("convbn", "adam")
    onet, rng = _oracle(specs, shape, 5)
    bnet = b.Net(ctx, specs, shape, max_batch=4, precision=b.FP32)
    assert bnet.num_params() == onet.num_params()
    assert np.all(bnet.get_param("p1", "W", 8 * 4 * 4) == 0) and np.all(bnet.get_param("p2", "W", 12) == 0)     # a new PReLU is a ReLU
    push_params(onet, bnet)
    np.testing.assert_array_equal(bnet.params(), onet.params_flat().astype(np.float32))
    for name, l in (("p1", onet.layer("p1")), ("p2", onet.layer("p2"))):
        w = l.params["W"].astype(np.float32).ravel()          # 'c' order [C, H, W] with the shared axes of extent 1
        np.testing.assert_array_equal(bnet.get_param(name, "W", w.size), w)
        new = rng.uniform(-1, 1, w.size).astype(np.float32)
        bnet.set_param(name, "W", new)
        np.testing.assert_array_equal(bnet.get_param(name, "W", w.size), new)
        l.params["W"] = new.reshape(l.alpha_shape).astype(np.float64)
    np.testing.assert_array_equal(bnet.params(), onet.params_flat().astype(np.float32))
    bnet.close()


def test_weight_init_and_refusals(b200):
    b, ctx = b200
    specs, shape = _specs("convbn", "adam", reg=False)
    bnet = b.Net(ctx, specs, shape, max_batch=4, precision=b.FP32)
    w_c1 = bnet.get_param("c1", "W", 8 * 3 * 9)
    bnet.init_weights(m.weight_init("ones"), "p2")
    assert np.all(bnet.get_param("p2", "W", 12) == 1)
    bnet.init_weights(m.weight_init("distribution", m.uniform(0.1, 0.3)), "p1")
    np.testing.assert_array_equal(bnet.get_param("p1", "W", 128), o.weight_init_draw("uniform", 0.1, 0.3, 128, 666, 1))
    bnet.init_weights(m.weight_init("xavier"))             # the global form leaves PReLU layers alone
    assert np.all(bnet.get_param("p2", "W", 12) == 1) and not np.array_equal(bnet.get_param("c1", "W", w_c1.size), w_c1)
    wi = engine.weight_init_struct(m.weight_init("relu"))
    assert ctx.lib.b2g_net_init_weights(bnet.h, b"p1", ctypes.byref(wi)) == -1
    arr = (_lib.Constraint * 1)(engine.constraint_struct(m.non_negative()))
    assert ctx.lib.b2g_net_set_constraints(bnet.h, b"p1", b"W", arr, 1) == -1
    with pytest.raises(b.B200GanError) as e:
        bnet.set_weight_noise(m.drop_connect(0.9), "p1")
    assert e.value.code == -1
    bnet.set_weight_noise(m.drop_connect(0.9))              # the global form skips PReLU layers
    bnet.set_weight_noise(None)
    bnet.close()
    for bad, code in (([{"type": "dense", "name": "d", "n_out": 4}, m.prelu((2,), "p")], -1),
                      ([{"type": "dense", "name": "d", "n_out": 4}, m.prelu((), "p", input_shape=(5,))], -2),
                      ([m.prelu((), "p", input_shape=(3, 8, 4))], -2)):
        with pytest.raises(b.B200GanError) as e:
            b.Net(ctx, bad + [{"type": "output", "name": "out", "n_out": 1}], (3, 8, 8) if len(bad) == 1 else (6,), max_batch=2)
        assert e.value.code == code, bad


def test_bf16_nets(b200):
    """BF16 conv + BatchNorm + PReLU fit: three steps stay within 5e-2 of the oracle's parameters (relative to their largest magnitude)."""
    b, ctx = b200
    specs, shape = _specs("convbn", "adam")
    onet, bnet = _fit_and_compare(b, ctx, specs, shape, precision=b.BF16)
    assert rel_err(bnet.params(), onet.params_flat()) < 5e-2, rel_err(bnet.params(), onet.params_flat())
    bnet.close()


# ------------------------------------------------------------------ the GAN step -------------------------------------------------------------
def _gan_pair(gs, ds, size=16, z=12):
    rng = np.random.default_rng(5)
    G = o.net_from_specs(gs, (z,), seed=1); D = o.net_from_specs(ds, (3, size, size), seed=2)
    randomize(G, rng); randomize(D, rng)
    for net in (G, D):
        for l in net.layers:
            if isinstance(l, o.PReLU):
                l.params["W"] = rng.uniform(0.05, 0.3, l.alpha_shape)
    return G, D


def test_gan_step_matches_oracle(b200):
    b, ctx = b200
    lr = 2e-3
    gs, ds = m.dcgan_generator(16, 12, 8, 3, lr=lr, activation="prelu"), m.dcgan_discriminator(16, 8, 3, lr=lr, activation="prelu")
    G, D = _gan_pair(gs, ds)
    data = [a.astype(np.float64) for a in o.synthetic_batch(4, 16, 3, 12, seed=3)]
    gan_step_parity(b, ctx, gs, ds, G, D, data, data[3:], lr, "prelu dcgan")
    # a generator ending in a PReLU (identity last deconv): not folded into D's first input-gradient kernel
    gs2 = copy.deepcopy(gs)
    gs2[-1].pop("activation")
    gs2.append(dict(m.prelu((2, 3), "gen_out_act"), updater=m.adam(lr, 0.5)))
    G2, D2 = _gan_pair(gs2, ds)
    gan_step_parity(b, ctx, gs2, ds, G2, D2, data, data[3:], lr, "generator ending in a PReLU")


def test_g_step_leaves_d_slopes_alone(b200):
    """D's PReLU layers on lr 0: after GAN steps their slopes are the bits they started with, although the G step back-propagates through them."""
    b, ctx = b200
    gs = m.dcgan_generator(16, 12, 8, 3, lr=2e-3, activation="prelu")
    ds = m.dcgan_discriminator(16, 8, 3, lr=2e-3, activation="prelu")
    for s in ds:
        if s["type"] == "prelu":
            s["updater"] = m.adam(0.0, 0.5)
    G, D = _gan_pair(gs, ds)
    bG = b.Net(ctx, gs, (12,), max_batch=4, precision=b.FP32); bD = b.Net(ctx, ds, (3, 16, 16), max_batch=8, precision=b.FP32, bn_groups=2)
    push_params(G, bG); push_params(D, bD)
    names = [s["name"] for s in ds if s["type"] == "prelu"]
    before = {nm: bD.get_param(nm, "W", D.layer(nm).params["W"].size) for nm in names}
    g_before = bG.params()
    gan = b.Gan(bG, bD, use_cuda_graph=True)
    data = o.synthetic_batch(4, 16, 3, 12, seed=3)
    for _ in range(3):
        gan.step(*data)
    for nm in names:
        np.testing.assert_array_equal(bD.get_param(nm, "W", before[nm].size), before[nm], err_msg=nm)
    assert not np.array_equal(bG.params(), g_before)
    gan.close(); bG.close(); bD.close()


def _as_elu_layers(specs):
    return [{"type": "activation", "name": s["name"], "activation": "elu"} if s["type"] == "prelu" else s for s in specs]


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_launch_count(b200, prec):
    """A PReLU layer launches what an ActivationLayer of codes 5-16 at its place launches (one forward, one backward per pass: neither is fused);
    the slope gradients ride the backward pass's reduce-list launch: in BF16 nets that launch is there already (the tensor-core weight
    gradients queue into it), in FP32 nets it is added once per backward that trains a PReLU: twice per GAN step (D step and G step)."""
    b, ctx = b200
    p = b.FP32 if prec == "fp32" else b.BF16
    size, z, nf, n = (16, 12, 8, 4) if prec == "fp32" else (64, 100, 64, 16)
    gs, ds = m.dcgan_generator(size, z, nf, 3, activation="prelu"), m.dcgan_discriminator(size, nf, 3, activation="prelu")
    data = o.synthetic_batch(n, size, 3, z, seed=3)
    counts = []
    for g_specs, d_specs in ((gs, ds), (_as_elu_layers(gs), _as_elu_layers(ds))):
        G = b.Net(ctx, g_specs, (z,), max_batch=n, precision=p, xent_clip_eps=0.0)
        D = b.Net(ctx, d_specs, (3, size, size), max_batch=2 * n, precision=p, xent_clip_eps=0.0, bn_groups=2)
        gan = b.Gan(G, D, use_cuda_graph=True)
        gan.upload(*data)
        counts.append(launches_per_step(ctx, gan, n))
        if p == b.BF16 and g_specs is gs:
            check_weight_operands(b, G, gs, "bf16 prelu G"); check_weight_operands(b, D, ds, "bf16 prelu D")
            assert np.isfinite(gan.losses()).all()
        gan.close(); G.close(); D.close()
    assert counts[0] == counts[1] + (2 if p == b.FP32 else 0), counts
