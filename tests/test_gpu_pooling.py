"""Average, sum and p-norm pooling on the GPU: the pool2d / global_pool kernels through their production wrappers (b2g_test_ew ops pool2d /
global_pool) against the oracle's restatement in both precisions on the vector, C % 8 != 0 and misaligned paths, with poisoned outputs and a global
map large enough to be split over blocks; fp32 AVG / SUM forwards bit for bit against an fp32 emulation of the documented summation order; FP32
nets with every kind against the float64 oracle over 3 fit iterations (one of them a ragged batch); BF16 nets layer by layer; the BF16 GAN step
with a global-pooling-head discriminator (graph replay == eager, two fresh nets equal, bit for bit); launches per pass; argument checks."""
import ctypes as C

import numpy as np
import pytest

from gan_deeplearning4j_b200 import models as m
from helpers import b200, bf16_round, check_bf16, fp32_gan_pair, oracle_gan_pair, pclose, push_params, randomize, rel_err
from oracle import dl4j_oracle as o

pytestmark = pytest.mark.gpu
TOL = 1e-3
U = 2.0 ** -24


def _nchw(a_nhwc):
    return np.ascontiguousarray(np.asarray(a_nhwc).transpose(0, 3, 1, 2))


def _nhwc(a_nchw):
    return np.ascontiguousarray(np.asarray(a_nchw).transpose(0, 2, 3, 1))


def _within(got, ref, mag, u_out, k, what):
    got, ref, mag = (np.asarray(v, np.float64) for v in (got, ref, mag))
    assert np.isfinite(got).all(), (what, "non-finite (an unwritten element reads back as NaN)")
    tol = u_out * np.abs(ref) + k * U * mag + 1e-30
    bad = np.abs(got - ref) > tol
    assert not bad.any(), (what, int(bad.sum()), got[bad][:4], ref[bad][:4])


# ------------------------------------------------------------------ the kernels against float64 -----------------------------------------
POOL2D_KINDS = [("avg", 2), ("sum", 2), ("pnorm", 1), ("pnorm", 2), ("pnorm", 3)]
PATHS = {"vector": (16, 0), "c13": (13, 0), "offset": (16, 3)}      # (C, element offset of every operand)


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("kind,p", POOL2D_KINDS)
def test_pool2d_kernels_against_float64(b200, kind, p, prec, path):
    b, ctx = b200
    P = b.FP32 if prec == "fp32" else b.BF16
    c, off = PATHS[path]
    u_out = U if P == b.FP32 else 2.0 ** -8
    rng = np.random.default_rng(o.POOL_CODES[kind] * 10 + p)
    for (kh, kw), (sh, sw), (ph, pw), h, w in [((3, 3), (2, 2), (1, 1), 9, 7), ((2, 3), (3, 1), (1, 2), 7, 6)]:
        n = 3
        oh, ow = (h + 2 * ph - kh) // sh + 1, (w + 2 * pw - kw) // sw + 1
        x = rng.uniform(-2, 2, (n, h, w, c)).astype(np.float32)
        e = rng.uniform(-2, 2, (n, oh, ow, c)).astype(np.float32)
        (y, dx, _), info = b.test_pool(ctx, P, "pool2d", x, e, (n * oh * ow * c, n * h * w * c, 0), pooling=kind, N=n, H=h, W=w, C=c, KH=kh, KW=kw,
                                     SH=sh, SW=sw, PH=ph, PW=pw, pnorm=float(p), offset=off, poison=True)
        assert info["kernel"] == f"pool2d_fwd_kernel<{kind}>,pool2d_bwd_kernel<{kind}>", info
        xs, es = (x, e) if P == b.FP32 else (bf16_round(x), bf16_round(e))
        xs, es = _nchw(xs.astype(np.float64)), _nchw(es.astype(np.float64))
        geo = ((kh, kw), (sh, sw), (ph, pw))
        y_ref = o.pool2d_forward(kind, xs, *geo, p)
        y_mag = y_ref if kind == "pnorm" else o.pool2d_forward(kind, np.abs(xs), *geo, p)
        _within(_nchw(y.reshape(n, oh, ow, c)), y_ref, y_mag, u_out, 32, (kind, p, prec, path, "y"))
        y_dev = _nchw(y.reshape(n, oh, ow, c).astype(np.float64))          # the backward reads the stored y
        dx_ref = o.pool2d_backward(kind, xs, y_dev, es, *geo, p)
        dx_mag = o.pool2d_backward(kind, np.abs(xs), y_dev, np.abs(es), *geo, p)
        _within(_nchw(dx.reshape(n, h, w, c)), dx_ref, dx_mag, u_out, 64, (kind, p, prec, path, "dx"))


def gp_plan(prec_bytes, n, hw, c, vec):
    """kernels_pool.cu gp_plan: (lanes per channel vector, splits)."""
    cv = c // (16 // prec_bytes) if vec else c
    cw = min(cv, 32); rows = 256 // cw; chunks = -(-cv // cw)
    blocks = n * chunks
    s = 1 if blocks >= 264 else -(-264 // blocks)
    s = min(s, max(1, hw // (rows * 4)))
    return rows, max(1, min(s, 64))


GLOBAL_KINDS = [("max", 2), ("avg", 2), ("sum", 2), ("pnorm", 1), ("pnorm", 3)]


@pytest.mark.parametrize("shape", ["small", "split"])
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("kind,p", GLOBAL_KINDS)
def test_global_kernels_against_float64(b200, kind, p, prec, path, shape):
    b, ctx = b200
    P = b.FP32 if prec == "fp32" else b.BF16
    c, off = PATHS[path]
    u_out = U if P == b.FP32 else 2.0 ** -8
    n, h, w = (5, 4, 3) if shape == "small" else (2, 64, 48)
    rng = np.random.default_rng(o.POOL_CODES[kind] * 10 + p + (shape == "split"))
    x = rng.uniform(-2, 2, (n, h, w, c)).astype(np.float32)
    e = rng.uniform(-2, 2, (n, c)).astype(np.float32)
    (y, dx, idx), info = b.test_pool(ctx, P, "global_pool", x, e, (n * c, n * h * w * c, n * c), pooling=kind, N=n, H=h, W=w, C=c, pnorm=float(p),
                                   offset=off, poison=True)
    assert info["kernel"] == f"global_pool_fwd_kernel<{kind}>,global_pool_bwd_kernel<{kind}>", info
    want_splits = gp_plan(4 if P == b.FP32 else 2, n, h * w, c, c % (4 if P == b.FP32 else 8) == 0 and off == 0)[1]
    assert info["splits"] == want_splits and (want_splits > 1) == (shape == "split"), (info, want_splits)
    xs, es = (x, e) if P == b.FP32 else (bf16_round(x), bf16_round(e))
    xs, es = _nchw(xs.astype(np.float64)), es.astype(np.float64)
    y_ref, i_ref = o.global_forward(kind, xs, p)
    if kind == "max":
        assert np.array_equal(idx.reshape(n, c), i_ref) and np.array_equal(y.reshape(n, c), y_ref), (kind, prec, path, shape)
    else:
        assert (idx == -1).all()
        y_mag = y_ref if kind == "pnorm" else o.global_forward(kind, np.abs(xs), p)[0]
        _within(y.reshape(n, c), y_ref, y_mag, u_out, 128, (kind, p, prec, path, shape, "y"))
    y_dev = y.reshape(n, c).astype(np.float64)
    dx_ref = o.global_backward(kind, xs, y_dev, i_ref, es, p)
    dx_mag = o.global_backward(kind, np.abs(xs), y_dev, i_ref, np.abs(es), p)
    _within(_nchw(dx.reshape(n, h, w, c)), dx_ref, dx_mag, u_out, 8, (kind, p, prec, path, shape, "dx"))


def _emulate_pool2d(kind, x, k, s, pad):
    """fp32, in the documented order: the window's in-range elements added in row-major window order, then / (kh*kw) for AVG."""
    (kh, kw), (sh, sw), (ph, pw) = k, s, pad
    n, h, w, c = x.shape
    oh, ow = (h + 2 * ph - kh) // sh + 1, (w + 2 * pw - kw) // sw + 1
    xp = np.zeros((n, h + 2 * ph, w + 2 * pw, c), np.float32); xp[:, ph:ph + h, pw:pw + w] = x
    valid = np.zeros((h + 2 * ph, w + 2 * pw), bool); valid[ph:ph + h, pw:pw + w] = True
    acc = np.zeros((n, oh, ow, c), np.float32)
    for r in range(kh):
        for q in range(kw):
            v = xp[:, r:r + sh * oh:sh, q:q + sw * ow:sw][:, :oh, :ow]
            m = valid[r:r + sh * oh:sh, q:q + sw * ow:sw][:oh, :ow][None, :, :, None]
            acc = np.where(m, acc + v, acc).astype(np.float32)
    return acc / np.float32(kh * kw) if kind == "avg" else acc


def _emulate_global(kind, x, rows, splits):
    """fp32: lane t of a split sums pixels t, t + rows, ...; lanes fold in order; splits fold in order; AVG / (H*W)."""
    n, hw, c = x.shape
    parts = []
    for sp in range(splits):
        p0, p1 = hw * sp // splits, hw * (sp + 1) // splits
        lanes = []
        for t in range(rows):
            a = np.zeros((n, c), np.float32)
            for pix in range(p0 + t, p1, rows):
                a = (a + x[:, pix]).astype(np.float32)
            lanes.append(a)
        a = lanes[0]
        for l in lanes[1:]:
            a = (a + l).astype(np.float32)
        parts.append(a)
    a = parts[0]
    for q in parts[1:]:
        a = (a + q).astype(np.float32)
    return a / np.float32(hw) if kind == "avg" else a


@pytest.mark.parametrize("kind", ["avg", "sum"])
def test_fp32_forward_bit_identical_to_the_documented_order(b200, kind):
    b, ctx = b200
    rng = np.random.default_rng(1)
    for c, off in ((16, 0), (13, 0)):
        x = rng.standard_normal((2, 9, 7, c)).astype(np.float32)
        geo = ((3, 3), (2, 2), (1, 1))
        oh, ow = 5, 4
        (y, _, _), _ = b.test_pool(ctx, b.FP32, "pool2d", x, np.zeros((2, oh, ow, c), np.float32), (2 * oh * ow * c, 0, 0), pooling=kind, N=2, H=9, W=7,
                                 C=c, KH=3, KW=3, SH=2, SW=2, PH=1, PW=1, offset=off)
        assert np.array_equal(y.reshape(2, oh, ow, c), _emulate_pool2d(kind, x, *geo)), (kind, c)
        for n, h, w in ((3, 5, 4), (2, 40, 30)):
            x = rng.standard_normal((n, h, w, c)).astype(np.float32)
            (y, _, _), info = b.test_pool(ctx, b.FP32, "global_pool", x, np.zeros((n, c), np.float32), (n * c, 0, 0), pooling=kind, N=n, H=h, W=w, C=c)
            rows, splits = gp_plan(4, n, h * w, c, c % 4 == 0)
            assert info["splits"] == splits
            assert np.array_equal(y.reshape(n, c), _emulate_global(kind, x.reshape(n, h * w, c), rows, splits)), (kind, c, n, h, w)


# ------------------------------------------------------------------ FP32 nets against the oracle ----------------------------------------
def _sub_net(pool, p):
    return [{"type": "conv2d", "name": "c1", "n_out": 8, "kernel": (3, 3), "stride": (1, 1), "padding": (1, 1), "activation": "tanh", "updater": m.sgd(0.05)},
            dict(m.subsampling(pool, (3, 3), (2, 2), (1, 1), pnorm=p if pool == "pnorm" else None), name="s1"),
            {"type": "conv2d", "name": "c2", "n_out": 6, "kernel": (2, 2), "stride": (1, 1), "activation": "tanh", "updater": m.adam(1e-2)},
            {"type": "cnn_to_ff", "name": "ff"},
            {"type": "dense", "name": "d1", "n_out": 7, "activation": "tanh", "updater": m.sgd(0.05), "l2": 1e-3},
            {"type": "output", "name": "out", "n_out": 3, "loss": "mse", "updater": m.sgd(0.05)}], (3, 9, 7)


def _global_net(pool, p):
    return [{"type": "conv2d", "name": "c1", "n_out": 8, "kernel": (3, 3), "stride": (2, 2), "padding": (1, 1), "activation": "tanh", "updater": m.sgd(0.05)},
            {"type": "batchnorm", "name": "bn1", "updater": m.sgd(0.05)},
            {"type": "activation", "name": "a1", "activation": "lrelu", "alpha": 0.2},
            dict(m.global_pooling(pool, p), name="g1"),
            {"type": "dense", "name": "d1", "n_out": 7, "activation": "tanh", "updater": m.sgd(0.05)},
            {"type": "output", "name": "out", "n_out": 3, "loss": "mse", "updater": m.sgd(0.05)}], (3, 9, 7)


NETS = [("sub", "avg", 2), ("sub", "sum", 2), ("sub", "pnorm", 2), ("sub", "pnorm", 3),
        ("global", "max", 2), ("global", "avg", 2), ("global", "sum", 2), ("global", "pnorm", 2), ("global", "pnorm", 1)]


@pytest.mark.parametrize("net,pool,p", NETS)
def test_fp32_nets_match_oracle(b200, net, pool, p):
    """Every activation, every gradient, the score, the post-update parameters and b2g_net_output within DESIGN 1's 1e-3 over 3 fit iterations;
    the second on a ragged batch of 5 (max_batch 6)."""
    b, ctx = b200
    specs, shape = (_sub_net if net == "sub" else _global_net)(pool, p)
    rng = np.random.default_rng(o.POOL_CODES[pool] * 10 + p)
    onet = o.net_from_specs(specs, shape, seed=2, flat_input=False); randomize(onet, rng)
    bnet = b.Net(ctx, specs, shape, max_batch=6, precision=b.FP32)
    push_params(onet, bnet)
    for it, mb in enumerate((6, 5, 6)):
        x = rng.uniform(-1.5, 1.5, (mb,) + shape); y = rng.uniform(-1, 1, (mb, 3))
        s_o, acts, _, _ = onet.compute_gradient_and_score(x, y, collect=True)
        s_b = bnet.compute_gradient_and_score(x, y)
        assert abs(s_b - s_o) <= TOL * abs(s_o), (net, pool, it, s_b, s_o)
        for i, a in enumerate(acts[:-1]):
            if specs[i]["type"] == "batchnorm" and specs[i + 1]["type"] == "activation":
                a = acts[i + 1]                          # the engine stores BatchNorm + activation as one tensor
            assert rel_err(bnet.activation(i, mb), a.reshape(mb, -1)) <= TOL, (net, pool, it, "activation", i)
        assert rel_err(bnet.gradients(), onet.grads_flat()) <= TOL, (net, pool, it, "gradients")
        s_o = onet.fit(x, y); s_b = bnet.fit(x, y)
        assert abs(s_b - s_o) <= TOL * abs(s_o), (net, pool, it, s_b, s_o)
        assert rel_err(bnet.params(), onet.params_flat()) <= TOL, (net, pool, it, "params")
        xo = rng.uniform(-1.5, 1.5, (4,) + shape)
        assert rel_err(bnet.output(xo), onet.output(xo).reshape(4, -1)) <= TOL, (net, pool, it, "output")
    bnet.close()


# ------------------------------------------------------------------ BF16 nets, layer by layer -------------------------------------------
@pytest.mark.parametrize("pool,p", [("avg", 2), ("sum", 2), ("pnorm", 2), ("max", 2)])
def test_bf16_nets_layer_by_layer(b200, pool, p):
    """A 16x16 DCGAN discriminator with a global-pooling head, and a conv -> subsampling -> conv -> global net: each layer against the oracle's
    layer run on the GPU's own input to it (check_bf16)."""
    b, ctx = b200
    n = 16
    sub = "avg" if pool == "max" else pool
    specs2 = [{"type": "conv2d", "name": "c1", "n_out": 64, "kernel": (4, 4), "stride": (2, 2), "padding": (1, 1), "activation": "lrelu", "alpha": 0.2},
              dict(m.subsampling(sub, (3, 3), (2, 2), (1, 1), pnorm=p if sub == "pnorm" else None), name="s1"),
              {"type": "conv2d", "name": "c2", "n_out": 128, "kernel": (3, 3), "stride": (1, 1), "padding": (1, 1), "has_bias": False},
              {"type": "batchnorm", "name": "bn2"}, {"type": "activation", "name": "a2", "activation": "lrelu", "alpha": 0.2},
              dict(m.global_pooling(pool, p), name="g"), {"type": "output", "name": "out", "n_out": 1}]
    rng = np.random.default_rng(o.POOL_CODES[pool])
    for specs in (m.dcgan_discriminator(16, 64, 3, global_pooling=pool), specs2):
        x = bf16_round(rng.uniform(-1, 1, (n, 3, 16, 16)))
        onet = o.net_from_specs(specs, (3, 16, 16), seed=3, flat_input=False); randomize(onet, rng)
        for l in onet.layers:
            if l.has_params and "W" in l.params:
                l.params["W"] = bf16_round(l.params["W"]).astype(np.float64)
        bnet = b.Net(ctx, specs, (3, 16, 16), max_batch=n, precision=b.BF16)
        push_params(onet, bnet)
        bnet.output(x, train=True)
        cur, i = x.astype(np.float64), 0
        while i < len(specs) - 1:
            ref = onet.layers[i].forward(cur, True)
            fused = specs[i]["type"] == "batchnorm" and specs[i + 1]["type"] == "activation"      # stored as one tensor
            if fused:
                ref = onet.layers[i + 1].forward(ref, True)
            got = bnet.activation(i, n).reshape(ref.shape)
            check_bf16(got, ref, f"{pool} {specs[i]['name']}")
            cur = got.astype(np.float64)
            i += 2 if fused else 1
        bnet.close()


# ------------------------------------------------------------------ the GAN step with a global-pooling head ------------------------------
def _gan_run(b, ctx, gs, ds, G, D, data, n, size, z, graph, steps=3):
    bG = b.Net(ctx, gs, (z,), max_batch=n, precision=b.BF16)
    bD = b.Net(ctx, ds, (3, size, size), max_batch=2 * n, precision=b.BF16, bn_groups=2)
    push_params(G, bG); push_params(D, bD)
    gan = b.Gan(bG, bD, use_cuda_graph=graph)
    losses = [gan.step(*data) for _ in range(steps)]
    out = (np.array(losses), bG.params(), bD.params(), bD.updater_state())
    gan.close(); bG.close(); bD.close()
    return out


@pytest.mark.parametrize("pool", ["sum", "avg"])
def test_bf16_gan_step_with_global_pooling_head_is_reproducible(b200, pool):
    """Graph replay equals eager execution and two fresh nets equal each other, bit for bit (the split global-pooling reduction folds in a fixed
    order); the losses stay finite and near the FP32 oracle's first step."""
    b, ctx = b200
    size, z, nf, n = 32, 16, 32, 16
    gs = m.dcgan_generator(size, z, nf, 3, lr=2e-4)
    ds = m.dcgan_discriminator(size, nf, 3, lr=2e-4, global_pooling=pool)
    data = [a.astype(np.float32) for a in o.synthetic_batch(n, size, 3, z, seed=3)]
    G, D = oracle_gan_pair(gs, ds, size, z)
    runs = [_gan_run(b, ctx, gs, ds, G, D, data, n, size, z, graph) for graph in (True, False, True)]
    for a, c in ((runs[0], runs[1]), (runs[0], runs[2])):
        for u, v in zip(a, c):
            assert np.array_equal(u, v), pool
    assert np.isfinite(runs[0][0]).all()
    r = o.gan_step(G, D, *[v.astype(np.float64) for v in data])
    want = np.array([r["loss_d_real"], r["loss_d_fake"], r["loss_g"]])
    assert np.all(np.abs(runs[0][0][0] - want) < 0.1 * np.maximum(1, np.abs(want))), (runs[0][0][0], want)


def test_fp32_gan_step_with_global_pooling_head_matches_oracle(b200):
    b, ctx = b200
    n, lr_ = 8, 2e-3
    gs = m.dcgan_generator(16, 12, 8, 3, lr=lr_)
    ds = m.dcgan_discriminator(16, 8, 3, lr=lr_, global_pooling="sum")
    G, D, bG, bD, data = fp32_gan_pair(b, ctx, gs, ds, n)
    gan = b.Gan(bG, bD, use_cuda_graph=True)
    for it in range(3):
        r = o.gan_step(G, D, *data)
        lo = gan.step(*data)
        want = np.array([r["loss_d_real"], r["loss_d_fake"], r["loss_g"]])
        assert np.all(np.abs(lo - want) < TOL * np.maximum(1, np.abs(want))), (it, lo, want)
        assert pclose(bD.params(), D.params_flat(), 2 * lr_), (it, "D", rel_err(bD.params(), D.params_flat()))
        assert pclose(bG.params(), G.params_flat(), 2 * lr_), (it, "G", rel_err(bG.params(), G.params_flat()))
    gan.close(); bG.close(); bD.close()


# ------------------------------------------------------------------ launches per pass ----------------------------------------------------
def _fit_launches(b, ctx, specs, shape, mb=4):
    net = b.Net(ctx, specs, shape, max_batch=mb, precision=b.FP32)
    rng = np.random.default_rng(0)
    x, y = rng.uniform(-1, 1, (mb,) + shape), rng.uniform(-1, 1, (mb, 3))
    net.fit(x, y)
    ctx.sync(); l0 = ctx.launch_count()
    net.fit(x, y)
    ctx.sync(); l1 = ctx.launch_count()
    net.output(x); ctx.sync(); l2 = ctx.launch_count()
    net.close()
    return l1 - l0, l2 - l1


def test_launches_per_pass(b200):
    """One forward launch per pooling layer, and one backward launch where a trainable layer sits below it: a first-layer pooling layer against
    the same net fed the pooled features directly, and a global / subsampling layer in the middle against MAXPOOL of the same geometry (one
    launch each way)."""
    b, ctx = b200
    head = lambda: [{"type": "dense", "name": "d", "n_out": 5, "activation": "tanh", "updater": m.sgd(0.1)},
                    {"type": "output", "name": "o", "n_out": 3, "loss": "mse", "updater": m.sgd(0.1)}]
    conv = lambda frozen=False: {"type": "conv2d", "name": "c", "n_out": 8, "kernel": (3, 3), "padding": (1, 1), "activation": "tanh", "updater": m.sgd(0.1),
                                 "frozen": frozen}
    for pool in ("max", "avg", "sum", "pnorm"):
        g = dict(m.global_pooling(pool), name="g")
        fit_a, out_a = _fit_launches(b, ctx, [g] + head(), (8, 4, 4))
        fit_b, out_b = _fit_launches(b, ctx, head(), (8,))
        assert (fit_a, out_a) == (fit_b + 1, out_b + 1), (pool, fit_a, fit_b)            # forward only: nothing trainable below
        whole = {"type": "maxpool", "name": "g", "kernel": (4, 4), "stride": (1, 1)}
        for frozen, extra in ((False, 0), (True, 0)):
            fa = _fit_launches(b, ctx, [conv(frozen), g] + head(), (3, 4, 4))
            fb = _fit_launches(b, ctx, [conv(frozen), whole, {"type": "cnn_to_ff", "name": "ff"}] + head(), (3, 4, 4))
            assert fa == fb, (pool, frozen, fa, fb)
    for pool in ("avg", "sum", "pnorm"):
        s = dict(m.subsampling(pool, (2, 2), (2, 2), pnorm=2 if pool == "pnorm" else None), name="s")
        mp = {"type": "maxpool", "name": "s", "kernel": (2, 2), "stride": (2, 2)}
        tail = [{"type": "cnn_to_ff", "name": "ff"}] + head()
        for frozen in (False, True):
            assert _fit_launches(b, ctx, [conv(frozen), s] + tail, (3, 6, 6)) == _fit_launches(b, ctx, [conv(frozen), mp] + tail, (3, 6, 6)), (pool, frozen)
        fit_a, _ = _fit_launches(b, ctx, [s] + tail, (3, 6, 6))
        fit_b, _ = _fit_launches(b, ctx, [mp] + tail, (3, 6, 6))
        assert fit_a == fit_b, pool


# ------------------------------------------------------------------ argument checks -------------------------------------------------------
def test_rejections(b200):
    b, ctx = b200
    from gan_deeplearning4j_b200 import engine, _lib

    def create(spec_list, mutate=None, shape=(4, 6, 6)):
        descs = [engine.layer_desc(s) for s in spec_list]
        if mutate:
            mutate(descs)
        arr = (_lib.LayerDesc * len(descs))(*descs)
        cfg = _lib.NetConfig(shape[1], shape[2], shape[0], 4, b.FP32, 0.0, 1e-5, 1, 666)
        h = C.c_void_p()
        rc = ctx.lib.b2g_net_create(ctx.h, C.byref(cfg), arr, len(descs), C.byref(h))
        if rc == 0:
            ctx.lib.b2g_net_destroy(h)
        return rc

    sub = [dict(m.subsampling("pnorm", (3, 3), (2, 2), (1, 1), pnorm=3), name="s"), {"type": "cnn_to_ff", "name": "f"},
           {"type": "output", "name": "o", "n_out": 2, "loss": "mse"}]
    glb = [dict(m.global_pooling("pnorm", 2), name="g"), {"type": "output", "name": "o", "n_out": 2, "loss": "mse"}]
    assert create(sub) == 0 and create(glb) == 0

    def setf(field, v):
        def mut(d): setattr(d[0], field, v)
        return mut
    for bad in (0, 4, -1):                                   # MAX on SUBSAMPLING, unknown kinds
        assert create(sub, setf("act", bad)) == -1, bad
    for bad in (4, -1):
        assert create(glb, setf("act", bad)) == -1, bad
    for bad in (0.0, 0.5, 2.5, -3.0, float("nan"), float("inf")):     # p not a whole number >= 1
        assert create(sub, setf("act_alpha", bad)) == -1, bad
        assert create(glb, setf("act_alpha", bad)) == -1, bad
    for field, bad in (("k_h", 0), ("s_w", 0), ("p_h", -1), ("p_w", 3), ("p_h", 3)):   # kernel / stride < 1, padding < 0 or >= kernel
        assert create(sub, setf(field, bad)) == -2, (field, bad)
    assert create(sub, setf("k_h", 9)) == -2                # empty output: 6 + 2 < 9
    with pytest.raises(b.B200GanError):
        b.test_pool(ctx, b.FP32, "pool2d", np.zeros(16, np.float32), np.zeros(4, np.float32), (4, 16, 0), pooling="max", N=1, H=4, W=4, C=1, KH=2, KW=2,
                  SH=2, SW=2)
    with pytest.raises(b.B200GanError):
        b.test_pool(ctx, b.FP32, "global_pool", np.zeros(16, np.float32), np.zeros(1, np.float32), (1, 16, 0), pooling="pnorm", pnorm=1.5, N=1, H=4, W=4, C=1)
