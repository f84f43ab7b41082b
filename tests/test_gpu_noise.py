"""GaussianDropout, GaussianNoise, AlphaDropout and SpatialDropout on the GPU: the kernels against the restatement's draws (Bernoulli kinds
exactly, Gaussian noise within 8 fp32 ulps) and the stated fp32 formulas on the device's own draws bit for bit; FP32 nets against the oracle
under identical draws; the identity cases; BF16 nets against the same nets without the layers; the CUDA-graph GAN step with instance noise;
checkpoint resume."""
from fractions import Fraction

import numpy as np
import pytest

from gan_deeplearning4j_b200 import models as m
from helpers import b200, bf16_round, push_params, randomize, rel_err
from oracle import dl4j_oracle as o

pytestmark = pytest.mark.gpu
TOL = 1e-3
SEED, LAYER, RANK, PASS = 1234567890123, 5, 3, (1 << 32) + 17
NS = [1, 7, 8, 4097, (1 << 20) + 3]


def _f32_nearest(F: Fraction) -> np.float32:
    """The fp32 nearest the exact value F, ties to even."""
    f = np.float32(float(F))
    cands = [np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))]
    best = min(cands, key=lambda c: (abs(Fraction(float(c)) - F), int(np.float32(c).view(np.uint32)) & 1))
    return np.float32(best)


def fma32(a, b, c):
    """fmaf(a, b, c) elementwise on fp32 arrays: one rounding of the exact a*b + c.  a*b is exact in float64; TwoSum gives the float64 sum
    and its error, and only a sum that is inexact and lands on an fp32 rounding midpoint (where rounding twice can differ from once) is
    redone exactly."""
    a, b, c = (np.broadcast_to(np.asarray(v, np.float32), np.broadcast(a, b, c).shape).astype(np.float64).ravel() for v in (a, b, c))
    p = a * b
    s = p + c
    bv = s - p
    err = (p - (s - bv)) + (c - bv)
    out = s.astype(np.float32)
    d = np.abs(s - out.astype(np.float64))
    sp = np.spacing(np.abs(out)).astype(np.float64)
    for i in np.flatnonzero((err != 0) & ((2 * d == sp) | (4 * d == sp))):
        out[i] = _f32_nearest(Fraction(p[i]) + Fraction(c[i]))
    return out


def _hook(b, ctx, P, kind, x, dy, v, **kw):
    return b.test_dropout_kind(ctx, P, kind, x, dy, v, **dict(dict(seed=SEED, layer=LAYER, rank=RANK, pass_=PASS), **kw))


def _inputs(n, shape=None):
    rng = np.random.default_rng(n)
    shape = shape or (1, 1, 1, n)
    x = (rng.uniform(0.5, 2.0, n) * rng.choice([-1.0, 1.0], n)).astype(np.float32).reshape(shape)      # no zeros: dx == 0 <=> dropped
    dy = (rng.uniform(0.5, 2.0, n) * rng.choice([-1.0, 1.0], n)).astype(np.float32).reshape(shape)
    return x, dy


@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("kind,sigma", [("gaussian_noise", 0.3), ("gaussian_dropout", 0.5)])
def test_gaussian_kernels(b200, kind, sigma, prec, n):
    b, ctx = b200
    P = b.BF16 if prec == "bf16" else b.FP32
    rnd = bf16_round if prec == "bf16" else (lambda a: np.asarray(a, np.float32))
    x, dy = _inputs(n)
    z64 = o.dropout_normals(SEED, RANK, LAYER, PASS, 1, 1, 1, n).ravel()
    if kind == "gaussian_noise":
        z_dev, _ = _hook(b, ctx, b.FP32, kind, np.zeros_like(x), dy, 1.0)      # fmaf(1, z, 0) = z: the device's own draws
        noise, _ = _hook(b, ctx, b.FP32, kind, np.zeros_like(x), dy, sigma)    # read through x = 0
        s = np.float32(sigma)
        ref = s * z64
    else:
        noise, _ = _hook(b, ctx, b.FP32, kind, np.ones_like(x), dy, sigma)     # y = 1 * m: read through x = 1
        s = o.gaussian_sigma(sigma)
        ref = 1 + np.float64(s) * z64
    noise = noise.ravel()
    tol = 8 * np.spacing(np.maximum(1, np.abs(z64)).astype(np.float32) * s).astype(np.float64)
    assert np.all(np.abs(noise - ref) <= tol), np.max(np.abs(noise - ref) / tol)
    y, dx = _hook(b, ctx, P, kind, x, dy, sigma)
    y2, dx2 = _hook(b, ctx, P, kind, x, dy, sigma)
    assert np.array_equal(y, y2) and np.array_equal(dx, dx2)          # the same pass draws the same noise
    xs, es = rnd(x).ravel(), rnd(dy).ravel()
    if kind == "gaussian_noise":
        assert np.array_equal(y.ravel(), rnd(fma32(s, z_dev.ravel(), xs)))
        assert np.array_equal(dx.ravel(), es)                              # the identity
    else:
        m_dev = noise.astype(np.float32)
        assert np.array_equal(y.ravel(), rnd(xs * m_dev)) and np.array_equal(dx.ravel(), rnd(es * m_dev))
    if n > 4096:
        zz = (noise - (0 if kind == "gaussian_noise" else 1)) / s
        assert abs(zz.mean()) < 5 / np.sqrt(n) and abs(zz.var() - 1) < 5 * np.sqrt(2 / n)
    y3, _ = _hook(b, ctx, P, kind, x, dy, sigma, pass_=PASS + 1)
    assert not np.array_equal(y, y3)


def _check_alpha(y, dx, x, dy, keep, p, rnd):
    a, bb, ap = o.alpha_coefficients(p)
    xs, es = rnd(x).ravel(), rnd(dy).ravel()
    assert np.array_equal(dx.ravel() != 0, keep)
    assert np.array_equal(dx.ravel(), np.where(keep, rnd(es * a), 0).astype(np.float32))
    ref = fma32(a, np.where(keep, xs, ap).astype(np.float32), bb)
    lo, hi = np.nextafter(ref, np.float32(-np.inf)), np.nextafter(ref, np.float32(np.inf))
    got = y.ravel()
    assert np.all((got == rnd(ref)) | (got == rnd(lo)) | (got == rnd(hi)))    # within 1 ulp of the fma, then the activation's rounding


@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("kind,p", [("alpha_dropout", 0.5), ("alpha_dropout", 0.9), ("spatial_dropout", 0.5)])
def test_bernoulli_kernels(b200, kind, p, prec, n):
    b, ctx = b200
    P = b.BF16 if prec == "bf16" else b.FP32
    rnd = bf16_round if prec == "bf16" else (lambda a: np.asarray(a, np.float32))
    x, dy = _inputs(n)
    y, dx = _hook(b, ctx, P, kind, x, dy, p)
    if kind == "alpha_dropout":
        keep = o.dropout_mask(SEED, RANK, LAYER, PASS, 1, 1, 1, n, p).ravel()
        _check_alpha(y, dx, x, dy, keep, p, rnd)
    else:
        keep = o.spatial_mask(SEED, RANK, LAYER, PASS, 1, n, p).ravel()         # one row of n channels: j = c
        s = np.float32(1) / np.float32(p)
        assert np.array_equal(y.ravel(), np.where(keep, rnd(rnd(x).ravel() * s), 0).astype(np.float32))
        assert np.array_equal(dx.ravel(), np.where(keep, rnd(rnd(dy).ravel() * s), 0).astype(np.float32))
    if n > 4096:
        assert abs(keep.mean() - p) < 5 * np.sqrt(p * (1 - p) / n)


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("C", [1, 3, 64])
def test_spatial_kernels_on_odd_maps(b200, C, prec):
    b, ctx = b200
    P = b.BF16 if prec == "bf16" else b.FP32
    rnd = bf16_round if prec == "bf16" else (lambda a: np.asarray(a, np.float32))
    rows, h, w, p = 37, 5, 3, 0.6
    x, dy = _inputs(rows * h * w * C, (rows, h, w, C))
    y, dx = _hook(b, ctx, P, "spatial_dropout", x, dy, p)
    keep = o.spatial_mask(SEED, RANK, LAYER, PASS, rows, C, p)[:, None, None, :]
    s = np.float32(1) / np.float32(p)
    assert np.array_equal(y, np.where(keep, rnd(rnd(x) * s), 0).astype(np.float32))
    assert np.array_equal(dx, np.where(keep, rnd(rnd(dy) * s), 0).astype(np.float32))
    assert 0 < keep.sum() < keep.size


def test_hook_identity_and_bad_arguments(b200):
    b, ctx = b200
    x, dy = _inputs(64)
    for kind, v in (("gaussian_noise", 0.0), ("gaussian_dropout", 0.0), ("alpha_dropout", 1.0), ("spatial_dropout", 1.0)):
        l0 = ctx.launch_count()
        y, dx = _hook(b, ctx, b.FP32, kind, x, dy, v)
        assert ctx.launch_count() == l0 and np.array_equal(y, x) and np.array_equal(dx, dy)
    for kind, bad in (("gaussian_noise", [-0.1, float("inf"), float("nan")]), ("gaussian_dropout", [-0.1, 1.0]),
                      ("alpha_dropout", [0.0, 1.5]), ("spatial_dropout", [0.0, 1.5])):
        for v in bad:
            with pytest.raises(b.B200GanError) as e:
                _hook(b, ctx, b.FP32, kind, x, dy, v)
            assert e.value.code == -1
            with pytest.raises(b.B200GanError) as e:
                b.Net(ctx, [{"type": "conv2d", "n_out": 4, "kernel": (1, 1)}, {"type": "dropout", "kind": kind, o.VALUE_KEY[kind]: v},
                            {"type": "cnn_to_ff"}, {"type": "output", "n_out": 1}], (3, 4, 4), max_batch=2)
            assert e.value.code == -1
    with pytest.raises(b.B200GanError) as e:          # SpatialDropout on a feed-forward input
        b.Net(ctx, [{"type": "dense", "n_out": 4}, m.spatial_dropout(0.5), {"type": "output", "n_out": 1}], (4,), max_batch=2)
    assert e.value.code == -2


def _chain_specs(kind, value, frozen=False):
    u = m.adam(1e-2)
    noise = lambda name, where: ([] if kind is None or (kind == "spatial_dropout" and where == "ff") else
                                 [{"type": "dropout", "name": name, "kind": kind, o.VALUE_KEY[kind]: value, "frozen": frozen}])
    return (noise("n0", "map") +
            [{"type": "conv2d", "name": "c1", "n_out": 8, "kernel": (3, 3), "stride": (2, 2), "padding": (1, 1), "updater": u},
             {"type": "activation", "name": "a1", "activation": "lrelu", "alpha": 0.2}] + noise("n1", "map") +
            [{"type": "conv2d", "name": "c2", "n_out": 12, "kernel": (3, 3), "stride": (1, 1), "padding": (1, 1), "has_bias": False, "updater": u},
             {"type": "batchnorm", "name": "bn2", "updater": u}, {"type": "activation", "name": "a2", "activation": "tanh"}] + noise("n2", "map") +
            [{"type": "cnn_to_ff", "name": "flat"},
             {"type": "dense", "name": "fc", "n_out": 10, "activation": "tanh", "updater": u}] + noise("n3", "ff") +
            [{"type": "output", "name": "out", "n_out": 1, "updater": u}])


KIND_VALUES = [("gaussian_noise", 0.2), ("gaussian_dropout", 0.3), ("alpha_dropout", 0.7), ("spatial_dropout", 0.6)]


@pytest.mark.parametrize("kind,value", KIND_VALUES)
def test_fp32_chain_matches_oracle_under_identical_draws(b200, kind, value):
    """A DropoutLayer of the kind on the net input and after each hidden activation: activations, zero patterns, score and gradients
    over two passes."""
    b, ctx = b200
    specs = _chain_specs(kind, value)
    rng = np.random.default_rng(3)
    onet = o.net_from_specs(specs, (3, 8, 8), mask_seed=41, seed=2); randomize(onet, rng)
    bnet = b.Net(ctx, specs, (3, 8, 8), max_batch=6, precision=b.FP32, seed=41)
    push_params(onet, bnet)
    x = rng.uniform(-1, 1, (6, 3, 8, 8)); y = rng.uniform(0, 1, (6, 1))
    for step in range(2):
        score_o, acts, _, _ = onet.compute_gradient_and_score(x, y, collect=True)
        score_b = bnet.compute_gradient_and_score(x, y)
        assert bnet.dropout_pass() == onet.dropout.pass_ == step + 1
        assert abs(score_b - score_o) < TOL * abs(score_o)
        for li, s in enumerate(specs):
            if s["type"] == "output" or (s["type"] == "batchnorm" and specs[li + 1]["type"] == "activation"):
                continue
            got, want = bnet.activation(li, 6), acts[li + 1].reshape(6, -1)
            assert rel_err(got, want) < TOL, (step, li, s["name"])
            if s["type"] == "dropout" and kind == "spatial_dropout":
                assert np.array_equal(got == 0, want == 0), (step, s["name"])
                assert 0 < (got == 0).mean() < 1
        g_b, g_o = bnet.gradients(), onet.grads_flat(); off = 0
        for li, name, pn, shape, _ in onet.param_table():
            k = int(np.prod(shape))
            assert rel_err(g_b[off:off + k], g_o[off:off + k]) < TOL, (step, name, pn)
            off += k
    bnet.close()


def test_identity_cases_launch_nothing_and_match_the_plain_net(b200):
    b, ctx = b200
    rng = np.random.default_rng(4)
    plain = _chain_specs(None, 0)
    variants = [_chain_specs(k, v) for k, v in (("gaussian_noise", 0.0), ("gaussian_dropout", 0.0), ("alpha_dropout", 1.0), ("spatial_dropout", 1.0))]
    variants += [_chain_specs(k, v, frozen=True) for k, v in KIND_VALUES]
    onet = o.net_from_specs(plain, (3, 8, 8), seed=2); randomize(onet, rng)
    x = rng.uniform(-1, 1, (6, 3, 8, 8)); y = rng.uniform(0, 1, (6, 1))
    base = b.Net(ctx, plain, (3, 8, 8), max_batch=6, precision=b.FP32); push_params(onet, base)
    l0 = ctx.launch_count(); out0 = base.output(x); la0 = ctx.launch_count() - l0
    s0 = base.compute_gradient_and_score(x, y); g0 = base.gradients()
    l0 = ctx.launch_count(); base.compute_gradient_and_score(x, y); lt0 = ctx.launch_count() - l0
    for specs in variants:
        n = b.Net(ctx, specs, (3, 8, 8), max_batch=6, precision=b.FP32); push_params(onet, n)
        l0 = ctx.launch_count(); out = n.output(x); la = ctx.launch_count() - l0
        assert np.array_equal(out, out0) and la == la0
        s = n.compute_gradient_and_score(x, y)
        assert s == s0 and np.array_equal(n.gradients(), g0)
        l0 = ctx.launch_count(); n.compute_gradient_and_score(x, y); assert ctx.launch_count() - l0 == lt0
        assert n.dropout_pass() == 0
        n.close()
    base.close()


def _bf16_grad_err(b, ctx, specs, in_shape, n, seed, rng_seed):
    rng = np.random.default_rng(rng_seed)
    onet = o.net_from_specs(specs, in_shape, mask_seed=seed, quirks=o.Quirks(xent_clip_eps=0.0), seed=2); randomize(onet, rng)
    bnet = b.Net(ctx, specs, in_shape, max_batch=n, precision=b.BF16, xent_clip_eps=0.0, seed=seed)
    push_params(onet, bnet)
    x = rng.uniform(-1, 1, (n,) + tuple(in_shape)); y = rng.uniform(0, 1, (n, 1))
    onet.compute_gradient_and_score(x, y); bnet.compute_gradient_and_score(x, y)
    g_b, g_o = bnet.gradients(), onet.grads_flat()
    bnet.close()
    return float(np.linalg.norm(g_b - g_o) / np.linalg.norm(g_o))


def _with_after_lrelu(specs, make):
    out = []
    for s in specs:
        out.append(s)
        if s.get("activation") == "lrelu":
            out.append(make(s["name"] + "_noise"))
    return out


def test_bf16_nets_with_noise_track_the_oracle(b200):
    """BF16 MLP D (tensor-core sizes) and 32x32 DCGAN D with instance noise, and each hidden kind after every LeakyReLU: the gradient error
    against the oracle under identical draws stays within 2x that of the same nets without the layers."""
    b, ctx = b200
    mlp, dc = m.mlp_discriminator(128, 256, lr=1e-3), m.dcgan_discriminator(32, 64, 3, lr=1e-3)
    cases = [("mlp", mlp, m.mlp_discriminator(128, 256, lr=1e-3, instance_noise=0.1), (128,), 256),
             ("mlp_gd", mlp, _with_after_lrelu(mlp, lambda nm: m.gaussian_dropout(0.5, nm)), (128,), 256),
             ("mlp_ad", mlp, _with_after_lrelu(mlp, lambda nm: m.alpha_dropout(0.9, nm)), (128,), 256),
             ("dcgan32", dc, m.dcgan_discriminator(32, 64, 3, lr=1e-3, instance_noise=0.1), (3, 32, 32), 8),
             ("dcgan32_sd", dc, _with_after_lrelu(dc, lambda nm: m.spatial_dropout(0.8, nm)), (3, 32, 32), 8)]
    for name, plain, noisy, shape, n in cases:
        e0 = _bf16_grad_err(b, ctx, plain, shape, n, 77, 6)
        e1 = _bf16_grad_err(b, ctx, noisy, shape, n, 77, 6)
        print(f"{name}: gradient error without the layers {e0:.3e}, with them {e1:.3e}")
        assert e1 <= 2 * e0, (name, e0, e1)


def _noisy_dcgan_d(size, nf, lr, instance_noise=0.2):
    """dcgan_discriminator with instance noise on the input and AlphaDropout, SpatialDropout and GaussianDropout after the hidden LeakyReLUs."""
    out, makers = [], [lambda nm: m.alpha_dropout(0.8, nm), lambda nm: m.spatial_dropout(0.7, nm), lambda nm: m.gaussian_dropout(0.3, nm)]
    for s in m.dcgan_discriminator(size, nf, 3, lr=lr, instance_noise=instance_noise):
        out.append(s)
        if s.get("activation") == "lrelu" and makers:
            out.append(makers.pop(0)(s["name"] + "_noise"))
    return out


def test_fp32_gan_step_with_instance_noise_graph_eager_and_oracle(b200):
    b, ctx = b200
    n, z, size = 8, 12, 16
    gs, ds = m.dcgan_generator(size, z, 8, 3, lr=2e-3), _noisy_dcgan_d(size, 8, 2e-3)
    kinds = sorted({s.get("kind") for s in ds if s["type"] == "dropout"})
    assert len([s for s in ds if s["type"] == "dropout"]) >= 3 and "gaussian_noise" in kinds
    runs = []
    for graph in (False, True):
        rng = np.random.default_rng(5)
        G = o.net_from_specs(gs, (z,), seed=1)
        D = o.net_from_specs(ds, (3, size, size), seed=2, mask_seed=667)
        randomize(G, rng); randomize(D, rng)
        bG = b.Net(ctx, gs, (z,), max_batch=n, precision=b.FP32)
        bD = b.Net(ctx, ds, (3, size, size), max_batch=2 * n, bn_groups=2, precision=b.FP32, seed=667)
        push_params(G, bG); push_params(D, bD)
        data = [a.astype(np.float64) for a in o.synthetic_batch(n, size, 3, z, seed=3)]
        gan = b.Gan(bG, bD, use_cuda_graph=graph)
        acts, losses = [], []
        for it in range(3):
            r = o.gan_step(G, D, *data)
            lo = gan.step(*data); losses.append(lo)
            want = np.array([r["loss_d_real"], r["loss_d_fake"], r["loss_g"]])
            assert np.all(np.abs(lo - want) < TOL * np.maximum(1, np.abs(want))), (graph, it, lo, want)
            for onet, bnet, tag in ((D, bD, "D"), (G, bG, "G")):
                p_b, p_o = bnet.params(), onet.params_flat(); off = 0
                for li, name, pn, shape, _ in onet.param_table():
                    k = int(np.prod(shape))
                    assert rel_err(p_b[off:off + k], p_o[off:off + k]) < 2 * TOL, (graph, it, tag, name, pn)
                    off += k
            assert bD.dropout_pass() == D.dropout.pass_ == 2 * (it + 1)
            acts.append(bD.activation(0, n))          # the instance noise of the generator step's D pass
        assert not np.array_equal(acts[0], acts[1]) and not np.array_equal(acts[1], acts[2])      # new noise on every step and replay
        runs.append((np.array(losses), bG.params(), bD.params()))
        gan.close(); bG.close(); bD.close()
    assert np.array_equal(runs[0][0], runs[1][0]) and np.array_equal(runs[0][1], runs[1][1]) and np.array_equal(runs[0][2], runs[1][2])


def test_checkpoint_resume_with_kinds(b200, tmp_path):
    b, ctx = b200
    specs = _chain_specs("gaussian_dropout", 0.3)
    specs = specs[:1] + [m.alpha_dropout(0.8, "ad"), m.spatial_dropout(0.7, "sd")] + specs[1:]
    rng = np.random.default_rng(5)
    x = rng.uniform(-1, 1, (6, 3, 8, 8)).astype(np.float32); y = rng.uniform(0, 1, (6, 1)).astype(np.float32)
    for prec in (b.FP32, b.BF16):
        u = b.Net(ctx, specs, (3, 8, 8), max_batch=6, precision=prec, seed=8)
        c = b.Net(ctx, specs, (3, 8, 8), max_batch=6, precision=prec, seed=8)
        c.set_params(u.params())
        for _ in range(5):
            u.fit(x, y)
        for _ in range(3):
            c.fit(x, y)
        path = str(tmp_path / f"ck{prec}.zip"); c.save(path)
        r = b.Net(ctx, specs, (3, 8, 8), max_batch=6, precision=prec, seed=8)
        meta = r.restore(path)
        assert meta["meta"]["dropout_pass"] == 3 and r.dropout_pass() == 3
        for _ in range(2):
            r.fit(x, y)
        assert np.array_equal(r.params(), u.params()) and r.dropout_pass() == u.dropout_pass() == 5
        for n in (u, c, r):
            n.close()


def test_scheduled_instance_noise_gan_step(b200):
    """A 16x16 FP32 DCGAN whose D has an Exponential-scheduled GaussianNoise on its input and Alpha / Spatial / GaussianDropout on hidden
    layers, three iterations against the oracle's step: eager and CUDA graph bit for bit, new noise every replay, dropout_value following the
    oracle each iteration without a re-capture; then an EPOCH schedule following set_epoch in a replay."""
    b, ctx = b200
    n, z, size = 8, 12, 16
    gs, ds = m.dcgan_generator(size, z, 8, 3, lr=2e-3), _noisy_dcgan_d(size, 8, 2e-3, instance_noise=m.exponential_schedule(0.3, 0.5))
    runs = []
    for graph in (False, True):
        rng = np.random.default_rng(5)
        G = o.net_from_specs(gs, (z,), seed=1)
        D = o.net_from_specs(ds, (3, size, size), seed=2, mask_seed=667)
        randomize(G, rng); randomize(D, rng)
        bG = b.Net(ctx, gs, (z,), max_batch=n, precision=b.FP32)
        bD = b.Net(ctx, ds, (3, size, size), max_batch=2 * n, bn_groups=2, precision=b.FP32, seed=667)
        push_params(G, bG); push_params(D, bD)
        data = [a.astype(np.float64) for a in o.synthetic_batch(n, size, 3, z, seed=3)]
        gan = b.Gan(bG, bD, use_cuda_graph=graph)

        def step(it, what):
            assert bD.dropout_value("dis_instance_noise") == D.dropout_value("dis_instance_noise"), (graph, what, it)
            r = o.gan_step(G, D, *data)
            lo = gan.step(*data)
            want = np.array([r["loss_d_real"], r["loss_d_fake"], r["loss_g"]])
            assert np.all(np.abs(lo - want) < TOL * np.maximum(1, np.abs(want))), (graph, what, it, lo, want)
            for onet, bnet, tag in ((D, bD, "D"), (G, bG, "G")):
                assert rel_err(bnet.params(), onet.params_flat()) < 2 * TOL, (graph, what, it, tag)
            return lo

        losses, acts = [], []
        for it in range(3):
            losses.append(step(it, "iteration"))
            acts.append(bD.activation(0, n))
        assert bD.dropout_value("dis_instance_noise") == np.float32(0.3 * 0.5 ** 3)
        assert not np.array_equal(acts[0], acts[1]) and not np.array_equal(acts[1], acts[2])
        # EPOCH schedule: set once (a re-capture), then set_epoch on both nets moves the value inside the replays
        sched = m.step_schedule(0.25, 0.5, 1, type="epoch")
        bD.set_dropout_schedule(sched, "dis_instance_noise"); D.set_dropout_schedule(sched, "dis_instance_noise")
        assert bD.specs[0]["stddev"] == sched
        for ep in (0, 2):
            for net in (bD, bG, D, G):
                net.set_epoch(ep)
            assert bD.dropout_value("dis_instance_noise") == np.float32(0.25 * 0.5 ** ep)
            losses.append(step(ep, "epoch"))
        bD.set_dropout_schedule(None, "dis_instance_noise")
        assert bD.dropout_value("dis_instance_noise") == np.float32(0.3) and bD.specs[0]["stddev"] == 0.3
        runs.append((np.array(losses), bG.params(), bD.params()))
        gan.close(); bG.close(); bD.close()
    assert np.array_equal(runs[0][0], runs[1][0]) and np.array_equal(runs[0][1], runs[1][1]) and np.array_equal(runs[0][2], runs[1][2])


def test_scheduled_dropout_kinds_match_the_oracle(b200):
    """Dropout(p) and each other kind with a schedule (the scheduled kernels, Dropout's included) in an FP32 chain: two fits against the
    oracle's, with a value clamped (a rate schedule going below 0: sigma 0, still drawn)."""
    b, ctx = b200
    for kind, sched in (("dropout", m.exponential_schedule(0.7, 0.9)), ("gaussian_dropout", m.map_schedule({0: 0.3, 1: -0.5})),
                        ("alpha_dropout", m.exponential_schedule(0.8, 0.9)), ("spatial_dropout", m.exponential_schedule(0.6, 1.1)),
                        ("gaussian_noise", m.exponential_schedule(0.2, 0.5))):
        specs = _chain_specs(kind, 0.5)
        for sp in specs:
            if sp["type"] == "dropout":
                sp[o.VALUE_KEY[kind]] = sched
        rng = np.random.default_rng(3)
        onet = o.net_from_specs(specs, (3, 8, 8), mask_seed=41, seed=2); randomize(onet, rng)
        bnet = b.Net(ctx, specs, (3, 8, 8), max_batch=6, precision=b.FP32, seed=41)
        push_params(onet, bnet)
        x = rng.uniform(-1, 1, (6, 3, 8, 8)); y = rng.uniform(0, 1, (6, 1))
        for it in range(2):
            assert bnet.dropout_value("n1") == onet.dropout_value("n1"), (kind, it)
            so, sb = onet.fit(x, y), bnet.fit(x, y)
            assert abs(sb - so) < TOL * max(1, abs(so)), (kind, it, sb, so)
            assert rel_err(bnet.params(), onet.params_flat()) < 2 * TOL, (kind, it)
        assert bnet.dropout_pass() == onet.dropout.pass_ == 2
        bnet.close()


def test_two_ranks_share_parameters_but_not_noise(tmp_path):
    from helpers import run_two_ranks
    d = run_two_ranks("dp_check.py", tmp_path / "noise_dp.json", 29548, args=("noise",))
    assert d["world"] == 2 and d["d_params_identical"] is True and d["noise_differs"] is True
    assert d["scheduled_value"] == np.float32(0.2 * 0.9 ** 3)
