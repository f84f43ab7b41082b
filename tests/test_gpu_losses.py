"""DL4J's MSE, L1, L2, MAE, Hinge, SquaredHinge and Wasserstein losses on the GPU: the loss kernel through its production wrapper (b2g_test_ew op
"loss") for every loss x activation x precision against float64, FP32 fit and output of an MLP OutputLayer(MSE, nOut = 7) and a conv net ending
in LossLayer(HINGE) against the oracle's score_and_grad, the FP32 GAN step (least-squares, hinge, Wasserstein) against the oracle's gan_step, BF16 graph
replay against eager with the XENT discriminator's launch counts, the argument checks and checkpoint / resume."""
import numpy as np
import pytest

from gan_deeplearning4j_b200 import models as m
from helpers import b200, bf16_gan, bf16_round, fp32_gan_pair, launches_per_step, pclose, push_params, randomize, rel_err
from oracle import dl4j_oracle as o

pytestmark = pytest.mark.gpu
TOL = 1e-3
U = 2.0 ** -24            # fp32 unit roundoff
ACTS = o.ACTS


# ------------------------------------------------------------------ the kernel against float64 ------------------------------------------
SHAPES = [(1, 1, 1, 0), (127, 3, 2, 1), (127, 256, 1, 3), (8192, 1, 2, 0), (8192, 256, 1, 5), (8192, 3, 2, 2)]   # rows, nOut, groups, offset


def _dlda_and_sens(loss, act, a, y, n_out, alpha):
    """float64 dL/da (with the / nOut), and |d(dL/dz)/da| = |g' h| + |g h'| (h = act'(a)): how far dz moves per unit error in a."""
    e, m = a - y, 1 - y * a
    per = 1.0 / n_out if o.per_output(loss) else 1.0
    if loss in ("mse", "l2"):
        g, gp = 2 * e * per, np.full_like(a, 2 * per)
    elif loss in ("l1", "mae"):
        g, gp = np.sign(e) * per, np.zeros_like(a)
    elif loss == "hinge":
        g, gp = np.where(m > 0, -y, 0.0), np.zeros_like(a)
    elif loss == "squared_hinge":
        g, gp = -2 * y * np.maximum(m, 0), np.where(m > 0, 2 * y * y, 0.0)
    else:
        g, gp = y * per, np.zeros_like(a)
    h = o.act_grad_from_out(act, a, alpha)
    hp = {"tanh": -2 * a, "sigmoid": 1 - 2 * a}.get(act, np.zeros_like(a))
    return g, np.abs(gp * h) + np.abs(g * hp)


def _near_kink(loss, a, y):
    """Elements within 1e-3 of a kink of L1 / MAE (a = y) or the hinges (1 - y a = 0), where fp32 and float64 may take different sides."""
    if loss in ("l1", "mae"):
        return np.abs(a - y) < 1e-3
    if loss in ("hinge", "squared_hinge"):
        return np.abs(1 - y * a) < 1e-3
    return np.zeros(a.shape, bool)


def _labels(loss, rng, shape):
    return rng.choice([-1.0, 1.0], shape) if loss in ("hinge", "squared_hinge") else rng.uniform(-1.5, 1.5, shape)


def _run(b, ctx, prec, loss, act, z, y, rows, n_out, groups, offset, alpha=0.2, poison=True):
    (dz, sums, _), info = b.test_ew(ctx, prec, "loss", z, y, (z.size, groups, 0), act=act, loss=loss, rows=rows, cols=n_out, groups=groups,
                                    alpha=alpha, offset=offset, poison=poison)
    return dz, sums, info["kernel"]


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("loss", o.LOSSES)
def test_loss_kernel_against_float64(b200, loss, act, prec):
    """dz within one bf16 ulp (bf16) or 8u (|dz| + sens (|a| + 1)) (fp32, sens = |d dz / da|: a = act(z) carries a few ulp of tanhf / expf and
    each later operation one rounding); loss sums within 2u|S| + 8u sum |dL/da| (|a| + 1); no poisoned element survives."""
    b, ctx = b200
    P = b.BF16 if prec == "bf16" else b.FP32
    rng = np.random.default_rng(o.LOSS_CODES[loss] * 100 + ACTS.index(act) * 10 + P)
    for rows, n_out, groups, offset in SHAPES:
        shape = (groups * rows, n_out)
        z = rng.uniform(-3, 3, shape).astype(np.float32); y = _labels(loss, rng, shape).astype(np.float32)
        dz, sums, kernel = _run(b, ctx, P, loss, act, z, y, rows, n_out, groups, offset)
        assert kernel == "loss_kernel"
        assert np.isfinite(dz).all() and np.isfinite(sums).all(), "poisoned output survived"
        zd = (bf16_round(z) if P == b.BF16 else z).astype(np.float64)
        a = o.act_forward(act, zd, 0.2)
        y64 = y.astype(np.float64)
        g, sens = _dlda_and_sens(loss, act, a, y64, n_out, 0.2)
        ref = g * o.act_grad_from_out(act, a, 0.2)
        ok = ~_near_kink(loss, a, y64)
        d = np.abs(dz.reshape(shape) - ref)
        if P == b.BF16:
            ulp = 2.0 ** (np.floor(np.log2(np.maximum(np.abs(ref), 2.0 ** -126))) - 7)
            tol = ulp + 8 * U * (np.abs(ref) + sens * (np.abs(a) + 1))
        else:
            tol = 8 * U * (np.abs(ref) + sens * (np.abs(a) + 1))
        bad = ok & ~(d <= tol)
        assert not bad.any(), (loss, act, prec, rows, n_out, groups, int(bad.sum()), float(d[bad].max()))
        for gi in range(groups):
            sl = slice(gi * rows, (gi + 1) * rows)
            s_ref, _ = o.score_and_grad(loss, act, 0.2, zd[sl], y64[sl])
            bound = 2 * U * abs(s_ref) + 8 * U * float((np.abs(g[sl]) * (np.abs(a[sl]) + 1)).sum()) + 1e-30
            assert abs(sums[gi] - s_ref) <= bound, (loss, act, prec, rows, n_out, groups, gi, sums[gi], s_ref, bound)


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("loss", o.LOSSES)
def test_small_integers_give_exact_sums(b200, loss, prec):
    """Small-integer z and y, identity: every score is an integer summed exactly in double, then divided by nOut once and rounded to fp32."""
    b, ctx = b200
    P = b.BF16 if prec == "bf16" else b.FP32
    rng = np.random.default_rng(o.LOSS_CODES[loss] + 50 * P)
    for rows, n_out, groups, offset in SHAPES:
        shape = (groups * rows, n_out)
        z = rng.integers(-4, 5, shape).astype(np.float32)
        y = (rng.choice([-1.0, 1.0], shape) if loss in ("hinge", "squared_hinge") else rng.integers(-4, 5, shape)).astype(np.float32)
        dz, sums, _ = _run(b, ctx, P, loss, "identity", z, y, rows, n_out, groups, offset)
        z64, y64 = z.astype(np.float64), y.astype(np.float64)
        for gi in range(groups):
            sl = slice(gi * rows, (gi + 1) * rows)
            e, m = z64[sl] - y64[sl], 1 - y64[sl] * z64[sl]
            raw = {"mse": (e * e).sum(), "l2": (e * e).sum(), "l1": np.abs(e).sum(), "mae": np.abs(e).sum(), "hinge": np.maximum(m, 0).sum(),
                   "squared_hinge": (np.maximum(m, 0) ** 2).sum(), "wasserstein": (y64[sl] * z64[sl]).sum()}[loss]
            want = np.float32(raw / n_out if o.per_output(loss) else raw)
            assert sums[gi] == want, (loss, prec, rows, n_out, groups, gi, sums[gi], want)
        if loss in ("l1", "mae", "hinge"):        # the kinks: a = y gives 0, a margin of exactly 0 gives 0
            _, ref = o.score_and_grad(loss, "identity", 0.0, z64, y64)
            assert np.array_equal(dz.reshape(shape), (bf16_round(ref) if P == b.BF16 else ref.astype(np.float32)))


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_multi_block_sums_are_bit_reproducible(b200, prec):
    b, ctx = b200
    P = b.BF16 if prec == "bf16" else b.FP32
    rng = np.random.default_rng(7)
    rows, n_out, groups = 8192, 256, 2
    z = rng.standard_normal((groups * rows, n_out)).astype(np.float32); y = rng.standard_normal(z.shape).astype(np.float32)
    for loss in ("mse", "wasserstein"):
        r1 = _run(b, ctx, P, loss, "tanh", z, y, rows, n_out, groups, 0)
        r2 = _run(b, ctx, P, loss, "tanh", z, y, rows, n_out, groups, 0)
        assert np.array_equal(r1[0].view(np.uint32), r2[0].view(np.uint32)) and np.array_equal(r1[1].view(np.uint32), r2[1].view(np.uint32))


# ------------------------------------------------------------------ FP32 fit and output against the oracle -------------------------------
def _mlp(act):
    return [{"type": "dense", "name": "d1", "n_out": 32, "activation": "tanh", "updater": m.sgd(0.05), "l2": 1e-3},
            {"type": "output", "name": "out", "n_out": 7, "loss": "mse", "activation": act, "updater": m.sgd(0.05)}], (16,)


def _conv_hinge():
    return [{"type": "conv2d", "name": "c1", "n_out": 8, "kernel": (3, 3), "stride": (2, 2), "padding": (1, 1), "activation": "lrelu", "alpha": 0.2,
             "updater": m.sgd(0.05), "l2": 1e-3},
            {"type": "conv2d", "name": "c2", "n_out": 6, "kernel": (3, 3), "stride": (1, 1), "padding": (1, 1), "has_bias": False, "updater": m.sgd(0.05)},
            {"type": "batchnorm", "name": "bn2", "updater": m.sgd(0.05)}, {"type": "activation", "name": "a2", "activation": "tanh"},
            {"type": "conv2d", "name": "c3", "n_out": 2, "kernel": (4, 4), "updater": m.sgd(0.05)},
            {"type": "loss", "name": "hinge", "loss": "hinge", "activation": "tanh"}], (3, 8, 8)


@pytest.mark.parametrize("net", ["mlp_identity", "mlp_tanh", "mlp_sigmoid", "conv_hinge"])
def test_fp32_fit_matches_oracle(b200, net):
    b, ctx = b200
    specs, shape = _mlp(net.split("_")[1]) if net.startswith("mlp") else _conv_hinge()
    rng = np.random.default_rng(3)
    onet = o.net_from_specs(specs, shape, seed=2); randomize(onet, rng)
    bnet = b.Net(ctx, specs, shape, max_batch=6, precision=b.FP32)
    push_params(onet, bnet)
    n_out = 7 if net.startswith("mlp") else 2
    for it in range(3):
        x = rng.uniform(-1, 1, (6,) + shape)
        y = rng.choice([-1.0, 1.0], (6, n_out)) if net == "conv_hinge" else rng.uniform(0, 1, (6, n_out))
        s_o = onet.compute_gradient_and_score(x, y); s_b = bnet.compute_gradient_and_score(x, y)
        assert abs(s_b - s_o) <= TOL * abs(s_o), (net, it, s_b, s_o)
        assert rel_err(bnet.gradients(), onet.grads_flat()) <= TOL, (net, it)
        s_o = onet.fit(x, y); s_b = bnet.fit(x, y)
        assert abs(s_b - s_o) <= TOL * abs(s_o), (net, it, s_b, s_o)
        assert rel_err(bnet.params(), onet.params_flat()) <= TOL, (net, it)
        xo = rng.uniform(-1, 1, (5,) + shape)
        out_o = onet.output(xo).reshape(5, -1)
        assert rel_err(bnet.output(xo), out_o) <= TOL, (net, it, "output")
    bnet.close()


# ------------------------------------------------------------------ the GAN step ---------------------------------------------------------
GAN_LOSSES = {"lsgan": ("mse", "identity", (1.0, 0.0, 1.0)), "hinge": ("hinge", "identity", (1.0, -1.0, 1.0)),
              "wasserstein": ("wasserstein", "identity", (-1.0, 1.0, -1.0))}


@pytest.mark.parametrize("kind", list(GAN_LOSSES))
def test_fp32_gan_step_matches_oracle(b200, kind):
    b, ctx = b200
    loss, act, (yr, yf, yg) = GAN_LOSSES[kind]
    n, lr_ = 8, 2e-3
    gs, ds = m.dcgan_generator(16, 12, 8, 3, lr=lr_), m.dcgan_discriminator(16, 8, 3, lr=lr_, loss=loss, out_activation=act)
    G, D, bG, bD, (x, zd, zg, _, _, _) = fp32_gan_pair(b, ctx, gs, ds, n)
    ys = [np.full((n, 1), v) for v in (yr, yf, yg)]
    gan = b.Gan(bG, bD, use_cuda_graph=True)
    for it in range(3):
        r = o.gan_step(G, D, x, zd, zg, *ys)
        lo = gan.step(x, zd, zg, *ys)
        want = np.array([r["loss_d_real"], r["loss_d_fake"], r["loss_g"]])
        assert np.all(np.abs(lo - want) < TOL * np.maximum(1, np.abs(want))), (kind, it, lo, want)
        assert pclose(bD.params(), D.params_flat(), 2 * lr_), (kind, it, "D", rel_err(bD.params(), D.params_flat()))
        assert pclose(bG.params(), G.params_flat(), 2 * lr_), (kind, it, "G", rel_err(bG.params(), G.params_flat()))
    gan.close(); bG.close(); bD.close()


def test_bf16_graph_replay_matches_eager(b200):
    b, ctx = b200
    n = 8
    for loss, (yr, yf, yg) in (("mse", (1.0, 0.0, 1.0)), ("hinge", (1.0, -1.0, 1.0))):
        runs = []
        for graph in (False, True):
            G, D = bf16_gan(b, ctx, m.dcgan_generator(32, 16, 64, 3), m.dcgan_discriminator(32, 64, 3, loss=loss), (16,), (3, 32, 32), n)
            data = [a.astype(np.float32) for a in o.synthetic_batch(n, 32, 3, 16, seed=3)][:3] + [np.full((n, 1), v, np.float32) for v in (yr, yf, yg)]
            gan = b.Gan(G, D, use_cuda_graph=graph)
            losses = np.array([gan.step(*data) for _ in range(4)])
            runs.append((losses, G.params(), D.params(), D.updater_state()))
            gan.close(); G.close(); D.close()
        assert np.isfinite(runs[0][0]).all()
        for a, c in zip(*runs):
            assert np.array_equal(a, c), loss


def test_launches_per_step_equal_the_xent_discriminators(b200):
    """C2 (DCGAN 64x64, bf16, batch 128) launches 83 kernels per step and a C5-shaped MLP-GAN 46, with D on XENT and on every new loss."""
    b, ctx = b200
    rng = np.random.default_rng(1)

    def per_step(gs, ds, gin, din, n, ys):
        G, D = bf16_gan(b, ctx, gs, ds, gin, din, n)
        gan = b.Gan(G, D, use_cuda_graph=True)
        gan.upload(rng.uniform(-1, 1, (n,) + tuple(din)), rng.uniform(-1, 1, (n,) + tuple(gin)), rng.uniform(-1, 1, (n,) + tuple(gin)),
                   *[np.full((n, 1), v) for v in ys])
        out = launches_per_step(ctx, gan, n)
        losses = gan.losses()
        gan.close(); G.close(); D.close()
        return out, losses

    for loss in ("xent",) + o.LOSSES:
        ys = (1.0, -1.0, 1.0) if loss in ("hinge", "squared_hinge", "wasserstein") else (1.0, 0.0, 1.0)
        c2, l2 = per_step(m.dcgan_generator(64, 100, 64, 3), m.dcgan_discriminator(64, 64, 3, loss=loss), (100,), (3, 64, 64), 128, ys)
        c5, l5 = per_step(m.mlp_generator(128, 1024, 256), m.mlp_discriminator(256, 1024, loss=loss), (128,), (256,), 8192, ys)
        assert (c2, c5) == (83, 46), loss
        assert np.isfinite(l2).all() and np.isfinite(l5).all(), loss


# ------------------------------------------------------------------ argument checks, checkpoint ---------------------------------------------
def _create(b, ctx, specs, shape, mutate=None, **cfg_kw):
    import ctypes as C
    from gan_deeplearning4j_b200 import _lib, engine
    descs = [engine.layer_desc(s) for s in specs]
    if mutate:
        mutate(descs)
    arr = (_lib.LayerDesc * len(descs))(*descs)
    c, h, w = shape if len(shape) == 3 else (shape[0], 1, 1)
    cfg = _lib.NetConfig(h, w, c, 4, 0, 0.0, 1e-5, 1, 666)
    hnd = C.c_void_p()
    r = ctx.lib.b2g_net_create(ctx.h, C.byref(cfg), arr, len(descs), C.byref(hnd))
    if r == 0:
        ctx.lib.b2g_net_destroy(hnd)
    return r, ctx.lib.b2g_last_error()


def test_rejections(b200):
    b, ctx = b200
    specs, shape = _mlp("identity")
    for bad in (9, -1, 100):
        def mut(d, bad=bad): d[-1].loss = bad
        r, msg = _create(b, ctx, specs, shape, mut)
        assert r == -1 and b"unknown loss" in msg, bad
        hs, hshape = _conv_hinge()
        r, msg = _create(b, ctx, hs, hshape, mut)
        assert r == -1 and b"unknown loss" in msg, bad
    hs, hshape = _conv_hinge()
    r, _ = _create(b, ctx, hs, hshape, lambda d: setattr(d[-1], "loss", 1))            # MCXENT on a LossLayer
    assert r == -6
    onmap = hs[:-2] + [{"type": "loss", "name": "l", "loss": "mse"}]                      # the loss on the 4x4x6 map
    r, msg = _create(b, ctx, onmap, hshape)
    assert r == -6 and b"map" in msg
    r, _ = _create(b, ctx, [dict(specs[0]), dict(specs[1], loss="xent")], shape)         # XENT with nOut = 7
    assert r == -6
    assert _create(b, ctx, specs, shape)[0] == 0
    # the GAN step: MCXENT or more than one output per example is refused
    gs = m.mlp_generator(16, 32, 24)
    G = b.Net(ctx, gs, (16,), max_batch=4, precision=b.FP32)
    for ds in (m.mlp_discriminator(24, 32)[:-1] + [dict(m.mlp_discriminator(24, 32)[-1], loss="mcxent", n_out=3)],
               m.mlp_discriminator(24, 32)[:-1] + [dict(m.mlp_discriminator(24, 32)[-1], loss="mse", n_out=3)]):
        D = b.Net(ctx, ds, (24,), max_batch=8, precision=b.FP32, bn_groups=2)
        with pytest.raises(b.B200GanError) as e:
            b.Gan(G, D)
        assert e.value.code == -6
        D.close()
    D = b.Net(ctx, m.mlp_discriminator(24, 32, loss="squared_hinge", out_activation="tanh"), (24,), max_batch=8, precision=b.FP32, bn_groups=2)
    b.Gan(G, D).close()
    D.close(); G.close()


def test_mse_output_checkpoint_resume_is_bit_identical(b200, tmp_path):
    b, ctx = b200
    from gan_deeplearning4j_b200 import serializer
    specs = [{"type": "dense", "name": "d1", "n_out": 32, "activation": "tanh", "updater": m.adam(2e-3)},
             {"type": "output", "name": "out", "n_out": 7, "loss": "mse", "activation": "sigmoid", "updater": m.adam(2e-3)}]
    rng = np.random.default_rng(4)
    batches = [(rng.uniform(-1, 1, (6, 16)), rng.uniform(0, 1, (6, 7))) for _ in range(6)]
    full = b.Net(ctx, specs, (16,), max_batch=6, precision=b.FP32, seed=9)
    scores = [full.fit(x, y) for x, y in batches]
    first = b.Net(ctx, specs, (16,), max_batch=6, precision=b.FP32, seed=9)
    for x, y in batches[:3]:
        first.fit(x, y)
    path = str(tmp_path / "ckpt.zip")
    first.save(path)
    saved = serializer.read_model(path)
    assert saved["specs"][-1]["loss"] == "mse" and saved["specs"][-1]["activation"] == "sigmoid"
    resumed = b.Net(ctx, saved["specs"], (16,), max_batch=6, precision=b.FP32, seed=1)
    resumed.restore(path)
    rs = [resumed.fit(x, y) for x, y in batches[3:]]
    assert rs == scores[3:]
    assert np.array_equal(full.params(), resumed.params()) and np.array_equal(full.updater_state(), resumed.updater_state())
    for net in (full, first, resumed):
        net.close()
