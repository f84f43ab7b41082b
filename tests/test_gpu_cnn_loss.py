"""CnnLossLayer on the GPU: the per-pixel loss kernels (b2g_test_ew ops cnn_xent / cnn_softmax_xent) against fp32 / float64 emulations of their
documented formulas and order, on one block and many, groups 1 and 2, C in {1, 3, 5, 16}, aligned and odd offsets, poisoned outputs -- the
vector and scalar paths give the same bits and so do two runs; FP32 nets ending in CnnLossLayer against the oracle over 3 fit iterations; a
BF16 net; the adversarial step with a PatchGAN discriminator against the oracle, graph replay
against eager, per-image labels against the same labels as maps, and the refusals."""
import numpy as np
import pytest

from gan_deeplearning4j_b200 import models as m
from helpers import b200, bf16_round, check_bf16, gan_step_parity, oracle_gan_pair, push_params, randomize, rel_err
from oracle import dl4j_oracle as o

pytestmark = pytest.mark.gpu
TOL = 1e-3


# ------------------------------------------------------------------ the loss kernels -----------------------------------------------------
def _xent_ref(z, y, clip):
    """xent_kernel's per-element formulas in fp32 (numpy's exp / log: within an ulp or two of the device's)."""
    z, y = z.astype(np.float32), y.astype(np.float32)
    one = np.float32(1)
    with np.errstate(over="ignore"):
        sg = one / (one + np.exp(-z))
    if clip > 0:
        p = np.minimum(np.maximum(sg, np.float32(clip)), one - np.float32(clip))
        return -(y * np.log(p) + (one - y) * np.log(one - p)), (p - y) / (p * (one - p)) * sg * (one - sg)
    return np.maximum(z, 0) + np.log1p(np.exp(-np.abs(z))) - y * z, sg - y


def _sm_ref(z, y):
    z = z.astype(np.float32)
    e = np.exp(z - z.max(1, keepdims=True))
    p = e / e.sum(1, keepdims=True, dtype=np.float32)
    loss = None if y is None else -(y * np.log(np.clip(p, np.float32(1e-10), np.float32(1 - 1e-10)).astype(np.float64))).sum(1)
    return p, loss


def _close(got, ref, rtol, atol, what):
    """Within rtol |ref| + atol: the device's expf / logf and numpy's differ by an ulp or two, which 1 - sigmoid and p - y can magnify."""
    got, ref = np.asarray(got, np.float64).ravel(), np.asarray(ref, np.float64).ravel()
    assert np.isfinite(got).all(), (what, "non-finite: an element left unwritten reads back as NaN")
    bad = np.abs(got - ref) > rtol * np.abs(ref) + atol
    assert not bad.any(), (what, int(bad.sum()), got[bad][:4], ref[bad][:4])


SHAPES = [(1, 1, 37), (1, 3, 300), (2, 5, 211), (2, 16, 4096), (1, 3, 120000), (2, 1, 150001)]    # (groups, C, pixels per group)


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("clip", [1e-5, 0.0])
@pytest.mark.parametrize("shape", SHAPES)
def test_cnn_xent_kernel(b200, shape, clip, prec):
    b, ctx = b200
    groups, c, rows = shape
    P = b.FP32 if prec == "fp32" else b.BF16
    rng = np.random.default_rng(groups * 1000 + c * 10 + rows % 7)
    n = groups * rows * c
    z = rng.uniform(-6, 6, n).astype(np.float32)
    if P == b.BF16:
        z = bf16_round(z)
    y = rng.uniform(0, 1, n).astype(np.float32)
    runs = {}
    for off in (0, 3, 0):
        outs, info = b.test_ew(ctx, P, "cnn_xent", z, y, (n, groups, 0), rows=rows, cols=c, groups=groups, clip_eps=clip, offset=off, poison=True)
        assert info["kernel"].startswith("cnn_xent_kernel"), info
        runs.setdefault(off, []).append(outs)
    dz0, ls0 = runs[0][0][0], runs[0][0][1]
    for dz, ls in [(r[0], r[1]) for rr in runs.values() for r in rr]:
        assert np.array_equal(dz, dz0) and np.array_equal(ls, ls0), "the loss sums and dz do not depend on the path or the run"
    lref, gref = _xent_ref(z, y, clip)
    if P == b.FP32:
        _close(dz0, gref, 1e-4, 1e-6, "dz")
    else:
        check_bf16(dz0, gref, "dz")
    want = lref.astype(np.float64).reshape(groups, -1).sum(1)
    assert np.all(np.abs(ls0 - want) <= 1e-5 * np.abs(want) + 1e-5), (ls0, want)


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("shape", SHAPES[:5])
def test_cnn_softmax_xent_kernel(b200, shape, prec):
    b, ctx = b200
    groups, c, rows = shape
    P = b.FP32 if prec == "fp32" else b.BF16
    rng = np.random.default_rng(groups * 100 + c)
    n = groups * rows * c
    z = rng.uniform(-5, 5, (groups * rows, c)).astype(np.float32)
    if P == b.BF16:
        z = bf16_round(z)
    y = np.eye(c, dtype=np.float32)[rng.integers(0, c, groups * rows)]
    if c > 1:
        y[::7] = rng.dirichlet(np.ones(c), len(y[::7]))          # soft labels too
    outs = [b.test_ew(ctx, P, "cnn_softmax_xent", z, y, (n, groups, n), rows=rows, cols=c, groups=groups, offset=off, poison=True)[0] for off in (0, 3, 0)]
    for u in outs[1:]:
        for a, bb in zip(outs[0], u):
            assert np.array_equal(a, bb)
    dz, ls, p = outs[0]
    pref, lref = _sm_ref(z, y)
    if P == b.FP32:
        _close(p, pref.ravel(), 1e-6, 1e-9, "p")
        _close(dz, (pref - y).ravel(), 0.0, 1e-6, "dz")
    else:
        check_bf16(p, pref.ravel(), "p"); check_bf16(dz, (pref - y).ravel(), "dz")
    want = lref.reshape(groups, -1).sum(1)
    assert np.all(np.abs(ls - want) <= 1e-5 * np.abs(want) + 1e-5), (ls, want)
    inf, info = b.test_ew(ctx, P, "cnn_softmax_xent", z, None, (0, 0, n), rows=rows, cols=c, groups=groups, poison=True)
    assert np.array_equal(inf[2], p), "the inference call's probabilities"
    assert info["kernel"] == "cnn_softmax_xent_kernel"


# ------------------------------------------------------------------ nets ----------------------------------------------------------------
NET_LOSSES = [("xent", "identity", 1), ("xent", "identity", 3), ("mcxent", "identity", 3), ("mse", "tanh", 2), ("l1", "identity", 1),
              ("hinge", "identity", 2), ("wasserstein", "identity", 1), ("squared_hinge", "elu", 2)]


def _labels(loss, rng, shape):
    if loss == "xent":
        return rng.uniform(0.05, 0.95, shape)
    if loss == "mcxent":
        n, c, h, w = shape
        return np.moveaxis(np.eye(c)[rng.integers(0, c, (n, h, w))], -1, 1)
    if loss in ("hinge", "squared_hinge", "wasserstein"):
        return rng.choice([-1.0, 1.0], shape)
    return rng.uniform(-1, 1, shape)


def _specs(loss, act, c):
    return [{"type": "conv2d", "name": "c1", "n_out": 8, "kernel": (3, 3), "stride": (1, 1), "padding": (1, 1), "has_bias": False, "updater": m.sgd(0.05)},
            {"type": "batchnorm", "name": "bn1", "updater": m.sgd(0.05)},
            {"type": "activation", "name": "a1", "activation": "lrelu", "alpha": 0.2},
            {"type": "conv2d", "name": "c2", "n_out": c, "kernel": (3, 3), "stride": (2, 2), "padding": (1, 1), "updater": m.sgd(0.05)},
            dict(m.cnn_loss(loss, act), name="cl")], (3, 9, 7)


@pytest.mark.parametrize("loss,act,c", NET_LOSSES)
def test_fp32_nets_match_oracle(b200, loss, act, c):
    """Activations, gradients, the score, the parameters after fit and b2g_net_output (the activated map in NCHW) within 1e-3 over 3 fit
    iterations, the second on a ragged batch."""
    b, ctx = b200
    specs, shape = _specs(loss, act, c)
    rng = np.random.default_rng(c * 13 + len(loss))
    onet = o.net_from_specs(specs, shape, seed=2, flat_input=False); randomize(onet, rng)
    bnet = b.Net(ctx, specs, shape, max_batch=6, precision=b.FP32)
    push_params(onet, bnet)
    assert bnet.out_elems == c * 5 * 4
    for it, mb in enumerate((6, 5, 6)):
        x = rng.uniform(-1.5, 1.5, (mb,) + shape); y = _labels(loss, rng, (mb, c, 5, 4))
        s_o, acts, _, _ = onet.compute_gradient_and_score(x, y, collect=True)
        s_b = bnet.compute_gradient_and_score(x, y)
        assert abs(s_b - s_o) <= TOL * abs(s_o), (loss, it, s_b, s_o)
        for i in (0, 2, 3):
            assert rel_err(bnet.activation(i, mb), acts[i].reshape(mb, -1)) <= TOL, (loss, it, "activation", i)
        assert rel_err(bnet.gradients(), onet.grads_flat()) <= TOL, (loss, it, "gradients")
        s_o = onet.fit(x, y); s_b = bnet.fit(x, y)
        assert abs(s_b - s_o) <= TOL * abs(s_o), (loss, it, s_b, s_o)
        assert rel_err(bnet.params(), onet.params_flat()) <= TOL, (loss, it, "params")
        xo = rng.uniform(-1.5, 1.5, (4,) + shape)
        assert rel_err(bnet.output(xo), onet.output(xo).reshape(4, -1)) <= TOL, (loss, it, "output")
    bnet.close()


@pytest.mark.parametrize("loss,act,c", [("xent", "identity", 1), ("mcxent", "identity", 3), ("mse", "identity", 2)])
def test_bf16_nets_match_oracle_loosely(b200, loss, act, c):
    b, ctx = b200
    specs, shape = _specs(loss, act, c)
    specs[0]["n_out"] = 64
    rng = np.random.default_rng(7)
    onet = o.net_from_specs(specs, shape, seed=2, flat_input=False); randomize(onet, rng)
    for l in onet.layers:
        if l.has_params and "W" in l.params:
            l.params["W"] = bf16_round(l.params["W"]).astype(np.float64)
    bnet = b.Net(ctx, specs, shape, max_batch=8, precision=b.BF16)
    push_params(onet, bnet)
    x = bf16_round(rng.uniform(-1, 1, (8,) + shape)); y = _labels(loss, rng, (8, c, 5, 4))
    s_o = onet.compute_gradient_and_score(x, y)
    s_b = bnet.compute_gradient_and_score(x, y)
    assert abs(s_b - s_o) <= 3e-2 * abs(s_o), (s_b, s_o)
    assert rel_err(bnet.gradients(), onet.grads_flat()) <= 5e-2
    # a whole bf16 forward (no layer-by-layer injection): the rounding of every layer accumulates, so the output is held to 2e-2 of its max
    assert rel_err(bnet.output(x).reshape(8, -1), onet.output(x).reshape(8, -1)) <= 2e-2
    bnet.close()


# ------------------------------------------------------------------ the adversarial step -------------------------------------------------
@pytest.mark.parametrize("loss", ["xent", "mse"])
def test_fp32_patch_gan_step_matches_oracle(b200, loss):
    """A 16x16 DCGAN with a 4x4-patch discriminator (XENT; MSE with labels 1 / 0 / 1): losses and both nets' parameters over 3 steps; graph
    replay equals the eager step bit for bit.  Gan.step takes the per-image labels and broadcasts them over the patch map."""
    b, ctx = b200
    size, z, n, lr_ = 16, 12, 8, 2e-3
    gs, ds = m.dcgan_generator(size, z, 8, 3, lr=lr_), m.dcgan_discriminator(size, 8, 3, lr=lr_, loss=loss, patch=True)
    G, D = oracle_gan_pair(gs, ds, size, z)
    data = [a.astype(np.float64) for a in o.synthetic_batch(n, size, 3, z, seed=3)]
    if loss == "mse":
        data[3], data[4], data[5] = np.ones((n, 1)), np.zeros((n, 1)), np.ones((n, 1))
    maps = [np.broadcast_to(v.reshape(n, 1, 1, 1), (n, 1, 4, 4)).copy() for v in data[3:]]
    gan_step_parity(b, ctx, gs, ds, G, D, data, maps, lr_, loss)


def _bf16_run(b, ctx, gs, ds, G, D, data, n, size, z, graph=True, steps=2):
    bG = b.Net(ctx, gs, (z,), max_batch=n, precision=b.BF16)
    bD = b.Net(ctx, ds, (3, size, size), max_batch=2 * n, precision=b.BF16, bn_groups=2)
    push_params(G, bG); push_params(D, bD)
    gan = b.Gan(bG, bD, use_cuda_graph=graph)
    gan.step(*data)
    s0 = bG.simt_gemm_calls() + bD.simt_gemm_calls()
    losses = [gan.step(*data) for _ in range(steps)]
    simt = (bG.simt_gemm_calls() + bD.simt_gemm_calls() - s0) / steps
    out = (np.array(losses), bG.params(), bD.params())
    gan.close(); bG.close(); bD.close()
    return out, simt


def test_bf16_patch_step_head_adds_no_simt_calls_and_label_broadcast(b200):
    """At the C2 shapes (64x64, nf 64; a small batch) the patch step reports fewer SIMT calls per step than the C2 step: the C2 head's dense
    kernels count, the patch head's few-output kernels do not.  Per-image labels broadcast by Gan.step give the same bits as the same labels as
    full maps."""
    b, ctx = b200
    size, z, nf, n = 64, 100, 64, 16
    gs = m.dcgan_generator(size, z, nf, 3)
    data = [a.astype(np.float32) for a in o.synthetic_batch(n, size, 3, z, seed=3)]
    rng = np.random.default_rng(5)
    simt = {}
    for patch in (False, True):
        ds = m.dcgan_discriminator(size, nf, 3, patch=patch)
        G = o.net_from_specs(gs, (z,), seed=1); D = o.net_from_specs(ds, (3, size, size), seed=2)
        randomize(G, rng); randomize(D, rng)
        out, simt[patch] = _bf16_run(b, ctx, gs, ds, G, D, data, n, size, z)
        assert np.isfinite(out[0]).all()
        if patch:
            maps = [np.broadcast_to(v.reshape(n, 1, 1, 1), (n, 1, 4, 4)).copy() for v in data[3:]]
            out2, _ = _bf16_run(b, ctx, gs, ds, G, D, data[:3] + maps, n, size, z)
            for u, v in zip(out, out2):
                assert np.array_equal(u, v), "per-image labels == the same labels as maps"
    # the C2 head runs dense_small_o forward / weight gradient / input gradient in the D step and forward / input gradient in the G step
    assert simt[True] == simt[False] - 5, simt


def test_bf16_head_conv_adds_no_simt_calls(b200):
    """BatchNorm -> the 3x3 s1 p1 head onto 1 channel -> CnnLossLayer: the head's forward, weight gradient and input gradient (the BatchNorm
    below is trainable) all run on the few-output kernels."""
    b, ctx = b200
    specs = [{"type": "batchnorm", "name": "bn", "updater": m.sgd(0.01)},
             {"type": "conv2d", "name": "head", "n_out": 1, "kernel": (3, 3), "stride": (1, 1), "padding": (1, 1), "updater": m.sgd(0.01)},
             dict(m.cnn_loss("xent"), name="cl")]
    net = b.Net(ctx, specs, (64, 4, 4), max_batch=8, precision=b.BF16)
    rng = np.random.default_rng(0)
    net.fit(rng.uniform(-1, 1, (8, 64, 4, 4)), rng.uniform(0, 1, (8, 1, 4, 4)))
    assert net.simt_gemm_calls() == 0
    net.close()


# ------------------------------------------------------------------ the few-output head conv kernels (impl 5) ------------------------------
HEAD_GEOMS = [(3, 3, 1, 1), (4, 4, 1, 1), (4, 4, 2, 1), (5, 5, 1, 2)]        # (kh, kw, stride, pad)


@pytest.mark.parametrize("o_", [1, 2, 3, 4])
@pytest.mark.parametrize("geom", HEAD_GEOMS)
def test_head_conv_kernels_bit_exact_on_integers(b200, geom, o_):
    """Forward with bias + activation, input gradient (with and without bias + activation), weight gradient at the production split count, one
    split, three, and more splits than pixels (empty splits), dw at an odd parameter offset, bias gradient: against float64 on small integer
    operands (every fp32 sum exact), after the same bf16 rounding of the stored outputs, with poisoned outputs."""
    torch = pytest.importorskip("torch")
    b, ctx = b200
    kh, kw, st, pd = geom
    nb, h, w, c = 2, 7, 5, 24
    oh, ow = (h + 2 * pd - kh) // st + 1, (w + 2 * pd - kw) // st + 1
    g = dict(n=nb, h=h, w=w, c=c, oh=oh, ow=ow, o=o_, kh=kh, kw=kw, sh=st, sw=st, ph=pd, pw=pd)
    rng = np.random.default_rng(kh * 10 + st + o_)
    x = rng.integers(-2, 3, (nb, c, h, w)).astype(np.float64)
    wt = rng.integers(-2, 3, (o_, c, kh, kw)).astype(np.float64)
    bias = rng.integers(-3, 4, o_).astype(np.float64)
    dy = rng.integers(-2, 3, (nb, o_, oh, ow)).astype(np.float64)
    xt = torch.tensor(x, requires_grad=True); wtt = torch.tensor(wt, requires_grad=True); bt = torch.tensor(bias, requires_grad=True)
    y = torch.nn.functional.conv2d(xt, wtt, bt, stride=st, padding=pd)
    y.backward(torch.tensor(dy))
    nhwc = lambda a: np.ascontiguousarray(np.asarray(a).transpose(0, 2, 3, 1))
    wn = nhwc(wt)                                                            # [O][KH][KW][C]
    yref = y.detach().numpy()
    for act, f in (("identity", lambda v: v), ("lrelu", lambda v: np.where(v > 0, v, 0.25 * v))):
        got, _, kern, _ = b.test_conv_ex(ctx, 0, g, nhwc(x), wn, yref.size, impl=5, bias=bias, act=act, alpha=0.25, poison=True)
        assert kern == "head_conv_fwd_kernel"
        assert np.array_equal(got, bf16_round(nhwc(f(yref))).ravel()), ("fprop", act)
    got, _, kern, _ = b.test_conv_ex(ctx, 1, g, nhwc(dy), wn, x.size, impl=5, poison=True)
    assert kern == "head_conv_dgrad_kernel"
    assert np.array_equal(got, bf16_round(nhwc(xt.grad.numpy())).ravel()), "dgrad"
    cb = rng.integers(-3, 4, c).astype(np.float64)
    got, _, _, _ = b.test_conv_ex(ctx, 1, g, nhwc(dy), wn, x.size, impl=5, bias=cb, act="relu", poison=True)
    assert np.array_equal(got, bf16_round(nhwc(np.maximum(xt.grad.numpy() + cb[None, :, None, None], 0))).ravel()), "dgrad + bias + relu"
    dw_ref = nhwc(wtt.grad.numpy()).ravel()
    P = nb * oh * ow
    for splits in (0, 1, 3, P + 5):
        info, db = {}, np.zeros(o_, np.float32)
        got, _, kern, _ = b.test_conv_ex(ctx, 2, g, nhwc(x), nhwc(dy), dw_ref.size, impl=5, splits=splits, poison=True, param_offset=3, db=db, info=info)
        assert kern == "head_conv_wgrad_kernel"
        assert splits == 0 or info["splits"] == splits
        assert np.array_equal(got, dw_ref.astype(np.float32)), ("wgrad", splits)
        assert np.array_equal(db, bt.grad.numpy().astype(np.float32)), ("db", splits)


def test_head_conv_refusals(b200):
    b, ctx = b200
    g = dict(n=1, h=5, w=5, c=12, oh=5, ow=5, o=1, kh=3, kw=3, sh=1, sw=1, ph=1, pw=1)          # C % 8 != 0
    with pytest.raises(b.B200GanError):
        b.test_conv_ex(ctx, 0, g, np.zeros(300), np.zeros(108), 25, impl=5)
    g = dict(n=1, h=5, w=5, c=16, oh=5, ow=5, o=1, kh=3, kw=3, sh=1, sw=1, ph=1, pw=1)
    with pytest.raises(b.B200GanError):
        b.test_conv_ex(ctx, 0, g, np.zeros(400), np.zeros(144), 25, impl=5, precision=b.FP32)


# ------------------------------------------------------------------ loss sums count every element ------------------------------------------
@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("shape", SHAPES)
def test_loss_sums_count_every_element(b200, shape, prec):
    """Every element's score is at least ~0.97 (XENT: the logit on the wrong side of its 0 / 1 label by >= 0.5; MCXENT: the label on the
    smallest logit, score >= log C), so a dropped or doubled element moves a group's sum by more than the 0.4 allowed here, which covers the
    fp32 rounding of the sum and the ulp differences of expf / logf."""
    b, ctx = b200
    groups, c, rows = shape
    P = b.FP32 if prec == "fp32" else b.BF16
    rng = np.random.default_rng(rows)
    n = groups * rows * c
    y = rng.integers(0, 2, n).astype(np.float32)
    z = (rng.uniform(0.5, 6, n) * np.where(y > 0, -1, 1)).astype(np.float32)
    if P == b.BF16:
        z = bf16_round(z)
    for clip in (1e-5, 0.0):
        (dz, ls, _), _ = b.test_ew(ctx, P, "cnn_xent", z, y, (n, groups, 0), rows=rows, cols=c, groups=groups, clip_eps=clip)
        lref, _ = _xent_ref(z, y, clip)
        assert lref.min() > 0.9
        want = lref.astype(np.float64).reshape(groups, -1).sum(1)
        assert np.all(np.abs(ls - want) <= 0.4), ("xent", clip, ls, want)
    if c == 1 or rows > 50000:
        return
    zs = rng.uniform(-5, 5, (groups * rows, c)).astype(np.float32)
    if P == b.BF16:
        zs = bf16_round(zs)
    ys = np.eye(c, dtype=np.float32)[zs.argmin(1)]
    (_, ls, _), _ = b.test_ew(ctx, P, "cnn_softmax_xent", zs, ys, (n, groups, n), rows=rows, cols=c, groups=groups)
    _, lref = _sm_ref(zs, ys)
    assert lref.min() >= np.log(c) - 1e-6
    want = lref.reshape(groups, -1).sum(1)
    assert np.all(np.abs(ls - want) <= 0.4), ("mcxent", ls, want)


def test_refusals(b200):
    b, ctx = b200
    size, z, nf, n = 16, 12, 8, 4
    bG = b.Net(ctx, m.dcgan_generator(size, z, nf, 3), (z,), max_batch=n, precision=b.FP32)
    ds = m.dcgan_discriminator(size, nf, 3, patch=True)
    ds[-1] = dict(m.cnn_loss("mcxent"), name="dis_loss")
    bD = b.Net(ctx, ds, (3, size, size), max_batch=2 * n, precision=b.FP32, bn_groups=2)
    with pytest.raises(b.B200GanError, match="MCXENT"):
        b.Gan(bG, bD)
    bD.close()
    bD = b.Net(ctx, m.dcgan_discriminator(size, nf, 3, patch=True), (3, size, size), max_batch=2 * n, precision=b.FP32, bn_groups=2)
    gan = b.Gan(bG, bD)
    data = [a.astype(np.float32) for a in o.synthetic_batch(n, size, 3, z, seed=3)]
    with pytest.raises(ValueError):
        gan.step(*data[:3], np.ones((n, 5)), data[4], data[5])      # 5 labels per image for a 16-patch map
    gan.close(); bD.close(); bG.close()
