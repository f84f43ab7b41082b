"""Spine-plus-skip graphs on the GPU: the vertex kernels (b2g_test_ew ops vertex_fwd / vertex_bwd / merge_fwd / merge_bwd / skip_add) bit for
bit against fp32 / bf16 emulations on the vector and scalar paths with poisoned outputs, written and accumulated; FP32 residual, U-Net,
shared-source and feed-forward merge nets against the float64 oracle over fit iterations; BF16 nets, one per
single-consumer fusion the engine turns off at a skip source; the adversarial step with residual nets against oracle gan_step, graph replay
against eager; and the launch budget."""
import numpy as np
import pytest

from gan_deeplearning4j_b200 import models as m
from helpers import b200, bf16_round, gan_step_parity, oracle_gan_pair, push_params, randomize, rel_err
from oracle import dl4j_oracle as o

pytestmark = pytest.mark.gpu
TOL = 1e-3


# ------------------------------------------------------------------ the vertex kernels ---------------------------------------------------
def _t(a, bf):
    a = np.asarray(a, np.float32)
    return bf16_round(a) if bf else a


def _ew_ref(op, a, b):
    """ew_forward in fp32 (every op is one fp32 operation on the inputs, AVERAGE (a + b) * 0.5)."""
    a, b = a.astype(np.float32), b.astype(np.float32)
    return o.ew_forward(op, a, b).astype(np.float32)


@pytest.mark.parametrize("prec", [0, 1])
@pytest.mark.parametrize("offset,n", [(0, 4096 + 24), (0, 4096 + 3), (1, 1000 + 3)])
@pytest.mark.parametrize("op", o.EW_OPS)
def test_elementwise_kernels_bit_exact(b200, prec, offset, n, op):
    b, ctx = b200
    bf = prec == b.BF16
    rng = np.random.default_rng(11)
    sp, sk, e, acc0 = (rng.standard_normal(n) for _ in range(4))
    sp[::7] = sk[::7]                              # exact ties (MAX sends them to the first input)
    sp, sk, e = _t(sp, bf), _t(sk, bf), _t(e, bf)
    acc0 = acc0.astype(np.float32)
    vec = "vec" if offset == 0 else "scalar"
    for order in (0, 1):
        a, c = (sp, sk) if order == 0 else (sk, sp)
        (y, _, _), info = b.test_ew(ctx, prec, "vertex_fwd", sp, sk, (n, 0, 0), act=op, n=n, groups=order, offset=offset, poison=True)
        assert info["kernel"] == f"vertex_ew_fwd_kernel<{vec}>"
        assert np.array_equal(y, _t(_ew_ref(op, a, c), bf)), (op, order)
        da, db = o.ew_backward(op, e, a, c)
        da, db = da.astype(np.float32), db.astype(np.float32)
        sp_share, sk_share = (da, db) if order == 0 else (db, da)
        for accumulate in (0, 1):
            (eo, acc, _), info = b.test_ew(ctx, prec, "vertex_bwd", np.concatenate([sp, sk]), np.concatenate([e, acc0]), (n, n, 0), act=op, n=n,
                                           groups=order, offset=offset, accumulate=accumulate, poison=not accumulate)
            assert info["kernel"] == f"vertex_ew_bwd_kernel<{vec}>"
            assert np.array_equal(eo, _t(sp_share, bf)), (op, order, accumulate, "spine")
            want = (acc0 + sk_share).astype(np.float32) if accumulate else sk_share
            assert np.array_equal(acc, want), (op, order, accumulate, "skip")


@pytest.mark.parametrize("prec", [0, 1])
@pytest.mark.parametrize("P,cs,ck,offset", [(300, 64, 32, 0), (77, 8, 16, 0), (50, 5, 3, 0), (64, 64, 64, 1)])
def test_merge_kernels_bit_exact(b200, prec, P, cs, ck, offset):
    b, ctx = b200
    bf = prec == b.BF16
    rng = np.random.default_rng(12)
    sp, sk = _t(rng.standard_normal((P, cs)), bf), _t(rng.standard_normal((P, ck)), bf)
    e = _t(rng.standard_normal((P, cs + ck)), bf)
    acc0 = rng.standard_normal((P, ck)).astype(np.float32)
    V = 8 if bf else 4
    vec = "vec" if offset == 0 and cs % V == 0 and ck % V == 0 else "scalar"
    for order in (0, 1):
        (y, _, _), info = b.test_ew(ctx, prec, "merge_fwd", sp, sk, (P * (cs + ck), 0, 0), rows=P, cols=cs, C=ck, groups=order, offset=offset, poison=True)
        assert info["kernel"] == f"merge_fwd_kernel<{vec}>"
        assert np.array_equal(y.reshape(P, -1), np.concatenate((sp, sk) if order == 0 else (sk, sp), 1)), order
        first, second = (e[:, :cs], e[:, cs:]) if order == 0 else (e[:, :ck], e[:, ck:])
        spine, skip = (first, second) if order == 0 else (second, first)
        for accumulate in (0, 1):
            (d, acc, _), info = b.test_ew(ctx, prec, "merge_bwd", e, acc0 if accumulate else None, (P * cs, P * ck, 0), rows=P, cols=cs, C=ck,
                                          groups=order, offset=offset, accumulate=accumulate, poison=not accumulate)
            assert info["kernel"] == f"merge_bwd_kernel<{vec}>"
            assert np.array_equal(d.reshape(P, cs), spine)
            assert np.array_equal(acc.reshape(P, ck), (acc0 + skip).astype(np.float32) if accumulate else skip.astype(np.float32))


@pytest.mark.parametrize("prec", [0, 1])
@pytest.mark.parametrize("offset,n", [(0, 8192), (0, 8195), (3, 999)])
def test_skip_add_bit_exact(b200, prec, offset, n):
    b, ctx = b200
    bf = prec == b.BF16
    rng = np.random.default_rng(13)
    e, acc = _t(rng.standard_normal(n), bf), rng.standard_normal(n).astype(np.float32)
    (out, _, _), info = b.test_ew(ctx, prec, "skip_add", e, acc, (n, 0, 0), n=n, offset=offset)
    assert info["kernel"] == ("skip_add_kernel<vec>" if offset == 0 else "skip_add_kernel<scalar>")
    assert np.array_equal(out, _t(e + acc, bf))


# ------------------------------------------------------------------ nets against the oracle ---------------------------------------------
def _dense(name, n_out, act="tanh", lr=0.05):
    return {"type": "dense", "name": name, "n_out": n_out, "activation": act, "updater": m.adam(lr)}


def _conv(name, c_in, c_out, k=3, s=1, p=1, act="identity", lr=0.01):
    return {"type": "conv2d", "name": name, "n_in": c_in, "n_out": c_out, "kernel": (k, k), "stride": (s, s), "padding": (p, p), "activation": act,
            "has_bias": False, "updater": m.adam(lr)}


def _nets(kind, ch=8):
    """(specs, input shape, loss) of the graphs the parity tests run."""
    if kind == "residual":
        return ([_conv("stem", 3, ch, act="tanh")] + m.residual_block("rb", ch, "stem", lr=0.01) +
                [_conv("head", ch, 2, k=1, p=0), m.cnn_loss("mse", name="loss")], (3, 8, 8), "mse")
    if kind == "unet":
        return m.unet(size=16, nc=3, n_classes=3, nf=ch, depth=2, lr=0.01), (3, 16, 16), "mcxent"
    if kind == "shared":
        return ([_conv("c1", 3, ch, act="tanh"), _conv("c2", ch, ch, act="sigmoid"), m.elementwise("max", ["c1", "c2"], name="a1"),
                 _conv("c3", ch, ch, act="tanh"), m.merge(["c1", "c3"], name="m1"), _conv("c4", 2 * ch, ch, act="tanh"), m.elementwise("product", ["c4", "c1"], name="p1"), _conv("head", ch, 3, k=1, p=0),
                 m.cnn_loss("mcxent", name="loss")], (3, 6, 6), "mcxent")
    if kind == "ff_merge":
        return ([_dense("d1", 16), _dense("d2", 24, "sigmoid"), m.merge(["d1", "d2"], name="mg"), _dense("d3", 12),
                 m.elementwise("average", ["d3", "d3"], name="av"),
                 {"type": "output", "name": "out", "n_out": 3, "loss": "mse", "activation": "identity", "updater": m.adam(0.05)}], (10,), "mse")
    raise ValueError(kind)


def _labels(loss, rng, shape):
    if loss == "mcxent":
        lab = rng.integers(0, shape[1], (shape[0],) + tuple(shape[2:]))
        return np.ascontiguousarray(np.moveaxis(np.eye(shape[1])[lab], -1, 1))
    return rng.standard_normal(shape)


@pytest.mark.parametrize("kind", ["residual", "unet", "shared", "ff_merge"])
def test_fp32_graph_nets_match_oracle(b200, kind):
    b, ctx = b200
    specs, shape, loss = _nets(kind)
    rng = np.random.default_rng(21)
    onet = o.net_from_specs(specs, shape, seed=2, flat_input=False); randomize(onet, rng)
    bnet = b.Net(ctx, specs, shape, max_batch=6, precision=b.FP32)
    push_params(onet, bnet)
    for it, mb in enumerate((6, 5, 6)):
        x = rng.uniform(-1.5, 1.5, (mb,) + shape)
        out = onet.forward(x, False)
        y = _labels(loss, rng, (mb,) + out.shape[1:])
        s_o, acts, _, _ = onet.compute_gradient_and_score(x, y, collect=True)
        s_b = bnet.compute_gradient_and_score(x, y)
        assert abs(s_b - s_o) <= TOL * abs(s_o), (kind, it, s_b, s_o)
        for i, sp in enumerate(specs):
            if sp["type"] in ("elementwise", "merge", "conv2d", "dense", "deconv2d"):
                assert rel_err(bnet.activation(i, mb), acts[i].reshape(mb, -1)) <= TOL, (kind, it, "activation", i, sp["name"])
        assert rel_err(bnet.gradients(), onet.grads_flat()) <= TOL, (kind, it, "gradients")
        s_o = onet.fit(x, y); s_b = bnet.fit(x, y)
        assert abs(s_b - s_o) <= TOL * abs(s_o), (kind, it, s_b, s_o)
        assert rel_err(bnet.params(), onet.params_flat()) <= TOL, (kind, it, "params")
        xo = rng.uniform(-1.5, 1.5, (4,) + shape)
        assert rel_err(bnet.output(xo), onet.output(xo).reshape(4, -1)) <= TOL, (kind, it, "output")
    bnet.close()


def _bf16_pair(b, ctx, specs, shape, seed=7, batch=8):
    rng = np.random.default_rng(seed)
    onet = o.net_from_specs(specs, shape, seed=2, flat_input=False); randomize(onet, rng)
    for l in onet.layers:
        if l.has_params and "W" in l.params:
            l.params["W"] = bf16_round(l.params["W"]).astype(np.float64)
    bnet = b.Net(ctx, specs, shape, max_batch=batch, precision=b.BF16)
    push_params(onet, bnet)
    return onet, bnet, rng


def _bf16_check(onet, bnet, x, y, what, gbar=5e-2):
    """The bars of the BF16 net tests elsewhere (test_gpu_cnn_loss.py): score 3e-2, gradients 5e-2, a whole inference forward 2e-2 of the max.
    The inference forward runs on a fresh input of another batch size, so no buffer the train pass left behind can stand in for one it skips."""
    s_o = onet.compute_gradient_and_score(x, y)
    s_b = bnet.compute_gradient_and_score(x, y)
    assert abs(s_b - s_o) <= 3e-2 * abs(s_o), (what, s_b, s_o)
    assert rel_err(bnet.gradients(), onet.grads_flat()) <= gbar, (what, rel_err(bnet.gradients(), onet.grads_flat()))
    x2 = bf16_round(np.random.default_rng(99).uniform(-1, 1, (x.shape[0] - 3,) + x.shape[1:]))
    assert rel_err(bnet.output(x2), onet.output(x2).reshape(x2.shape[0], -1)) <= 2e-2, (what, "output")


@pytest.mark.parametrize("kind", ["residual", "unet", "shared", "ff_merge"])
def test_bf16_graph_nets_match_oracle_loosely(b200, kind):
    b, ctx = b200
    specs, shape, loss = _nets(kind, ch=64)
    onet, bnet, rng = _bf16_pair(b, ctx, specs, shape)
    x = bf16_round(rng.uniform(-1, 1, (8,) + shape))
    y = _labels(loss, rng, (8,) + onet.forward(x, False).shape[1:])
    # the residual block's two BatchNorms compound the bf16 rounding of a whole pass (no layer-by-layer injection) to ~5.1e-2 of the largest
    # gradient element; the FP32 test of the same net pins the arithmetic at 1e-3
    _bf16_check(onet, bnet, x, y, kind, gbar=6e-2 if kind == "residual" else 5e-2)
    bnet.close()


# One BF16 net per single-consumer fusion the engine turns off at a skip source; each would compute another function with the fusion on.
def _guard_net(guard, ch=64):
    u = lambda: m.adam(0.01)
    if guard == "bn_act":           # the BatchNorm is the source: fused with its ReLU, the vertex would read relu(bn) for bn
        body = [_conv("c1", 3, ch), {"type": "batchnorm", "name": "bn1", "updater": u()}, {"type": "activation", "name": "a1", "activation": "relu"},
                _conv("c2", ch, ch), m.elementwise("add", ["c2", "bn1"], name="v")]
    elif guard == "fold":           # the GEMM is the source: folded with the inference BatchNorm after it, its own output would never be written
        body = [_conv("c0", 3, ch, act="tanh"), _conv("c1", ch, ch), {"type": "batchnorm", "name": "bn1", "updater": u()},
                {"type": "activation", "name": "a1", "activation": "relu"}, _conv("c2", ch, ch), m.elementwise("add", ["c2", "c1"], name="v")]
    else:                           # "bwd": c2's tensor-core input gradient (4x4 s2 p1) would premultiply bn1 / a1's derivative (EPI_BNBWD)
        body = [_conv("c0", 3, ch, act="tanh"), _conv("c1", ch, ch), {"type": "batchnorm", "name": "bn1", "updater": u()},   # before the share arrived
                {"type": "activation", "name": "a1", "activation": "lrelu", "alpha": 0.2}, _conv("c2", ch, ch, k=4, s=2, p=1, act="tanh"),
                {"type": "deconv2d", "name": "d3", "n_in": ch, "n_out": ch, "kernel": (4, 4), "stride": (2, 2), "padding": (1, 1), "has_bias": False,
                 "updater": u()}, m.elementwise("add", ["d3", "a1"], name="v")]
    return body + [_conv("head", ch, 2, k=1, p=0), m.cnn_loss("mse", name="loss")], (3, 8, 8)


@pytest.mark.parametrize("guard", ["bn_act", "fold", "bwd"])
def test_bf16_fusion_guards(b200, guard):
    b, ctx = b200
    specs, shape = _guard_net(guard)
    onet, bnet, rng = _bf16_pair(b, ctx, specs, shape)
    x = bf16_round(rng.uniform(-1, 1, (8,) + shape)); y = rng.standard_normal((8, 2, 8, 8))
    _bf16_check(onet, bnet, x, y, guard)      # "fold": the inference forward on the fresh input is where the fold would happen
    bnet.close()


# ------------------------------------------------------------------ the adversarial step -------------------------------------------------
def _residual(size=16, z=12, nf=8, patch=False):
    return m.dcgan_generator(size, z, nf, 3, lr=2e-3, residual=True), m.dcgan_discriminator(size, nf, 3, lr=2e-3, residual=True, patch=patch)


@pytest.mark.parametrize("patch", [False, True])
def test_fp32_residual_gan_step_matches_oracle(b200, patch):
    b, ctx = b200
    size, z, n, lr_ = 16, 12, 8, 2e-3
    gs, ds = _residual(patch=patch)
    G, D = oracle_gan_pair(gs, ds, size, z)
    data = [a.astype(np.float64) for a in o.synthetic_batch(n, size, 3, z, seed=3)]
    labels = [np.broadcast_to(v.reshape(n, 1, 1, 1), (n, 1, 4, 4)).copy() if patch else v for v in data[3:]]
    gan_step_parity(b, ctx, gs, ds, G, D, data, labels, lr_, patch)


def test_bf16_residual_gan_step_runs_and_replays(b200):
    b, ctx = b200
    size, z, n = 32, 16, 16
    gs, ds = _residual(size, z, 64)
    G, D = oracle_gan_pair(gs, ds, size, z)
    data = [a.astype(np.float32) for a in o.synthetic_batch(n, size, 3, z, seed=3)]
    out = {}
    for graph in (True, False):
        bG = b.Net(ctx, gs, (z,), max_batch=n, precision=b.BF16)
        bD = b.Net(ctx, ds, (3, size, size), max_batch=2 * n, precision=b.BF16, bn_groups=2)
        push_params(G, bG); push_params(D, bD)
        gan = b.Gan(bG, bD, use_cuda_graph=graph)
        out[graph] = (np.array([gan.step(*data) for _ in range(3)]), bG.params(), bD.params())
        gan.close(); bG.close(); bD.close()
    assert np.isfinite(out[True][0]).all()
    for u, v in zip(out[True], out[False]):
        assert np.array_equal(u, v), "graph replay == eager"


def test_launch_budget(b200):
    """A vertex costs one launch in the forward; in the backward one plus one per skip source.  The same net with an identity ActivationLayer
    in the vertex's place (one launch each way) is the yardstick."""
    b, ctx = b200
    out = {"type": "output", "name": "out", "n_out": 3, "loss": "mse", "activation": "identity", "updater": m.sgd(0.1)}
    base = [_dense("d1", 16), _dense("d2", 16)]
    vert = base + [m.elementwise("add", ["d2", "d1"], name="v"), _dense("d3", 8), out]
    ident = base + [{"type": "activation", "name": "v", "activation": "identity"}, _dense("d3", 8), out]
    rng = np.random.default_rng(3)
    x, y = rng.standard_normal((4, 10)), rng.standard_normal((4, 3))
    counts = {}
    for name, specs in (("vertex", vert), ("identity", ident)):
        net = b.Net(ctx, specs, (10,), max_batch=4, precision=b.FP32)
        net.output(x); c0 = ctx.launch_count(); net.output(x); c1 = ctx.launch_count()
        net.compute_gradient_and_score(x, y); c2 = ctx.launch_count(); net.compute_gradient_and_score(x, y); c3 = ctx.launch_count()
        counts[name] = (c1 - c0, c3 - c2)
        net.close()
    assert counts["vertex"][0] == counts["identity"][0]
    assert counts["vertex"][1] == counts["identity"][1] + 1       # one skip source


def test_residual_gan_step_launch_budget(b200):
    """The captured adversarial step with residual G and D launches what the same nets launch with a launch-free layer (DropoutLayer p = 1) in
    place of every Add, plus the budget: per forward one launch per vertex, per backward one per vertex and one per skip source.  The step runs
    G forward twice (x_fake, then the G step), D forward twice and backward twice (D step, then the G step through D), G backward once.  FP32,
    so no tensor-core epilogue fusion (the guards' business) enters either count."""
    b, ctx = b200
    size, z, nf, n = 16, 12, 8, 8
    gs = m.dcgan_generator(size, z, nf, 3, residual=True)
    ds = m.dcgan_discriminator(size, nf, 3, residual=True)
    plain = lambda specs: [{"type": "dropout", "name": s["name"], "p": 1.0} if s["type"] == "elementwise" else s for s in specs]
    vs = lambda specs: (sum(s["type"] == "elementwise" for s in specs), len({s["inputs"][1] for s in specs if s["type"] == "elementwise"}))
    (vg, sg), (vd, sd) = vs(gs), vs(ds)
    assert vg == 2 and vd == 2
    data = [a.astype(np.float32) for a in o.synthetic_batch(n, size, 3, z, seed=3)]
    per_step = {}
    for name, (g_specs, d_specs) in (("residual", (gs, ds)), ("plain", (plain(gs), plain(ds)))):
        bG = b.Net(ctx, g_specs, (z,), max_batch=n, precision=b.FP32)
        bD = b.Net(ctx, d_specs, (3, size, size), max_batch=2 * n, precision=b.FP32, bn_groups=2)
        gan = b.Gan(bG, bD, use_cuda_graph=True)
        gan.upload(*data)
        gan.step_resident(n); ctx.sync()
        c0 = ctx.launch_count()
        for _ in range(3):
            gan.step_resident(n)
        ctx.sync()
        per_step[name] = (ctx.launch_count() - c0) / 3
        gan.close(); bG.close(); bD.close()
    budget = 2 * vg + 2 * vd + 2 * (vd + sd) + (vg + sg)
    assert per_step["residual"] == per_step["plain"] + budget, (per_step, budget)


def test_checkpoint_round_trip_restores_the_graph(b200, tmp_path):
    """A checkpoint stores the specs, vertex inputs included: a net built from the file's specs and restored computes what the saved one does."""
    from gan_deeplearning4j_b200 import serializer
    b, ctx = b200
    specs, shape, loss = _nets("unet")
    rng = np.random.default_rng(31)
    net = b.Net(ctx, specs, shape, max_batch=4, precision=b.FP32)
    x = rng.uniform(-1, 1, (4,) + shape)
    y = _labels(loss, rng, (4, 3) + shape[1:])
    net.fit(x, y)
    path = str(tmp_path / "unet.zip")
    net.save(path)
    saved = serializer.read_model(path)
    net2 = b.Net(ctx, saved["specs"], saved["input_shape"], max_batch=4, precision=b.FP32)
    net2.restore(path)
    assert [s.get("inputs") for s in saved["specs"]] == [s.get("inputs") for s in specs]
    assert np.array_equal(net2.output(x), net.output(x))
    assert net2.fit(x, y) == net.fit(x, y)
    net.close(); net2.close()
