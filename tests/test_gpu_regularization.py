"""DL4J's l1, l2, l1Bias and l2Bias on the device (b2g_net_set_regularization): FP32 fit of every updater kind against the oracle on the MLP,
conv + BatchNorm and odd-width (scalar updater path) nets, also with a schedule, gradient normalization and constraints; the score and
calcL1 / calcL2 against the oracle; nets without the new terms unchanged bit for bit and launch for launch; the GAN step against the oracle
(graph replay == eager) and a change between replays; the bf16 weight operands; two ranks."""
import numpy as np
import pytest

from gan_deeplearning4j_b200 import models as m
from helpers import (b200, bf16_gan, check_weight_operands, compare_params_and_state, gan_step_parity, launches_per_step,  # noqa: F401
                     mlp_convbn_specs, oracle_gan_pair, pclose, push_params, randomize, rel_err, run_two_ranks)
from oracle import dl4j_oracle as o

pytestmark = pytest.mark.gpu
TOL = 1e-3
KINDS = ("sgd", "rmsprop", "adam", "noop") + o.EXT_UPDATERS
# l1 comparable to the updater steps, so that weights near 0 cross it within three updates
REG = {"l1": 2e-3, "l2": 1e-2, "l1_bias": 1e-3, "l2_bias": 5e-3}
GEMM = ("conv2d", "deconv2d", "dense", "output")


def _upd(kind):
    if kind == "noop":
        return m.noop()
    if kind == "adadelta":
        return m.adadelta(0.95, 1e-6)
    if kind == "sgd":
        return m.sgd(0.05)
    if kind in ("nesterovs", "adagrad"):
        return getattr(m, kind)(0.02)
    if kind == "nadam":
        return m.nadam(2e-4)
    return getattr(m, kind)(2e-3)


def _bound(kind):
    """Twice the largest step an element with a numerically zero gradient can take (as in test_gpu_updaters), plus 2 l1: an element the
    update leaves within rounding of 0 may take the other sign of l1 on the device."""
    step = {"nesterovs": 0.02, "adagrad": 0.02, "adamax": 2e-3, "nadam": 2e-4 * 1.9 / np.sqrt(1e-3), "amsgrad": 2e-3, "adam": 2e-3,
            "adadelta": np.sqrt(1e-6 / 0.05), "rmsprop": 2e-3 / np.sqrt(0.05), "sgd": 0.0, "noop": 0.0}[kind]
    return 2 * step + 2 * REG["l1"]


def _specs(net, kind, reg=REG):
    """'mlp' / 'convbn' / 'odd' (every segment of odd length: the updater's scalar path), every layer on `kind`, every GEMM layer with reg;
    the BatchNorm spec carries reg too, which BatchNorm ignores."""
    u = lambda: _upd(kind)
    if net == "odd":
        specs, shape = [{"type": "dense", "name": "d1", "n_out": 37, "activation": "tanh", "updater": u()},
                        {"type": "dense", "name": "d2", "n_out": 23, "activation": "lrelu", "alpha": 0.2, "updater": u()},
                        {"type": "output", "name": "out", "n_out": 1, "updater": u()}], (13,)
    else:
        specs, shape = mlp_convbn_specs(net, u)
    for s in specs:
        if s["type"] in GEMM + ("batchnorm",):
            s.update(reg)
    return specs, shape


def _oracle(specs, shape, seed, grad_clip):
    """The oracle net with random biases / BatchNorm parameters and every 11th weight exactly 0 (sign 0)."""
    rng = np.random.default_rng(seed)
    onet = o.net_from_specs(specs, shape, seed=2, grad_clip=grad_clip)
    randomize(onet, rng)
    for l in onet.layers:
        if getattr(l, "params", None) and "W" in l.params:
            l.params["W"].reshape(-1)[::11] = 0.0
    return onet, rng


def _fit_and_compare(b, ctx, specs, shape, steps=3, grad_clip=0.5, seed=11, oracle_grad_norm=None, **net_kw):
    onet, rng = _oracle(specs, shape, seed, grad_clip)
    if oracle_grad_norm:
        onet.set_gradient_normalization(*oracle_grad_norm)
    bnet = b.Net(ctx, specs, shape, max_batch=6, precision=b.FP32, grad_clip=grad_clip, **net_kw)
    push_params(onet, bnet)
    w0 = bnet.params()
    bounds = {s["name"]: _bound(s["updater"]["kind"]) for s in specs if s.get("updater")}
    for it in range(steps):
        x, y = rng.uniform(-1, 1, (6,) + shape), rng.uniform(0, 1, (6, 1))
        onet.fit(x, y); bnet.fit(x, y)
        compare_params_and_state(onet, bnet, it, TOL, bounds)
    assert np.any((w0 > 0) & (bnet.params() < 0)) or np.any((w0 < 0) & (bnet.params() > 0)), "no weight crossed 0"
    return onet, bnet


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("net", ["mlp", "convbn", "odd"])
def test_fp32_fit_matches_oracle(b200, net, kind):
    b, ctx = b200
    specs, shape = _specs(net, kind)
    _, bnet = _fit_and_compare(b, ctx, specs, shape)
    bnet.close()


@pytest.mark.parametrize("kind", ["adam", "nesterovs", "amsgrad"])
def test_fp32_fit_with_schedule_gradient_normalization_and_constraints(b200, kind):
    b, ctx = b200
    specs, shape = _specs("mlp", kind)
    for s in specs:
        s["updater"]["lr"] = m.exponential_schedule(s["updater"]["lr"], 0.8)
    _fit_and_compare(b, ctx, specs, shape)[1].close()
    specs, shape = _specs("convbn", kind)
    _fit_and_compare(b, ctx, specs, shape, grad_clip=0.0, gradient_normalization="clip_l2_per_layer", gradient_normalization_threshold=0.05,
                     oracle_grad_norm=("clip_l2_per_layer", 0.05))[1].close()
    specs, shape = _specs("mlp", kind)
    for s in specs:
        s["constraints"] = [m.max_norm(1.0, (0,))]
    _fit_and_compare(b, ctx, specs, shape)[1].close()


def test_score_and_calc_regularization_match_the_oracle(b200):
    b, ctx = b200
    cases = [{k: REG[k]} for k in REG] + [REG]
    for reg in cases:
        specs, shape = _specs("convbn", "adam", reg)
        specs[0]["frozen"] = True                           # a FrozenLayer takes no term
        onet, rng = _oracle(specs, shape, 3, 0.0)
        bnet = b.Net(ctx, specs, shape, max_batch=6, precision=b.FP32)
        push_params(onet, bnet)
        x, y = rng.uniform(-1, 1, (6,) + shape), rng.uniform(0, 1, (6, 1))
        want = onet.compute_gradient_and_score(x, y)
        got = bnet.compute_gradient_and_score(x, y)
        assert abs(got - want) <= 1e-5 * abs(want), (reg, got, want)
        l1, l2 = bnet.calc_regularization()
        assert abs(l1 - onet.calc_l1()) <= 1e-6 * max(onet.calc_l1(), 1e-30) and abs(l2 - onet.calc_l2()) <= 1e-6 * max(onet.calc_l2(), 1e-30), reg
        assert (l1 > 0) == bool(reg.get("l1") or reg.get("l1_bias")) and (l2 > 0) == bool(reg.get("l2") or reg.get("l2_bias")), reg
        bnet.close()


def _fit_run(b, ctx, specs, shape, setup=None, steps=3):
    """Scores, final parameters and kernel launches of `steps` fits from the same data and parameters."""
    rng = np.random.default_rng(8)
    net = b.Net(ctx, specs, shape, max_batch=6, precision=b.FP32, seed=4)
    if setup:
        setup(net)
    ctx.sync(); l0 = ctx.launch_count()
    scores = [net.fit(rng.uniform(-1, 1, (6,) + shape), rng.uniform(0, 1, (6, 1))) for _ in range(steps)]
    ctx.sync()
    out = (np.array(scores), net.params(), net.updater_state(), ctx.launch_count() - l0)
    net.close()
    return out


def _same(u, v):
    for a, c in zip(u, v):
        assert np.array_equal(a, c), (a, c)


def test_unused_settings_change_nothing(b200):
    """A net given all-zero coefficients equals one never given any, bit for bit and launch for launch; set_regularization(l2=x) equals the
    desc's l2 = x; the named form replaces one layer's coefficients only."""
    b, ctx = b200
    specs, shape = mlp_convbn_specs("convbn", lambda: m.adam(2e-3))
    plain = _fit_run(b, ctx, specs, shape)
    _same(plain, _fit_run(b, ctx, specs, shape, lambda n: n.set_regularization()))
    _same(plain, _fit_run(b, ctx, specs, shape, lambda n: n.set_regularization(l1=0.0, l2=0.0, layer="c1")))
    with_l2 = [dict(s, l2=1e-2) if s["type"] in GEMM else s for s in specs]
    desc = _fit_run(b, ctx, with_l2, shape)
    _same(desc, _fit_run(b, ctx, specs, shape, lambda n: n.set_regularization(l2=1e-2)))
    assert not np.array_equal(desc[1], plain[1]) and desc[3] == plain[3] + 3          # the l2 sum of each fit's score
    full = _fit_run(b, ctx, specs, shape, lambda n: n.set_regularization(**REG))
    assert full[3] == desc[3] + 3, "one more score launch (the l1 sum) per fit, nothing else"
    one = _fit_run(b, ctx, specs, shape, lambda n: n.set_regularization(l2=1e-2, layer="fc"))
    net = b.Net(ctx, specs, shape, max_batch=6)
    net.set_regularization(l2=1e-2, layer="fc")
    assert net.get_regularization("fc") == {"l1": 0.0, "l2": np.float32(1e-2), "l1_bias": 0.0, "l2_bias": 0.0}
    assert net.get_regularization("c1") == {"l1": 0.0, "l2": 0.0, "l1_bias": 0.0, "l2_bias": 0.0}
    assert [s.get("l2") for s in net.specs] == [None] * 6 + [1e-2, None]
    net.close()
    assert not np.array_equal(one[1], plain[1])


def test_rejections(b200):
    b, ctx = b200
    import ctypes as C
    from gan_deeplearning4j_b200 import engine
    specs, shape = mlp_convbn_specs("convbn", lambda: m.adam(2e-3))
    net = b.Net(ctx, specs, shape, max_batch=4)
    for bad in (-1e-4, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            net.set_regularization(l1_bias=bad)
        r = engine.regularization_struct({"l2": bad})
        assert ctx.lib.b2g_net_set_regularization(net.h, None, C.byref(r)) == -1
    for layer in (b"nope", b"bn2", b"a1"):          # unknown, BatchNorm, no parameters
        r = engine.regularization_struct(REG)
        assert ctx.lib.b2g_net_set_regularization(net.h, layer, C.byref(r)) == -1, layer
        assert ctx.lib.b2g_net_get_regularization(net.h, layer, C.byref(r)) == -1, layer
    assert net.calc_regularization() == (0.0, 0.0)
    with pytest.raises(ValueError):
        b.Net(ctx, specs, shape, max_batch=4, regularization={"l3": 1.0})
    net.close()


def _reg_gan_specs(reg_g, reg_d):
    gs, ds = m.dcgan_generator(16, 12, 8, 3, lr=2e-3), m.dcgan_discriminator(16, 8, 3, lr=2e-3)
    for specs, reg in ((gs, reg_g), (ds, reg_d)):
        for s in specs:
            if s["type"] in GEMM:
                s.update(reg)
    return gs, ds


def test_gan_step_matches_oracle_graph_and_eager(b200):
    b, ctx = b200
    gs, ds = _reg_gan_specs(REG, {"l1": 1e-3, "l2": 2e-2, "l1_bias": 2e-3, "l2_bias": 1e-2})
    G, D = oracle_gan_pair(gs, ds)
    data = [a.astype(np.float64) for a in o.synthetic_batch(8, 16, 3, 12, seed=3)]
    gan_step_parity(b, ctx, gs, ds, G, D, data, data[3:], 2e-3 + REG["l1"], "regularized G and D")


def test_a_change_between_replays_takes_effect(b200):
    b, ctx = b200
    gs, ds = _reg_gan_specs({}, {"l2": 1e-2})
    G, D = oracle_gan_pair(gs, ds)
    data = [a.astype(np.float64) for a in o.synthetic_batch(8, 16, 3, 12, seed=3)]
    bG = b.Net(ctx, gs, (12,), max_batch=8); bD = b.Net(ctx, ds, (3, 16, 16), max_batch=16, bn_groups=2)
    push_params(G, bG); push_params(D, bD)
    gan = b.Gan(bG, bD, use_cuda_graph=True)
    last = [s["name"] for s in gs if s["type"] in GEMM][-1]
    for it in range(4):
        if it == 2:                     # the step is captured by now: the new values must reach the replay
            bD.set_regularization(**REG); bG.set_regularization(l1=5e-3, layer=last)
            for l in D.layers:
                if isinstance(l, (o.Conv2D, o.Dense)):
                    l.l2 = REG["l2"]
                    D.layer_regularization[l.name] = (REG["l1"], REG["l1_bias"], REG["l2_bias"])
            G.layer_regularization[last] = (5e-3,) + G.layer_regularization.get(last, (0.0, 0.0, 0.0))[1:]
        o.gan_step(G, D, *data)
        gan.step(*data)
        assert pclose(bD.params(), D.params_flat(), 2 * (2e-3 + REG["l1"])), (it, rel_err(bD.params(), D.params_flat()))
        assert pclose(bG.params(), G.params_flat(), 2 * (2e-3 + 5e-3)), (it, rel_err(bG.params(), G.params_flat()))
    assert bD.specs[0]["l1"] == REG["l1"] and [s.get("l1") for s in bG.specs if s["type"] in GEMM][-2:] == [None, 5e-3]
    gan.close(); bG.close(); bD.close()


def test_bf16_operands_and_launch_counts(b200):
    """BF16 DCGAN 32x32 (the last deconv takes the packed pixel-shuffle operand): after regularized steps every bf16 weight operand equals
    bf16(master); a regularized step launches what an l2-only one does; two identical runs give identical bits."""
    b, ctx = b200
    runs = []
    for reg in ({"l2": 1e-4}, REG, REG):
        gs, ds = m.dcgan_generator(32, 16, 64, 3, lr=2e-3), m.dcgan_discriminator(32, 64, 3, lr=2e-3)
        G, D = bf16_gan(b, ctx, gs, ds, (16,), (3, 32, 32), 8)
        G.set_regularization(**reg); D.set_regularization(**reg)
        gan = b.Gan(G, D, use_cuda_graph=True)
        gan.upload(*o.synthetic_batch(8, 32, 3, 16, seed=3))
        n = launches_per_step(ctx, gan, 8)
        assert check_weight_operands(b, G, gs, "G") == 1
        check_weight_operands(b, D, ds, "D")
        runs.append((G.params(), D.params(), n))
        gan.close(); G.close(); D.close()
    assert runs[0][2] == runs[1][2] == runs[2][2]
    assert np.array_equal(runs[1][0], runs[2][0]) and np.array_equal(runs[1][1], runs[2][1])
    assert not np.array_equal(runs[0][1], runs[1][1])


def test_two_ranks_match_one_gpu(tmp_path):
    d = run_two_ranks("dp_check.py", tmp_path / "regularization_dp.json", 29571, args=("regularization",))
    assert d["world"] == 2 and d["params_identical_across_ranks"] is True and d["max_rel_err_vs_one_gpu"] < 1e-5
