"""DL4J's Nesterovs, AdaGrad, AdaMax, Nadam, AMSGrad and AdaDelta on the GPU: FP32 fit of every kind against the oracle on an MLP and a
conv+BatchNorm net (parameters and every state slot), a net that mixes kinds per layer, odd widths (the scalar path), gradient normalization
and schedules, the FP32 GAN step against the oracle, BF16 graph replay against eager and the bf16 weight copies, AMSGrad checkpoint / resume,
parameter averaging, launch counts and argument checks."""
import copy

import numpy as np
import pytest

from gan_deeplearning4j_b200 import models as m
from helpers import (b200, bf16_gan, check_weight_operands, compare_params_and_state, fp32_gan_pair, launches_per_step, mlp_convbn_specs,
                     push_params, randomize, run_two_ranks)
from oracle import dl4j_oracle as o

pytestmark = pytest.mark.gpu
TOL = 1e-3
KINDS = o.EXT_UPDATERS


def _upd(kind, lr=None):
    """One updater spec of `kind` at test-sized hyperparameters (lr may be a schedule; AdaDelta has none)."""
    lr = copy.deepcopy(lr)
    if kind == "nesterovs":
        return m.nesterovs(0.02 if lr is None else lr, 0.9)
    if kind == "adagrad":
        return m.adagrad(0.02 if lr is None else lr)
    if kind == "adadelta":
        return m.adadelta(0.95, 1e-6)
    if kind == "nadam":
        return m.nadam(2e-4 if lr is None else lr)
    return getattr(m, kind)(2e-3 if lr is None else lr)


def _step_bound(kind):
    """Twice the largest step an element whose gradient is numerically zero can take (the sign of such a gradient is not reproducible in
    fp32): about lr for the sign-like first steps, 1.9 / sqrt(1 - b2) lr for Nadam's, sqrt(eps / (1 - rho)) for AdaDelta's."""
    return 2 * {"nesterovs": 0.02, "adagrad": 0.02, "adamax": 2e-3, "nadam": 2e-4 * 1.9 / np.sqrt(1e-3), "amsgrad": 2e-3,
                "adadelta": np.sqrt(1e-6 / 0.05), "adam": 2e-3, "sgd": 0.0}[kind]


def _specs(net, kinds):
    """net 'mlp' / 'convbn' / 'odd'; kinds: one kind for every layer, or a list cycled over the layers with parameters."""
    ks = [kinds] if isinstance(kinds, str) else list(kinds)
    it = iter(ks * 8)
    u = lambda: _upd(next(it))
    if net == "odd":          # every segment length odd: the updater's scalar path
        return [{"type": "dense", "name": "d1", "n_out": 37, "activation": "tanh", "updater": u(), "l2": 1e-3},
                {"type": "dense", "name": "d2", "n_out": 23, "activation": "lrelu", "alpha": 0.2, "updater": u()},
                {"type": "output", "name": "out", "n_out": 1, "updater": u()}], (13,)
    specs, shape = mlp_convbn_specs(net, u)
    if net == "convbn":
        specs[0]["l2"] = 1e-3
    return specs, shape


def _with_kind(specs, kind):
    """specs with every updater replaced by one of `kind`; Adam's specs as they are."""
    return specs if kind == "adam" else [dict(s, updater=_upd(kind)) if s.get("updater") else s for s in specs]


def _bounds(specs):
    return {s["name"]: _step_bound(s["updater"]["kind"]) for s in specs if s.get("updater")}


def _fit_and_compare(b, ctx, specs, shape, steps=6, grad_clip=0.5, seed=11, **net_kw):
    rng = np.random.default_rng(seed)
    onet = o.net_from_specs(specs, shape, seed=2, grad_clip=grad_clip); randomize(onet, rng)
    if "oracle_grad_norm" in net_kw:
        onet.set_gradient_normalization(*net_kw.pop("oracle_grad_norm"))
    bnet = b.Net(ctx, specs, shape, max_batch=6, precision=b.FP32, grad_clip=grad_clip, **net_kw)
    push_params(onet, bnet)
    for it in range(steps):
        x, y = rng.uniform(-1, 1, (6,) + shape), rng.uniform(0, 1, (6, 1))
        onet.fit(x, y); bnet.fit(x, y)
        compare_params_and_state(onet, bnet, it, TOL, _bounds(specs))
    assert bnet.iteration() == steps
    return onet, bnet


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("net", ["mlp", "convbn"])
def test_fp32_fit_matches_oracle(b200, net, kind):
    b, ctx = b200
    specs, shape = _specs(net, kind)
    _, bnet = _fit_and_compare(b, ctx, specs, shape)
    assert bnet.updater_state_size() == (3 if kind == "amsgrad" else 2) * bnet.num_params()
    bnet.close()


def test_fp32_fit_mixed_kinds_per_layer(b200):
    b, ctx = b200
    specs, shape = _specs("convbn", ["amsgrad", "nesterovs", "adadelta", "adamax", "nadam", "adagrad"])
    _, bnet = _fit_and_compare(b, ctx, specs, shape, steps=5)
    bnet.close()
    specs, shape = _specs("mlp", "adagrad")
    specs[0]["updater"], specs[2]["updater"] = m.adam(2e-3), m.sgd(0.05)      # existing kinds beside a new one, one updater pass
    _, bnet = _fit_and_compare(b, ctx, specs, shape, steps=4)
    bnet.close()


@pytest.mark.parametrize("kind", KINDS)
def test_fp32_fit_odd_widths_take_the_scalar_path(b200, kind):
    b, ctx = b200
    specs, shape = _specs("odd", kind)
    _, bnet = _fit_and_compare(b, ctx, specs, shape, steps=5)
    bnet.close()


@pytest.mark.parametrize("kind", KINDS)
def test_clip_l2_per_layer_and_exponential_schedule(b200, kind):
    b, ctx = b200
    specs, shape = _specs("mlp", kind)
    if kind != "adadelta":
        for s in specs:
            s["updater"]["lr"] = m.exponential_schedule(s["updater"]["lr"], 0.8)
    _, bnet = _fit_and_compare(b, ctx, specs, shape, steps=5, grad_clip=0.0, gradient_normalization="clip_l2_per_layer",
                               gradient_normalization_threshold=0.05, oracle_grad_norm=("clip_l2_per_layer", 0.05))
    if kind != "adadelta":
        assert abs(bnet.learning_rate("d1") - np.float32(_upd(kind)["lr"] * 0.8 ** 5)) <= 1e-6 * _upd(kind)["lr"]
    bnet.close()


def test_adadelta_refuses_a_learning_rate_schedule(b200):
    b, ctx = b200
    specs, shape = _specs("mlp", ["adadelta", "adam", "adadelta"])
    net = b.Net(ctx, specs, shape, max_batch=4)
    for layer in ("d1", "out"):
        with pytest.raises(b.B200GanError) as e:
            net.set_lr_schedule(m.exponential_schedule(1e-2, 0.9), layer)
        assert e.value.code == -1
        with pytest.raises(b.B200GanError):
            net.learning_rate(layer)
    net.set_lr_schedule(m.exponential_schedule(1e-2, 0.9))             # every layer with a learning rate: d2 only
    assert net.learning_rate("d2") == np.float32(1e-2)
    assert "lr" not in net.specs[0]["updater"] and net.specs[1]["updater"]["lr"]["schedule"] == "exponential"
    net.close()


def test_fp32_gan_step_matches_oracle(b200):
    """G on Nesterovs, D on AMSGrad (three state slots), CUDA-graph replay after the first step."""
    b, ctx = b200
    n = 8
    gs, ds = _with_kind(m.dcgan_generator(16, 12, 8, 3), "nesterovs"), _with_kind(m.dcgan_discriminator(16, 8, 3), "amsgrad")
    G, D, bG, bD, data = fp32_gan_pair(b, ctx, gs, ds, n)
    gan = b.Gan(bG, bD, use_cuda_graph=True)
    for it in range(5):
        r = o.gan_step(G, D, *data)
        lo = gan.step(*data)
        want = np.array([r["loss_d_real"], r["loss_d_fake"], r["loss_g"]])
        assert np.all(np.abs(lo - want) < TOL * np.maximum(1, np.abs(want))), (it, lo, want)
        compare_params_and_state(D, bD, (it, "D"), 2 * TOL, _bounds(ds)); compare_params_and_state(G, bG, (it, "G"), 2 * TOL, _bounds(gs))
    assert bD.updater_state_size() == 3 * bD.num_params() and bG.updater_state_size() == 2 * bG.num_params()
    gan.close(); bG.close(); bD.close()


def _bf16_dcgan(b, ctx, n, gkinds, dkinds, size=32):
    z, nf = 16, 64
    gs, ds = m.dcgan_generator(size, z, nf, 3), m.dcgan_discriminator(size, nf, 3)
    for specs, kinds in ((gs, gkinds), (ds, dkinds)):
        it = iter(list(kinds) * 8)
        for s in specs:
            if s.get("updater"):
                s["updater"] = _upd(next(it))
    G = b.Net(ctx, gs, (z,), max_batch=n, precision=b.BF16, xent_clip_eps=0.0)
    D = b.Net(ctx, ds, (3, size, size), max_batch=2 * n, precision=b.BF16, xent_clip_eps=0.0, bn_groups=2)
    data = [a.astype(np.float32) for a in o.synthetic_batch(n, size, 3, z, seed=3)]
    return gs, ds, G, D, data


GK, DK = ("nesterovs", "adamax", "adagrad", "amsgrad"), ("nadam", "adadelta", "amsgrad")


def test_bf16_graph_replay_matches_eager(b200):
    b, ctx = b200
    n = 8
    runs = []
    for graph in (False, True):
        _, _, G, D, data = _bf16_dcgan(b, ctx, n, GK, DK)
        gan = b.Gan(G, D, use_cuda_graph=graph)
        losses = [gan.step(*data) for _ in range(5)]
        runs.append((np.array(losses), G.params(), D.params(), G.updater_state(), D.updater_state(), G.iteration(), D.iteration()))
        gan.close(); G.close(); D.close()
    for a, c in zip(*runs):
        assert np.array_equal(a, c)
    assert np.abs(runs[0][1]).max() > 0 and runs[0][5] == 5


def test_bf16_weight_copies_track_the_master(b200):
    b, ctx = b200
    for gk, dk in ((GK, DK), (("amsgrad",), ("adadelta", "nesterovs"))):
        gs, ds, G, D, data = _bf16_dcgan(b, ctx, 8, gk, dk)
        gan = b.Gan(G, D, use_cuda_graph=True)
        g0 = G.params()
        for it in range(3):
            gan.step(*data)
            assert check_weight_operands(b, G, gs, f"G step {it}") == 1      # G's last layer: the packed pixel-shuffle operand
            check_weight_operands(b, D, ds, f"D step {it}")
        assert np.abs(G.params() - g0).max() > 0
        gan.close(); G.close(); D.close()


def test_amsgrad_checkpoint_resume_is_bit_identical(b200, tmp_path):
    b, ctx = b200
    from gan_deeplearning4j_b200 import serializer
    specs, shape = _specs("convbn", ["amsgrad", "amsgrad", "nadam", "amsgrad", "adagrad"])
    rng = np.random.default_rng(4)
    batches = [(rng.uniform(-1, 1, (6,) + shape), rng.uniform(0, 1, (6, 1))) for _ in range(7)]
    full = b.Net(ctx, specs, shape, max_batch=6, precision=b.FP32, seed=9)
    for x, y in batches:
        full.fit(x, y)
    first = b.Net(ctx, specs, shape, max_batch=6, precision=b.FP32, seed=9)
    for x, y in batches[:4]:
        first.fit(x, y)
    path = str(tmp_path / "ckpt.zip")
    first.save(path)
    saved = serializer.read_model(path)
    assert saved["updater_state"].size == 3 * first.num_params() and saved["meta"]["iteration"] == 4
    assert [s.get("updater", {}).get("kind") for s in saved["specs"]] == [s.get("updater", {}).get("kind") for s in specs]
    resumed = b.Net(ctx, saved["specs"], shape, max_batch=6, precision=b.FP32, seed=1)
    resumed.restore(path)
    assert resumed.iteration() == 4 and np.array_equal(resumed.updater_state(), first.updater_state())
    for x, y in batches[4:]:
        resumed.fit(x, y)
    assert np.array_equal(full.params(), resumed.params()) and np.array_equal(full.updater_state(), resumed.updater_state())
    assert resumed.iteration() == full.iteration() == 7
    n = full.num_params()
    assert np.abs(full.updater_state()[2 * n:]).max() > 0                 # the third slot holds AMSGrad's v-hat
    for net in (full, first, resumed):
        net.close()


def test_single_process_parameter_averaging_with_amsgrad_matches_oracle(b200):
    b, ctx = b200
    from gan_deeplearning4j_b200 import parallel
    specs, shape = _specs("mlp", "amsgrad")
    rng = np.random.default_rng(17)
    onet = o.net_from_specs(specs, shape, seed=2, grad_clip=0.5); randomize(onet, rng)
    bnet = b.Net(ctx, specs, shape, max_batch=8, precision=b.FP32, grad_clip=0.5)
    push_params(onet, bnet)
    for rnd in range(2):
        d = [(rng.uniform(-1, 1, (8,) + shape), rng.uniform(0, 1, (8, 1))) for _ in range(2)]
        w0, w1 = copy.deepcopy(onet), copy.deepcopy(onet)
        w0.fit(*d[0]); w1.fit(*d[1])
        o.parameter_average([w0, w1], onet); onet.iteration = w0.iteration
        parallel.fit_parameter_averaging(bnet, d, averaging_frequency=10)
        compare_params_and_state(onet, bnet, ("averaging", rnd), TOL, _bounds(specs))
    assert bnet.iteration() == 2
    bnet.close()


def test_launch_counts_do_not_change(b200):
    """C2 (bench.py's DCGAN 64x64, bf16, batch 128) launches 83 kernels per step and a C5-shaped MLP-GAN 46, with Adam and with every new kind."""
    b, ctx = b200
    rng = np.random.default_rng(1)

    def per_step(gs, ds, gin, din, n):
        G, D = bf16_gan(b, ctx, gs, ds, gin, din, n)
        gan = b.Gan(G, D, use_cuda_graph=True)
        x = rng.uniform(-1, 1, (n,) + tuple(din))
        gan.upload(x, rng.uniform(-1, 1, (n,) + tuple(gin)), rng.uniform(-1, 1, (n,) + tuple(gin)), np.ones((n, 1)), np.zeros((n, 1)), np.ones((n, 1)))
        out = launches_per_step(ctx, gan, n)
        gan.close(); G.close(); D.close()
        return out

    for kind in ("adam",) + KINDS:
        assert per_step(_with_kind(m.dcgan_generator(64, 100, 64, 3), kind), _with_kind(m.dcgan_discriminator(64, 64, 3), kind), (100,), (3, 64, 64), 128) == 83, kind
        assert per_step(_with_kind(m.mlp_generator(128, 1024, 256), kind), _with_kind(m.mlp_discriminator(256, 1024), kind), (128,), (256,), 8192) == 46, kind


def test_rejections(b200):
    b, ctx = b200
    import ctypes as C
    from gan_deeplearning4j_b200 import _lib, engine
    specs, shape = _specs("mlp", "amsgrad")
    for bad in (10, -1, 1000):
        descs = [engine.layer_desc(s) for s in specs]
        descs[1].updater = bad
        arr = (_lib.LayerDesc * len(descs))(*descs)
        cfg = _lib.NetConfig(1, 1, shape[0], 4, 0, 0.0, 1e-5, 1, 666)
        h = C.c_void_p()
        assert ctx.lib.b2g_net_create(ctx.h, C.byref(cfg), arr, len(descs), C.byref(h)) == -1, bad
        assert b"unknown updater" in ctx.lib.b2g_last_error()
    with pytest.raises(KeyError):
        b.Net(ctx, [dict(specs[0], updater={"kind": "lamb", "lr": 1e-3})], shape, max_batch=4)
    net = b.Net(ctx, specs, shape, max_batch=4)
    n = net.num_params()
    assert net.updater_state_size() == 3 * n
    with pytest.raises(b.B200GanError):
        net.set_updater_state(np.zeros(2 * n, np.float32))                # an AMSGrad net takes three slots
    net.close()


def test_two_ranks_average_every_state_slot(tmp_path):
    d = run_two_ranks("dp_check.py", tmp_path / "updater_dp.json", 29551, args=("updater",))
    assert d["world"] == 2 and d["state_slots"] == 3 and d["ranks_differed"] is True
    assert d["max_rel_err_params"] < 1e-6 and max(d["max_rel_err_slot"]) < 1e-6
