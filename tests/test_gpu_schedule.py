"""Learning-rate schedules on the GPU: the device-evaluated rate of every kind and type against the oracle's lr_at, FP32 fit and the fused
GAN step against the oracle, CUDA-graph replay against eager bit for bit (an epoch change without a re-capture, a schedule change with one),
identity schedules, checkpoint / resume, the bf16 weight copies, launch counts and argument checks."""
import copy

import numpy as np
import pytest

from gan_deeplearning4j_b200 import models as m
from helpers import (b200, bf16_gan, check_weight_operands, compare_params_and_state, fp32_gan_pair, launches_per_step, mlp_convbn_specs,
                     push_params, randomize)
from oracle import dl4j_oracle as o

pytestmark = pytest.mark.gpu
TOL = 1e-3


def _specs(kind, upd, lr):
    mk = {"sgd": lambda: m.sgd(copy.deepcopy(lr)), "rmsprop": lambda: m.rmsprop(copy.deepcopy(lr), 0.9, 1e-8), "adam": lambda: m.adam(copy.deepcopy(lr))}[upd]
    return mlp_convbn_specs(kind, mk)


def _f32_close(got, want) -> bool:
    """The device evaluates pow / exp in double like the restatement; after the one rounding to fp32 they may differ by one fp32 ulp."""
    want = np.float32(want)
    return abs(np.float32(got) - want) <= np.spacing(want)


def _all_schedules(type_):
    return [m.exponential_schedule(0.1, 0.97, type=type_), m.inverse_schedule(0.1, 0.01, 0.75, type=type_),
            m.sigmoid_schedule(0.1, 0.05, 10, type=type_), m.step_schedule(0.1, 0.5, 10, type=type_), m.step_schedule(0.3, 0.7, 2.5, type=type_),
            m.map_schedule({0: 0.1, 10: 0.05, 100: 0.01, 12345: 1e-4}, type=type_)]


@pytest.mark.parametrize("type_", ["iteration", "epoch"])
def test_learning_rate_of_every_kind_matches_the_restatement(b200, type_):
    b, ctx = b200
    specs, shape = _specs("mlp", "adam", 0.02)
    net = b.Net(ctx, specs, shape, max_batch=4)
    counters = (0, 1, 2, 9, 10, 11, 12, 99, 100, 101, 12344, 12345, 100000)
    for sched in _all_schedules(type_):
        net.set_lr_schedule(sched, "d2")
        for c in counters:
            other = 7 + c % 5                      # the counter the schedule does not read must not matter
            net.set_iteration(c if type_ == "iteration" else other); net.set_epoch(c if type_ == "epoch" else other)
            got, want = net.learning_rate("d2"), o.lr_at(sched, c if type_ == "iteration" else other, c if type_ == "epoch" else other)
            assert _f32_close(got, want), (sched, c, got, want)
            assert net.learning_rate("d1") == np.float32(0.02)        # unscheduled layers keep their constant lr
    net.set_lr_schedule(None, "d2")
    assert net.learning_rate("d2") == np.float32(0.02)
    net.close()


def _fit_run(b, ctx, kind, upd, sched_name):
    lr0 = 0.05 if upd == "sgd" else 1e-2
    sched = m.step_schedule(lr0, 0.5, 3) if sched_name == "step" else m.map_schedule({0: lr0, 2: 0.3 * lr0, 5: 0.6 * lr0})
    specs, shape = _specs(kind, upd, sched)
    rng = np.random.default_rng(11)
    onet = o.net_from_specs(specs, shape, seed=2); randomize(onet, rng)
    bnet = b.Net(ctx, specs, shape, max_batch=6, precision=b.FP32)
    push_params(onet, bnet)
    return onet, bnet, shape, rng


@pytest.mark.parametrize("sched_name", ["step", "map"])
@pytest.mark.parametrize("upd", ["sgd", "rmsprop", "adam"])
@pytest.mark.parametrize("kind", ["mlp", "convbn"])
def test_fp32_fit_matches_oracle(b200, kind, upd, sched_name):
    b, ctx = b200
    onet, bnet, shape, rng = _fit_run(b, ctx, kind, upd, sched_name)
    seen = set()
    for it in range(8):
        x, y = rng.uniform(-1, 1, (6,) + shape), rng.uniform(0, 1, (6, 1))
        name = onet.layers[-1].name
        assert _f32_close(bnet.learning_rate(name), onet.learning_rate(name))
        seen.add(float(bnet.learning_rate(name)))
        onet.fit(x, y); bnet.fit(x, y)
        compare_params_and_state(onet, bnet, (kind, upd, sched_name, it), TOL)
    assert len(seen) == 3, seen                    # the run crossed two schedule boundaries
    bnet.close()


def test_set_and_clear_mid_run_take_effect_at_the_next_update(b200):
    b, ctx = b200
    specs, shape = _specs("mlp", "adam", 1e-2)
    rng = np.random.default_rng(3)
    onet = o.net_from_specs(specs, shape, seed=2); randomize(onet, rng)
    bnet = b.Net(ctx, specs, shape, max_batch=6, precision=b.FP32)
    push_params(onet, bnet)
    names = ["d1", "d2", "out"]
    plan = [None, None, ("all", m.exponential_schedule(2e-2, 0.8)), None, ("d2", m.map_schedule({0: 1e-3, 4: 5e-3}, type="epoch")), None,
            ("all", "clear"), None]
    for it, change in enumerate(plan):
        if change is not None:
            layer, sched = change
            sched = None if sched == "clear" else sched
            bnet.set_lr_schedule(sched, None if layer == "all" else layer)
            onet.set_lr_schedule(sched, None if layer == "all" else layer)
        if it == 5:
            bnet.set_epoch(4); onet.set_epoch(4)
        x, y = rng.uniform(-1, 1, (6,) + shape), rng.uniform(0, 1, (6, 1))
        onet.fit(x, y); bnet.fit(x, y)
        compare_params_and_state(onet, bnet, ("plan", it), TOL)
    assert bnet.learning_rate("d2") == np.float32(1e-2)
    bnet.close()


def test_fp32_gan_step_matches_oracle(b200):
    b, ctx = b200
    n = 8
    gs, ds = m.dcgan_generator(16, 12, 8, 3, lr=m.exponential_schedule(2e-3, 0.8)), m.dcgan_discriminator(16, 8, 3, lr=m.step_schedule(2e-3, 0.5, 2))
    G, D, bG, bD, data = fp32_gan_pair(b, ctx, gs, ds, n)
    gan = b.Gan(bG, bD, use_cuda_graph=True)
    for it in range(5):
        r = o.gan_step(G, D, *data)
        lo = gan.step(*data)
        want = np.array([r["loss_d_real"], r["loss_d_fake"], r["loss_g"]])
        assert np.all(np.abs(lo - want) < TOL * np.maximum(1, np.abs(want))), (it, lo, want)
        compare_params_and_state(D, bD, (it, "D"), 2 * TOL); compare_params_and_state(G, bG, (it, "G"), 2 * TOL)
    assert _f32_close(bD.learning_rate("dis_conv_1"), 2e-3 * 0.25) and _f32_close(bG.learning_rate("gen_deconv_1"), 2e-3 * 0.8 ** 5)
    gan.close(); bG.close(); bD.close()


def _bf16_dcgan(b, ctx, n, size=32, gsched=2e-3, dsched=2e-3):
    z, nf = 16, 64
    gs, ds = m.dcgan_generator(size, z, nf, 3, lr=gsched), m.dcgan_discriminator(size, nf, 3, lr=dsched)
    G = b.Net(ctx, gs, (z,), max_batch=n, precision=b.BF16, xent_clip_eps=0.0)
    D = b.Net(ctx, ds, (3, size, size), max_batch=2 * n, precision=b.BF16, xent_clip_eps=0.0, bn_groups=2)
    data = [a.astype(np.float32) for a in o.synthetic_batch(n, size, 3, z, seed=3)]
    return gs, ds, G, D, data


def test_graph_replay_matches_eager_with_epoch_and_schedule_changes(b200):
    """BF16 GAN steps, eager and from CUDA graphs: an EPOCH schedule on G whose epoch changes between replays (no re-capture needed), and a
    schedule set on D mid-run and cleared again (re-captures).  Losses, parameters and updater state agree bit for bit."""
    b, ctx = b200
    n = 8
    gsched = m.step_schedule(2e-3, 0.5, 1, type="epoch")
    runs = []
    for graph in (False, True):
        _, _, G, D, data = _bf16_dcgan(b, ctx, n, gsched=gsched)
        gan = b.Gan(G, D, use_cuda_graph=graph)
        losses, g_lrs = [], []
        for it in range(7):
            G.set_epoch(it // 2)
            if it == 2:
                D.set_lr_schedule(m.inverse_schedule(4e-3, 0.5, 1.0))
            if it == 5:
                D.set_lr_schedule(None)
            g_lrs.append(G.learning_rate("gen_deconv_1"))
            losses.append(gan.step(*data))
        runs.append((np.array(losses), G.params(), D.params(), G.updater_state(), D.updater_state(), g_lrs))
        gan.close(); G.close(); D.close()
    (le, ge, de, sge, sde, lre), (lg, gg, dg, sgg, sdg, lrg) = runs
    assert np.array_equal(le, lg) and np.array_equal(ge, gg) and np.array_equal(de, dg) and np.array_equal(sge, sgg) and np.array_equal(sde, sdg)
    assert lre == lrg and all(_f32_close(v, 2e-3 * 0.5 ** (it // 2)) for it, v in enumerate(lre)), lre


def test_identity_schedules_are_bit_identical_to_none_through_the_graph(b200):
    b, ctx = b200
    n = 8
    runs = []
    for g_lr, d_lr in ((2e-3, 2e-3), (m.exponential_schedule(2e-3, 1.0), m.map_schedule({0: 2e-3}, type="epoch"))):
        _, _, G, D, data = _bf16_dcgan(b, ctx, n, gsched=g_lr, dsched=d_lr)
        D.set_epoch(3)
        gan = b.Gan(G, D, use_cuda_graph=True)
        losses = [gan.step(*data) for _ in range(4)]
        runs.append((np.array(losses), G.params(), D.params(), G.updater_state(), D.updater_state()))
        gan.close(); G.close(); D.close()
    for a, c in zip(*runs):
        assert np.array_equal(a, c)


def test_checkpoint_resume_is_bit_identical(b200, tmp_path):
    """Save after k fits (the schedules live in the checkpoint's specs, the epoch in its metadata), restore into a fresh net built from the
    checkpoint's specs, continue: the same parameters and state as an uninterrupted run."""
    b, ctx = b200
    from gan_deeplearning4j_b200 import serializer
    specs, shape = _specs("mlp", "adam", m.step_schedule(1e-2, 0.5, 2))
    rng = np.random.default_rng(4)
    batches = [(rng.uniform(-1, 1, (6,) + shape), rng.uniform(0, 1, (6, 1))) for _ in range(7)]

    def start():
        net = b.Net(ctx, specs, shape, max_batch=6, precision=b.FP32, seed=9)
        net.set_lr_schedule(m.map_schedule({0: 3e-3, 2: 1e-3}, type="epoch"), "out")
        return net

    full = start()
    for i, (x, y) in enumerate(batches):
        full.set_epoch(i // 3); full.fit(x, y)
    first = start()
    for i, (x, y) in enumerate(batches[:4]):
        first.set_epoch(i // 3); first.fit(x, y)
    path = str(tmp_path / "ckpt.zip")
    first.save(path)
    saved = serializer.read_model(path)
    assert saved["meta"]["epoch"] == 1 and saved["meta"]["iteration"] == 4
    assert saved["specs"][2]["updater"]["lr"] == {"schedule": "map", "type": "epoch", "values": [[0, 3e-3], [2, 1e-3]]}
    assert saved["specs"][0]["updater"]["lr"]["schedule"] == "step"
    resumed = b.Net(ctx, saved["specs"], shape, max_batch=6, precision=b.FP32, seed=1)
    resumed.restore(path)
    assert resumed.epoch() == 1 and resumed.iteration() == 4
    for i, (x, y) in enumerate(batches[4:], start=4):
        resumed.set_epoch(i // 3); resumed.fit(x, y)
    assert np.array_equal(full.params(), resumed.params()) and np.array_equal(full.updater_state(), resumed.updater_state())
    assert resumed.learning_rate("out") == np.float32(1e-3) and _f32_close(resumed.learning_rate("d1"), 1e-2 * 0.5 ** 3)
    for net in (full, first, resumed):
        net.close()


def test_bf16_weight_copies_track_the_master(b200):
    b, ctx = b200
    gs, ds, G, D, data = _bf16_dcgan(b, ctx, 8, gsched=m.sigmoid_schedule(4e-3, 0.5, 2), dsched=m.map_schedule({0: 2e-3, 2: 5e-3}))
    gan = b.Gan(G, D, use_cuda_graph=True)
    g0 = G.params()
    for it in range(4):
        gan.step(*data)
        check_weight_operands(b, G, gs, f"G step {it}"); check_weight_operands(b, D, ds, f"D step {it}")
    assert np.abs(G.params() - g0).max() > 0
    gan.close(); G.close(); D.close()


def test_launch_counts(b200):
    """C2 (bench.py's DCGAN 64x64, bf16, batch 128) launches 83 kernels per step with and without schedules; fit launches the same."""
    b, ctx = b200
    n = 128
    G, D = bf16_gan(b, ctx, m.dcgan_generator(64, 100, 64, 3), m.dcgan_discriminator(64, 64, 3), (100,), (3, 64, 64), n)
    gan = b.Gan(G, D, use_cuda_graph=True)
    rng = np.random.default_rng(1)
    gan.upload(rng.uniform(-1, 1, (n, 3, 64, 64)), rng.uniform(-1, 1, (n, 100)), rng.uniform(-1, 1, (n, 100)), np.ones((n, 1)), np.zeros((n, 1)), np.ones((n, 1)))
    assert launches_per_step(ctx, gan, n) == 83
    G.set_lr_schedule(m.exponential_schedule(2e-4, 0.999)); D.set_lr_schedule(m.map_schedule({0: 2e-4, 3: 1e-4}, type="epoch"))
    assert launches_per_step(ctx, gan, n) == 83
    G.set_lr_schedule(None); D.set_lr_schedule(None)
    assert launches_per_step(ctx, gan, n) == 83
    gan.close(); G.close(); D.close()
    specs, shape = _specs("mlp", "adam", 1e-3)
    net = b.Net(ctx, specs, shape, max_batch=4, precision=b.FP32)
    x, y = rng.uniform(-1, 1, (4,) + shape), rng.uniform(0, 1, (4, 1))
    counts = []
    for sched in (None, m.step_schedule(1e-3, 0.5, 1), None):
        net.set_lr_schedule(sched)
        l0 = ctx.launch_count(); net.fit(x, y); counts.append(ctx.launch_count() - l0)
    assert counts[0] == counts[1] == counts[2]
    net.close()


def test_rejections(b200):
    b, ctx = b200
    import ctypes as C
    from gan_deeplearning4j_b200 import _lib
    specs = [{"type": "dense", "name": "d1", "n_out": 8, "activation": "tanh", "updater": m.adam(1e-3), "frozen": True},
             {"type": "dense", "name": "d2", "n_out": 8, "activation": "tanh", "updater": {"kind": "noop"}},
             {"type": "activation", "name": "act", "activation": "relu"},
             {"type": "output", "name": "out", "n_out": 1, "updater": m.sgd(0.1)}]
    net = b.Net(ctx, specs, (4,), max_batch=4)

    def raw(layer=b"out", **kw):
        s = _lib.LrSchedule(); s.kind, s.type, s.initial, s.gamma, s.power, s.step, s.decay_rate = 1, 0, 0.1, 0.9, 1.0, 1.0, 0.5
        keys = (C.c_int32 * 3)(0, 5, 9); vals = (C.c_double * 3)(0.1, 0.2, 0.3)
        s.n_map, s.map_keys, s.map_values = 3, keys, vals
        for k, v in kw.items():
            setattr(s, k, v)
        return net.lib.b2g_net_set_lr_schedule(net.h, layer, C.byref(s))

    assert raw() == 0 and raw(kind=5) == 0 and raw(kind=4) == 0 and raw(kind=2) == 0 and raw(kind=3, step=-4.0) == 0 and raw(type=1) == 0
    assert raw(layer=None) == 0                   # every layer with a learning rate: only "out" here
    for kw in (dict(kind=6), dict(kind=-1), dict(kind=100), dict(type=2), dict(type=-1), dict(initial=float("nan")), dict(gamma=float("inf")),
               dict(power=float("nan")), dict(step=float("-inf")), dict(decay_rate=float("nan")), dict(kind=4, step=0.0), dict(kind=4, step=-1.0),
               dict(kind=2, gamma=-0.1), dict(kind=5, n_map=0)):
        assert raw(**kw) == -1, kw
    bad_maps = (((1, 5, 9), (0.1, 0.2, 0.3)), ((0, 5, 5), (0.1, 0.2, 0.3)), ((0, 9, 5), (0.1, 0.2, 0.3)), ((0, 5, 9), (0.1, float("nan"), 0.3)))
    for keys, vals in bad_maps:
        assert raw(kind=5, map_keys=(C.c_int32 * 3)(*keys), map_values=(C.c_double * 3)(*vals)) == -1, (keys, vals)
    for layer in (b"nope", b"d1", b"d2", b"act"):          # unknown, frozen, NoOp, no parameters
        assert raw(layer=layer) == -1, layer
        assert net.lib.b2g_net_get_learning_rate(net.h, layer, C.byref(C.c_float())) == -1, layer
    assert net.lib.b2g_net_set_lr_schedule(net.h, b"out", None) == 0
    assert net.lib.b2g_net_set_epoch(net.h, -1) == -1
    with pytest.raises(ValueError):
        net.set_lr_schedule({"schedule": "poly", "initial": 0.1})
    with pytest.raises(b.B200GanError) as e:
        net.set_lr_schedule(m.map_schedule({1: 0.1}))
    assert e.value.code == -1
    assert net.learning_rate("out") == np.float32(0.1)     # failed calls left the constant lr
    net.close()
