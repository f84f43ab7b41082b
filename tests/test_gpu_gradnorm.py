"""L2 gradient normalization on the GPU: FP32 fit and the fused GAN step against the oracle's restatement for all four
modes, eager against CUDA-graph replay bit for bit (a mode change re-captures), the bf16 weight copies after normalized updates, launch counts,
argument checks and two ranks."""
import copy

import numpy as np
import pytest

from gan_deeplearning4j_b200 import models as m
from helpers import (b200, bf16_gan, check_weight_operands, compare_params_and_state, fp32_gan_pair, launches_per_step, mlp_convbn_specs,
                     push_params, randomize, run_two_ranks)
from oracle import dl4j_oracle as o

pytestmark = pytest.mark.gpu
TOL = 1e-3
L2_MODES = ("renormalize_l2_per_layer", "renormalize_l2_per_param_type", "clip_l2_per_layer", "clip_l2_per_param_type")


def _specs(kind, upd):
    u = lambda: m.sgd(0.05) if upd == "sgd" else m.adam(1e-2)
    if kind == "ragged":       # 7 -> 999 -> 33 -> 1: segments at offsets 6993, 7992, ... (not multiples of 4): the scalar branches
        return [{"type": "dense", "name": "d1", "n_out": 999, "activation": "tanh", "updater": u()},
                {"type": "dense", "name": "d2", "n_out": 33, "activation": "relu", "updater": u(), "l2": 1e-3},
                {"type": "output", "name": "out", "n_out": 1, "updater": u()}], (7,)
    return mlp_convbn_specs(kind, u)


def _threshold_between(norms):
    """A ClipL2 threshold strictly between the smallest and the largest group norm, so that both branches run."""
    lo, hi = min(n for n in norms if n > 0), max(norms)
    assert hi > 1.5 * lo, norms
    return float(np.sqrt(lo * hi))


@pytest.mark.parametrize("mode", L2_MODES)
@pytest.mark.parametrize("upd", ["sgd", "adam"])
@pytest.mark.parametrize("kind", ["mlp", "ragged", "convbn"])
def test_fp32_fit_matches_oracle(b200, kind, upd, mode):
    b, ctx = b200
    specs, shape = _specs(kind, upd)
    rng = np.random.default_rng(11)
    onet = o.net_from_specs(specs, shape, seed=2); randomize(onet, rng)
    n = 6
    xs = [rng.uniform(-1, 1, (n,) + shape) for _ in range(3)]; ys = [rng.uniform(0, 1, (n, 1)) for _ in range(3)]
    thr = 1.0
    if mode.startswith("clip"):        # dry run: the first update's group norms
        probe = copy.deepcopy(onet); probe.set_gradient_normalization(mode, 1e30)
        probe.fit(xs[0], ys[0])
        thr = _threshold_between(probe.grad_norm_last_norms)
    onet.set_gradient_normalization(mode, thr)
    bnet = b.Net(ctx, specs, shape, max_batch=n, precision=b.FP32, gradient_normalization=mode, gradient_normalization_threshold=thr)
    push_params(onet, bnet)
    clipped = []
    for it in range(3):
        onet.fit(xs[it], ys[it]); bnet.fit(xs[it], ys[it])
        if mode.startswith("clip"):
            clipped += [nm > thr for nm in onet.grad_norm_last_norms]
        compare_params_and_state(onet, bnet, (kind, upd, mode, it), TOL)
    if mode.startswith("clip"):
        assert any(clipped) and not all(clipped), clipped
    bnet.close()


def _normalized_pair(b, ctx, n, gmode, dmode, gthr=1.0, dthr=1.0):
    """fp32_gan_pair of the 16x16 DCGAN with G's gradient normalization (mode, threshold) gmode, gthr and D's dmode, dthr on both sides."""
    gs, ds = m.dcgan_generator(16, 12, 8, 3, lr=2e-3), m.dcgan_discriminator(16, 8, 3, lr=2e-3)
    G, D, bG, bD, data = fp32_gan_pair(b, ctx, gs, ds, n, g_kw=dict(gradient_normalization=gmode, gradient_normalization_threshold=gthr),
                                       d_kw=dict(gradient_normalization=dmode, gradient_normalization_threshold=dthr))
    G.set_gradient_normalization(gmode, gthr); D.set_gradient_normalization(dmode, dthr)
    return G, D, bG, bD, data


def _gan_norms(b, ctx, n, mode):
    """The group norms of the first step's D and G updates (oracle), for a threshold between them."""
    G, D, bG, bD, data = _normalized_pair(b, ctx, n, mode, mode, 1e30, 1e30)
    bG.close(); bD.close()
    o.gan_step(G, D, *data)
    return G.grad_norm_last_norms, D.grad_norm_last_norms


@pytest.mark.parametrize("mode", L2_MODES)
def test_fp32_gan_step_matches_oracle(b200, mode):
    b, ctx = b200
    n = 8
    gthr = dthr = 1.0
    if mode.startswith("clip"):
        gn, dn = _gan_norms(b, ctx, n, mode)
        gthr, dthr = _threshold_between(gn), _threshold_between(dn)
    G, D, bG, bD, data = _normalized_pair(b, ctx, n, mode, mode, gthr, dthr)
    gan = b.Gan(bG, bD, use_cuda_graph=True)
    for it in range(3):
        r = o.gan_step(G, D, *data)
        lo = gan.step(*data)
        want = np.array([r["loss_d_real"], r["loss_d_fake"], r["loss_g"]])
        assert np.all(np.abs(lo - want) < TOL * np.maximum(1, np.abs(want))), (mode, it, lo, want)
        compare_params_and_state(D, bD, (mode, it, "D"), 2 * TOL); compare_params_and_state(G, bG, (mode, it, "G"), 2 * TOL)
    gan.close(); bG.close(); bD.close()


def test_mnist_example_configuration_with_dropout(b200):
    """DL4J's MNIST GAN example: mlp_generator + mlp_discriminator(dropout=0.5), RenormalizeL2PerLayer on both nets, FP32, under the masks of
    the oracle's dropout_mask."""
    b, ctx = b200
    n, z, hid, d = 16, 24, 64, 48
    gs, ds = m.mlp_generator(z, hid, d, lr=1e-3), m.mlp_discriminator(d, hid, lr=1e-3, dropout=0.5)
    rng = np.random.default_rng(9)
    G = o.net_from_specs(gs, (z,), seed=1); D = o.net_from_specs(ds, (d,), mask_seed=667, seed=2)
    randomize(G, rng); randomize(D, rng)
    mode = "renormalize_l2_per_layer"
    G.set_gradient_normalization(mode); D.set_gradient_normalization(mode)
    bG = b.Net(ctx, gs, (z,), max_batch=n, precision=b.FP32, gradient_normalization=mode)
    bD = b.Net(ctx, ds, (d,), max_batch=2 * n, precision=b.FP32, bn_groups=2, seed=667, gradient_normalization=mode)
    push_params(G, bG); push_params(D, bD)
    gan = b.Gan(bG, bD, use_cuda_graph=True)
    data = [rng.uniform(-1, 1, (n, d)), rng.uniform(-1, 1, (n, z)), rng.uniform(-1, 1, (n, z)),
            1 + 0.05 * rng.standard_normal((n, 1)), 0.05 * rng.standard_normal((n, 1)), np.ones((n, 1))]
    for it in range(3):
        r = o.gan_step(G, D, *data)
        lo = gan.step(*data)
        want = np.array([r["loss_d_real"], r["loss_d_fake"], r["loss_g"]])
        assert np.all(np.abs(lo - want) < TOL * np.maximum(1, np.abs(want))), (it, lo, want)
        compare_params_and_state(D, bD, (it, "D"), 2 * TOL); compare_params_and_state(G, bG, (it, "G"), 2 * TOL)
        assert len(D.grad_norm_last_norms) == 3 and len(G.grad_norm_last_norms) == 3
    gan.close(); bG.close(); bD.close()


def test_graph_replay_matches_eager_and_recaptures_on_a_mode_change(b200):
    """The same sequence of steps and mode changes, eager and from CUDA graphs: identical losses and parameters bit for bit.  A changed mode
    re-captures: the launch count per step follows the mode."""
    b, ctx = b200
    n = 8
    plan = [("renormalize_l2_per_layer", 1.0)] * 2 + [("clip_l2_per_param_type", 0.05)] * 2 + [("none", 1.0)] + [("clip_l2_per_layer", 0.2)] * 2
    runs = []
    for graph in (False, True):
        G, D, bG, bD, data = _normalized_pair(b, ctx, n, "none", "none")
        gan = b.Gan(bG, bD, use_cuda_graph=graph)
        losses, launches = [], []
        for mode, thr in plan:
            bG.set_gradient_normalization(mode, thr); bD.set_gradient_normalization(mode, thr)
            l0 = ctx.launch_count()
            losses.append(gan.step(*data))
            launches.append(ctx.launch_count() - l0)
        runs.append((np.array(losses), bG.params(), bD.params(), bG.updater_state(), bD.updater_state(), launches))
        gan.close(); bG.close(); bD.close()
    (le, ge, de, se_g, se_d, ne), (lg, gg, dg, sg_g, sg_d, ng) = runs
    assert np.array_equal(le, lg) and np.array_equal(ge, gg) and np.array_equal(de, dg) and np.array_equal(se_g, sg_g) and np.array_equal(se_d, sg_d)
    assert ne == ng, (ne, ng)
    none_step = ne[4]
    for (mode, _), k in zip(plan, ne):
        assert k == none_step + (0 if mode == "none" else 2), (mode, k, none_step)


def test_launch_counts(b200):
    """C2 (bench.py's DCGAN 64x64, bf16, batch 128) launches 83 kernels per step without a mode, 85 with an L2 mode on both nets (one norm
    kernel per update); fit adds exactly one launch."""
    b, ctx = b200
    n = 128
    G, D = bf16_gan(b, ctx, m.dcgan_generator(64, 100, 64, 3), m.dcgan_discriminator(64, 64, 3), (100,), (3, 64, 64), n)
    gan = b.Gan(G, D, use_cuda_graph=True)
    rng = np.random.default_rng(1)
    gan.upload(rng.uniform(-1, 1, (n, 3, 64, 64)), rng.uniform(-1, 1, (n, 100)), rng.uniform(-1, 1, (n, 100)), np.ones((n, 1)), np.zeros((n, 1)), np.ones((n, 1)))
    assert launches_per_step(ctx, gan, n) == 83
    G.set_gradient_normalization("clip_l2_per_layer", 1.0); D.set_gradient_normalization("renormalize_l2_per_layer")
    assert launches_per_step(ctx, gan, n) == 85
    G.set_gradient_normalization("none"); D.set_gradient_normalization("none")
    assert launches_per_step(ctx, gan, n) == 83
    gan.close(); G.close(); D.close()
    specs, shape = _specs("mlp", "adam")
    net = b.Net(ctx, specs, shape, max_batch=4, precision=b.FP32)
    x, y = rng.uniform(-1, 1, (4,) + shape), rng.uniform(0, 1, (4, 1))
    counts = []
    for mode in ("none", "renormalize_l2_per_param_type", "none"):
        net.set_gradient_normalization(mode)
        l0 = ctx.launch_count(); net.fit(x, y); counts.append(ctx.launch_count() - l0)
    assert counts[1] == counts[0] + 1 and counts[2] == counts[0]
    net.close()


def test_bf16_weight_copies_track_the_master(b200):
    """BF16 DCGAN 32x32 (G-last on the pixel-shuffle operand) with L2 modes through graph steps, and a fit net whose pixel-shuffle W sits at
    flat offset 3 (the updater's scalar branch): every bf16 weight copy equals the rounded fp32 master."""
    b, ctx = b200
    size, z, nf, n = 32, 16, 64, 8
    gs, ds = m.dcgan_generator(size, z, nf, 3, lr=2e-3), m.dcgan_discriminator(size, nf, 3, lr=2e-3)
    G = b.Net(ctx, gs, (z,), max_batch=n, precision=b.BF16, xent_clip_eps=0.0, gradient_normalization="renormalize_l2_per_layer")
    D = b.Net(ctx, ds, (3, size, size), max_batch=2 * n, precision=b.BF16, xent_clip_eps=0.0, bn_groups=2,
              gradient_normalization="clip_l2_per_param_type", gradient_normalization_threshold=0.01)
    gan = b.Gan(G, D, use_cuda_graph=True)
    data = [a.astype(np.float32) for a in o.synthetic_batch(n, size, 3, z, seed=3)]
    g0 = G.params()
    for it in range(3):
        gan.step(*data)
        check_weight_operands(b, G, gs, f"G step {it}"); check_weight_operands(b, D, ds, f"D step {it}")
    assert np.abs(G.params() - g0).max() > 0
    gan.close(); G.close(); D.close()
    u = m.adam(1e-3)
    specs = [{"type": "deconv2d", "name": "ps", "n_in": 64, "n_out": 3, "kernel": (4, 4), "stride": (2, 2), "padding": (1, 1), "has_bias": True,
              "activation": "tanh", "updater": u, "l2": 1e-3},
             {"type": "conv2d", "name": "c1", "n_in": 3, "n_out": 64, "kernel": (4, 4), "stride": (2, 2), "padding": (1, 1), "activation": "lrelu",
              "alpha": 0.2, "updater": u},
             {"type": "conv2d", "name": "c2", "n_in": 64, "n_out": 1, "kernel": (8, 8), "updater": u},
             {"type": "loss", "name": "loss"}]
    rng = np.random.default_rng(8)
    for mode in ("renormalize_l2_per_param_type", "clip_l2_per_layer"):
        net = b.Net(ctx, specs, (64, 8, 8), max_batch=6, precision=b.BF16, gradient_normalization=mode, gradient_normalization_threshold=0.05)
        for it in range(3):
            net.fit(rng.standard_normal((6, 64, 8, 8)).astype(np.float32), rng.uniform(0, 1, (6, 1)).astype(np.float32))
            check_weight_operands(b, net, specs, f"{mode} fit {it}")
        net.close()


def test_rejections(b200):
    b, ctx = b200
    specs, shape = _specs("mlp", "sgd")
    net = b.Net(ctx, specs, shape, max_batch=4)
    set_raw = lambda mode, thr: net.lib.b2g_net_set_gradient_normalization(net.h, mode, thr)
    assert set_raw(3, 1.0) == -1 and "grad_clip" in net.lib.b2g_last_error().decode()
    for mode in (-1, 6, 7, 100):
        assert set_raw(mode, 1.0) == -1
    for mode in (4, 5):
        for thr in (0.0, -1.0, float("nan"), float("inf")):
            assert set_raw(mode, thr) == -1, (mode, thr)
    for mode in (0, 1, 2):
        assert set_raw(mode, 0.0) == 0           # the renormalize modes ignore the threshold
    with pytest.raises(ValueError):
        net.set_gradient_normalization("clip_element_wise_absolute_value")
    with pytest.raises(b.B200GanError) as e:
        net.set_gradient_normalization("clip_l2_per_layer", 0.0)
    assert e.value.code == -1
    net.close()
    clipped = b.Net(ctx, specs, shape, max_batch=4, grad_clip=1.0)
    for mode in (1, 2, 4, 5):
        assert clipped.lib.b2g_net_set_gradient_normalization(clipped.h, mode, 1.0) == -1
    assert clipped.lib.b2g_net_set_gradient_normalization(clipped.h, 0, 1.0) == 0
    clipped.close()
    with pytest.raises(b.B200GanError) as e:
        b.Net(ctx, specs, shape, max_batch=4, grad_clip=1.0, gradient_normalization="renormalize_l2_per_layer")
    assert e.value.code == -1


def test_two_ranks_match_one_gpu(tmp_path):
    d = run_two_ranks("dp_check.py", tmp_path / "gradnorm_dp.json", 29549, args=("gradnorm",))
    assert d["world"] == 2 and d["params_identical_across_ranks"] is True and d["max_rel_err_vs_one_gpu"] < 1e-5
