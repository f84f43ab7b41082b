"""DL4J's weight constraints on the device (b2g_net_set_constraints / apply_constraints, kernels_constraint.cu): every kind and dims pattern
bit for bit against the emulation of the documented summation order (ew_ref.device_apply), fit and the FP32 GAN step against the oracle,
the bf16 weight operands after constrained updates, and the launches a constraint adds."""
import copy

import numpy as np
import pytest

from helpers import (b200, bf16_gan, check_weight_operands, gan_step_parity, launches_per_step, oracle_gan_pair, pclose, push_params, rel_err,  # noqa: F401
                     run_two_ranks)
from oracle import dl4j_oracle as o
import ew_ref as er
from gan_deeplearning4j_b200 import models as m

pytestmark = pytest.mark.gpu

# odd channel counts (not multiples of 8) and biases of odd length, so W starts at odd offsets of the flattened vector
ODD = [
    {"type": "conv2d", "name": "c1", "n_in": 5, "n_out": 7, "kernel": (3, 3), "stride": (1, 1), "padding": (1, 1), "activation": "relu"},
    {"type": "batchnorm", "name": "bn"},
    {"type": "deconv2d", "name": "d1", "n_in": 7, "n_out": 3, "kernel": (4, 4), "stride": (2, 2), "padding": (1, 1)},
    {"type": "cnn_to_ff", "name": "flat"},
    {"type": "dense", "name": "fc", "n_in": 3 * 12 * 12, "n_out": 37},
    {"type": "output", "name": "out", "n_in": 37, "n_out": 1, "loss": "xent"},
]
KIND = {"c1": "conv", "d1": "conv", "fc": "dense", "out": "dense", "big": "dense"}
PATTERNS = [("c1", "weights", d) for d in ((1, 2, 3), (0,), (2, 3), (), (1,), (0, 1), (0, 3))] + \
           [("d1", "weights", d) for d in ((0, 2, 3), (1, 2, 3))] + \
           [("fc", "weights", d) for d in ((0,), (1,), ())] + \
           [("c1", "bias", d) for d in ((0,), (1,))] + [("bn", "all", (1,))]
BIG = [{"type": "dense", "name": "big", "n_in": 1024, "n_out": 1031}, {"type": "output", "name": "out", "n_in": 1031, "n_out": 1, "loss": "xent"}]


def _tensors(specs, shape, flat):
    on = o.net_from_specs(specs, shape, flat_input=False)
    on.set_params_flat(np.asarray(flat, np.float64))
    return {(l.name, p): np.asarray(v, np.float32) for l in on.layers if l.has_params for p, v in l.params.items()}


def _kinds(rng, norms):
    lo, mid, hi = np.quantile(norms, [0.25, 0.5, 0.75])
    return [m.max_norm(mid, ()), m.min_max_norm(lo, hi, ()), m.min_max_norm(lo, hi, (), rate=0.5), m.unit_norm(()), m.non_negative()]


def _check_apply(b, ctx, specs, shape, cases, rng):
    net = b.Net(ctx, specs, shape, max_batch=4)
    try:
        for layer, on, dims in cases:
            p0 = (rng.standard_normal(net.num_params()) * rng.uniform(0.2, 3.0)).astype(np.float32)
            p0[rng.integers(0, p0.size, 16)] = -0.0
            before = _tensors(specs, shape, p0)
            targets = b.engine.constraint_params(next(s for s in specs if s["name"] == layer), on)
            kind = {p: KIND[layer] if p == "W" else "vector" for p in targets}
            s, _ = er.group_sums(kind[targets[0]], before[(layer, targets[0])], dims)
            for c in _kinds(rng, np.sqrt(s)):
                c = dict(c, dims=list(dims), on=on)
                net.set_params(p0)
                net.set_constraints([c], layer)
                net.apply_constraints()
                got = _tensors(specs, shape, net.params())
                for k, v in got.items():
                    want = er.device_apply(kind[k[1]], before[k], c) if k[0] == layer and k[1] in targets else before[k]   # nothing else moves
                    bad = v.view(np.uint32) != want.view(np.uint32)
                    assert not bad.any(), (layer, k, dims, c, int(bad.sum()), bad.size)
                net.set_constraints(None, layer)
    finally:
        net.close()


def test_apply_constraints_bit_exact_every_kind_and_pattern(b200):
    b, ctx = b200
    _check_apply(b, ctx, ODD, (5, 6, 6), PATTERNS, np.random.default_rng(1))


def test_whole_tensor_group_of_a_million_takes_the_two_launch_path(b200):
    b, ctx = b200
    _check_apply(b, ctx, BIG, (1024,), [("big", "weights", ()), ("big", "weights", (1,))], np.random.default_rng(2))


def _fit_parity(b, ctx, updater):
    specs = m.dcgan_discriminator(16, 8, 3, lr=2e-3)
    for sp in specs:
        if sp.get("updater"):
            sp["updater"] = copy.deepcopy(updater)
    cons = [m.max_norm(0.6, (1, 2, 3)), m.non_negative(on="bias")]
    rng = np.random.default_rng(3)
    on = o.net_from_specs(specs, (3, 16, 16), seed=2, constraints=cons)
    from helpers import randomize
    randomize(on, rng)
    bn = b.Net(ctx, specs, (3, 16, 16), max_batch=8, constraints=cons)
    assert {sp["name"]: r for sp in bn.specs if (r := b.engine.resolve_constraints(sp))} == on.layer_constraints      # the global rule
    push_params(on, bn)
    x = rng.uniform(-1, 1, (8, 3 * 16 * 16)); y = rng.integers(0, 2, (8, 1)).astype(np.float64)
    for it in range(3):
        on.fit(x, y); bn.fit(x, y)
        assert pclose(bn.params(), on.params_flat(), 2 * 2e-3), (updater["kind"], it, rel_err(bn.params(), on.params_flat()))
    # the constraint did bind: every conv W's output units are within the bound
    for l in on.layers:
        if getattr(l, "params", None) and "W" in l.params:
            assert np.sqrt((l.params["W"] ** 2).sum(axis=(1, 2, 3))).max() <= 0.6 + 1e-9
    bn.close()


@pytest.mark.parametrize("updater", [m.adam(2e-3, 0.5), m.rmsprop(2e-3, 0.95, 1e-8)], ids=["adam", "rmsprop"])
def test_fit_parity_with_the_oracle(b200, updater):
    b, ctx = b200
    _fit_parity(b, ctx, updater)


def _wgan_specs(d_cons, g_cons=None):
    gs = m.dcgan_generator(16, 12, 8, 3, lr=2e-3)
    ds = m.dcgan_discriminator(16, 8, 3, lr=2e-3, loss="wasserstein", out_activation="identity")
    for specs, cons in ((ds, d_cons), (gs, g_cons)):
        for sp in specs:
            if cons and sp["type"] in ("conv2d", "deconv2d"):
                sp["constraints"] = copy.deepcopy(cons)
    return gs, ds


WGAN_LABELS = [np.ones((8, 1)), -np.ones((8, 1)), np.ones((8, 1))]


def test_wasserstein_gan_step_parity_with_max_norm_critic(b200):
    """D under MaxNorm per output unit, G per output unit of its deconvs ({0, 2, 3}: strided groups), CUDA graph and eager."""
    b, ctx = b200
    gs, ds = _wgan_specs([m.max_norm(0.5, (1, 2, 3))], [m.max_norm(0.8, (0, 2, 3))])
    G, D = oracle_gan_pair(gs, ds)
    data = [a.astype(np.float64) for a in o.synthetic_batch(8, 16, 3, 12, seed=3)]
    gan_step_parity(b, ctx, gs, ds, G, D, data[:3] + WGAN_LABELS, WGAN_LABELS, 2e-3, "wgan max-norm")


def test_changing_a_constraint_recaptures_the_graph(b200):
    b, ctx = b200
    gs, ds = _wgan_specs([m.max_norm(0.5, (1, 2, 3))])
    G, D = oracle_gan_pair(gs, ds)
    data = [a.astype(np.float64) for a in o.synthetic_batch(8, 16, 3, 12, seed=3)]
    bG = b.Net(ctx, gs, (12,), max_batch=8); bD = b.Net(ctx, ds, (3, 16, 16), max_batch=16, bn_groups=2)
    push_params(G, bG); push_params(D, bD)
    gan = b.Gan(bG, bD, use_cuda_graph=True)
    tighter = [m.max_norm(0.2, (1, 2, 3))]
    for it in range(4):
        if it == 2:
            bD.set_constraints(tighter)
            D.set_constraints(tighter)
        o.gan_step(G, D, *data[:3], *WGAN_LABELS)
        gan.step(*data[:3], *WGAN_LABELS)
        assert pclose(bD.params(), D.params_flat(), 4e-3), (it, rel_err(bD.params(), D.params_flat()))
        assert pclose(bG.params(), G.params_flat(), 4e-3), (it, rel_err(bG.params(), G.params_flat()))
    w = [l.params["W"] for l in D.layers if getattr(l, "params", None) and "W" in l.params]
    assert max(np.sqrt((x ** 2).sum(axis=(1, 2, 3))).max() for x in w) <= 0.2 + 1e-6
    assert all(sp.get("constraints") == tighter for sp in bD.specs if sp["type"] == "conv2d")
    gan.close(); bG.close(); bD.close()


def _bf16_run(b, ctx, d_cons, g_cons, steps=3):
    """BF16 DCGAN 32x32 whose last deconv (64 -> 3 channels) takes the pixel-shuffle operand."""
    gs = m.dcgan_generator(32, 16, 64, 3, lr=2e-3)
    ds = m.dcgan_discriminator(32, 64, 3, lr=2e-3)
    G, D = bf16_gan(b, ctx, gs, ds, (16,), (3, 32, 32), 8)
    if d_cons:
        D.set_constraints(d_cons)
    if g_cons:
        G.set_constraints(g_cons)
    gan = b.Gan(G, D, use_cuda_graph=True)
    data = o.synthetic_batch(8, 32, 3, 16, seed=3)
    gan.upload(*data)
    n = launches_per_step(ctx, gan, 8)
    for _ in range(steps):
        gan.step_resident(8)
    ctx.sync()
    return gs, ds, G, D, gan, n


def _expected_launches(specs, input_shape, cons):
    """Per update of one net given the global constraints cons: 1 if some tensor has a NonNegative or a one-pass group, + 2 if some tensor has
    a two-launch group (one constraint per tensor here: one round)."""
    net = o.net_from_specs(specs, input_shape)
    net.set_constraints(cons)
    paths = set()
    for name, per in net.layer_constraints.items():
        l = net.layer(name)
        for p, (c,) in per.items():
            kind = "vector" if p != "W" else "dense" if isinstance(l, o.Dense) else "conv"
            paths.add("one-pass" if c["constraint"] == "non_negative" else er.constraint_path(kind, l.params[p].shape, c["dims"]))
    return ("one-pass" in paths) + 2 * ("two-launch" in paths)


def test_bf16_operands_follow_the_constrained_master_and_launch_counts(b200):
    """After constrained BF16 updates the straight and packed pixel-shuffle bf16 copies equal bf16(master) bit for bit; a constrained GAN step
    launches what an unconstrained one does plus the stated rounds; two identical runs give identical bits."""
    b, ctx = b200
    # D: whole-tensor groups (conv 3->64: 3072 elements, one pass; the others above 4096: two launches, contiguous); G: per output unit of its
    # deconvs, strided groups (two launches; the last deconv's scale pass writes the packed pixel-shuffle operand)
    d_cons, g_cons = [m.max_norm(1.0, ())], [m.max_norm(0.8, (0, 2, 3))]
    gs, ds, G0, D0, gan0, n0 = _bf16_run(b, ctx, None, None)
    assert _expected_launches(ds, (3, 32, 32), d_cons) == 3 and _expected_launches(gs, (16,), g_cons) == 2       # every path runs
    gan0.close(); G0.close(); D0.close()
    runs = []
    for _ in range(2):
        gs, ds, G, D, gan, n = _bf16_run(b, ctx, d_cons, g_cons)
        assert check_weight_operands(b, G, gs, "G") >= 1           # the pixel-shuffle last deconv was checked
        check_weight_operands(b, D, ds, "D")
        runs.append((G.params(), D.params(), n))
        gan.close(); G.close(); D.close()
    assert np.array_equal(runs[0][0], runs[1][0]) and np.array_equal(runs[0][1], runs[1][1])
    assert runs[0][2] == n0 + _expected_launches(ds, (3, 32, 32), d_cons) + _expected_launches(gs, (16,), g_cons), (n0, runs[0][2])


def test_two_ranks_match_one_gpu(tmp_path):
    d = run_two_ranks("dp_check.py", tmp_path / "constraint_dp.json", 29563, args=("constraint",))
    assert d["world"] == 2 and d["params_identical_across_ranks"] is True and d["max_rel_err_vs_one_gpu"] < 1e-5
