"""Weight noise (DropConnect, WeightNoise; b2g_weight_noise in include/b200gan.h) on the GPU against the oracle's restatement: the noisy
operands bit for bit (the Normal draws within the fp32 Box-Muller tolerance), FP32 training parity through every GEMM route of a small chain,
the BF16 nets loosely, the adversarial step graph-replayed, eager and restated, and the launches and pass counter of the identity cases."""
import numpy as np
import pytest

from helpers import (b200, bf16_gan, bf16_round, fp32_gan_pair, gan_step_parity, launches_per_step, oracle_gan_pair, pack_deconv_ps, pclose,
                     push_params, randomize, rel_err, w_internal)
from oracle import dl4j_oracle as o

pytestmark = pytest.mark.gpu
_ = b200

DC = {"weight_noise": "drop_connect", "p": 0.7, "apply_to_bias": True}
UNI = {"weight_noise": "weight_noise", "distribution": {"distribution": "uniform", "lower": 0.5, "upper": 1.5}, "apply_to_bias": True, "additive": False}
NORMAL = {"weight_noise": "weight_noise", "distribution": {"distribution": "normal", "mean": 0.01, "std": 0.05}, "apply_to_bias": True, "additive": True}
SCHED = {"weight_noise": "drop_connect", "p": {"schedule": "exponential", "initial": 0.8, "gamma": 0.5, "type": "iteration"}, "apply_to_bias": True}


def _operand_specs(wn):
    """conv (5 biases first: W at an odd parameter offset) -> conv onto 64 channels -> the 4x4 s2 p1 deconv onto 3 channels (packed pixel-shuffle
    operand in BF16 nets) -> dense -> output, every GEMM layer noisy."""
    return [{"type": "conv2d", "name": "c1", "n_in": 3, "n_out": 5, "kernel": (3, 3), "padding": (1, 1), "activation": "lrelu", "alpha": 0.2, "weight_noise": wn},
            {"type": "conv2d", "name": "c2", "n_in": 5, "n_out": 64, "kernel": (4, 4), "stride": (2, 2), "padding": (1, 1), "activation": "relu", "weight_noise": wn},
            {"type": "deconv2d", "name": "dc", "n_in": 64, "n_out": 3, "kernel": (4, 4), "stride": (2, 2), "padding": (1, 1), "activation": "tanh", "weight_noise": wn},
            {"type": "cnn_to_ff", "name": "flat"},
            {"type": "dense", "name": "d", "n_in": 192, "n_out": 16, "activation": "tanh", "weight_noise": wn},
            {"type": "output", "name": "out", "n_in": 16, "n_out": 1, "weight_noise": wn}]


def _sizes(s):
    k = s.get("kernel", (1, 1))
    return s["n_in"] * s["n_out"] * k[0] * k[1], s["n_out"]


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("name,wn", [("dropconnect", DC), ("scheduled", SCHED), ("uniform", UNI), ("normal", NORMAL)])
def test_noisy_operands_match_the_restatement(b200, prec, name, wn):
    """After two fits (passes P = 0, 1; a scheduled p at iterations 0 and 1) every layer's W', packed W' and b' are the restatement's of the
    second pass from the library's own parameters of that pass: bit for bit, or for Normal within 8 fp32 ulps of the noise (bf16: within the
    bf16 rounding of the restated value)."""
    b, ctx = b200
    precision = b.BF16 if prec == "bf16" else b.FP32
    specs = _operand_specs(wn)
    net = b.Net(ctx, specs, (3, 8, 8), max_batch=4, precision=precision, seed=21)
    rng = np.random.default_rng(3)
    x = rng.uniform(-1, 1, (4, 3, 8, 8)); y = rng.uniform(0, 1, (4, 1))
    net.fit(x, y)
    theta = {s["name"]: (net.get_param(s["name"], "W", _sizes(s)[0]), net.get_param(s["name"], "b", _sizes(s)[1])) for s in specs if "n_out" in s}
    net.compute_gradient_and_score(x, y)          # the second pass draws from theta (compute_gradient_and_score does not update)
    assert net.dropout_pass() == 2
    packed = 0
    for li, s in enumerate(specs):
        if "n_out" not in s:
            continue
        nw, nb = _sizes(s)
        w = w_internal(s, theta[s["name"]][0]).astype(np.float32)
        bias = theta[s["name"]][1].astype(np.float32)
        p = o.drop_connect_p(wn, (1, 0)) if wn["weight_noise"] == "drop_connect" else None
        ref_w = o.weight_noise_apply(wn, w, o.weight_noise_draw(wn, nw, 0, 21, 0, li, 1, p), p)
        ref_b = o.weight_noise_apply(wn, bias, o.weight_noise_draw(wn, nb, o.bias_j0(nw), 21, 0, li, 1, p), p)
        got_w, got_b = net.noisy_operand(li, 0, nw), net.noisy_operand(li, 2, nb)
        for got, ref, what, bf in ((got_w, ref_w, "W", prec == "bf16"), (got_b, ref_b, "b", False)):
            want = bf16_round(ref) if bf else ref
            if name == "normal":
                # the fp32 Box-Muller of the device (8 ulps of |std z| <= 0.3, as the GaussianNoise tests allow), then one rounding of w + n
                tol = 8 * np.spacing(np.float32(0.3)) + 2 * np.spacing(np.abs(ref).astype(np.float32)) + (2.0 ** -8 * np.abs(ref) if bf else 0)
                assert np.all(np.abs(got - want) <= tol), (s["name"], what, np.max(np.abs(got - want)))
            else:
                assert np.array_equal(got, want), (prec, name, s["name"], what, rel_err(got, want))
        if prec == "bf16" and s["type"] == "deconv2d":
            got = net.noisy_operand(li, 1, 144 * 64)
            want = pack_deconv_ps(bf16_round(ref_w).reshape(64, 4, 4, 3))
            if name == "normal":
                assert np.all(np.abs(got - want) <= 2.0 ** -8 * np.abs(want) + 1e-30)
            else:
                assert np.array_equal(got, want), (name, "packed")
            packed += 1
    assert packed == (1 if prec == "bf16" else 0)
    net.close()


def _chain(wn):
    return [{"type": "conv2d", "name": "c1", "n_out": 5, "kernel": (3, 3), "stride": (2, 2), "padding": (1, 1), "weight_noise": wn, "updater": {"kind": "sgd", "lr": 0.05}},
            {"type": "activation", "name": "a1", "activation": "lrelu", "alpha": 0.2},
            {"type": "conv2d", "name": "c2", "n_out": 6, "kernel": (3, 3), "padding": (1, 1), "has_bias": False, "weight_noise": wn, "updater": {"kind": "sgd", "lr": 0.05}},
            {"type": "batchnorm", "name": "bn", "updater": {"kind": "sgd", "lr": 0.05}}, {"type": "activation", "name": "a2", "activation": "tanh"},
            {"type": "cnn_to_ff", "name": "flat"},
            {"type": "dense", "name": "d", "n_out": 8, "activation": "tanh", "weight_noise": wn, "updater": {"kind": "sgd", "lr": 0.05}},
            {"type": "output", "name": "out", "n_out": 1, "weight_noise": wn, "updater": {"kind": "sgd", "lr": 0.05}}]


@pytest.mark.parametrize("name,wn", [("dropconnect", DC), ("scheduled", SCHED), ("uniform", UNI), ("normal", NORMAL)])
def test_fp32_chain_follows_the_restatement(b200, name, wn):
    """FP32: three fits' scores, the gradients of a fourth pass and the updated parameters against the restatement (pclose at the FP32 bars)."""
    b, ctx = b200
    specs = _chain(wn)
    rng = np.random.default_rng(5)
    onet = o.net_from_specs(specs, (2, 8, 8), seed=3, mask_seed=11); randomize(onet, rng)
    net = b.Net(ctx, specs, (2, 8, 8), max_batch=6, precision=b.FP32, seed=11)
    push_params(onet, net)
    x = rng.uniform(-1, 1, (6, 2, 8, 8)); y = rng.uniform(0, 1, (6, 1))
    for it in range(3):
        s_o, s_b = onet.fit(x, y), net.fit(x, y)
        assert abs(s_b - s_o) < 1e-4 * max(1, abs(s_o)), (name, it, s_b, s_o)
        assert pclose(net.params(), onet.params_flat(), 0.1, 1e-3), (name, it, rel_err(net.params(), onet.params_flat()))
    s_o, s_b = onet.compute_gradient_and_score(x, y), net.compute_gradient_and_score(x, y)
    assert abs(s_b - s_o) < 1e-4 * max(1, abs(s_o))
    assert pclose(net.gradients(), onet.grads_flat(), 1e-3, 2e-3), (name, rel_err(net.gradients(), onet.grads_flat()))
    assert net.dropout_pass() == onet.dropout.pass_ == 4
    net.close()


def test_bf16_chain_follows_the_restatement_loosely(b200):
    """BF16: the operand net's scores over three fits follow the restatement's within the bf16 budget."""
    b, ctx = b200
    specs = _operand_specs(DC)
    rng = np.random.default_rng(6)
    onet = o.net_from_specs(specs, (3, 8, 8), seed=3, mask_seed=21); randomize(onet, rng)
    net = b.Net(ctx, specs, (3, 8, 8), max_batch=8, precision=b.BF16, seed=21)
    push_params(onet, net)
    x = rng.uniform(-1, 1, (8, 3, 8, 8)); y = rng.uniform(0, 1, (8, 1))
    for it in range(3):
        s_o, s_b = onet.fit(x, y), net.fit(x, y)
        assert abs(s_b - s_o) < 3e-2 * max(1, abs(s_o)), (it, s_b, s_o)
    assert rel_err(net.params(), onet.params_flat()) < 3e-2
    net.close()


def test_gan_step_graph_eager_and_oracle_agree(b200):
    """FP32 16x16 GAN, DropConnect(0.9) on D and WeightNoise(Normal(0, 0.01)) on G, both read from the specs: graph replay, eager and the
    oracle over 3 steps, each step drawing anew (D's real | fake pass P, the generator pass P + 1)."""
    from gan_deeplearning4j_b200 import models as m
    b, ctx = b200
    gs = [dict(s, weight_noise=m.weight_noise(m.normal(0, 0.01))) if s["type"] in ("deconv2d", "dense") else s for s in m.dcgan_generator(16, 12, 8, 3, lr=2e-3)]
    ds = m.dcgan_discriminator(16, 8, 3, lr=2e-3, drop_connect=0.9)
    G, D = oracle_gan_pair(gs, ds)
    data = [a.astype(np.float64) for a in o.synthetic_batch(8, 16, 3, 12, seed=3)]
    labels = tuple(data[3:])
    gan_step_parity(b, ctx, gs, ds, G, D, data, labels, 2e-3, "weight noise")
    # every step drew new operands: D's counter moved by two per step
    _, _, bG, bD, _ = fp32_gan_pair(b, ctx, gs, ds, 8)
    gan = b.Gan(bG, bD, use_cuda_graph=True)
    seen = []
    for _ in range(3):
        gan.step(*data)
        seen.append(bD.noisy_operand(0, 0, 8 * 3 * 16))
    assert bD.dropout_pass() == 6 and not np.array_equal(seen[0], seen[1]) and not np.array_equal(seen[1], seen[2])
    gan.close(); bG.close(); bD.close()


def test_identity_cases_launch_nothing_and_a_noisy_d_adds_two_launches(b200):
    """DropConnect(1) launches nothing and leaves P alone; DropConnect(0.9) on D adds one launch per D pass (2 per GAN step) and advances P by 2;
    an inference pass and a frozen layer draw nothing."""
    from gan_deeplearning4j_b200 import models as m
    b, ctx = b200
    rng = np.random.default_rng(1)
    n, gin, din = 16, (32,), (3, 16, 16)

    def run(drop_connect):
        G, D = bf16_gan(b, ctx, m.dcgan_generator(16, 32, 16, 3), m.dcgan_discriminator(16, 16, 3, drop_connect=drop_connect), gin, din, n)
        gan = b.Gan(G, D, use_cuda_graph=True)
        gan.upload(rng.uniform(-1, 1, (n,) + din), rng.uniform(-1, 1, (n,) + gin), rng.uniform(-1, 1, (n,) + gin), *[np.full((n, 1), v) for v in (1.0, 0.0, 1.0)])
        out = launches_per_step(ctx, gan, n), D.dropout_pass()
        x = rng.uniform(-1, 1, (n,) + din)
        ctx.sync(); l0 = ctx.launch_count(); D.output(x); ctx.sync()
        infer = ctx.launch_count() - l0
        assert D.dropout_pass() == out[1] and np.isfinite(gan.losses()).all()
        gan.close(); G.close(); D.close()
        return out + (infer,)

    plain, one, noisy = run(None), run(1.0), run(0.9)
    assert plain[1] == one[1] == 0 and one[0] == plain[0] and one[2] == plain[2]
    assert noisy[0] == plain[0] + 2 and noisy[1] == 2 * 5 and noisy[2] == plain[2]
    # a frozen layer draws nothing, even when named
    specs = [{"type": "dense", "name": "d1", "n_out": 8, "frozen": True}, {"type": "dense", "name": "d2", "n_out": 8, "activation": "tanh"},
             {"type": "output", "name": "out", "n_out": 1}]
    net = b.Net(ctx, specs, (6,), max_batch=4, precision=b.FP32, weight_noise={"weight_noise": "drop_connect", "p": 0.5})
    assert "weight_noise" not in net.specs[0] and net.specs[1]["weight_noise"]["p"] == 0.5
    net.set_weight_noise({"weight_noise": "drop_connect", "p": 0.5}, "d1")
    net.set_weight_noise(None, "d2"); net.set_weight_noise(None, "out")
    net.fit(rng.uniform(-1, 1, (4, 6)), rng.uniform(0, 1, (4, 1)))
    assert net.dropout_pass() == 0
    with pytest.raises(b.B200GanError) as e:
        net.noisy_operand(0, 0, 48)
    assert e.value.code == -6
    for bad in ({"weight_noise": "drop_connect", "p": 0.0}, {"weight_noise": "drop_connect", "p": 1.5},
                {"weight_noise": "weight_noise", "distribution": {"distribution": "normal", "mean": 0.0, "std": -1.0}},
                {"weight_noise": "weight_noise", "distribution": {"distribution": "uniform", "lower": 1.0, "upper": 0.0}},
                {"weight_noise": "weight_noise", "distribution": {"distribution": "normal", "mean": float("nan"), "std": 1.0}}):
        with pytest.raises(b.B200GanError) as e:
            net.set_weight_noise(bad)
        assert e.value.code == -1, bad
    net.close()
