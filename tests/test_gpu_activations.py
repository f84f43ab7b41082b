"""The activations of b2g_activation codes 5-16 on the GPU: the act_ext kernels through their production wrappers (b2g_test_ew ops act_ext_fwd /
act_ext_bwd) for every kind x precision x {vector, offset} path against float64 of the same stored z; FP32 nets with the new kinds in every
placement (Dense -> Dense -> OutputLayer(MSE), Conv2D -> BatchNorm -> ActivationLayer -> Deconv2D -> BatchNorm -> LossLayer) against
the oracle's restatement; BF16 16x16 DCGAN nets with ELU / SELU / Swish layer by layer on injected inputs; the FP32 GAN step (G: ELU hidden,
HardTanh output; D: SELU) against the oracle's gan_step in graph replay and eager mode with its launches per step; and the argument checks."""
import ctypes as C

import numpy as np
import pytest

from gan_deeplearning4j_b200 import models as m
from helpers import b200, bf16_round, check_bf16, fp32_gan_pair, launches_per_step, pclose, push_params, randomize, rel_err
from oracle import dl4j_oracle as o

pytestmark = pytest.mark.gpu
TOL = 1e-3
U = 2.0 ** -24


# ------------------------------------------------------------------ the kernels against float64 -----------------------------------------
BOUNDARIES = np.array([0.0, -0.0, 1.0, -1.0, 2.5, -2.5, 6.0, -6.0, 0.5, -0.5, 1.5, 2.0, 3.0, 100.0, -100.0, 99.5, -99.5, 20.0, -20.0, 88.0, -88.0, 0.75, -0.75])


def _inputs(n, rng):
    z = np.concatenate([BOUNDARIES, np.nextafter(BOUNDARIES.astype(np.float32), np.float32(np.inf)),
                        np.nextafter(BOUNDARIES.astype(np.float32), np.float32(-np.inf)), rng.uniform(-8, 8, n), rng.uniform(-100, 100, n // 4)])
    return rng.permutation(z).astype(np.float32)


@pytest.mark.parametrize("offset", [0, 3])
@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("kind", o.EXT_ACTS)
def test_kernels_against_float64(b200, kind, prec, offset):
    """f and eps * f' within one rounding of the output type (2^-8 relative for bf16, the bound of the other bf16 tests) plus the fp32
    evaluation's few units of 2^-24 on the terms it combines; no inf / NaN anywhere, no element left unwritten (the outputs are poisoned)."""
    b, ctx = b200
    p = b.FP32 if prec == "fp32" else b.BF16
    rng = np.random.default_rng(o.ACT_CODES[kind] * 7 + offset)
    z = _inputs(4099, rng)
    e = rng.uniform(-2, 2, z.size).astype(np.float32)
    alpha = 0.75 if kind in ("elu", "thresholdedrelu") else 0.0
    zs, es = (z, e) if p == b.FP32 else (bf16_round(z), bf16_round(e))
    zs, es = zs.astype(np.float64), es.astype(np.float64)
    u_out = U if p == b.FP32 else 2.0 ** -8
    (fwd, _, _), info_f = b.test_ew(ctx, p, "act_ext_fwd", z, None, (z.size, 0, 0), act=kind, alpha=alpha, n=z.size, offset=offset, poison=True)
    (bwd, _, _), info_b = b.test_ew(ctx, p, "act_ext_bwd", z, e, (z.size, 0, 0), act=kind, alpha=alpha, n=z.size, offset=offset)
    assert info_f["kernel"] == f"act_ext_fwd_kernel<{kind}>" and info_b["kernel"] == f"act_ext_bwd_kernel<{kind}>"
    f_ref = o.forward(kind, zs, alpha)
    d_ref = es * o.derivative(kind, zs, alpha)
    for got, ref, scale, what in ((fwd, f_ref, 1.0, "f"), (bwd, d_ref, np.abs(es), "eps*f'")):
        assert np.isfinite(got).all(), (kind, prec, what, "non-finite")
        tol = u_out * np.abs(ref) + 16 * U * (np.abs(ref) + scale)
        bad = np.abs(got - ref) > tol
        assert not bad.any(), (kind, prec, offset, what, zs[bad][:5], got[bad][:5], ref[bad][:5])


# ------------------------------------------------------------------ FP32 nets against the oracle ----------------------------------------
# Cube composes to z^27 through three layers: its MLP takes small steps on small inputs, so that it trains instead of overflowing; its conv
# net (Cube around two BatchNorms) has gradients near 1e10 on the first step, so its layers run their updates with lr 0
def _lr(kind, lr, conv=False):
    return (0.0 if conv else lr * 1e-3) if kind == "cube" else lr


def _mlp(kind):
    return [{"type": "dense", "name": "d1", "n_out": 24, "activation": kind, "updater": m.sgd(_lr(kind, 0.05)), "l2": 1e-3},
            {"type": "dense", "name": "d2", "n_out": 16, "activation": kind, "updater": m.adam(_lr(kind, 1e-2))},
            {"type": "output", "name": "out", "n_out": 5, "loss": "mse", "activation": kind, "updater": m.sgd(_lr(kind, 0.05))}], (12,), 5


def _conv(kind):
    return [{"type": "conv2d", "name": "c1", "n_out": 8, "kernel": (3, 3), "stride": (2, 2), "padding": (1, 1), "activation": kind, "updater": m.sgd(_lr(kind, 0.05, True))},
            {"type": "batchnorm", "name": "bn1", "updater": m.sgd(_lr(kind, 0.05, True))},
            {"type": "activation", "name": "a1", "activation": kind},
            {"type": "deconv2d", "name": "dc2", "n_out": 6, "kernel": (4, 4), "stride": (2, 2), "padding": (1, 1), "activation": kind, "updater": m.sgd(_lr(kind, 0.05, True))},
            {"type": "batchnorm", "name": "bn2", "updater": m.sgd(_lr(kind, 0.05, True))},
            {"type": "conv2d", "name": "c3", "n_out": 2, "kernel": (8, 8), "updater": m.adam(_lr(kind, 1e-2, True))},
            {"type": "loss", "name": "loss", "loss": "mse", "activation": kind}], (3, 8, 8), 2


@pytest.mark.parametrize("net", ["mlp", "conv"])
@pytest.mark.parametrize("kind", o.EXT_ACTS)
def test_fp32_nets_match_oracle(b200, kind, net):
    """Every activation, every gradient, the score, the post-update parameters and b2g_net_output (inference: the BatchNorm after a GEMM of a new
    kind is not folded into it; train mode: batch statistics) within DESIGN 1's 1e-3."""
    b, ctx = b200
    specs, shape, n_out = (_mlp if net == "mlp" else _conv)(kind)
    rng = np.random.default_rng(o.ACT_CODES[kind])
    onet = o.net_from_specs(specs, shape, seed=2, flat_input=False); randomize(onet, rng)
    bnet = b.Net(ctx, specs, shape, max_batch=6, precision=b.FP32)
    push_params(onet, bnet)
    r = 0.5 if kind == "cube" and net == "mlp" else 1.5
    for it in range(3):
        x = rng.uniform(-r, r, (6,) + shape); y = rng.uniform(-1, 1, (6, n_out))
        s_o, acts, _, _ = onet.compute_gradient_and_score(x, y, collect=True)
        s_b = bnet.compute_gradient_and_score(x, y)
        assert abs(s_b - s_o) <= TOL * abs(s_o), (kind, net, it, s_b, s_o)
        for i, a in enumerate(acts[:-1]):
            assert rel_err(bnet.activation(i, 6), a.reshape(6, -1)) <= TOL, (kind, net, it, "activation", i)
        assert rel_err(bnet.gradients(), onet.grads_flat()) <= TOL, (kind, net, it, "gradients")
        s_o = onet.fit(x, y); s_b = bnet.fit(x, y)
        assert abs(s_b - s_o) <= TOL * abs(s_o), (kind, net, it, s_b, s_o)
        assert rel_err(bnet.params(), onet.params_flat()) <= TOL, (kind, net, it, "params")
        xo = rng.uniform(-r, r, (5,) + shape)
        assert rel_err(bnet.output(xo), onet.output(xo).reshape(5, -1)) <= TOL, (kind, net, it, "output")
        assert rel_err(bnet.output(xo, train=True), onet.forward(xo, True).reshape(5, -1)) <= TOL, (kind, net, it, "train output")
    bnet.close()


# ------------------------------------------------------------------ BF16 DCGAN-shaped nets ----------------------------------------------
def _check_ext_gemm(got, ref, z, kind, what):
    """A GEMM layer of a new kind in bf16: its z is rounded to bf16 once before f (b2g_activation), so beside check_bf16's bound on a the
    rounding of z moves the result by up to |f'(z)| 2^-8 |z|."""
    got, ref, z = (np.asarray(v, np.float64) for v in (got, ref, z))
    tol = 2.0 ** -8 * (np.abs(ref) + np.abs(o.derivative(kind, z) * z)) + 2e-3 * np.sqrt(np.mean(ref ** 2))
    bad = ~(np.abs(got - ref) <= tol)
    assert not bad.any(), (what, int(bad.sum()), bad.size, float(np.abs(got - ref)[bad].max()))


@pytest.mark.parametrize("kind", ["elu", "selu", "swish"])
def test_bf16_dcgan_layers_on_injected_inputs(b200, kind):
    """Each layer of a 16x16 DCGAN generator / discriminator with `kind` in place of ReLU / LeakyReLU against the oracle's layer run on the GPU's
    own input to it (check_bf16; a GEMM of a new kind also allows the rounding of its stored z, _check_ext_gemm), and the same number of SIMT
    GEMM calls as the ReLU / LeakyReLU nets: the GEMMs stay on tensor cores."""
    b, ctx = b200
    n, z = 16, 32
    rng = np.random.default_rng(9)
    cases = [(m.dcgan_generator(16, z, 64, 3, activation=kind), m.dcgan_generator(16, z, 64, 3), (z,)),
             (m.dcgan_discriminator(16, 64, 3, activation=kind), m.dcgan_discriminator(16, 64, 3), (3, 16, 16))]
    for specs, base, shape in cases:
        x = bf16_round(rng.uniform(-1, 1, (n,) + shape))
        onet = o.net_from_specs(specs, shape, seed=3, flat_input=False); randomize(onet, rng)
        for l in onet.layers:          # the tensor-core path reads bf16 weights: the oracle takes the same operands
            if l.has_params and "W" in l.params:
                l.params["W"] = bf16_round(l.params["W"]).astype(np.float64)
        calls = []
        for sp in (specs, base):
            bnet = b.Net(ctx, sp, shape, max_batch=n, precision=b.BF16)
            push_params(onet, bnet)
            bnet.output(x, train=True)
            if sp is specs:
                cur = x.astype(np.float64)
                for i, l in enumerate(onet.layers):
                    if i + 1 == len(onet.layers) and sp[i]["type"] == "loss":
                        break
                    ref = l.forward(cur, True)
                    got = bnet.activation(i, n).reshape(ref.shape)
                    if sp[i]["type"] != "activation" and sp[i].get("activation") in o.EXT_ACTS:
                        _check_ext_gemm(got, ref, l._z, sp[i]["activation"], f"{kind} {sp[i]['name']}")
                    else:
                        check_bf16(got, ref, f"{kind} {sp[i]['name']}")
                    cur = got.astype(np.float64)
            calls.append(bnet.simt_gemm_calls())
            bnet.close()
        assert calls[0] == calls[1], (kind, calls)


# ------------------------------------------------------------------ the fused GAN step, FP32 --------------------------------------------
# launches per FP32 16x16 step (nf 8, z 12, batch 8) of the ELU / HardTanh generator with the SELU discriminator, and of the same nets on
# ReLU / tanh and LeakyReLU (DESIGN.md 3.1: 14 more): per G forward (2 a step) 3 act_ext_fwd, per D forward (2) 2; G backward 2 more launches (its
# unfused ActivationLayers; HardTanh's act_ext_bwd replaces tanh's), each D backward 1 more (its unfused ActivationLayer)
EXTRA_LAUNCHES = 2 * 3 + 2 * 2 + 2 + 2 * 1


def test_fp32_gan_step_matches_oracle(b200):
    b, ctx = b200
    size, z, nf, n, lr_ = 16, 12, 8, 8, 2e-3
    gs = m.dcgan_generator(size, z, nf, 3, lr=lr_, activation="elu", out_activation="hardtanh")
    ds = m.dcgan_discriminator(size, nf, 3, lr=lr_, activation="selu")
    counts = {}
    for graph in (True, False):
        G, D, bG, bD, data = fp32_gan_pair(b, ctx, gs, ds, n)
        gan = b.Gan(bG, bD, use_cuda_graph=graph)
        for it in range(3):
            r = o.gan_step(G, D, *data)
            lo = gan.step(*data)
            want = np.array([r["loss_d_real"], r["loss_d_fake"], r["loss_g"]])
            assert np.all(np.abs(lo - want) < TOL * np.maximum(1, np.abs(want))), (graph, it, lo, want)
            assert pclose(bD.params(), D.params_flat(), 2 * lr_), (graph, it, "D", rel_err(bD.params(), D.params_flat()))
            assert pclose(bG.params(), G.params_flat(), 2 * lr_), (graph, it, "G", rel_err(bG.params(), G.params_flat()))
        gan.upload(*[a.astype(np.float32) for a in data])
        counts[graph] = launches_per_step(ctx, gan, n)
        gan.close(); bG.close(); bD.close()
    bG = b.Net(ctx, m.dcgan_generator(size, z, nf, 3, lr=lr_), (z,), max_batch=n, precision=b.FP32)
    bD = b.Net(ctx, m.dcgan_discriminator(size, nf, 3, lr=lr_), (3, size, size), max_batch=2 * n, precision=b.FP32, bn_groups=2)
    gan = b.Gan(bG, bD, use_cuda_graph=True)
    gan.upload(*[a.astype(np.float32) for a in data])
    base = launches_per_step(ctx, gan, n)
    gan.close(); bG.close(); bD.close()
    assert counts[True] == counts[False] == base + EXTRA_LAUNCHES, (counts, base)


# ------------------------------------------------------------------ argument checks -------------------------------------------------------
def test_rejections(b200):
    b, ctx = b200
    from gan_deeplearning4j_b200 import engine, _lib

    def create(spec_list, mutate=None):
        descs = [engine.layer_desc(s) for s in spec_list]
        if mutate:
            mutate(descs)
        arr = (_lib.LayerDesc * len(descs))(*descs)
        cfg = _lib.NetConfig(1, 1, 6, 4, b.FP32, 0.0, 1e-5, 1, 666)
        h = C.c_void_p()
        rc = ctx.lib.b2g_net_create(ctx.h, C.byref(cfg), arr, len(descs), C.byref(h))
        if rc == 0:
            ctx.lib.b2g_net_destroy(h)
        return rc

    specs = [{"type": "dense", "name": "d", "n_out": 4, "activation": "elu"}, {"type": "output", "name": "o", "n_out": 2, "loss": "mse", "activation": "selu"}]
    assert create(specs) == 0
    for li, bad in ((0, 17), (0, -1), (1, 17), (0, 99)):
        def mut(d, li=li, bad=bad): d[li].act = bad
        assert create(specs, mut) == -1, (li, bad)
    def nan_alpha(d): d[0].act_alpha = float("nan")
    def inf_alpha(d): d[1].act_alpha = float("inf")
    assert create(specs, nan_alpha) == -1 and create(specs, inf_alpha) == -1
    z = np.zeros(8, np.float32)
    with pytest.raises(b.B200GanError):
        b.test_ew(ctx, b.FP32, "act_ext_fwd", z, None, (8, 0, 0), act="relu", n=8)           # codes 0-4 are not the extended kernels'
    with pytest.raises(b.B200GanError):
        b.test_ew(ctx, b.FP32, "act_ext_bwd", z, None, (8, 0, 0), act="elu", n=8)            # eps missing
