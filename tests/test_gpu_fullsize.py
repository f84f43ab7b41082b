"""Parity of the BENCHMARKED path at the BENCHMARKED sizes (VERDICT round 1, weak #1): every wgmma kernel variant that the C2 step
(64x64x3 DCGAN, batch 128; reference call sites J:135-150, J:203-219) dispatches -- one-CTA-per-tile conv with 64- and 128-column tiles, pixel-shuffle deconv,
folded-BatchNorm (AFFINE) epilogue, the fused BatchNorm epilogues (EPI_STATS / EPI_BNBWD / EPI_ACTBWD), two-thirds-wave split-K weight gradient,
the 3-channel edge kernels -- runs here through the C-ABI test hook with the PRODUCTION dispatch, the hook reports
which kernel ran (asserted), and the result is compared with the CPU oracle (oracle/dl4j_oracle.py ConvolutionLayer / Deconvolution2D
semantics) on the same bf16-rounded operands:
    bf16 outputs:  |got - ref| <= 2^-8 |ref| + 2e-3 rms(ref)        (one bf16 rounding is 2^-9 relative; fp32 accumulation order)
    fp32 wgrad:    max|got - ref| <= 1e-4 max|ref|
The tensor-core fprop / dgrad GEMMs are compared on every element of the whole batch with the float64 reference of tests/conv_ref.py
(pinned to the oracle by tests/test_conv_ref.py), on an output poisoned with NaN before the launch, and their production epilogue is
re-run at one CTA and at one CTA per tile (bit-identical).  The oracle evaluates whole sampled images (first / last, a few in the middle,
the real|fake group boundary) for the edge kernels, and the full batch in image chunks (the weight gradient is a sum over images) for wgrad.
"""
import copy

import numpy as np
import pytest

import conv_ref
import tc_schedule
from helpers import (b200, bf16_round, bf16_weights, check_bf16, check_generator_step_grads, check_grads_against_oracle, flat_order,
                     grads_by_tensor, inject_forward, rel_fro)
from oracle import dl4j_oracle as o
from tc_schedule import pick_row_tile as _pick_row_tile

pytestmark = pytest.mark.gpu

N = 128     # C2 per-GPU batch; the D step runs 2N


def sample_images(n):
    return sorted(set(i for i in (0, 1, 36, 37, 73, 74, n // 2 - 1, n // 2, n - 2, n - 1) if 0 <= i < n))


def conv_layer(c, oc, wt):
    l = o.Conv2D(c, oc, (4, 4), (2, 2), (1, 1), has_bias=False); l.init(np.random.default_rng(0), np.float64); l.params["W"] = wt.astype(np.float64); return l


def geom_of(n, h, c, oc):
    return dict(n=n, h=h, w=h, c=c, oh=h // 2, ow=h // 2, o=oc, kh=4, kw=4, sh=2, sw=2, ph=1, pw=1)


def act_fwd(name, z, alpha):
    return {"identity": lambda: z, "relu": lambda: np.maximum(z, 0), "lrelu": lambda: np.where(z > 0, z, alpha * z), "tanh": lambda: np.tanh(z)}[name]()


_REF = {}


def _full_ref(key, fn):
    """float64 GEMM of a whole batch (conv_ref), computed once per shape: every epilogue of a case shares its operands."""
    if key not in _REF:
        _REF[key] = fn()
    return _REF[key]


def _check_schedule_invariance(b, ctx, kind, g, a, wt, size, kw, out, stats, kernel, what):
    """The production epilogue of a shape once more at one CTA (every tile through one CTA's rings and park slots) and at one CTA per tile:
    output and statistics bit-identical to the production grid's."""
    bn = int(kernel.split("<")[1].split(",")[0])
    geo = tc_schedule.geometry("fprop" if kind == 0 else "dgrad", g["n"], g["h"], g["w"], g["c"], g["o"], 4, 2, 1, bn)
    for mc in (1, geo["tiles"]):
        o2, s2, k2, _ = b.test_conv_ex(ctx, kind, g, a, wt, size, poison=True, max_ctas=mc, **kw)
        assert k2 == kernel, (what, mc, k2)
        assert np.array_equal(o2.view(np.uint32), out.view(np.uint32)), f"{what}: max_ctas={mc} output differs from the production grid's"
        if stats is not None:
            assert np.array_equal(s2, stats), f"{what}: max_ctas={mc} statistics differ from the production grid's"


# (name, batch, conv-input size h, c, o, expected kernel, the epilogue the step runs this GEMM with)
# conv geometry 4x4 s2 p1: x [n,h,h,c] -> y [n,h/2,h/2,o]
FPROP = [
    ("D2 fprop, D step (2N, real|fake)", 2 * N, 32, 64, 128, "tc_conv_kernel<128,4>", "stats"),
    ("D3 fprop, D step", 2 * N, 16, 128, 256, "tc_conv_kernel<128,4>", "stats"),
    ("D4 fprop, D step", 2 * N, 8, 256, 512, "tc_conv_kernel<64,4>", "stats"),
    ("D2 fprop, G step / G4 input gradient", N, 32, 64, 128, "tc_conv_kernel<128,4>", "bnbwd_relu"),
    ("D3 fprop, G step / G3 input gradient", N, 16, 128, 256, "tc_conv_kernel<64,4>", "bnbwd_relu"),
    ("D4 fprop, G step / G2 input gradient", N, 8, 256, 512, "tc_conv_kernel<64,4>", "bnbwd_relu"),
]


@pytest.mark.parametrize("case", FPROP, ids=[c[0] for c in FPROP])
@pytest.mark.parametrize("epi", ["stats", "bnbwd_relu", "plain_bias_lrelu"])
def test_fprop_production_dispatch(b200, case, epi):
    """conv forward (D2-D4) with the BatchNorm statistics epilogue, and the same kernel as the generator's input-gradient GEMM with the
    BatchNorm-backward epilogue (J:197-199 BatchNormalization + ReLU below each transposed conv).  Every element of the whole batch against
    the float64 reference; the output is poisoned (bf16 NaN) before each launch, so an unwritten tile fails."""
    b, ctx = b200
    name, n, h, c, oc, kernel, prod_epi = case
    rng = np.random.default_rng(11)
    x = bf16_round(rng.standard_normal((n, h, h, c))); wt = bf16_round(rng.standard_normal((oc, 4, 4, c)) / np.sqrt(16 * c))
    g = geom_of(n, h, c, oc); oh = h // 2
    groups = 2 if n == 2 * N else 1
    ref = _full_ref(("fprop", name), lambda: conv_ref.conv2d(x, wt, 2, 1))        # [n, oh, oh, oc]
    size = n * oh * oh * oc
    if epi == "stats":
        kw = dict(epi=b.EPI_STATS, groups=groups)
        out, stats, k, _ = b.test_conv_ex(ctx, 0, g, x, wt, size, poison=True, **kw)
        check_bf16(out.reshape(n, oh, oh, oc), ref, name)
        # the statistics are those of the STORED bf16 tensor, per (group, channel): exact up to fp32 summation order inside a 128-row tile
        og = out.reshape(groups, -1, oc).astype(np.float64)
        np.testing.assert_allclose(stats[:, 0, :], og.sum(1), rtol=2e-5, atol=2e-3)
        np.testing.assert_allclose(stats[:, 1, :], (og ** 2).sum(1), rtol=2e-5, atol=2e-3)
    elif epi == "plain_bias_lrelu":
        bias = rng.standard_normal(oc).astype(np.float32) * 0.1
        kw = dict(act="lrelu", alpha=0.2, bias=bias)
        out, stats, k, _ = b.test_conv_ex(ctx, 0, g, x, wt, size, poison=True, **kw)
        check_bf16(out.reshape(n, oh, oh, oc), act_fwd("lrelu", ref + bias.astype(np.float64), 0.2), name)
    else:
        # the GEMM result is the epsilon w.r.t. the output y of BatchNorm+ReLU; z = that BatchNorm's input: out = eps * relu'(y), statistics sum out, sum out*z
        z = bf16_round(rng.standard_normal((n, oh, oh, oc)))
        y = bf16_round(np.maximum(z * rng.uniform(0.5, 1.5, oc) + rng.standard_normal(oc) * 0.3, 0))
        kw = dict(epi=b.EPI_BNBWD, act="relu", groups=groups, aux=y, aux2=z)
        out, stats, k, _ = b.test_conv_ex(ctx, 0, g, x, wt, size, poison=True, **kw)
        check_bf16(out.reshape(n, oh, oh, oc), ref * (y > 0), name)
        zg = z.reshape(groups, -1, oc).astype(np.float64); og = out.reshape(groups, -1, oc).astype(np.float64)
        np.testing.assert_allclose(stats[:, 0, :], og.sum(1), rtol=2e-5, atol=2e-3)
        np.testing.assert_allclose(stats[:, 1, :], (og * zg).sum(1), rtol=2e-5, atol=5e-3)
    assert k == kernel, f"{name}: dispatched {k}, the C2 step is expected to run {kernel}"
    if epi == prod_epi:
        _check_schedule_invariance(b, ctx, 0, g, x, wt, size, kw, out, stats, kernel, name)


# conv geometry: dy [n,h/2,h/2,o] -> dx [n,h,h,c]  (= transposed-conv forward o -> c)
DGRAD = [
    ("D2 dgrad, D step (2N)", 2 * N, 32, 64, 128, "tc_conv_kernel<64,4>", "actbwd_lrelu"),
    ("D3 dgrad, D step", 2 * N, 16, 128, 256, "tc_conv_kernel<128,4>", "bnbwd_lrelu"),
    ("D4 dgrad, D step", 2 * N, 8, 256, 512, "tc_conv_kernel<128,4>", "bnbwd_lrelu"),
    ("G4 forward / D2 dgrad, G step (N)", N, 32, 64, 128, "tc_conv_kernel<64,4>", "stats"),
    ("G3 forward / D3 dgrad, G step", N, 16, 128, 256, "tc_conv_kernel<128,4>", "stats"),
    ("G2 forward / D4 dgrad, G step", N, 8, 256, 512, "tc_conv_kernel<64,4>", "stats"),
]


@pytest.mark.parametrize("case", DGRAD, ids=[c[0] for c in DGRAD])
@pytest.mark.parametrize("epi", ["stats", "bnbwd_lrelu", "affine_relu", "actbwd_lrelu"])
def test_dgrad_production_dispatch(b200, case, epi):
    """Deconvolution2D forward = conv input gradient in sub-pixel phase form, weights read as MN-major tiles from the straight [O][16][C] copy:
    train-mode generator forward (statistics epilogue), inference-mode generator forward (folded BatchNorm + ReLU: gen.output, J:420),
    discriminator input gradients with the BatchNorm-backward / LeakyReLU-backward epilogues.  Whole batch, poisoned output, as above."""
    b, ctx = b200
    name, n, h, c, oc, kernel, prod_epi = case
    rng = np.random.default_rng(12)
    dy = bf16_round(rng.standard_normal((n, h // 2, h // 2, oc))); wt = bf16_round(rng.standard_normal((oc, 4, 4, c)) / np.sqrt(4 * oc))
    g = geom_of(n, h, c, oc)
    groups = 2 if n == 2 * N else 1
    ref = _full_ref(("dgrad", name), lambda: conv_ref.conv2d_input_grad(dy, wt, (h, h), 2, 1))     # [n, h, h, c]
    size = n * h * h * c
    stats = None
    if epi == "stats":
        kw = dict(epi=b.EPI_STATS, groups=groups)
        out, stats, k, _ = b.test_conv_ex(ctx, 1, g, dy, wt, size, poison=True, **kw)
        check_bf16(out.reshape(n, h, h, c), ref, name)
        og = out.reshape(groups, -1, c).astype(np.float64)
        np.testing.assert_allclose(stats[:, 0, :], og.sum(1), rtol=2e-5, atol=2e-3)
        np.testing.assert_allclose(stats[:, 1, :], (og ** 2).sum(1), rtol=2e-5, atol=2e-3)
    elif epi == "affine_relu":
        scale = rng.uniform(0.5, 1.5, c).astype(np.float32); shift = (rng.standard_normal(c) * 0.2).astype(np.float32)
        kw = dict(act="relu", bias=shift, scale=scale)
        out, _, k, _ = b.test_conv_ex(ctx, 1, g, dy, wt, size, poison=True, **kw)
        check_bf16(out.reshape(n, h, h, c), act_fwd("relu", ref * scale.astype(np.float64) + shift.astype(np.float64), 0.0), name)
    elif epi == "actbwd_lrelu":
        a = bf16_round(rng.standard_normal((n, h, h, c)))
        kw = dict(epi=b.EPI_ACTBWD, act="lrelu", alpha=0.2, aux=a)
        out, _, k, _ = b.test_conv_ex(ctx, 1, g, dy, wt, size, poison=True, **kw)
        check_bf16(out.reshape(n, h, h, c), ref * np.where(a > 0, 1.0, 0.2), name)
    else:
        z = bf16_round(rng.standard_normal((n, h, h, c)))
        u = z * rng.uniform(0.5, 1.5, c) + rng.standard_normal(c) * 0.3
        y = bf16_round(np.where(u > 0, u, 0.2 * u))
        kw = dict(epi=b.EPI_BNBWD, act="lrelu", alpha=0.2, groups=groups, aux=y, aux2=z)
        out, stats, k, _ = b.test_conv_ex(ctx, 1, g, dy, wt, size, poison=True, **kw)
        check_bf16(out.reshape(n, h, h, c), ref * np.where(y > 0, 1.0, 0.2), name)
        zg = z.reshape(groups, -1, c).astype(np.float64); og = out.reshape(groups, -1, c).astype(np.float64)
        np.testing.assert_allclose(stats[:, 0, :], og.sum(1), rtol=2e-5, atol=2e-3)
        np.testing.assert_allclose(stats[:, 1, :], (og * zg).sum(1), rtol=2e-5, atol=5e-3)
    assert k == kernel, f"{name}: dispatched {k}, the C2 step is expected to run {kernel}"
    if epi == prod_epi:
        _check_schedule_invariance(b, ctx, 1, g, dy, wt, size, kw, out, stats, kernel, name)


WGRAD = [
    ("D2 wgrad, D step (2N)", 2 * N, 32, 64, 128, "tc_wgrad_kernel<128,4>"),
    ("D3 wgrad, D step", 2 * N, 16, 128, 256, "tc_wgrad_kernel<128,4>"),
    ("D4 wgrad, D step", 2 * N, 8, 256, 512, "tc_wgrad_kernel<128,4>"),
    ("G4 wgrad (N)", N, 32, 64, 128, "tc_wgrad_kernel<128,4>"),
    ("G3 wgrad", N, 16, 128, 256, "tc_wgrad_kernel<128,4>"),
    ("G2 wgrad", N, 8, 256, 512, "tc_wgrad_kernel<128,4>"),
]


@pytest.mark.parametrize("case", WGRAD, ids=[c[0] for c in WGRAD])
def test_wgrad_production_dispatch(b200, case):
    """dW = sum over the whole batch: split-K grids of at most 96 CTAs (beside the input-gradient chain) with fp32 partials and the fixed-order
    reduction.  Oracle: ConvolutionLayer.backpropGradient on image chunks, summed (dW is linear in the batch)."""
    b, ctx = b200
    name, n, h, c, oc, kernel = case
    rng = np.random.default_rng(13)
    x = bf16_round(rng.standard_normal((n, h, h, c))); dy = bf16_round(rng.standard_normal((n, h // 2, h // 2, oc)))
    g = geom_of(n, h, c, oc)
    opts = b._lib.TestConvOpts()
    import ctypes as C
    out = np.empty(oc * 16 * c, np.float32); ms = C.c_float()
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    xa, da = np.ascontiguousarray(x.ravel()), np.ascontiguousarray(dy.ravel())
    b.engine.check(ctx.lib.b2g_test_conv_ex(ctx.h, 2, 1, b.BF16, C.byref(b._lib.ConvGeom(**g)), fp(xa), fp(da), fp(out), 1, C.byref(ms), C.byref(opts)))
    lay = conv_layer(c, oc, np.zeros((oc, c, 4, 4)))
    ref = np.zeros((oc, c, 4, 4))
    for i0 in range(0, n, 32):
        lay.forward(x[i0:i0 + 32].transpose(0, 3, 1, 2).astype(np.float64), True)
        lay.backward(dy[i0:i0 + 32].transpose(0, 3, 1, 2).astype(np.float64)); ref += lay.grads["W"]
    ref = ref.transpose(0, 2, 3, 1)
    err = np.abs(out.reshape(oc, 4, 4, c) - ref).max() / np.abs(ref).max()
    assert err < 1e-4, (name, err)
    assert opts.kernel.decode() == kernel, f"{name}: dispatched {opts.kernel.decode()}, expected {kernel}"


def test_edge_kernels_full_size(b200):
    """D1 (3 -> 64 image channels, J:135-140 analogue in the 64x64 DCGAN) and G-last at the C2 batch: tensor-core edge kernels (impl 3)."""
    b, ctx = b200
    rng = np.random.default_rng(14)
    n, h, c, oc = 2 * N, 64, 3, 64
    x = bf16_round(rng.uniform(-1, 1, (n, h, h, c))); wt = bf16_round(rng.standard_normal((oc, 4, 4, c)) / np.sqrt(16 * c)); dy = bf16_round(rng.standard_normal((n, h // 2, h // 2, oc)))
    g = geom_of(n, h, c, oc); idx = sample_images(n)
    lay = conv_layer(c, oc, wt.transpose(0, 3, 1, 2))
    y = lay.forward(x[idx].transpose(0, 3, 1, 2).astype(np.float64), True).transpose(0, 2, 3, 1)
    dx = lay.backward(dy[idx].transpose(0, 3, 1, 2).astype(np.float64)).transpose(0, 2, 3, 1)
    got, _ = b.test_conv(ctx, 0, 3, b.BF16, g, x, wt, n * 32 * 32 * oc); check_bf16(got.reshape(n, 32, 32, oc)[idx], y, "D1 fprop (tc_edge_conv_kernel)")
    got, _ = b.test_conv(ctx, 1, 3, b.BF16, g, dy, wt, n * h * h * c); check_bf16(got.reshape(n, h, h, c)[idx], dx, "D1 dgrad / G-last forward (pixel-shuffle tensor-core conv)")
    ref = np.zeros((oc, c, 4, 4))
    for i0 in range(0, n, 64):
        lay.forward(x[i0:i0 + 64].transpose(0, 3, 1, 2).astype(np.float64), True); lay.backward(dy[i0:i0 + 64].transpose(0, 3, 1, 2).astype(np.float64)); ref += lay.grads["W"]
    got, _ = b.test_conv(ctx, 2, 3, b.BF16, g, x, dy, oc * 16 * c)
    assert np.abs(got.reshape(oc, 4, 4, c) - ref.transpose(0, 2, 3, 1)).max() / np.abs(ref).max() < 1e-4


# ------------------------------------------------------------------------------------------------
# Whole step in BF16 at the BASELINE sizes, layer by layer with injected inputs (VERDICT round 1, next-round item 1):
# every layer's oracle is evaluated on the GPU's OWN input to that layer, so one layer's bf16 rounding never hides in the next one's
# tolerance; the backward pass is the oracle's exact backward through the layers whose caches hold those injected activations.
# ------------------------------------------------------------------------------------------------
STEP_CASES = [("c2", 64, 100, 64, 128), ("c4", 128, 100, 64, 32), ("c5", 0, 128, 1024, 8192)]


@pytest.mark.parametrize("case", STEP_CASES, ids=[c[0] for c in STEP_CASES])
def test_bf16_whole_step_layer_by_layer(b200, case):
    """BASELINE configs[1] / [3] per GPU: D's train pass (computeGradientAndScore on 2N images) and the generator step through D, BF16.
    Forward: every conv / transposed conv / BatchNorm(+activation) tensor within one bf16 rounding of the oracle on the same input.
    Backward: every gradient tensor against the oracle's exact backward from the injected activations: relative Frobenius error <= 3e-2
    (ten bf16-rounded epsilon tensors deep), cosine >= 0.999."""
    b, ctx = b200
    from gan_deeplearning4j_b200 import models as m
    from helpers import push_params, randomize
    name, size, z, nf, n = case
    rng = np.random.default_rng(21)
    if name == "c5":        # MLP-GAN (BASELINE configs[4]): dense tensor-core path, samples of d = 256 features
        gs, ds, dshape = m.mlp_generator(z, nf, 256), m.mlp_discriminator(256, nf), (256,)
        data = [rng.uniform(-1, 1, (n, 256)), rng.uniform(-1, 1, (n, z)), rng.uniform(-1, 1, (n, z)), 1 + 0.05 * rng.standard_normal((n, 1)), 0.05 * rng.standard_normal((n, 1)), np.ones((n, 1))]
        data = [np.asarray(a, np.float32) for a in data]
    else:
        gs, ds, dshape = m.dcgan_generator(size, z, nf, 3), m.dcgan_discriminator(size, nf, 3), (3, size, size)
        data = [np.asarray(a, np.float32) for a in o.synthetic_batch(n, size, 3, z, seed=5)]
    q = o.Quirks(xent_clip_eps=0.0)
    G = o.net_from_specs(gs, (z,), quirks=q, dtype=np.float32, seed=1); D = o.net_from_specs(ds, dshape, quirks=q, dtype=np.float32, seed=2, flat_input=False)
    randomize(G, rng); randomize(D, rng)
    bG = b.Net(ctx, gs, (z,), max_batch=n, precision=b.BF16, xent_clip_eps=0.0)
    bD = b.Net(ctx, ds, dshape, max_batch=2 * n, precision=b.BF16, xent_clip_eps=0.0, bn_groups=2)
    push_params(G, bG); push_params(D, bD)
    # ---- D alone on 2N images (one BatchNorm group): forward tensors and every D gradient
    x2 = np.concatenate([data[0], rng.uniform(-1, 1, data[0].shape).astype(np.float32)]); y2 = np.concatenate([data[3], data[4]])
    bD.compute_gradient_and_score(x2, y2)
    # the tensor-core path holds bf16 weights: the oracle must see the same operands
    bf16_weights(G); bf16_weights(D)
    inject_forward(D, bD, ds, bf16_round(x2), 2 * n, "D (2N)")
    loss_sum, eps = D.layers[-1].score_and_eps(y2.astype(np.float32))
    if isinstance(D.layers[-1], o.Output):
        eps = D.layers[-1].backward(eps)
    D.backward_from_prefix(eps)
    check_grads_against_oracle(D, bD.gradients(), ds, "D")
    # ---- the adversarial step: afterwards the nets hold the G-step pass (G train forward on z_g, D train forward on G's output)
    pD_before = bD.params()
    gan = b.Gan(bG, bD, use_cuda_graph=False)
    gan.step(*data)
    # D was updated once before the G step ran through it: give the oracle those parameters (G's are still the pre-update ones it ran with)
    D.set_params_flat(bD.params().astype(np.float32))
    bf16_weights(D)
    assert np.abs(bD.params() - pD_before).max() > 0
    check_generator_step_grads(G, D, bG, bD, gs, ds, data[2], data[5])
    assert bD.simt_gemm_calls() > 0        # the skinny layers (the logit; z -> 4x4 in the DCGANs) are SIMT by design, and counted
    gan.close(); bG.close(); bD.close()


# (name, batch, C, O): 1x1 geometry.  G-first (z -> 4x4 x nf*8 map, J:189-196 Deconvolution2D on the 1x1 latent "image") is the dgrad form
# with the reduction over O latent inputs; D-last (J:159-163 OutputLayer, one logit per image) is the fprop form with O = 1.
DENSE_K = [("G-first, C2 (z=100 -> 8192)", N, 8192, 100), ("G-first, ragged batch / odd latent size", 77, 1024, 13), ("G-first, batch 2N, z=128", 2 * N, 2048, 128)]
DENSE_O = [("D-last, D step (2N)", 2 * N, 8192, 1), ("D-last, ragged batch", 37, 1024, 1)]


def dense_geom(n, c, oc):
    return dict(n=n, h=1, w=1, c=c, oh=1, ow=1, o=oc, kh=1, kw=1, sh=1, sw=1, ph=0, pw=0)


@pytest.mark.parametrize("case", DENSE_K + DENSE_O, ids=[c[0] for c in DENSE_K + DENSE_O])
def test_dense_kernels(b200, case):
    """The 1x1-geometry layers at the ends of the stack through the C-ABI hook (impl 4): input-gradient form (= G-first forward),
    weight gradient, and for O = 1 the forward dot product; reference = float64 matmul of the same bf16-rounded operands."""
    b, ctx = b200
    name, n, c, oc = case
    rng = np.random.default_rng(5)
    g = dense_geom(n, c, oc)
    dy = bf16_round(rng.standard_normal((n, oc))); wt = bf16_round(rng.standard_normal((oc, c)) / np.sqrt(oc)); x = bf16_round(rng.standard_normal((n, c)))
    got, _ = b.test_conv(ctx, 1, 4, b.BF16, g, dy, wt, n * c)
    check_bf16(got.reshape(n, c), dy.astype(np.float64) @ wt.astype(np.float64), name + " dgrad form")
    got, _ = b.test_conv(ctx, 2, 4, b.BF16, g, x, dy, oc * c)
    ref = dy.astype(np.float64).T @ x.astype(np.float64)
    assert np.abs(got.reshape(oc, c) - ref).max() <= 1e-4 * np.abs(ref).max(), name + " wgrad"
    if oc <= 4:
        got, _ = b.test_conv(ctx, 0, 4, b.BF16, g, x, wt, n * oc)
        check_bf16(got.reshape(n, oc), x.astype(np.float64) @ wt.astype(np.float64).T, name + " fprop")


# ------------------------------------------------------------------------------------------------
# BF16 at ragged batches: which kernel a GEMM runs depends on the batch.  A tensor-core tile exists only when pick_row_tile (kernels_tc.cu)
# finds one for the batch; the fused BatchNorm epilogues (EPI_STATS / EPI_BNBWD) also need every tile inside one statistics group
# (tc_epi_ok: images per group % images per tile == 0).  Otherwise the SIMT kernels, or the tensor-core GEMM followed by the unfused
# k_bn_stats_acc / k_bn_bwd_stats_acc, take over.  DCGAN 32x32, nf = 64, z = 16 (every channel count tensor-core eligible), per-net batches
# N in {1, 3, 4, 8}: between them the layers of one step take all three routes.
# ------------------------------------------------------------------------------------------------
SWEEP_SIZE, SWEEP_Z, SWEEP_NF = 32, 16, 64


def _sweep_routes(n):
    """Route of every GEMM of the generator's train forward (n images, one statistics group) and of the discriminator's pass of the D
    update (2n images, two groups of n): "fused" (tensor core, BatchNorm statistics in the epilogue), "unfused" (tensor core, then
    k_bn_stats_acc), "tc" (tensor core, no BatchNorm after it), "simt".  (net, layer name, route)"""
    def bn_route(rows, groups, gh, gw):
        nt = _pick_row_tile(rows, gh, gw)
        if nt is None:
            return "simt"
        return "fused" if (rows // groups) % nt == 0 else "unfused"
    out = [("G", "gen_deconv_1", "simt"),                          # z -> 4x4: the 1x1 problem with a 16-long reduction (dense_small_k, by design)
           ("G", "gen_deconv_2", bn_route(n, 1, 4, 4)),             # conv-equivalent output grid = the 4x4 input map
           ("G", "gen_deconv_3", bn_route(n, 1, 8, 8)),
           ("G", "gen_deconv_4", "tc"),                             # pixel-shuffle conv over 16x16 blocks: a tile for every batch
           ("D", "dis_conv_1", "tc"),                               # 3-channel edge conv
           ("D", "dis_conv_2", bn_route(2 * n, 2, 8, 8)),
           ("D", "dis_conv_3", bn_route(2 * n, 2, 4, 4)),
           ("D", "dis_conv_4", "simt")]                             # the logit (one output unit, by design)
    return out


SWEEP_N = (1, 3, 4, 8)
# Largest relative Frobenius error of any gradient tensor checked on injected activations, measured at N = 8 (every BatchNorm fused) on an
# H100 80GB HBM3: 0.0364; bound = 2x that.  Every ragged N must meet the same bound: the fallback routes may not be less accurate than the
# fused one (measured at N = 1 / 3 / 4: 0.0069 / 0.0061 / 0.0069).
SWEEP_GRAD_FRO = 0.073
# The D pass of the step (two BatchNorm groups of N: the unfused routes) is compared with the oracle run on its own, not on injected
# activations, so rounding compounds through the layers and grows as the groups shrink.  Measured on the same H100: 0.051 / 0.080 / 0.090 /
# 0.123 at N = 8 / 4 / 3 / 1; bound = 2x the largest.  A wrong route (statistics of the wrong group, a missing term) is off by O(1).
SWEEP_STEP_D_FRO = 0.25


def test_ragged_batch_route_table_covers_every_route():
    routes = {r for n in SWEEP_N for _, _, r in _sweep_routes(n)}
    assert {"fused", "unfused", "simt"} <= routes, routes
    assert all(r == "fused" for _, name, r in _sweep_routes(8) if name in ("gen_deconv_2", "gen_deconv_3", "dis_conv_2", "dis_conv_3"))


def _oracle_grads(onet):
    out = {}
    for li, l in enumerate(onet.layers):
        if l.has_params:
            for pname, _, _ in l.param_specs():
                out[(li, pname)] = flat_order(l, pname)
    return out


def _check_grads(got_flat, want, onet, specs, what, fro_bound, errs, injected=True):
    """injected: the oracle ran on the GPU's own activations, so the running-statistic pseudo-gradients (1 - decay) * (running - batch
    statistic) must match to 1e-4 relative; otherwise they are held to the Frobenius bound like every other gradient."""
    got = grads_by_tensor(onet, got_flat)
    for (li, pname), gv in got.items():
        ref = want[(li, pname)]
        if injected and pname in ("mean", "var"):
            e = float(np.abs(gv - ref).max() / (np.abs(ref).max() + 1e-30))
            assert e <= 1e-4, (f"{what}: {specs[li].get('name')}.{pname}", e)
            continue
        fro = rel_fro(gv, ref); errs.append(fro)
        if fro_bound is not None:
            assert fro <= fro_bound, (f"{what}: {specs[li].get('name')}.{pname}", fro, fro_bound)


@pytest.mark.parametrize("n", SWEEP_N)
def test_bf16_ragged_batch_routes_layer_by_layer(b200, n):
    b, ctx = b200
    from gan_deeplearning4j_b200 import models as m
    from helpers import push_params, randomize
    size, z, nf = SWEEP_SIZE, SWEEP_Z, SWEEP_NF
    rng = np.random.default_rng(31 + n)
    gs, ds, dshape = m.dcgan_generator(size, z, nf, 3), m.dcgan_discriminator(size, nf, 3), (3, size, size)
    data = [np.asarray(a, np.float32) for a in o.synthetic_batch(n, size, 3, z, seed=40 + n)]
    q = o.Quirks(xent_clip_eps=0.0)
    G = o.net_from_specs(gs, (z,), quirks=q, dtype=np.float32, seed=1); D = o.net_from_specs(ds, dshape, quirks=q, dtype=np.float32, seed=2, flat_input=False)
    randomize(G, rng); randomize(D, rng)
    bG = b.Net(ctx, gs, (z,), max_batch=n, precision=b.BF16, xent_clip_eps=0.0)
    bD = b.Net(ctx, ds, dshape, max_batch=2 * n, precision=b.BF16, xent_clip_eps=0.0, bn_groups=2)
    push_params(G, bG); push_params(D, bD)
    bf16_weights(G); bf16_weights(D)
    routes = _sweep_routes(n)
    errs = []
    # ---- the SIMT count of a train-mode forward is the table's (the D pass and D.output see the same 2N rows)
    x2 = np.concatenate([data[0], rng.uniform(-1, 1, data[0].shape).astype(np.float32)])
    for net, tag, x in ((bG, "G", data[1]), (bD, "D", x2)):
        s0 = net.simt_gemm_calls(); net.output(x, train=True)
        assert net.simt_gemm_calls() - s0 == sum(r == "simt" for t, _, r in routes if t == tag), (tag, n, routes)
    # ---- inference-mode slicing invariance: the first k images of a batch through the kernels of batch k (other routes, same inputs)
    for net, specs, x in ((bG, gs, data[1]), (bD, ds, x2)):
        full = net.output(x)
        layers = [li for li, s in enumerate(specs) if s["type"] == "batchnorm" or
                  (s["type"] in ("conv2d", "deconv2d", "dense") and not (li + 1 < len(specs) and specs[li + 1]["type"] == "batchnorm"))]
        acts = {li: net.activation(li, x.shape[0]) for li in layers}
        for k in sorted({1, max(1, x.shape[0] - 1)}):
            if k == x.shape[0]:
                continue
            part = net.output(x[:k])
            tol = lambda ref: 2 * 2.0 ** -8 * np.abs(ref) + 2e-3 * np.sqrt(np.mean(ref.astype(np.float64) ** 2)) + 1e-30
            assert (np.abs(part - full[:k]) <= tol(full[:k])).all(), ("output", n, k)
            for li in layers:
                ref = acts[li][:k]
                assert (np.abs(net.activation(li, k) - ref) <= tol(ref)).all(), (specs[li]["name"], n, k)
    # ---- D's train pass on 2N images (one statistics group), layer by layer with injected activations; every gradient incl. mean / var
    y2 = np.concatenate([data[3], data[4]])
    bD.compute_gradient_and_score(x2, y2)
    inject_forward(D, bD, ds, bf16_round(x2), 2 * n, f"D (2N = {2 * n})")
    _, eps = D.layers[-1].score_and_eps(y2.astype(np.float32))
    D.backward_from_prefix(eps)
    _check_grads(bD.gradients(), _oracle_grads(D), D, ds, f"D train pass, N = {n}", SWEEP_GRAD_FRO, errs)
    # ---- the adversarial step.  Its D pass runs 2N images as two BatchNorm groups (the unfused routes): its gradients are still in D's
    # gradient buffer afterwards (the G step through D computes no D weight gradient); reference = the oracle on each group, summed
    x_fake = bG.output(data[1])                                     # gen.output(z_d): what the step feeds D as fakes (same kernels, same params)
    D0 = [copy.deepcopy(l) for l in D.layers]
    gan = b.Gan(bG, bD, use_cuda_graph=False)
    gan.step(*data)
    want = {}
    for gi, (xg_, yg_) in enumerate(((bf16_round(data[0]), data[3]), (bf16_round(x_fake.reshape(data[0].shape)), data[4]))):
        D.layers = [copy.deepcopy(l) for l in D0]
        cur = xg_.astype(np.float32)
        for l in D.layers:
            cur = l.forward(cur, True)
        _, eps = D.layers[-1].score_and_eps(yg_.astype(np.float32))
        D.backward_from_prefix(eps)
        for key, v in _oracle_grads(D).items():
            want[key] = want.get(key, 0) + (0.5 * v if key[1] in ("mean", "var") else v)
    step_errs = []
    _check_grads(bD.gradients(), want, D, ds, f"D pass of the step (two groups of N = {n})", SWEEP_STEP_D_FRO, step_errs, injected=False)
    # ---- the generator step: G train forward on z_g and D forward on its output, injected; every G gradient incl. mean / var
    D.layers = [copy.deepcopy(l) for l in D0]
    D.set_params_flat(bD.params().astype(np.float32))
    bf16_weights(D)
    xg = inject_forward(G, bG, gs, bf16_round(data[2]), n, f"G (train, N = {n})")
    inject_forward(D, bD, ds, xg, n, f"D (G step, N = {n})")
    _, eps = D.layers[-1].score_and_eps(data[5].astype(np.float32))
    eps_g = D.backward_from_prefix(eps).reshape(xg.shape)
    for l in reversed(G.layers):
        eps_g = l.backward(eps_g)
    _check_grads(bG.gradients(), _oracle_grads(G), G, gs, f"G step, N = {n}", SWEEP_GRAD_FRO, errs)
    print(f"ragged-batch sweep N={n}: largest relative Frobenius gradient error {max(errs):.4g} (injected), {max(step_errs):.4g} (D pass of the step)")
    gan.close(); bG.close(); bD.close()
