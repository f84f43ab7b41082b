"""GPU parity tests: the CUDA path (through the C-ABI, via ctypes) against the CPU oracle on identical inputs.

FP32 mode is the DL4J-parity mode: activations, gradients, scores and post-update parameters must match the
fp64 oracle within 1e-3 relative (north_star's tolerance; written as TOL below).  BF16 (tensor-core) mode is
compared kernel-by-kernel against the oracle evaluated on the same bf16-rounded operands (SURVEY.md section 7
"hard parts"), and end to end with a tolerance that reflects 8-bit mantissas.
"""
import numpy as np
import pytest

from gan_deeplearning4j_b200 import models as m
from helpers import (assert_close_up_to_sign_flips, b200, bf16_round, check_weight_operands, fp32_gan_pair, push_params, randomize, rel_err)
from oracle import dl4j_oracle as o

pytestmark = pytest.mark.gpu

TOL = 1e-3   # north_star: "within 1e-3 relative fp32"


def every_layer_specs(act="tanh"):
    u = m.adam(1e-2)
    return [
        {"type": "batchnorm", "name": "bn0", "updater": u},
        {"type": "conv2d", "name": "c1", "n_out": 8, "kernel": (3, 3), "stride": (2, 2), "padding": (1, 1), "activation": act, "alpha": 0.2, "updater": u, "l2": 1e-3},
        {"type": "maxpool", "name": "mp", "kernel": (2, 2), "stride": (1, 1)},
        {"type": "upsample2d", "name": "up", "size": 2},
        {"type": "deconv2d", "name": "d1", "n_out": 6, "kernel": (4, 4), "stride": (2, 2), "padding": (1, 1), "updater": m.rmsprop(1e-2, 0.9, 1e-6), "has_bias": False},
        {"type": "batchnorm", "name": "bn1", "updater": u}, {"type": "activation", "name": "a1", "activation": "lrelu", "alpha": 0.2},
        {"type": "conv2d", "name": "c2", "n_out": 2, "kernel": (5, 5), "stride": (1, 1), "padding": (2, 2), "activation": "sigmoid", "updater": m.sgd(0.05), "l2": 1e-3},
        {"type": "cnn_to_ff", "name": "flat"},
        {"type": "dense", "name": "fc", "n_out": 7, "activation": act, "alpha": 0.2, "updater": u, "l2": 1e-3},
        {"type": "output", "name": "out", "n_out": 1, "updater": m.rmsprop(2e-3, 1e-8, 1e-8)},
    ]


@pytest.mark.parametrize("act", ["tanh", "lrelu"])
def test_fp32_every_layer_activations_gradients_and_update(b200, act):
    b, ctx = b200
    specs = every_layer_specs(act)
    rng = np.random.default_rng(0)
    onet = o.net_from_specs(specs, (3, 9, 9), grad_clip=1.0); randomize(onet, rng)
    bnet = b.Net(ctx, specs, (3, 9, 9), max_batch=6, precision=b.FP32, grad_clip=1.0)
    assert bnet.num_params() == onet.num_params()
    push_params(onet, bnet)
    np.testing.assert_allclose(bnet.params(), onet.params_flat(), rtol=1e-6)       # set/get round trip in DL4J order
    x = rng.uniform(-1, 1, (6, 3, 9, 9)); y = rng.uniform(-0.1, 1.1, (6, 1))
    # inference-mode output (BN running stats)
    assert rel_err(bnet.output(x), onet.output(x).reshape(6, -1)) < TOL
    # train-mode forward: every layer's activations
    score_o, acts, epss, eps_in = onet.compute_gradient_and_score(x, y, collect=True)
    score_b = bnet.compute_gradient_and_score(x, y)
    assert abs(score_b - score_o) < TOL * abs(score_o)
    for li, s in enumerate(specs):
        if s["type"] in ("loss",) or (s["type"] == "batchnorm" and li + 1 < len(specs) and specs[li + 1]["type"] == "activation"):
            continue                                   # BN fused with the following ActivationLayer reports the fused output
        want = acts[li + 1].reshape(6, -1)             # +1: helpers prepend the input reshape
        if s["type"] == "output":
            continue
        assert rel_err(bnet.activation(li, 6), want) < TOL, (li, s["name"])
    # gradients (minibatch sums), DL4J flattened order
    g_b, g_o = bnet.gradients(), onet.grads_flat()
    off = 0
    for li, name, p, shape, _ in onet.param_table():
        n = int(np.prod(shape))
        assert rel_err(g_b[off:off + n], g_o[off:off + n]) < TOL, (name, p)
        off += n
    # one fit step: divide-by-mb -> clip -> updater -> +l2*W -> subtract
    onet.fit(x, y); bnet.fit(x, y)
    p_b, p_o = bnet.params(), onet.params_flat()
    off = 0
    for li, name, p, shape, _ in onet.param_table():
        n = int(np.prod(shape))
        assert rel_err(p_b[off:off + n], p_o[off:off + n]) < TOL, (name, p)
        off += n
    # second step exercises the updater state (Adam t=2, RmsProp cache)
    onet.fit(x, y); bnet.fit(x, y)
    assert rel_err(bnet.params(), onet.params_flat()) < TOL
    bnet.close()


def _dcgan(size, z, nf):
    return m.dcgan_generator(size, z, nf, 3, lr=2e-3), m.dcgan_discriminator(size, nf, 3, lr=2e-3)


@pytest.mark.parametrize("fake_bn_train", [False, True])
def test_fp32_gan_step_matches_oracle(b200, fake_bn_train):
    b, ctx = b200
    n = 8
    G, D, bG, bD, data = fp32_gan_pair(b, ctx, *_dcgan(16, 12, 8), n)
    gan = b.Gan(bG, bD, fake_bn_train=fake_bn_train, use_cuda_graph=False)
    for it in range(3):
        r = o.gan_step(G, D, *data, fake_bn_train=fake_bn_train)
        losses = gan.step(*data)
        assert abs(losses[0] - r["loss_d_real"]) < TOL * max(1, abs(r["loss_d_real"])), it
        assert abs(losses[1] - r["loss_d_fake"]) < TOL * max(1, abs(r["loss_d_fake"])), it
        assert abs(losses[2] - r["loss_g"]) < TOL * max(1, abs(r["loss_g"])), it
        for onet, bnet, tag in ((D, bD, "D"), (G, bG, "G")):
            p_b, p_o = bnet.params(), onet.params_flat(); off = 0
            for li, name, p, shape, _ in onet.param_table():
                k = int(np.prod(shape))
                assert rel_err(p_b[off:off + k], p_o[off:off + k]) < 2 * TOL, (it, tag, name, p)
                off += k
    # the generator's input gradient path: D's epsilon w.r.t. its input is what G back-propagates
    gan.close(); bG.close(); bD.close()


def test_cuda_graph_replay_equals_eager(b200):
    b, ctx = b200
    n = 8
    data = o.synthetic_batch(n, 16, 3, 12, seed=4)
    outs = []
    for graph in (False, True):
        _, _, bG, bD, _ = fp32_gan_pair(b, ctx, *_dcgan(16, 12, 8), n)
        gan = b.Gan(bG, bD, use_cuda_graph=graph)
        gan.upload(*data)
        for _ in range(3):
            gan.step_resident(n)
        outs.append((gan.losses().copy(), bG.params(), bD.params()))
        gan.close(); bG.close(); bD.close()
    np.testing.assert_allclose(outs[0][0], outs[1][0], rtol=1e-5)
    np.testing.assert_allclose(outs[0][1], outs[1][1], rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(outs[0][2], outs[1][2], rtol=1e-5, atol=1e-7)


def test_fp32_reference_graphs_replay_J408_510(b200):
    """The reference file's own graphs (C1) driven exactly like the Java loop body: dis fit by two parameter-averaged
    workers, 12 D->gan copies, gan fit, 16 gan->gen copies -- through getParam/setParam/fit/output only."""
    b, ctx = b200
    n, z = 8, 2
    dis_s, gen_s, gan_s = m.reference_discriminator(0.002), m.reference_generator(0.0, z), m.reference_gan(0.004, z)
    odis = o.net_from_specs(dis_s, (1, 28, 28), grad_clip=1.0, seed=1, flat_input=False); ogen = o.net_from_specs(gen_s, (z,), grad_clip=1.0, seed=2); ogan = o.net_from_specs(gan_s, (z,), grad_clip=1.0, seed=3)
    ng = len(gen_s)
    mk = lambda s, shp, mb: b.Net(ctx, s, shp, max_batch=mb, precision=b.FP32, grad_clip=1.0)
    bdis, bw0, bw1, bgen, bgan = mk(dis_s, (1, 28, 28), n), mk(dis_s, (1, 28, 28), n), mk(dis_s, (1, 28, 28), n), mk(gen_s, (z,), n), mk(gan_s, (z,), n)
    push_params(odis, bdis); push_params(ogen, bgen); push_params(ogan, bgan)
    rng = np.random.default_rng(0)
    x = np.round(rng.uniform(0, 1, (n, 784)), 2)
    z_d = rng.uniform(-1, 1, (n, z)); z_g = rng.uniform(-1, 1, (n, z))
    y_r = 1 + 0.05 * rng.standard_normal((n, 1)); y_f = 0.05 * rng.standard_normal((n, 1)); y_g = np.ones((n, 1))
    # the oracle's gan graph in helpers has an extra input reshape only for conv inputs -> gen part starts at index 0
    r = o.gan_iteration_reference(odis, ogen, ogan, ng, x.reshape(n, 1, 28, 28), z_d, z_g, y_r, y_f, y_g)
    # ---- CUDA replay
    x_fake = bgen.output(z_d)                                                 # gen.output(...)  J:420
    assert rel_err(x_fake, r["x_fake"].reshape(n, -1)) < TOL
    for w in (bw0, bw1):
        w.set_params(bdis.params()); w.set_updater_state(bdis.updater_state())
    s0 = bw0.fit(x, y_r); s1 = bw1.fit(x_fake, y_f)                           # two Spark workers, one minibatch each
    assert abs(s0 - r["score_d_real"]) < TOL * abs(r["score_d_real"]) and abs(s1 - r["score_d_fake"]) < TOL * abs(r["score_d_fake"])
    bdis.set_params(0.5 * (bw0.params() + bw1.params()))                      # ParameterAveragingTrainingMaster: params AND updater state
    bdis.set_updater_state(0.5 * (bw0.updater_state() + bw1.updater_state()))
    assert_close_up_to_sign_flips(bdis.params(), odis.params_flat(), 0.002, TOL)
    for s in dis_s:                                                           # J:429-460
        for p, cnt in _params_of(s, bdis):
            bgan.set_param(s["name"].replace("dis_", "gan_dis_", 1), p, bdis.get_param(s["name"], p, cnt))
    s2 = bgan.fit(z_g, y_g)                                                   # sparkGan.fit  J:471
    assert abs(s2 - r["score_gan"]) < TOL * abs(r["score_gan"])
    for s in gen_s:                                                           # J:474-510
        for p, cnt in _params_of(s, bgen):
            bgen.set_param(s["name"], p, bgan.get_param(s["name"].replace("gen_", "gan_", 1), p, cnt))
    assert_close_up_to_sign_flips(bgen.params(), ogen.params_flat(), 0.004, TOL)
    assert_close_up_to_sign_flips(bgan.params(), ogan.params_flat(), 0.004, TOL)
    for nn in (bdis, bw0, bw1, bgen, bgan):
        nn.close()


def _params_of(spec, net):
    t = spec["type"]
    if t == "batchnorm":
        c = net.get_param  # sizes are discovered by asking for a wrong size first is clumsy; use the spec tables instead
        size = {"dis_batch_layer_1": 1, "gen_batch_1": 2, "gen_batch_4": 6272}[spec["name"]]
        return [(p, size) for p in ("gamma", "beta", "mean", "var")]
    if t in ("conv2d", "dense", "output"):
        sizes = {"dis_conv2d_layer_2": (1600, 64), "dis_conv2d_layer_4": (204800, 128), "dis_dense_layer_6": (1152 * 1024, 1024), "dis_output_layer_7": (1024, 1),
                 "gen_dense_layer_2": (2 * 1024, 1024), "gen_dense_layer_3": (1024 * 6272, 6272), "gen_conv2d_6": (204800, 64), "gen_conv2d_8": (1600, 1)}[spec["name"]]
        return [("W", sizes[0]), ("b", sizes[1])]
    return []


# ------------------------------------------------------------------------------------------------
# bf16 / kernel-level parity
# ------------------------------------------------------------------------------------------------
CONV_CASES = [
    # n, h, w, c, o, k, s, p
    (2, 8, 8, 16, 24, 4, 2, 1), (3, 7, 9, 5, 6, 5, 2, 0), (2, 14, 14, 8, 4, 5, 1, 2), (4, 1, 1, 20, 12, 1, 1, 0), (2, 4, 4, 32, 1, 4, 1, 0),
]


def _conv_ref(n, h, w, c, oc, k, s, p, rng, rnd):
    x = rnd(rng.standard_normal((n, c, h, w))); wt = rnd(rng.standard_normal((oc, c, k, k)) / np.sqrt(c * k * k))
    l = o.Conv2D(c, oc, (k, k), (s, s), (p, p), has_bias=False); l.init(np.random.default_rng(0), np.float64)
    l.params["W"] = wt.astype(np.float64)
    y = l.forward(x.astype(np.float64), True)
    dy = rnd(rng.standard_normal(y.shape)).astype(np.float64)
    dx = l.backward(dy)
    return x, wt, y, dy, dx, l.grads["W"]


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("case", CONV_CASES)
def test_simt_conv_kernels_match_oracle(b200, case, prec):
    b, ctx = b200
    n, h, w, c, oc, k, s, p = case
    rng = np.random.default_rng(1)
    rnd = bf16_round if prec == "bf16" else (lambda a: np.asarray(a, np.float32))
    P = b.BF16 if prec == "bf16" else b.FP32
    tol = 1e-2 if prec == "bf16" else 1e-4            # bf16: outputs are rounded to bf16 (2^-9) on store
    x, wt, y, dy, dx, dw = _conv_ref(n, h, w, c, oc, k, s, p, rng, rnd)
    oh, ow = y.shape[2], y.shape[3]
    geom = dict(n=n, h=h, w=w, c=c, oh=oh, ow=ow, o=oc, kh=k, kw=k, sh=s, sw=s, ph=p, pw=p)
    x_nhwc = x.transpose(0, 2, 3, 1); w_int = wt.transpose(0, 2, 3, 1); dy_nhwc = dy.transpose(0, 2, 3, 1)
    out, _ = b.test_conv(ctx, 0, 0, P, geom, x_nhwc, w_int, y.size)
    assert rel_err(out.reshape(n, oh, ow, oc), y.transpose(0, 2, 3, 1)) < tol
    out, _ = b.test_conv(ctx, 1, 0, P, geom, dy_nhwc, w_int, dx.size)
    assert rel_err(out.reshape(n, h, w, c), dx.transpose(0, 2, 3, 1)) < tol
    out, _ = b.test_conv(ctx, 2, 0, P, geom, x_nhwc, dy_nhwc, dw.size)
    assert rel_err(out.reshape(oc, k, k, c), dw.transpose(0, 2, 3, 1)) < (1e-4 if prec == "fp32" else 1e-3)   # fp32 accumulate, fp32 out


def test_bf16_gan_step_tracks_oracle(b200):
    """End to end in tensor-core mode: same step, bf16 activations/weights, fp32 accumulation and master weights."""
    b, ctx = b200
    n = 16
    G, D, bG, bD, data = fp32_gan_pair(b, ctx, *_dcgan(16, 12, 8), n, quirks=o.Quirks(xent_clip_eps=0.0), precision=b.BF16, xent_clip_eps=0.0)
    gan = b.Gan(bG, bD, use_cuda_graph=False)
    r = o.gan_step(G, D, *data)
    losses = gan.step(*data)
    assert abs(losses[0] - r["loss_d_real"]) < 0.05 and abs(losses[1] - r["loss_d_fake"]) < 0.05 and abs(losses[2] - r["loss_g"]) < 0.05
    # Adam's first step moves every weight by ~lr*sign(g): compare the update direction where the gradient is not tiny
    gan.close(); bG.close(); bD.close()


def test_full_size_c2_step_properties(b200):
    """BASELINE config C2 (64x64x3, z=100, batch 128) at full size: size-independent properties."""
    b, ctx = b200
    n = 128
    gs, ds = m.dcgan_generator(64, 100, 64, 3), m.dcgan_discriminator(64, 64, 3)
    bG = b.Net(ctx, gs, (100,), max_batch=n, precision=b.BF16, xent_clip_eps=0.0)
    bD = b.Net(ctx, ds, (3, 64, 64), max_batch=2 * n, precision=b.BF16, xent_clip_eps=0.0, bn_groups=2)
    assert (bG.num_params(), bD.num_params()) == (3578627, 2767425)
    gan = b.Gan(bG, bD, use_cuda_graph=True)
    data = o.synthetic_batch(n, 64, 3, 100, seed=666)
    pG0, pD0 = bG.params(), bD.params()
    gan.upload(*data)
    first = None
    for it in range(6):
        gan.step_resident(n)
        l = gan.losses()
        assert np.all(np.isfinite(l)), l
        first = l if first is None else first
    pG1, pD1 = bG.params(), bD.params()
    assert np.all(np.isfinite(pG1)) and np.all(np.isfinite(pD1))
    # Adam with lr 2e-4: after 6 steps no weight moved by more than ~6*lr*(1+slack); BN running stats by at most the decay rule
    assert np.abs(pG1 - pG0).max() < 1.0 and 0 < np.abs(pD1 - pD0).max() < 1.0
    # the discriminator learns the fixed synthetic batch: its loss on it goes down
    assert l[0] + l[1] < first[0] + first[1]
    # generated images are in tanh range
    xg = bG.output(data[1][:8])
    assert xg.shape == (8, 3 * 64 * 64) and np.abs(xg).max() <= 1.0
    gan.close(); bG.close(); bD.close()


# ------------------------------------------------------------------------------------------------
# wgmma tensor-core kernels vs the oracle on bf16-rounded operands (and vs the SIMT kernel)
# ------------------------------------------------------------------------------------------------
TC_FPROP_CASES = [
    # n, h, w, c, o, k, s, p
    (2, 16, 16, 64, 64, 4, 2, 1),      # 8x8 out: two images per 128-row tile, BN=64
    (1, 32, 32, 64, 128, 4, 2, 1),     # 16x16 out: 8 rows of one image per tile, BN=128 (D2 shape, one image)
    (8, 8, 8, 128, 256, 4, 2, 1),      # 4x4 out: eight images per tile, two 64-channel chunks, BN=128 (D4-like)
    (2, 8, 8, 64, 64, 3, 1, 1),        # stride 1
    (4, 9, 9, 64, 128, 5, 2, 0),       # reference-style 5x5 s2 p0, Truncate: 3x3 out ... not tileable -> must be refused
    (128, 1, 1, 128, 64, 1, 1, 0),     # dense layer as 1x1 conv
]


@pytest.mark.parametrize("case", TC_FPROP_CASES)
def test_tc_fprop_matches_oracle(b200, case):
    b, ctx = b200
    n, h, w, c, oc, k, s, p = case
    rng = np.random.default_rng(2)
    x, wt, y, dy, dx, dw = _conv_ref(n, h, w, c, oc, k, s, p, rng, bf16_round)
    oh, ow = y.shape[2], y.shape[3]
    geom = dict(n=n, h=h, w=w, c=c, oh=oh, ow=ow, o=oc, kh=k, kw=k, sh=s, sw=s, ph=p, pw=p)
    x_nhwc = x.transpose(0, 2, 3, 1); w_int = wt.transpose(0, 2, 3, 1)
    if (oh * ow) % 128 and 128 % (oh * ow):
        with pytest.raises(b.B200GanError):
            b.test_conv(ctx, 0, 1, b.BF16, geom, x_nhwc, w_int, y.size)
        return
    out, _ = b.test_conv(ctx, 0, 1, b.BF16, geom, x_nhwc, w_int, y.size)
    assert rel_err(out.reshape(n, oh, ow, oc), y.transpose(0, 2, 3, 1)) < 1e-2     # bf16 store: 2^-9 relative per element
    ref, _ = b.test_conv(ctx, 0, 0, b.BF16, geom, x_nhwc, w_int, y.size)            # SIMT kernel, same operands
    assert rel_err(out, ref) < 1e-2


TC_DGRAD_CASES = [
    # conv geometry: n, h, w, c (dx), o (dy channels); dy is h/2 x w/2
    (2, 16, 16, 64, 64), (1, 32, 32, 128, 128), (8, 8, 8, 64, 256), (2, 64, 64, 64, 64),
]


@pytest.mark.parametrize("case", TC_DGRAD_CASES)
def test_tc_dgrad_phase_form_matches_oracle(b200, case):
    """conv input-gradient == Deconvolution2D forward (4x4 s2 p1) as four sub-pixel 2x2 convolutions."""
    b, ctx = b200
    n, h, w, c, oc = case
    rng = np.random.default_rng(3)
    x, wt, y, dy, dx, dw = _conv_ref(n, h, w, c, oc, 4, 2, 1, rng, bf16_round)
    geom = dict(n=n, h=h, w=w, c=c, oh=h // 2, ow=w // 2, o=oc, kh=4, kw=4, sh=2, sw=2, ph=1, pw=1)
    dy_nhwc = dy.transpose(0, 2, 3, 1); w_int = wt.transpose(0, 2, 3, 1)
    out, _ = b.test_conv(ctx, 1, 1, b.BF16, geom, dy_nhwc, w_int, dx.size)
    assert rel_err(out.reshape(n, h, w, c), dx.transpose(0, 2, 3, 1)) < 1e-2


# the tensor-core weight gradients are checked at every split schedule, bit for bit on integer operands, in tests/test_gpu_tc_wgrad.py


TC_EDGE_CASES = [
    # conv geometry 4x4 s2 p1 with <= 4 image channels: n, h, w, c (image side), o (feature side)
    (4, 64, 64, 3, 64),       # DCGAN D1 / G-last
    (2, 128, 128, 3, 64),     # C4: 128x128 images
    (8, 16, 16, 3, 128),      # two images per 128-pixel tile, two 64-channel K chunks
    (2, 32, 32, 4, 64), (2, 32, 32, 1, 64),
]


@pytest.mark.parametrize("case", TC_EDGE_CASES)
def test_tc_skinny_layer_kernels_match_oracle(b200, case):
    """Tensor-core versions of the <= 4-image-channel layers: transposed conv as ONE 3x3 conv over 2x2 output blocks (pixel-shuffle epilogue)."""
    b, ctx = b200
    n, h, w, c, oc = case
    rng = np.random.default_rng(5)
    x, wt, y, dy, dx, dw = _conv_ref(n, h, w, c, oc, 4, 2, 1, rng, bf16_round)
    geom = dict(n=n, h=h, w=w, c=c, oh=h // 2, ow=w // 2, o=oc, kh=4, kw=4, sh=2, sw=2, ph=1, pw=1)
    dy_nhwc = dy.transpose(0, 2, 3, 1); w_int = wt.transpose(0, 2, 3, 1)
    out, _ = b.test_conv(ctx, 1, 3, b.BF16, geom, dy_nhwc, w_int, dx.size)
    assert rel_err(out.reshape(n, h, w, c), dx.transpose(0, 2, 3, 1)) < 1e-2
    ref, _ = b.test_conv(ctx, 1, 2, b.BF16, geom, dy_nhwc, w_int, dx.size)           # SIMT skinny kernel, same operands
    assert rel_err(out, ref) < 1e-2
    # fprop: im2col rows built in shared memory (the 3-channel image cannot be gathered by TMA), one K = 64 MMA group per 128 pixels
    if w // 2 < 16:
        return        # 128-pixel tiles spanning several images are only implemented for the transposed-conv form
    x_nhwc = x.transpose(0, 2, 3, 1)
    out, _ = b.test_conv(ctx, 0, 3, b.BF16, geom, x_nhwc, w_int, y.size)
    assert rel_err(out.reshape(n, h // 2, w // 2, oc), y.transpose(0, 2, 3, 1)) < 1e-2
    if oc == 64:      # wgrad: MN-major operands, split over pixels, fp32 partials summed in fixed order
        out, _ = b.test_conv(ctx, 2, 3, b.BF16, geom, x_nhwc, dy_nhwc, dw.size)
        assert rel_err(out.reshape(oc, 4, 4, c), dw.transpose(0, 2, 3, 1)) < 1e-4


# ------------------------------------------------------------------------------------------------
# skinny-layer kernels (kernels_edge.cu) are reached through the engine: layer-level parity in both precisions
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_edge_layers_dcgan_ends(b200, prec):
    """D1 (3->64 conv), G-last (64->3 transposed conv + tanh), D-last (full-window conv -> 1 logit), G-first (z -> 4x4)
    at a size where every specialised kernel engages; fp32 vs oracle to TOL, bf16 vs oracle loosely."""
    b, ctx = b200
    P = b.BF16 if prec == "bf16" else b.FP32
    tol = 4e-2 if prec == "bf16" else TOL
    size, z, nf, n = 32, 16, 64, 8          # G: z->(4x4x256)->8x8x128->16x16x64->32x32x3 ; D: 32->16x16x64->8x8x128->4x4x256->1
    gs, ds = m.dcgan_generator(size, z, nf, 3, lr=1e-3), m.dcgan_discriminator(size, nf, 3, lr=1e-3)
    q = o.Quirks(xent_clip_eps=0.0)
    rng = np.random.default_rng(11)
    G = o.net_from_specs(gs, (z,), quirks=q, seed=1); D = o.net_from_specs(ds, (3, size, size), quirks=q, seed=2)
    randomize(G, rng); randomize(D, rng)
    bG = b.Net(ctx, gs, (z,), max_batch=n, precision=P, xent_clip_eps=0.0)
    bD = b.Net(ctx, ds, (3, size, size), max_batch=2 * n, precision=P, xent_clip_eps=0.0, bn_groups=2)
    push_params(G, bG); push_params(D, bD)
    x, z_d, z_g, y_r, y_f, y_g = [a.astype(np.float64) for a in o.synthetic_batch(n, size, 3, z, seed=5)]
    # forward of both nets (train mode)
    xg_o = G.forward(z_g, True); xg_b = bG.output(z_g, train=True)
    assert rel_err(xg_b, xg_o.reshape(n, -1)) < tol
    # D gradients on the real batch (exercises D1 fprop/wgrad, D-last fwd/dgrad/wgrad)
    s_o = D.compute_gradient_and_score(x, y_r); s_b = bD.compute_gradient_and_score(x, y_r)
    assert abs(s_b - s_o) < tol * max(1.0, abs(s_o))
    g_b, g_o = bD.gradients(), D.grads_flat(); off = 0
    for li, name, p, shape, _ in D.param_table():
        k = int(np.prod(shape))
        if p not in ("mean", "var"):
            if prec == "fp32":
                assert rel_err(g_b[off:off + k], g_o[off:off + k]) < tol, (name, p)
            else:   # bf16 activations through train-mode BN on 8 images: compare in the Frobenius norm
                d = np.linalg.norm(g_b[off:off + k] - g_o[off:off + k]) / (np.linalg.norm(g_o[off:off + k]) + 1e-30)
                assert d < 0.1, (name, p, d)
        off += k
    # full step: exercises G-last forward/wgrad/input-grad, D1 input-grad, G-first forward/wgrad
    gan = b.Gan(bG, bD, use_cuda_graph=False)
    r = o.gan_step(G, D, x, z_d, z_g, y_r, y_f, y_g)
    losses = gan.step(x, z_d, z_g, y_r, y_f, y_g)
    want = np.array([r["loss_d_real"], r["loss_d_fake"], r["loss_g"]])
    assert np.all(np.abs(losses - want) < (tol if prec == "fp32" else 0.1) * np.maximum(1.0, np.abs(want))), (losses, want)
    if prec == "fp32":
        for onet, bnet in ((D, bD), (G, bG)):
            p_b, p_o = bnet.params(), onet.params_flat(); off = 0
            for li, name, p, shape, _ in onet.param_table():
                k = int(np.prod(shape))
                if p in ("mean", "var"):
                    assert rel_err(p_b[off:off + k], p_o[off:off + k]) < 2 * TOL, (name, p)
                else:     # Adam's first step is lr*g/(|g|+eps'): elements with a numerically-zero gradient may land one step apart
                    assert_close_up_to_sign_flips(p_b[off:off + k], p_o[off:off + k], 1e-3, TOL)
                off += k
    gan.close(); bG.close(); bD.close()


# ------------------------------------------------------------------------------------------------
# C5: MLP-GAN (dense / OutputLayer path) and C4 (128x128, 5-stage) 
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_mlp_gan_step_matches_oracle(b200, prec):
    """Dense layers + OutputLayer(XENT): fp32 to TOL; bf16 at tensor-core-eligible sizes (batch 128, widths multiple of 128) loosely."""
    b, ctx = b200
    P = b.BF16 if prec == "bf16" else b.FP32
    n, z, hid, d = 128, 128, 256, 128
    gs, ds = m.mlp_generator(z, hid, d, lr=1e-3), m.mlp_discriminator(d, hid, lr=1e-3)
    q = o.Quirks(xent_clip_eps=0.0)
    rng = np.random.default_rng(21)
    G = o.net_from_specs(gs, (z,), quirks=q, seed=1); D = o.net_from_specs(ds, (d,), quirks=q, seed=2)
    randomize(G, rng); randomize(D, rng)
    bG = b.Net(ctx, gs, (z,), max_batch=n, precision=P, xent_clip_eps=0.0)
    bD = b.Net(ctx, ds, (d,), max_batch=2 * n, precision=P, xent_clip_eps=0.0, bn_groups=2)
    push_params(G, bG); push_params(D, bD)
    x = rng.uniform(-1, 1, (n, d)); z_d = rng.uniform(-1, 1, (n, z)); z_g = rng.uniform(-1, 1, (n, z))
    y_r = 1 + 0.05 * rng.standard_normal((n, 1)); y_f = 0.05 * rng.standard_normal((n, 1)); y_g = np.ones((n, 1))
    # gradients of D on the real batch
    s_o = D.compute_gradient_and_score(x, y_r); s_b = bD.compute_gradient_and_score(x, y_r)
    tol = TOL if prec == "fp32" else 3e-2
    assert abs(s_b - s_o) < tol * max(1.0, abs(s_o))
    g_b, g_o = bD.gradients(), D.grads_flat()
    err = np.linalg.norm(g_b - g_o) / np.linalg.norm(g_o)
    assert err < (TOL if prec == "fp32" else 3e-2), err
    gan = b.Gan(bG, bD, use_cuda_graph=False)
    r = o.gan_step(G, D, x, z_d, z_g, y_r, y_f, y_g)
    losses = gan.step(x, z_d, z_g, y_r, y_f, y_g)
    want = np.array([r["loss_d_real"], r["loss_d_fake"], r["loss_g"]])
    assert np.all(np.abs(losses - want) < tol * np.maximum(1.0, np.abs(want))), (losses, want)
    if prec == "fp32":
        assert_close_up_to_sign_flips(bD.params(), D.params_flat(), 1e-3, TOL)
        assert_close_up_to_sign_flips(bG.params(), G.params_flat(), 1e-3, TOL)
    gan.close(); bG.close(); bD.close()


def test_full_size_c4_and_c5_steps_run(b200):
    """BASELINE configs[3] (128x128x3, 32 per GPU) and configs[4] (MLP-GAN d=256, batch 8192) at full size: finite, learning, in range."""
    b, ctx = b200
    for name, gs, ds, gin, din, n in (("c4", m.dcgan_generator(128), m.dcgan_discriminator(128), (100,), (3, 128, 128), 32),
                                     ("c5", m.mlp_generator(128, 1024, 256), m.mlp_discriminator(256, 1024), (128,), (256,), 8192)):
        bG = b.Net(ctx, gs, gin, max_batch=n, precision=b.BF16, xent_clip_eps=0.0)
        bD = b.Net(ctx, ds, din, max_batch=2 * n, precision=b.BF16, xent_clip_eps=0.0, bn_groups=2)
        if name == "c4":
            assert m.forward_macs(gs, gin) == 551092224 and m.forward_macs(ds, din) == 549470208      # SURVEY.md 8d
        gan = b.Gan(bG, bD, use_cuda_graph=True)
        rng = np.random.default_rng(1)
        data = [rng.uniform(-1, 1, (n,) + din), rng.uniform(-1, 1, (n,) + gin), rng.uniform(-1, 1, (n,) + gin),
                1 + 0.05 * rng.standard_normal((n, 1)), 0.05 * rng.standard_normal((n, 1)), np.ones((n, 1))]
        gan.upload(*data)
        first = None
        for _ in range(5):
            gan.step_resident(n); l = gan.losses(); assert np.all(np.isfinite(l)), (name, l)
            first = l if first is None else first
        assert l[0] + l[1] < first[0] + first[1], (name, first, l)
        out = bG.output(data[1][:4]); assert np.all(np.isfinite(out)) and np.abs(out).max() <= 1.0
        gan.close(); bG.close(); bD.close()


# ------------------------------------------------------------------------------------------------
# error behaviour at the boundary (DL4J throws; the C-ABI returns codes that the mirrors raise)
# ------------------------------------------------------------------------------------------------
def test_boundary_error_codes(b200):
    b, ctx = b200
    specs = m.dcgan_discriminator(16, 8, 3)
    net = b.Net(ctx, specs, (3, 16, 16), max_batch=4, precision=b.FP32)
    with pytest.raises(b.B200GanError) as e:                     # batch larger than max_batch
        net.output(np.zeros((5, 3, 16, 16), np.float32))
    assert e.value.code == -2
    with pytest.raises(b.B200GanError) as e:                     # unknown layer
        net.set_param("no_such_layer", "W", np.zeros(3, np.float32))
    assert e.value.code == -1
    with pytest.raises(b.B200GanError) as e:                     # wrong element count (DL4J: shape mismatch on setParam)
        net.set_param("dis_conv_1", "W", np.zeros(7, np.float32))
    assert e.value.code == -2
    with pytest.raises(b.B200GanError) as e:                     # BN has no "W"
        net.get_param("dis_bn_2", "W", 4)
    assert e.value.code == -1
    with pytest.raises(b.B200GanError) as e:                     # nIn that contradicts the incoming shape
        b.Net(ctx, [{"type": "conv2d", "name": "c", "n_in": 5, "n_out": 4, "kernel": (3, 3)}], (3, 8, 8), max_batch=2)
    assert e.value.code == -2
    with pytest.raises(b.B200GanError) as e:                     # dense on a convolutional activation without CnnToFeedForward
        b.Net(ctx, [{"type": "dense", "name": "d", "n_out": 4}], (3, 8, 8), max_batch=2)
    assert e.value.code == -2
    with pytest.raises(b.B200GanError) as e:                     # fit needs a loss-bearing last layer
        b.Net(ctx, [{"type": "dense", "name": "d", "n_out": 4}], (8,), max_batch=2).fit(np.zeros((2, 8)), np.zeros((2, 1)))
    assert e.value.code == -6
    # ragged batches: every batch size from 1 up to max works and matches the oracle (falls back to non-tiled kernels)
    onet = o.net_from_specs(specs, (3, 16, 16)); push_params(onet, net)
    for bs in (1, 3, 4):
        x = np.random.default_rng(bs).uniform(-1, 1, (bs, 3, 16, 16))
        assert rel_err(net.output(x), onet.output(x).reshape(bs, -1)) < TOL
    net.close()


def test_fp32_transfer_learning_head_matches_oracle(b200):
    """SURVEY 8f #3 (J:337-364, 512-545): frozen D trunk + BatchNormalization(1024) + OutputLayer(MCXENT, softmax, 10)."""
    b, ctx = b200
    n = 8
    odis = o.net_from_specs(m.reference_discriminator(), (1, 28, 28), grad_clip=1.0, seed=1, flat_input=False)
    rng = np.random.default_rng(3); randomize(odis, rng)
    ocv = o.reference_computer_vision(odis)
    specs = m.reference_computer_vision()
    bcv = b.Net(ctx, specs, (1, 28, 28), max_batch=n, precision=b.FP32, grad_clip=1.0)
    assert bcv.num_params() == ocv.num_params()
    # the driver copies the trunk by name (J:516-542); the new layers get the oracle's init
    for s in specs:
        l = ocv.layer(s["name"]) if s["type"] in ("batchnorm", "conv2d", "dense", "output") else None
        if l is not None:
            for p, shape, order in l.param_specs():
                bcv.set_param(s["name"], p, l.params[p].ravel(order=order.upper()))
    np.testing.assert_allclose(bcv.params(), ocv.params_flat(), rtol=1e-6)
    x = np.round(rng.uniform(0, 1, (n, 784)), 2); y = np.eye(10)[rng.integers(0, 10, n)]
    xo = x.reshape(n, 1, 28, 28)
    assert rel_err(bcv.output(x), ocv.output(xo)) < TOL                       # softmax probabilities, test-mode trunk
    s_o = ocv.compute_gradient_and_score(xo, y); s_b = bcv.compute_gradient_and_score(x, y)
    assert abs(s_b - s_o) < TOL * abs(s_o)
    g_b, g_o = bcv.gradients(), ocv.grads_flat(); off = 0
    for li, name, p, shape, _ in ocv.param_table():
        k = int(np.prod(shape))
        if name in ("dis_batch", "dis_output_layer_7"):
            assert rel_err(g_b[off:off + k], g_o[off:off + k]) < TOL, (name, p)
        else:
            assert not np.any(g_b[off:off + k]), (name, p)                     # FrozenLayer: no gradient at all
        off += k
    p0 = bcv.params()
    ocv.fit(xo, y); bcv.fit(x, y)
    p1 = bcv.params(); off = 0
    for li, name, p, shape, _ in ocv.param_table():
        k = int(np.prod(shape))
        if name in ("dis_batch", "dis_output_layer_7"):
            assert_close_up_to_sign_flips(p1[off:off + k], ocv.params_flat()[off:off + k], 0.002, TOL)
        else:
            assert np.array_equal(p1[off:off + k], p0[off:off + k]), (name, p)  # not even l2-decayed
        off += k
    bcv.close()


def test_reference_program_replay_end_to_end(b200, tmp_path):
    """examples/gan_computer_vision.py = the Java main replayed: CSV in, two iterations, sample + prediction CSVs and parameter dumps out."""
    import subprocess, sys, os
    from gan_deeplearning4j_b200 import data
    rng = np.random.default_rng(0)
    data.write_csv(str(tmp_path / "train.csv"), rng.uniform(0, 1, (48, 784)), rng.integers(0, 10, 48))
    data.write_csv(str(tmp_path / "test.csv"), rng.uniform(0, 1, (30, 784)), rng.integers(0, 10, 30))
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "examples", "gan_computer_vision.py"), "--train-csv", str(tmp_path / "train.csv"),
                        "--test-csv", str(tmp_path / "test.csv"), "--out", str(tmp_path / "out"), "--iterations", "2", "--batch", "16"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "Completed Batch 2!" in r.stdout
    out = np.loadtxt(tmp_path / "out" / "mnist_out_2.csv", delimiter=","); pred = np.loadtxt(tmp_path / "out" / "mnist_test_predictions_2.csv", delimiter=",")
    assert out.shape == (100, 784) and np.all((out >= 0) & (out <= 1))            # sigmoid images of the 10x10 latent grid
    assert pred.shape == (30, 10) and np.allclose(pred.sum(1), 1, atol=1e-4)
    assert os.path.getsize(tmp_path / "out" / "dis_coefficients_2.bin") == 4 * 1388293


# ------------------------------------------------------------------------------------------------
# committed golden fixture (tests/golden): the CUDA path against fixed bytes
# ------------------------------------------------------------------------------------------------
def test_fp32_gan_step_matches_golden_fixture(b200):
    """The same step against the committed fixture tests/golden/gan_step_dcgan16.npz (inputs, initial parameters, and the oracle's losses and
    parameters after each of 3 steps; tests/golden/make_golden.py): the CUDA path is compared with fixed bytes, not with a live oracle run."""
    import os
    b, ctx = b200
    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gan_step_dcgan16.npz"))
    size, z, nf, n = 16, 12, 8, 8
    gs, ds = m.dcgan_generator(size, z, nf, 3, lr=2e-3), m.dcgan_discriminator(size, nf, 3, lr=2e-3)
    bG = b.Net(ctx, gs, (z,), max_batch=n, precision=b.FP32, xent_clip_eps=1e-5)
    bD = b.Net(ctx, ds, (3, size, size), max_batch=2 * n, precision=b.FP32, xent_clip_eps=1e-5, bn_groups=2)
    bG.set_params(gold["g_params0"].astype(np.float32)); bD.set_params(gold["d_params0"].astype(np.float32))
    gan = b.Gan(bG, bD, use_cuda_graph=False)
    data = [gold[k] for k in ("x_real", "z_d", "z_g", "y_real", "y_fake", "y_gen")]
    for it in range(1, 4):
        losses = gan.step(*data); want = gold[f"losses{it}"]
        assert np.all(np.abs(losses - want) < TOL * np.maximum(1.0, np.abs(want))), (it, losses, want)
        assert rel_err(bD.params(), gold[f"d_params{it}"]) < 2 * TOL, it
        assert rel_err(bG.params(), gold[f"g_params{it}"]) < 2 * TOL, it
    gan.close(); bG.close(); bD.close()


def test_checkpoint_resume_equals_uninterrupted_run(b200, tmp_path):
    """ModelSerializer.writeModel / restore (J:606-618) with the updater state AND the iteration counter: N steps, save, restore into a
    fresh net, M more steps == N+M uninterrupted steps, bit for bit (Adam's bias correction depends on t: ADVICE round 1)."""
    b, ctx = b200
    specs = m.dcgan_discriminator(16, 8, 3, lr=1e-2)
    rng = np.random.default_rng(9)
    xs = [rng.uniform(-1, 1, (8, 3, 16, 16)).astype(np.float32) for _ in range(5)]; ys = [rng.uniform(0, 1, (8, 1)).astype(np.float32) for _ in range(5)]
    for prec in (b.FP32, b.BF16):
        a = b.Net(ctx, specs, (3, 16, 16), max_batch=8, precision=prec, xent_clip_eps=0.0, seed=3)
        for i in range(5):
            a.fit(xs[i], ys[i])
        c = b.Net(ctx, specs, (3, 16, 16), max_batch=8, precision=prec, xent_clip_eps=0.0, seed=3)
        for i in range(3):
            c.fit(xs[i], ys[i])
        assert c.iteration() == 3
        path = str(tmp_path / f"ckpt_{prec}.zip"); c.save(path)
        r = b.Net(ctx, specs, (3, 16, 16), max_batch=8, precision=prec, xent_clip_eps=0.0, seed=99)       # different init: everything must come from the file
        meta = r.restore(path)
        assert r.iteration() == 3 and meta["meta"]["iteration"] == 3
        for i in range(3, 5):
            r.fit(xs[i], ys[i])
        assert np.array_equal(r.params(), a.params()) and np.array_equal(r.updater_state(), a.updater_state()) and r.iteration() == 5
        # without the counter the resumed Adam restarts its bias correction: the run must diverge (this is what the counter is for)
        w = b.Net(ctx, specs, (3, 16, 16), max_batch=8, precision=prec, xent_clip_eps=0.0, seed=99)
        w.set_params(c.params()); w.set_updater_state(c.updater_state())
        for i in range(3, 5):
            w.fit(xs[i], ys[i])
        assert not np.array_equal(w.params(), a.params())
        for net in (a, c, r, w):
            net.close()


def test_xavier_init_statistics(b200):
    """WeightInit.XAVIER (J:127): W ~ N(0, 2/(fanIn+fanOut)) with conv fanIn = nIn*kH*kW, fanOut = nOut*kH*kW/(sH*sW); biases 0;
    BatchNorm gamma 1, beta 0, mean 0, var 1 -- the formula the oracle's Layer.init restates (dl4j_oracle.Conv2D.fans)."""
    b, ctx = b200
    for specs, shape, onet in ((m.dcgan_discriminator(64, 64, 3), (3, 64, 64), o.dcgan_discriminator(64, 64, 3)), (m.dcgan_generator(64, 100, 64, 3), (100,), o.dcgan_generator(64, 100, 64, 3))):
        net = b.Net(ctx, specs, shape, max_batch=2, precision=b.FP32, seed=666)
        other = b.Net(ctx, specs, shape, max_batch=2, precision=b.FP32, seed=667)
        for s, l in zip(specs, onet.layers):
            if s["type"] in ("conv2d", "deconv2d"):
                fi, fo = l.fans()
                w = net.get_param(s["name"], "W", int(np.prod(l.params["W"].shape)))
                want = np.sqrt(2.0 / (fi + fo))
                if w.size >= 4096:
                    assert abs(w.std() / want - 1.0) < 0.05 and abs(w.mean()) < 0.05 * want, (s["name"], w.std(), want)
                assert not np.array_equal(w, other.get_param(s["name"], "W", w.size))          # the seed matters
                if s.get("has_bias", True):
                    assert np.all(net.get_param(s["name"], "b", s["n_out"]) == 0)
            elif s["type"] == "batchnorm":
                c = l.params["gamma"].size
                assert np.all(net.get_param(s["name"], "gamma", c) == 1) and np.all(net.get_param(s["name"], "beta", c) == 0)
                assert np.all(net.get_param(s["name"], "mean", c) == 0) and np.all(net.get_param(s["name"], "var", c) == 1)
        again = b.Net(ctx, specs, shape, max_batch=2, precision=b.FP32, seed=666)
        assert np.array_equal(again.params(), net.params())                                    # .seed(666): reproducible
        for n_ in (net, other, again):
            n_.close()


def test_single_process_parameter_averaging_matches_oracle(b200):
    """parallel.fit_parameter_averaging == SparkComputationGraph.fit with a ParameterAveragingTrainingMaster (J:325-333, J:426): two workers,
    one minibatch each, parameters AND updater state averaged -- against the oracle's parameter_average of two fitted copies (FP32 mode)."""
    import copy
    b, ctx = b200
    from gan_deeplearning4j_b200 import parallel
    specs = m.reference_discriminator(0.002)
    rng = np.random.default_rng(17)
    onet = o.net_from_specs(specs, (1, 28, 28), grad_clip=1.0); randomize(onet, rng)
    bnet = b.Net(ctx, specs, (1, 28, 28), max_batch=8, precision=b.FP32, grad_clip=1.0)
    push_params(onet, bnet)
    d = [(rng.uniform(0, 1, (8, 1, 28, 28)), 1 + 0.05 * rng.standard_normal((8, 1))), (rng.uniform(0, 1, (8, 1, 28, 28)), 0.05 * rng.standard_normal((8, 1)))]
    w0, w1 = copy.deepcopy(onet), copy.deepcopy(onet)
    w0.fit(*d[0]); w1.fit(*d[1])
    o.parameter_average([w0, w1], onet)
    parallel.fit_parameter_averaging(bnet, d, averaging_frequency=10)
    # RmsProp(lr, 1e-8, 1e-8) behaves like lr*sign(g): elements whose gradient is numerically zero may land one lr apart (see DESIGN.md 1)
    diff = np.abs(bnet.params() - onet.params_flat())
    assert diff.max() <= 2 * 0.002 + 1e-6 and (diff > 1e-5).mean() < 0.02, (diff.max(), (diff > 1e-5).mean())
    assert bnet.iteration() == 1
    bnet.close()


# ------------------------------------------------------------------------------------------------
# The bf16 weight operands a BF16 net's forward reads instead of the fp32 master: the straight copy of every GEMM weight, and the packed
# [(py,px,c)][(dyr,dxc)][O] operand of the pixel-shuffle transposed conv onto <= 4 channels.  After an update the updater kernel writes both
# itself (vector or scalar branch, through its own inverse of the packing map); setParam / setParams / parameter averaging rewrite them
# from the master.  Either way they must equal the master rounded to nearest even, bit for bit.
# ------------------------------------------------------------------------------------------------
def test_bf16_gan_weight_operands_track_the_master(b200):
    """DCGAN 32x32, nf = 64: G-last (64 -> 3) and D-first's input gradient run the pixel-shuffle tensor-core conv.  Three Gan.steps and a resident step replayed from the CUDA
    graph; after each, every GEMM layer's bf16 operands of both nets equal the rounded fp32 master."""
    b, ctx = b200
    size, z, nf, n = 32, 16, 64, 8
    gs, ds = _dcgan(size, z, nf)
    _, _, bG, bD, data = fp32_gan_pair(b, ctx, gs, ds, n, size, z, precision=b.BF16)
    assert check_weight_operands(b, bG, gs, "G after set_params") == 1 and check_weight_operands(b, bD, ds, "D after set_params") == 1
    gan = b.Gan(bG, bD, use_cuda_graph=True)
    g0 = bG.params()
    for it in range(3):
        gan.step(*data)
        assert check_weight_operands(b, bG, gs, f"G after step {it + 1}") == 1
        check_weight_operands(b, bD, ds, f"D after step {it + 1}")
    data2 = [a.astype(np.float32) for a in o.synthetic_batch(n, size, 3, z, seed=4)]
    gan.upload(*data2); gan.step_resident(n); ctx.sync()
    check_weight_operands(b, bG, gs, "G after a resident step"); check_weight_operands(b, bD, ds, "D after a resident step")
    assert np.abs(bG.params() - g0).max() > 0
    gan.close(); bG.close(); bD.close()


def _ps_fit_specs(updater, ps_bias):
    """A (64, 8, 8) map -> pixel-shuffle transposed conv to 3 channels -> conv -> whole-map conv -> logit.  With a bias the transposed conv's
    W segment starts at flat offset 3 ([b | W]): the updater writes it from its scalar branch; without, from its 16-byte branch."""
    return [{"type": "deconv2d", "name": "ps", "n_in": 64, "n_out": 3, "kernel": (4, 4), "stride": (2, 2), "padding": (1, 1), "has_bias": ps_bias,
             "activation": "tanh", "updater": updater, "l2": 1e-3},
            {"type": "conv2d", "name": "c1", "n_in": 3, "n_out": 64, "kernel": (4, 4), "stride": (2, 2), "padding": (1, 1), "activation": "lrelu", "alpha": 0.2,
             "updater": updater, "l2": 1e-3},
            {"type": "conv2d", "name": "c2", "n_in": 64, "n_out": 1, "kernel": (8, 8), "updater": updater, "l2": 1e-3},
            {"type": "loss", "name": "loss"}]


@pytest.mark.parametrize("ps_bias", [True, False], ids=["ps-W-at-offset-3", "ps-W-aligned"])
@pytest.mark.parametrize("upd", ["sgd", "rmsprop", "adam"])
def test_bf16_fit_weight_operands_track_the_master(b200, upd, ps_bias):
    b, ctx = b200
    u = {"sgd": m.sgd(0.05), "rmsprop": m.rmsprop(1e-3, 0.9, 1e-6), "adam": m.adam(1e-3)}[upd]
    specs = _ps_fit_specs(u, ps_bias)
    off = 0
    for li, name, p, shape, _ in o.net_from_specs(specs, (64, 8, 8)).param_table():
        if (name, p) == ("ps", "W"):
            break
        off += int(np.prod(shape))
    assert off == (3 if ps_bias else 0)
    net = b.Net(ctx, specs, (64, 8, 8), max_batch=6, precision=b.BF16, grad_clip=0.5)
    rng = np.random.default_rng(8)
    for it in range(3):
        net.fit(rng.standard_normal((6, 64, 8, 8)).astype(np.float32), rng.uniform(0, 1, (6, 1)).astype(np.float32))
        assert check_weight_operands(b, net, specs, f"{upd} fit {it + 1}") == 2
    net.close()


def test_bf16_weight_operands_after_set_params_set_param_restore_and_averaging(b200, tmp_path):
    """The host-side rewrites of the master: setParams (all layers), setParam of the packed layer alone (net_refresh_shadow's only_layer),
    restore from a checkpoint, and single-process parameter averaging."""
    b, ctx = b200
    from gan_deeplearning4j_b200 import parallel
    specs = _ps_fit_specs(m.adam(1e-3), True)
    net = b.Net(ctx, specs, (64, 8, 8), max_batch=6, precision=b.BF16)
    rng = np.random.default_rng(9)
    net.set_params((0.05 * rng.standard_normal(net.num_params())).astype(np.float32))
    check_weight_operands(b, net, specs, "set_params")
    net.set_param("ps", "W", (0.1 * rng.standard_normal(64 * 3 * 16)).astype(np.float32))
    check_weight_operands(b, net, specs, "set_param(ps, W)")
    path = str(tmp_path / "ps.zip"); net.save(path)
    other = b.Net(ctx, specs, (64, 8, 8), max_batch=6, precision=b.BF16, seed=5)
    other.restore(path)
    assert np.array_equal(other.params(), net.params())
    check_weight_operands(b, other, specs, "restore")
    d = [(rng.standard_normal((6, 64, 8, 8)).astype(np.float32), rng.uniform(0, 1, (6, 1)).astype(np.float32)) for _ in range(2)]
    parallel.fit_parameter_averaging(net, d, averaging_frequency=1)
    check_weight_operands(b, net, specs, "parameter averaging")
    net.close(); other.close()
