"""Per-output loss weights and labels masks on the GPU (semantics at b2g_loss in include/b200gan.h): FP32 nets against the oracle
over 3 fits with a ragged batch -- a weighted MCXENT classifier, a U-Net with weighted MCXENT and a per-pixel mask, a PatchGAN
discriminator with a mask, every loss code on OutputLayer / LossLayer / CnnLossLayer with per-example and per-output masks; all-ones weights and
mask give the unweighted bits; the masked PatchGAN step against the restatement, BF16 graph replay against eager, new mask contents without
re-capture, the unmasked step's launch count; and the refusals."""
import copy

import numpy as np
import pytest

from gan_deeplearning4j_b200 import models as m
from helpers import b200, launches_per_step, oracle_gan_pair, pclose, push_params, randomize, rel_err
from oracle import dl4j_oracle as o

pytestmark = pytest.mark.gpu
TOL = 1e-3


def _labels(loss, rng, shape):
    if loss == "mcxent":
        k = rng.integers(0, shape[1], (shape[0],) + tuple(shape[2:]))
        return np.ascontiguousarray(np.moveaxis(np.eye(shape[1])[k], -1, 1))
    if loss == "xent":
        return rng.uniform(0, 1, shape)
    if loss in ("hinge", "squared_hinge"):
        return rng.choice([-1.0, 1.0], shape)
    return rng.uniform(-1, 1, shape)


def _fits(b, onet, bnet, shape, loss, rng, mask_of, batches=(6, 5, 6), what="", lr=None):
    """3 fits (the middle one ragged): score, gradients (computeGradientAndScore) and parameters against the restatement (with lr: by pclose
    at 2 lr, for Adam nets, whose near-zero gradients move a parameter by up to lr on last-bit differences)."""
    for it, mb in enumerate(batches):
        x = rng.uniform(-1.5, 1.5, (mb,) + shape)
        out_shape = (mb,) + tuple(onet.output(x[:1]).shape[1:])
        y = _labels(loss, rng, out_shape)
        mk = mask_of(rng, out_shape)
        s_o = onet.compute_gradient_and_score(x, y, mask=mk)
        s_b = bnet.compute_gradient_and_score(x, y, mask=mk)
        assert abs(s_b - s_o) <= TOL * max(1.0, abs(s_o)), (what, it, s_b, s_o)
        assert rel_err(bnet.gradients(), onet.grads_flat()) <= TOL, (what, it, "gradients")
        s_o = onet.fit(x, y, mask=mk); s_b = bnet.fit(x, y, mask=mk)
        assert abs(s_b - s_o) <= TOL * max(1.0, abs(s_o)), (what, it, s_b, s_o)
        if lr is None:
            assert rel_err(bnet.params(), onet.params_flat()) <= TOL, (what, it, "params")
        else:
            assert pclose(bnet.params(), onet.params_flat(), 2 * lr), (what, it, "params", rel_err(bnet.params(), onet.params_flat()))


def test_weighted_mcxent_classifier(b200):
    """dense -> OutputLayer(MCXENT) with class weights and a per-example mask (0/1 and fractional)."""
    b, ctx = b200
    specs = [{"type": "dense", "name": "d", "n_out": 16, "activation": "tanh", "updater": m.adam(0.01)},
             {"type": "output", "name": "out", "n_out": 5, "loss": "mcxent", "updater": m.adam(0.01), "loss_weights": [0.5, 1.0, 2.0, 0.25, 1.5]}]
    rng = np.random.default_rng(1)
    onet = o.net_from_specs(specs, (12,), seed=2); randomize(onet, rng)
    bnet = b.Net(ctx, specs, (12,), max_batch=6, precision=b.FP32)
    push_params(onet, bnet)
    mask = lambda r, s: np.where(r.uniform(0, 1, (s[0], 1)) < 0.3, 0.0, r.uniform(0.2, 1.0, (s[0], 1)))
    _fits(b, onet, bnet, (12,), "mcxent", rng, mask, what="classifier", lr=0.01)
    bnet.close()


def test_unet_weighted_mcxent_per_pixel_mask(b200):
    b, ctx = b200
    specs = m.unet(size=16, nc=3, n_classes=3, nf=8, depth=2, lr=0.01)
    for sp in specs:              # SGD: Adam turns last-bit gradient differences on near-zero gradients into lr-sized steps
        if "updater" in sp:
            sp["updater"] = m.sgd(0.01)
    specs[-1]["loss_weights"] = [0.2, 1.0, 3.0]
    rng = np.random.default_rng(2)
    onet = o.net_from_specs(specs, (3, 16, 16), seed=2, flat_input=False); randomize(onet, rng)
    bnet = b.Net(ctx, specs, (3, 16, 16), max_batch=6, precision=b.FP32)
    push_params(onet, bnet)
    mask = lambda r, s: (r.uniform(0, 1, (s[0], 1) + s[2:]) > 0.25).astype(np.float64)      # "void" pixels
    _fits(b, onet, bnet, (3, 16, 16), "mcxent", rng, mask, what="unet")
    bnet.close()


def _small_specs(kind, loss, act, c):
    conv = {"type": "conv2d", "name": "c1", "n_out": 8, "kernel": (3, 3), "stride": (1, 1), "padding": (1, 1), "activation": "tanh",
            "updater": m.sgd(0.05)}
    if kind == "cnn_loss":
        head = {"type": "conv2d", "name": "c2", "n_out": c, "kernel": (1, 1), "stride": (1, 1), "padding": (0, 0), "activation": "identity",
                "updater": m.sgd(0.05)}
        return [conv, head, m.cnn_loss(loss, act if loss not in ("xent", "mcxent") else "identity", name="cl")], (3, 5, 7)
    if kind == "output":
        out = {"type": "output", "name": "out", "n_out": c, "loss": loss, "updater": m.sgd(0.05)}
        if loss not in ("xent", "mcxent"):
            out["activation"] = act
        return [{"type": "dense", "name": "d", "n_out": 8, "activation": "tanh", "updater": m.sgd(0.05)}, out], (6,)
    ll = {"type": "loss", "name": "ll", "loss": loss}
    if loss != "xent":
        ll["activation"] = act
    return [{"type": "dense", "name": "d", "n_out": c, "activation": "identity", "updater": m.sgd(0.05)}, ll], (6,)


CASES = [(k, l, a) for k in ("output", "loss", "cnn_loss") for l, a in
         (("xent", "identity"), ("mcxent", "identity"), ("mse", "tanh"), ("l1", "identity"), ("l2", "sigmoid"), ("mae", "softplus"),
          ("hinge", "identity"), ("squared_hinge", "tanh"), ("wasserstein", "identity"))
         if not (k == "loss" and l == "mcxent")]


@pytest.mark.parametrize("kind,loss,act", CASES)
def test_every_loss_weighted_and_masked(b200, kind, loss, act):
    """Weights (where the loss takes them) and a per-row, then a per-output mask (not MCXENT): a CnnLossLayer's NCHW per-output mask goes
    through the labels' NHWC conversion."""
    b, ctx = b200
    c = 1 if loss == "xent" and kind != "cnn_loss" else 3
    specs, shape = _small_specs(kind, loss, act, c)
    if loss not in o.DEFAULT_QUIRKS.weightless_losses:
        specs[-1]["loss_weights"] = [0.5, 2.0, 1.25][:c]
    rng = np.random.default_rng(len(kind) * 10 + len(loss))
    for per_output in ((False, True) if loss != "mcxent" else (False,)):
        onet = o.net_from_specs(specs, shape, seed=2, flat_input=False); randomize(onet, rng)
        bnet = b.Net(ctx, specs, shape, max_batch=6, precision=b.FP32)
        push_params(onet, bnet)
        mask = lambda r, s: r.uniform(0, 1, s if per_output else (s[0], 1) + tuple(s[2:]))
        _fits(b, onet, bnet, shape, loss, rng, mask, what=(kind, loss, per_output))
        bnet.close()


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("loss", ["xent", "mcxent", "mse"])
def test_all_ones_give_the_unweighted_bits(b200, loss, prec):
    """All-ones weights and an all-ones mask, one-hot labels for MCXENT: the weighted / masked instantiations give the unweighted kernels'
    scores and parameters bit for bit, on a CnnLossLayer and an OutputLayer."""
    b, ctx = b200
    P = b.FP32 if prec == "fp32" else b.BF16
    for kind in ("cnn_loss", "output"):
        c = 1 if loss == "xent" and kind == "output" else 3
        specs, shape = _small_specs(kind, loss, "tanh", c)
        rng = np.random.default_rng(4)
        onet = o.net_from_specs(specs, shape, seed=2, flat_input=False); randomize(onet, rng)
        runs = []
        for weighted in (False, True):
            bnet = b.Net(ctx, specs, shape, max_batch=6, precision=P)
            push_params(onet, bnet)
            if weighted:
                bnet.set_loss_weights(np.ones(c))
            r = np.random.default_rng(5)
            scores = []
            for mb in (6, 5):
                x = r.uniform(-1, 1, (mb,) + shape)
                y = _labels(loss, r, (mb,) + tuple(onet.output(x[:1]).shape[1:]))
                mk = np.ones((mb, 1) + tuple(y.shape[2:])) if weighted else None
                scores.append(bnet.fit(x, y, mask=mk))
            runs.append((np.array(scores), bnet.params()))
            bnet.close()
        assert np.array_equal(runs[0][0], runs[1][0]), (kind, loss, prec, "scores")
        assert np.array_equal(runs[0][1], runs[1][1]), (kind, loss, prec, "params")


def _patch_gan(size=16, z=12, lr_=2e-3):
    gs, ds = m.dcgan_generator(size, z, 8, 3, lr=lr_), m.dcgan_discriminator(size, 8, 3, lr=lr_, patch=True)
    return gs, ds


def test_patch_discriminator_fit_with_mask(b200):
    """The PatchGAN discriminator on its own: fit with a per-patch mask."""
    b, ctx = b200
    _, ds = _patch_gan()
    rng = np.random.default_rng(6)
    onet = o.net_from_specs(ds, (3, 16, 16), seed=2); randomize(onet, rng)
    bnet = b.Net(ctx, ds, (3, 16, 16), max_batch=6, precision=b.FP32)
    push_params(onet, bnet)
    mask = lambda r, s: (r.uniform(0, 1, s) > 0.4).astype(np.float64)
    _fits(b, onet, bnet, (3, 16, 16), "xent", rng, mask, what="patch D")
    bnet.close()


def test_fp32_masked_patch_gan_step_matches_restatement(b200):
    """3 masked steps: losses and both nets' parameters against the oracle's gan_step, graph replay and eager, the two bit for bit."""
    b, ctx = b200
    size, z, n, lr_ = 16, 12, 8, 2e-3
    gs, ds = _patch_gan(size, z, lr_)
    G, D = oracle_gan_pair(gs, ds, size, z)
    data = [a.astype(np.float64) for a in o.synthetic_batch(n, size, 3, z, seed=3)]
    maps = [np.broadcast_to(v.reshape(n, 1, 1, 1), (n, 1, 4, 4)).copy() for v in data[3:]]
    rng = np.random.default_rng(7)
    masks = [(rng.uniform(0, 1, (n, 1, 4, 4)) > 0.3) * rng.uniform(0.5, 1.0, (n, 1, 4, 4)) for _ in range(3)]
    results = {}
    for graph in (True, False):
        Gc, Dc = copy.deepcopy(G), copy.deepcopy(D)
        bG = b.Net(ctx, gs, (z,), max_batch=n, precision=b.FP32)
        bD = b.Net(ctx, ds, (3, size, size), max_batch=2 * n, precision=b.FP32, bn_groups=2)
        push_params(Gc, bG); push_params(Dc, bD)
        gan = b.Gan(bG, bD, use_cuda_graph=graph)
        gan.set_label_masks(*masks)
        ls = []
        for it in range(3):
            r = o.gan_step(Gc, Dc, *data[:3], *maps, m_real=masks[0], m_fake=masks[1], m_gen=masks[2])
            lo = gan.step(*data)
            ls.append(lo)
            want = np.array([r["loss_d_real"], r["loss_d_fake"], r["loss_g"]])
            assert np.all(np.abs(lo - want) < TOL * np.maximum(1, np.abs(want))), (graph, it, lo, want)
            assert pclose(bD.params(), Dc.params_flat(), 2 * lr_), (graph, it, "D")
            assert pclose(bG.params(), Gc.params_flat(), 2 * lr_), (graph, it, "G")
        results[graph] = (np.array(ls), bG.params(), bD.params())
        gan.close(); bG.close(); bD.close()
    for u, v in zip(results[True], results[False]):
        assert np.array_equal(u, v), "graph replay == eager"


def test_bf16_masked_step_replay_new_contents_and_launches(b200):
    """BF16 PatchGAN step: graph replay equals eager bit for bit with masks, new mask contents reach the replayed graph without a re-capture
    (the replay after set_label_masks equals an eager run with the same masks), and a masked step launches what the unmasked one does."""
    b, ctx = b200
    size, z, n = 16, 12, 8
    gs, ds = _patch_gan(size, z)
    G, D = oracle_gan_pair(gs, ds, size, z)
    data = [a.astype(np.float32) for a in o.synthetic_batch(n, size, 3, z, seed=3)]
    rng = np.random.default_rng(8)
    m1 = [rng.uniform(0, 1, (n, 1, 4, 4)) for _ in range(3)]
    m2 = [(rng.uniform(0, 1, (n, 1, 4, 4)) > 0.5).astype(np.float64) for _ in range(3)]
    outs, launches = {}, {}
    for graph in (True, False):
        bG = b.Net(ctx, gs, (z,), max_batch=n, precision=b.BF16)
        bD = b.Net(ctx, ds, (3, size, size), max_batch=2 * n, precision=b.BF16, bn_groups=2)
        push_params(G, bG); push_params(D, bD)
        gan = b.Gan(bG, bD, use_cuda_graph=graph)
        seq = []
        gan.set_label_masks(*m1)
        seq.append(gan.step(*data)); seq.append(gan.step(*data))
        gan.set_label_masks(*m2)              # same width: the captured graph is replayed with the new contents
        seq.append(gan.step(*data))
        outs[graph] = (np.array(seq), bG.params(), bD.params())
        if graph:
            gan.upload(*data)
            launches["masked"] = launches_per_step(ctx, gan, n)
            gan.set_label_masks(None, None, None)
            launches["unmasked"] = launches_per_step(ctx, gan, n)
        gan.close(); bG.close(); bD.close()
    for u, v in zip(outs[True], outs[False]):
        assert np.array_equal(u, v), "graph replay == eager"
    assert launches["masked"] == launches["unmasked"], launches


def test_refusals(b200):
    b, ctx = b200
    specs, shape = _small_specs("output", "hinge", "identity", 3)
    net = b.Net(ctx, specs, shape, max_batch=4, precision=b.FP32)
    with pytest.raises(b.B200GanError):
        net.set_loss_weights([1.0, 1.0, 1.0])                     # hinge has no weights
    net.close()
    specs, shape = _small_specs("output", "mse", "identity", 3)
    net = b.Net(ctx, specs, shape, max_batch=4, precision=b.FP32)
    for bad in ([1.0, 1.0], [1.0, np.nan, 1.0], [1.0, np.inf, 1.0]):
        with pytest.raises(b.B200GanError):
            net.set_loss_weights(bad)
    with pytest.raises(b.B200GanError):
        net.set_loss_weights([1.0, 1.0, 1.0], layer="d")          # not the loss layer
    x, y = np.zeros((4, 6)), np.zeros((4, 3))
    with pytest.raises(b.B200GanError):
        net.fit(x, y, mask=np.ones((4, 2)))                        # width neither 1 nor nOut
    net.set_loss_weights([1.0, 2.0, 3.0], layer="out"); net.set_loss_weights(None)
    net.close()
    specs, shape = _small_specs("output", "mcxent", "identity", 3)
    net = b.Net(ctx, specs, shape, max_batch=4, precision=b.FP32)
    with pytest.raises(b.B200GanError):
        net.fit(x, np.eye(3)[[0, 1, 2, 0]], mask=np.ones((4, 3)))  # per-output mask with MCXENT
    net.close()
    net = b.Net(ctx, [{"type": "dense", "name": "d", "n_out": 3, "updater": m.sgd(0.1)}], (6,), max_batch=4, precision=b.FP32)
    with pytest.raises(b.B200GanError):
        net.set_loss_weights([1.0, 1.0, 1.0])                     # no loss layer
    net.close()
    with pytest.raises(ValueError):
        b.Net(ctx, [{"type": "dense", "name": "d", "n_out": 3, "loss_weights": [1, 1, 1]}, {"type": "loss", "name": "l", "loss": "mse"}], (6,),
              max_batch=4, precision=b.FP32)
    gs, ds = _patch_gan()
    G, D = oracle_gan_pair(gs, ds)
    bG = b.Net(ctx, gs, (12,), max_batch=4, precision=b.FP32); bD = b.Net(ctx, ds, (3, 16, 16), max_batch=8, precision=b.FP32, bn_groups=2)
    gan = b.Gan(bG, bD, use_cuda_graph=False)
    ones = np.ones((4, 1, 4, 4))
    with pytest.raises(ValueError):
        gan.set_label_masks(ones, ones, np.ones((4, 2, 4, 4)))    # one shape for all three
    with pytest.raises(b.B200GanError):
        gan.set_label_masks(np.ones((4, 2, 4, 4)), np.ones((4, 2, 4, 4)), np.ones((4, 2, 4, 4)))    # width 2 on one channel
    gan.set_label_masks(ones, ones, ones)
    data = [a.astype(np.float32) for a in o.synthetic_batch(2, 16, 3, 12, seed=3)]
    with pytest.raises(b.B200GanError):
        gan.step(*data)                                           # masks set for batch 4, a step of 2
    gan.close(); bG.close(); bD.close()


def test_checkpoint_carries_loss_weights(b200, tmp_path):
    b, ctx = b200
    specs, shape = _small_specs("output", "mse", "identity", 3)
    net = b.Net(ctx, specs, shape, max_batch=4, precision=b.FP32)
    net.set_loss_weights([0.5, 1.0, 2.0])
    path = tmp_path / "net.zip"
    net.save(path)
    other = b.Net(ctx, specs, shape, max_batch=4, precision=b.FP32)
    other.restore(path)
    assert other.specs[-1]["loss_weights"] == [0.5, 1.0, 2.0]
    rng = np.random.default_rng(0)
    x, y = rng.uniform(-1, 1, (4, 6)), rng.uniform(-1, 1, (4, 3))
    assert net.compute_gradient_and_score(x, y) == other.compute_gradient_and_score(x, y)
    net.close(); other.close()


def test_restore_of_nets_without_a_loss_layer(b200, tmp_path):
    """A generator (ends in a deconvolution) and an MLP generator (ends in a dense layer) save and restore as before: clearing loss weights is
    a no-op on a net without a loss layer."""
    b, ctx = b200
    for specs, shape in ((m.dcgan_generator(16, 12, 8, 3), (12,)), (m.mlp_generator(8, 16, 10), (8,))):
        net = b.Net(ctx, specs, shape, max_batch=4, precision=b.FP32)
        rng = np.random.default_rng(0)
        net.set_params(rng.uniform(-0.1, 0.1, net.num_params()))
        path = tmp_path / "gen.zip"
        net.save(path)
        other = b.Net(ctx, specs, shape, max_batch=4, precision=b.FP32)
        other.restore(path)
        assert np.array_equal(other.params(), net.params())
        net.set_loss_weights(None)                    # a no-op, not an error
        with pytest.raises(b.B200GanError):
            net.set_loss_weights([1.0])               # weights need a loss layer
        net.close(); other.close()


def test_mask_shape_is_checked_before_the_copy(b200):
    """A mask that holds fewer values than its width asks the engine to read is refused in Python."""
    b, ctx = b200
    specs, shape = _small_specs("cnn_loss", "xent", "identity", 3)
    net = b.Net(ctx, specs, shape, max_batch=4, precision=b.FP32)
    x, y = np.zeros((4,) + shape), np.zeros((4, 3, 5, 7))
    for bad in (np.ones((4, 1)), np.ones(4), np.ones((4, 5, 7)), np.ones((4, 1, 5, 6))):
        with pytest.raises(ValueError):
            net.fit(x, y, mask=bad)
    net.fit(x, y, mask=np.ones((4, 1, 5, 7))); net.fit(x, y, mask=np.ones((4, 3, 5, 7)))
    net.close()
