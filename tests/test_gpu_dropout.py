"""DropoutLayer on the GPU: the dropout kernels against the oracle's mask element for element, FP32 nets against the oracle under identical
masks, BF16 nets against the same nets without dropout, the identity cases, the device pass counter (eager, CUDA graph, checkpoint) and
two ranks."""
import numpy as np
import pytest

from gan_deeplearning4j_b200 import models as m
from helpers import b200, bf16_round, fp32_gan_pair, push_params, randomize, rel_err, run_two_ranks
from oracle import dl4j_oracle as o

pytestmark = pytest.mark.gpu
TOL = 1e-3


@pytest.mark.parametrize("p", [0.5, 0.9, 1.0])
@pytest.mark.parametrize("n", [1, 7, 8, 4097, (1 << 20) + 3])
@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_dropout_kernels_match_the_oracle_mask_exactly(b200, prec, n, p):
    b, ctx = b200
    P = b.BF16 if prec == "bf16" else b.FP32
    rng = np.random.default_rng(n)
    x = (rng.uniform(0.5, 2.0, n) * rng.choice([-1.0, 1.0], n)).astype(np.float32).reshape(1, 1, 1, n)      # no zeros: y == 0 <=> dropped
    dy = (rng.uniform(0.5, 2.0, n) * rng.choice([-1.0, 1.0], n)).astype(np.float32).reshape(1, 1, 1, n)
    seed, layer, rank, pass_ = 1234567890123, 5, 3, (1 << 32) + 17
    y, dx = b.test_dropout(ctx, P, x, dy, p, seed=seed, layer=layer, rank=rank, pass_=pass_)
    keep = o.dropout_mask(seed, rank, layer, pass_, 1, 1, 1, n, p).ravel()
    assert np.array_equal(y.ravel() != 0, keep) and np.array_equal(dx.ravel() != 0, keep)
    s = np.float32(1) / np.float32(p)
    rnd = bf16_round if prec == "bf16" else (lambda a: np.asarray(a, np.float32))
    xs, es = rnd(x).ravel(), rnd(dy).ravel()
    assert np.array_equal(y.ravel(), np.where(keep, rnd(xs * s), 0).astype(np.float32))
    assert np.array_equal(dx.ravel(), np.where(keep, rnd(es * s), 0).astype(np.float32))
    if n > 4096:
        assert abs(keep.mean() - p) < 5 * np.sqrt(p * (1 - p) / n) + 1e-12


def test_dropout_rejects_bad_arguments(b200):
    b, ctx = b200
    x = np.ones((1, 1, 1, 8), np.float32)
    for p in (0.0, -0.5, 1.5, float("nan")):
        with pytest.raises(b.B200GanError) as e:
            b.test_dropout(ctx, b.FP32, x, x, p)
        assert e.value.code == -1
        with pytest.raises(b.B200GanError) as e:
            b.Net(ctx, [{"type": "dense", "n_out": 4}, {"type": "dropout", "p": p}, {"type": "output", "n_out": 1}], (4,), max_batch=2)
        assert e.value.code == -1
    with pytest.raises(b.B200GanError) as e:        # 2^34 + elements in one pass: the counter's element index would wrap
        b.Net(ctx, [{"type": "dense", "n_out": 1 << 20}, {"type": "dropout", "p": 0.5}, {"type": "output", "n_out": 1}], (1,), max_batch=(1 << 14) + 1)
    assert e.value.code == -6


def _chain_specs(p=0.7, frozen=False, with_dropout=True):
    u = m.adam(1e-2)
    drop = lambda name: [{"type": "dropout", "name": name, "p": p, "frozen": frozen}] if with_dropout else []
    return ([{"type": "conv2d", "name": "c1", "n_out": 8, "kernel": (3, 3), "stride": (2, 2), "padding": (1, 1), "updater": u},
             {"type": "activation", "name": "a1", "activation": "lrelu", "alpha": 0.2}] + drop("drop1") +
            [{"type": "conv2d", "name": "c2", "n_out": 12, "kernel": (3, 3), "stride": (1, 1), "padding": (1, 1), "has_bias": False, "updater": u},
             {"type": "batchnorm", "name": "bn2", "updater": u}, {"type": "activation", "name": "a2", "activation": "tanh"}] + drop("drop2") +
            [{"type": "cnn_to_ff", "name": "flat"},
             {"type": "dense", "name": "fc", "n_out": 10, "activation": "tanh", "updater": u},
             {"type": "output", "name": "out", "n_out": 1, "updater": u}])


def test_fp32_chain_matches_oracle_under_identical_masks(b200):
    """conv -> act -> dropout -> conv -> BN -> act -> dropout -> dense -> output: activations, zero patterns, score and gradients."""
    b, ctx = b200
    specs = _chain_specs()
    rng = np.random.default_rng(3)
    onet = o.net_from_specs(specs, (3, 8, 8), mask_seed=41, seed=2); randomize(onet, rng)
    bnet = b.Net(ctx, specs, (3, 8, 8), max_batch=6, precision=b.FP32, seed=41)
    push_params(onet, bnet)
    x = rng.uniform(-1, 1, (6, 3, 8, 8)); y = rng.uniform(0, 1, (6, 1))
    for step in range(2):              # pass 0, then pass 1: the counter moves the masks
        score_o, acts, _, _ = onet.compute_gradient_and_score(x, y, collect=True)
        score_b = bnet.compute_gradient_and_score(x, y)
        assert bnet.dropout_pass() == onet.dropout.pass_ == step + 1
        assert abs(score_b - score_o) < TOL * abs(score_o)
        for li, s in enumerate(specs):
            if s["type"] == "output" or (s["type"] == "batchnorm" and specs[li + 1]["type"] == "activation"):
                continue
            got, want = bnet.activation(li, 6), acts[li + 1].reshape(6, -1)
            assert rel_err(got, want) < TOL, (step, li, s["name"])
            if s["type"] == "dropout":
                assert np.array_equal(got == 0, want == 0), (step, s["name"])
                assert 0 < (got == 0).mean() < 1
        g_b, g_o = bnet.gradients(), onet.grads_flat(); off = 0
        for li, name, pn, shape, _ in onet.param_table():
            k = int(np.prod(shape))
            assert rel_err(g_b[off:off + k], g_o[off:off + k]) < TOL, (step, name, pn)
            off += k
    bnet.close()


def test_inference_and_frozen_dropout_are_the_identity(b200):
    b, ctx = b200
    rng = np.random.default_rng(4)
    plain, drop, frozen = _chain_specs(with_dropout=False), _chain_specs(), _chain_specs(frozen=True)
    onet = o.net_from_specs(plain, (3, 8, 8), seed=2); randomize(onet, rng)
    x = rng.uniform(-1, 1, (6, 3, 8, 8)); y = rng.uniform(0, 1, (6, 1))
    nets = [b.Net(ctx, s, (3, 8, 8), max_batch=6, precision=b.FP32) for s in (plain, drop, frozen)]
    for n in nets:
        push_params(onet, n)
    outs, launches = [], []
    for n in nets:
        l0 = ctx.launch_count(); outs.append(n.output(x)); launches.append(ctx.launch_count() - l0)
    assert np.array_equal(outs[0], outs[1]) and np.array_equal(outs[0], outs[2])
    assert launches[0] == launches[1] == launches[2]
    assert nets[1].dropout_pass() == 0
    assert np.array_equal(nets[1].activation(2, 6), nets[1].activation(1, 6))      # a pass-through layer reports its input
    # a frozen DropoutLayer runs in test mode: the train step equals the net without it, bit for bit, and counts no pass
    s0 = nets[0].compute_gradient_and_score(x, y); s2 = nets[2].compute_gradient_and_score(x, y)
    assert s0 == s2 and np.array_equal(nets[0].gradients(), nets[2].gradients())
    assert nets[2].dropout_pass() == 0
    for n in nets:
        n.close()


def test_pass_counter_and_checkpoint_resume(b200, tmp_path):
    b, ctx = b200
    specs = _chain_specs()
    rng = np.random.default_rng(5)
    x = rng.uniform(-1, 1, (6, 3, 8, 8)).astype(np.float32); y = rng.uniform(0, 1, (6, 1)).astype(np.float32)
    a = b.Net(ctx, specs, (3, 8, 8), max_batch=6, precision=b.FP32, seed=8)
    assert a.dropout_pass() == 0
    a.compute_gradient_and_score(x, y); assert a.dropout_pass() == 1
    a.output(x); assert a.dropout_pass() == 1
    a.output(x, train=True); assert a.dropout_pass() == 2
    a.set_dropout_pass(123456789012); assert a.dropout_pass() == 123456789012
    a.set_dropout_pass(0)
    for prec in (b.FP32, b.BF16):
        u = b.Net(ctx, specs, (3, 8, 8), max_batch=6, precision=prec, seed=8)
        c = b.Net(ctx, specs, (3, 8, 8), max_batch=6, precision=prec, seed=8)
        c.set_params(u.params())
        for _ in range(5):
            u.fit(x, y)
        for _ in range(3):
            c.fit(x, y)
        path = str(tmp_path / f"ck{prec}.zip"); c.save(path)
        r = b.Net(ctx, specs, (3, 8, 8), max_batch=6, precision=prec, seed=8)
        meta = r.restore(path)
        assert meta["meta"]["dropout_pass"] == 3 and r.dropout_pass() == 3
        for _ in range(2):
            r.fit(x, y)
        assert np.array_equal(r.params(), u.params()) and r.dropout_pass() == u.dropout_pass() == 5
        for n in (u, c, r):
            n.close()
    a.close()


def _dcgan_d_with_dropout(size, nf, lr, p):
    out = []
    for s in m.dcgan_discriminator(size, nf, 3, lr=lr):
        out.append(s)
        if s.get("activation") == "lrelu":
            out.append({"type": "dropout", "name": s["name"] + "_drop", "p": p})
    return out


def _bf16_grad_err(b, ctx, specs, in_shape, n, seed, rng_seed):
    rng = np.random.default_rng(rng_seed)
    onet = o.net_from_specs(specs, in_shape, mask_seed=seed, quirks=o.Quirks(xent_clip_eps=0.0), seed=2); randomize(onet, rng)
    bnet = b.Net(ctx, specs, in_shape, max_batch=n, precision=b.BF16, xent_clip_eps=0.0, seed=seed)
    push_params(onet, bnet)
    x = rng.uniform(-1, 1, (n,) + tuple(in_shape)); y = rng.uniform(0, 1, (n, 1))
    onet.compute_gradient_and_score(x, y); bnet.compute_gradient_and_score(x, y)
    g_b, g_o = bnet.gradients(), onet.grads_flat()
    bnet.close()
    return float(np.linalg.norm(g_b - g_o) / np.linalg.norm(g_o))


def test_bf16_nets_with_dropout_track_the_oracle(b200):
    """BF16 MLP D (tensor-core sizes) and 32x32 DCGAN D with dropout after each LeakyReLU: the gradient error against the oracle under
    identical masks stays within 2x that of the same nets without dropout.  The DCGAN D puts DropoutLayers between the fused BatchNorm
    epilogues and the next GEMM (the BatchNorm backward then runs the accumulator kernels on its own)."""
    b, ctx = b200
    cases = [("mlp", m.mlp_discriminator(128, 256, lr=1e-3), m.mlp_discriminator(128, 256, lr=1e-3, dropout=0.5), (128,), 256),
             ("dcgan32", m.dcgan_discriminator(32, 64, 3, lr=1e-3), _dcgan_d_with_dropout(32, 64, 1e-3, 0.5), (3, 32, 32), 8)]
    for name, plain, drop, shape, n in cases:
        e0 = _bf16_grad_err(b, ctx, plain, shape, n, 77, 6)
        e1 = _bf16_grad_err(b, ctx, drop, shape, n, 77, 6)
        print(f"{name}: gradient error without dropout {e0:.3e}, with dropout {e1:.3e}")
        assert e1 <= 2 * e0, (name, e0, e1)


def test_fp32_gan_step_with_dropout_graph_eager_and_oracle(b200):
    b, ctx = b200
    n = 8
    gs, ds = m.dcgan_generator(16, 12, 8, 3, lr=2e-3), _dcgan_d_with_dropout(16, 8, 2e-3, 0.7)
    runs = []
    for graph in (False, True):
        G, D, bG, bD, data = fp32_gan_pair(b, ctx, gs, ds, n, mask_seed=667, d_kw=dict(seed=667))
        gan = b.Gan(bG, bD, use_cuda_graph=graph)
        drop = [i for i, s in enumerate(ds) if s["type"] == "dropout"]
        masks, losses = [], []
        for it in range(3):
            r = o.gan_step(G, D, *data)
            lo = gan.step(*data); losses.append(lo)
            want = np.array([r["loss_d_real"], r["loss_d_fake"], r["loss_g"]])
            assert np.all(np.abs(lo - want) < TOL * np.maximum(1, np.abs(want))), (graph, it, lo, want)
            for onet, bnet, tag in ((D, bD, "D"), (G, bG, "G")):
                p_b, p_o = bnet.params(), onet.params_flat(); off = 0
                for li, name, pn, shape, _ in onet.param_table():
                    k = int(np.prod(shape))
                    assert rel_err(p_b[off:off + k], p_o[off:off + k]) < 2 * TOL, (graph, it, tag, name, pn)
                    off += k
            assert bD.dropout_pass() == D.dropout.pass_ == 2 * (it + 1)
            # the last D pass of the step is the generator step's (N rows, pass 2*it + 1): its zero pattern is that mask, drawn on the device
            step_masks = []
            for li in drop:
                got = bD.activation(li, n)
                want = D.layers[li + 1]._m != 0                     # +1: the oracle's prepended input reshape
                assert np.array_equal(got.reshape(want.shape) != 0, want), (graph, it, li)
                step_masks.append(got != 0)
            masks.append(step_masks)
        assert not all(np.array_equal(a, c) for a, c in zip(masks[0], masks[1]))    # step 2 drew new masks: P was not frozen into the graph
        runs.append((np.array(losses), bG.params(), bD.params()))
        gan.close(); bG.close(); bD.close()
    assert np.array_equal(runs[0][0], runs[1][0]) and np.array_equal(runs[0][1], runs[1][1]) and np.array_equal(runs[0][2], runs[1][2])


def test_two_ranks_share_parameters_but_not_masks(tmp_path):
    d = run_two_ranks("dp_check.py", tmp_path / "dropout_dp.json", 29547, args=("dropout",))
    assert d["world"] == 2 and d["d_params_identical"] is True and d["dropout_activations_differ"] is True and d["masks_match_oracle"] is True
