"""DropoutLayer on the CPU: the oracle's NumPy restatement -- Philox4x32-10 against Random123's known answers, the mask's statistics and inputs, the layer's
gradient, the GAN step's pass bookkeeping, and the host-side plumbing (spec -> desc, models, checkpoint metadata).  No GPU needed."""
import copy

import numpy as np
import pytest

from helpers import randomize
from oracle import dl4j_oracle as o


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
], ids=["zeros", "ones", "pi"])
def test_philox_known_answers(ctr, key, want):
    assert tuple(int(v) for v in o.philox4x32_10(ctr, key)) == want


def test_philox_vectorised_equals_scalar():
    g = np.arange(1000, 1010, dtype=np.uint64)
    vec = np.stack(o.philox4x32_10((g, 7, 1, 3 | (2 << 16)), (12345, 0)), -1)
    for i, c in enumerate(range(1000, 1010)):
        assert tuple(int(v) for v in o.philox4x32_10((c, 7, 1, 3 | (2 << 16)), (12345, 0))) == tuple(int(v) for v in vec[i])


@pytest.mark.parametrize("p", [0.1, 0.5, 0.8])
def test_keep_rate_within_5_sigma(p):
    n = 10 ** 6
    keep = o.dropout_mask(666, 0, 3, 11, 1000, 10, 10, 10, p)
    assert keep.size == n
    sigma = np.sqrt(n * p * (1 - p))
    assert abs(int(keep.sum()) - n * p) < 5 * sigma, (keep.sum(), n * p)


def test_mask_depends_on_every_input():
    base = dict(seed=666, rank=0, layer=2, pass_=5, rows=8, h=4, w=4, c=16, p=0.5)
    m0 = o.dropout_mask(**base)
    for k, v in (("seed", 667), ("rank", 1), ("layer", 3), ("pass_", 6), ("pass_", 5 + (1 << 32))):
        assert not np.array_equal(m0, o.dropout_mask(**dict(base, **{k: v}))), k
    assert np.array_equal(o.dropout_mask(**dict(base, seed=0)), o.dropout_mask(**dict(base, seed=666)))      # seed 0 means 666, as for Xavier
    assert o.dropout_mask(**dict(base, p=1.0)).all()


def test_mask_rows_of_a_pass_and_nchw_order():
    """Rows [r0, r0 + k) of a pass are the same slice of the whole pass's mask, and the NCHW result is the NHWC element order transposed."""
    full = o.dropout_mask(1, 0, 4, 9, 6, 3, 5, 7, 0.6)
    assert full.shape == (6, 7, 3, 5)
    assert np.array_equal(o.dropout_mask(1, 0, 4, 9, 2, 3, 5, 7, 0.6, row0=3), full[3:5])
    # element (row 1, c 2, y 1, x 3) is NHWC index ((1*3 + 1)*5 + 3)*7 + 2
    e = ((1 * 3 + 1) * 5 + 3) * 7 + 2
    words = o.philox4x32_10((e >> 2, 9, 0, 4), (1, 0))
    assert bool(full[1, 2, 1, 3]) == (int(words[e & 3]) < int(np.floor(float(np.float32(0.6)) * 2.0 ** 32)))


def test_dropout_layer_forward_backward_and_finite_differences():
    """Inverted dropout with a fixed mask: y = x * m, dx = dy * m; the net's gradient through it matches central differences."""
    rng = np.random.default_rng(0)
    specs = [{"type": "dense", "name": "d1", "n_out": 12, "activation": "tanh"},
             {"type": "dropout", "name": "drop", "p": 0.6},
             {"type": "dense", "name": "d2", "n_out": 5, "activation": "sigmoid"},
             {"type": "output", "name": "out", "n_out": 1}]
    net = o.net_from_specs(specs, (7,), mask_seed=3, seed=3); randomize(net, rng)
    assert net.layers[1].index == 1
    x = rng.uniform(-1, 1, (6, 7)); y = rng.uniform(0, 1, (6, 1))
    score = net.compute_gradient_and_score(x, y, pass_=4)
    keep = o.dropout_mask(3, 0, 1, 4, 6, 1, 1, 12, 0.6).reshape(6, 12)
    h = np.tanh(x @ net.layers[0].params["W"] + net.layers[0].params["b"])
    s = float(np.float32(1) / np.float32(0.6))
    assert np.allclose(h * net.layers[1]._m, h * keep * s)
    assert 0 < keep.sum() < keep.size
    g = net.grads_flat().copy()
    theta = net.params_flat().copy()
    for i in rng.choice(theta.size, 25, replace=False):
        tp, tm = theta.copy(), theta.copy(); tp[i] += 1e-6; tm[i] -= 1e-6
        net.set_params_flat(tp); sp = net.compute_gradient_and_score(x, y, pass_=4)
        net.set_params_flat(tm); sm = net.compute_gradient_and_score(x, y, pass_=4)
        fd = (sp - sm) / 2e-6 * x.shape[0]            # gradients are minibatch sums
        assert abs(fd - g[i]) <= 1e-5 * max(1.0, abs(fd)), (i, fd, g[i])
    net.set_params_flat(theta)
    assert net.dropout.pass_ == 0 and not net.dropout.queue       # an explicit pass leaves the counter alone
    net.compute_gradient_and_score(x, y); assert net.dropout.pass_ == 1
    net.output(x); assert net.dropout.pass_ == 1
    assert np.isfinite(score)


def test_frozen_and_inference_dropout_is_identity():
    d = o.Dropout(0.3, "d", index=0, state=o.DropoutState(1)); d.init(None, np.float64)
    x = np.random.default_rng(1).standard_normal((4, 3, 2, 2))
    assert d.forward(x, False) is x and d.backward(x) is x
    d.frozen = True
    assert not d.active()


def _mlp(dropout, seed):
    from gan_deeplearning4j_b200 import models as m
    n, z, hid, d = 8, 6, 16, 10
    gs, ds = m.mlp_generator(z, hid, d, lr=1e-2), m.mlp_discriminator(d, hid, lr=1e-2, dropout=dropout)
    q = o.Quirks(xent_clip_eps=0.0)
    rng = np.random.default_rng(seed)
    G = o.net_from_specs(gs, (z,), quirks=q, seed=1); D = o.net_from_specs(ds, (d,), quirks=q, seed=2)
    randomize(G, rng); randomize(D, rng)
    data = [rng.uniform(-1, 1, (n, d)), rng.uniform(-1, 1, (n, z)), rng.uniform(-1, 1, (n, z)),
            1 + 0.05 * rng.standard_normal((n, 1)), 0.05 * rng.standard_normal((n, 1)), np.ones((n, 1))]
    return G, D, data


def test_gan_step_with_p1_layers_equals_without_bit_for_bit():
    G0, D0, data = _mlp(None, 4)
    G1, D1, _ = _mlp(1.0, 4)
    D1.set_params_flat(D0.params_flat()); G1.set_params_flat(G0.params_flat())
    for _ in range(2):
        r0 = o.gan_step(G0, D0, *data); r1 = o.gan_step(G1, D1, *data)
        assert (r0["loss_d_real"], r0["loss_d_fake"], r0["loss_g"]) == (r1["loss_d_real"], r1["loss_d_fake"], r1["loss_g"])
        assert np.array_equal(D0.params_flat(), D1.params_flat()) and np.array_equal(G0.params_flat(), G1.params_flat())
    assert D1.dropout.pass_ == 0       # p = 1 masks nothing, so no pass is counted


def test_gan_step_draws_passes_p_and_p_plus_1():
    """The D step's real and fake minibatches are rows [0, N) and [N, 2N) of pass P; the G step's D pass is P + 1."""
    G, D, data = _mlp(0.5, 5)
    n = data[0].shape[0]
    Dc = copy.deepcopy(D)
    o.gan_step(G, D, *data)
    assert D.dropout.pass_ == 2 and not D.dropout.queue
    drop = [i for i, l in enumerate(D.layers) if isinstance(l, o.Dropout)]
    assert [D.layers[i].index for i in drop] == [1, 3]
    # the G step's D forward ran last: its masks are pass 1
    for i in drop:
        assert np.array_equal(D.layers[i]._m != 0, o.dropout_mask(Dc.dropout.seed, 0, D.layers[i].index, 1, n, 1, 1, 16, 0.5).reshape(n, 16))
    Dc.compute_gradient_and_score(data[0], data[3], pass_=0, row0=n)
    for i in drop:
        assert np.array_equal(Dc.layers[i]._m != 0, o.dropout_mask(Dc.dropout.seed, 0, D.layers[i].index, 0, 2 * n, 1, 1, 16, 0.5).reshape(2 * n, 16)[n:])


def test_specs_models_and_checkpoint_metadata(tmp_path):
    from gan_deeplearning4j_b200 import engine, models as m, serializer
    d = engine.layer_desc({"type": "dropout", "name": "drop", "p": 0.25})
    assert d.type == 11 and abs(d.act_alpha - 0.25) < 1e-7
    assert m.mlp_discriminator() == m.mlp_discriminator(dropout=None)
    assert [s["type"] for s in m.mlp_discriminator(dropout=0.5)] == ["dense", "dropout", "dense", "dropout", "output"]
    assert m.forward_macs(m.mlp_discriminator(dropout=0.5), (256,)) == m.forward_macs(m.mlp_discriminator(), (256,))

    class Fake:           # a net stand-in: what restore_into calls
        def __init__(self): self.p, self.set = np.arange(4, dtype=np.float32), {}
        def num_params(self): return 4
        def set_params(self, v): self.set["params"] = v
        def set_updater_state(self, v): self.set["state"] = v
        def set_iteration(self, v): self.set["iteration"] = v
        def set_dropout_pass(self, v): self.set["dropout_pass"] = v
    path = str(tmp_path / "ck.zip")
    serializer.write_model(path, [], (4,), np.arange(4, dtype=np.float32), np.zeros(8, np.float32), {"iteration": 3, "dropout_pass": 7})
    f = Fake(); serializer.restore_into(f, path)
    assert f.set["iteration"] == 3 and f.set["dropout_pass"] == 7
    serializer.write_model(path, [], (4,), np.arange(4, dtype=np.float32), None, {})
    f = Fake(); serializer.restore_into(f, path)
    assert "dropout_pass" not in f.set
