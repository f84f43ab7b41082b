"""ElementWiseVertex / MergeVertex on the CPU: the oracle's vertices and skip edges against finite differences at GradientCheckUtil's
tolerances and against torch.autograd, the oracle's vertex resolution against the library's, and the specs, builders and refusals of the
Python host layer."""
import numpy as np
import pytest
import torch

from gan_deeplearning4j_b200 import engine as E
from gan_deeplearning4j_b200 import models as m
from oracle import dl4j_oracle as o

FD_EPS, MAX_REL, MIN_ABS = 1e-6, 1e-3, 1e-8      # GradientCheckUtil.checkGradients(..., 1e-6, 1e-3, 1e-8, ...)


def fd_check(net, x, y, rng, n_check=60):
    """Central differences of the score against grads_flat / mb on n_check random parameters (every one if fewer)."""
    net.compute_gradient_and_score(x, y)
    g = net.grads_flat() / x.shape[0]
    p0 = net.params_flat().copy()
    # BatchNorm's running mean / var carry pseudo-gradients and no score dependence in train mode
    live = np.concatenate([np.full(int(np.prod(sh)), p not in net.layers[li].noop_names()) for li, _, p, sh, _ in net.param_table()])
    idx = np.flatnonzero(live)
    idx = idx if idx.size <= n_check else rng.choice(idx, n_check, replace=False)
    for k in idx:
        p = p0.copy(); p[k] += FD_EPS; net.set_params_flat(p); sp = net.compute_gradient_and_score(x, y)
        p[k] -= 2 * FD_EPS; net.set_params_flat(p); sm = net.compute_gradient_and_score(x, y)
        num = (sp - sm) / (2 * FD_EPS)
        if abs(num - g[k]) < MIN_ABS:
            continue
        rel = abs(num - g[k]) / (abs(num) + abs(g[k]))
        assert rel < MAX_REL, (k, num, g[k], rel)
    net.set_params_flat(p0)


def dense(name, n_out, act="tanh"):
    return {"type": "dense", "name": name, "n_out": n_out, "activation": act, "updater": m.sgd(0.1)}


def ff_graph(vertex, src="d1", order=0):
    """d1 -> d2 -> vertex(d2, src) -> d3 -> output(mse)."""
    ins = ["d2", src] if order == 0 else [src, "d2"]
    v = m.merge(ins, name="v") if vertex == "merge" else m.elementwise(vertex, ins, name="v")
    return [dense("d1", 6), dense("d2", 6, "sigmoid"), v, dense("d3", 5),
            {"type": "output", "name": "out", "n_out": 3, "loss": "mse", "activation": "identity", "updater": m.sgd(0.1)}]


def conv(name, c_in, c_out, k=3, s=1, p=1, act="identity"):
    return {"type": "conv2d", "name": name, "n_in": c_in, "n_out": c_out, "kernel": (k, k), "stride": (s, s), "padding": (p, p), "activation": act,
            "has_bias": False, "updater": m.sgd(0.1)}


def residual_net(ch=4):
    return ([conv("stem", 2, ch, act="tanh")] + m.residual_block("rb", ch, "stem", activation="tanh") +
            [conv("head", ch, 2, k=1, p=0), m.cnn_loss("mse", name="loss")])


def shared_source_net():
    """One source (c1) feeding two vertices: an Add and, later, a Merge."""
    return [conv("c1", 2, 4, act="tanh"), conv("c2", 4, 4, act="sigmoid"), m.elementwise("add", ["c2", "c1"], name="a1"),
            conv("c3", 4, 4, act="tanh"), m.merge(["c1", "c3"], name="m1"), conv("head", 8, 3, k=1, p=0), m.cnn_loss("mcxent", name="loss")]


def onehot_map(rng, n, c, h, w):
    lab = rng.integers(0, c, (n, h, w))
    return np.moveaxis(np.eye(c)[lab], -1, 1)


@pytest.mark.parametrize("op", o.EW_OPS)
@pytest.mark.parametrize("order", [0, 1])
def test_elementwise_finite_differences(op, order):
    rng = np.random.default_rng(1)
    net = o.net_from_specs(ff_graph(op, order=order), (4,))
    x, y = rng.standard_normal((5, 4)), rng.standard_normal((5, 3))
    fd_check(net, x, y, rng, n_check=10 ** 6)


@pytest.mark.parametrize("order", [0, 1])
def test_merge_finite_differences(order):
    rng = np.random.default_rng(2)
    net = o.net_from_specs(ff_graph("merge", order=order), (4,))
    x, y = rng.standard_normal((5, 4)), rng.standard_normal((5, 3))
    fd_check(net, x, y, rng, n_check=10 ** 6)


@pytest.mark.parametrize("op", o.EW_OPS)
def test_vertex_on_its_own_predecessor_exact_ties(op):
    """j = i - 1: both inputs are the same tensor, so MAX ties on every element (all of e goes to the first input; the sum is e either way)."""
    rng = np.random.default_rng(3)
    net = o.net_from_specs(ff_graph(op, src="d2"), (4,))
    x, y = rng.standard_normal((5, 4)), rng.standard_normal((5, 3))
    fd_check(net, x, y, rng, n_check=10 ** 6)


def test_max_tie_rule():
    a = np.array([1.0, 2.0, 3.0]); b = np.array([1.0, 5.0, 0.0]); e = np.array([10.0, 20.0, 30.0])
    da, db = o.ew_backward("max", e, a, b)
    assert list(da) == [10.0, 0.0, 30.0] and list(db) == [0.0, 20.0, 0.0]
    v = o.ElementWiseVertex("max", 0, 1)      # order 1: (skip, spine) -> the tie goes to the skip input
    v.forward(b, a, True)
    spine, skip = v.backward(e)
    assert list(spine) == [0.0, 20.0, 0.0] and list(skip) == [10.0, 0.0, 30.0]


@pytest.mark.parametrize("builder,shape,loss", [
    ("residual", (2, 6, 6), "mse"), ("unet", (2, 8, 8), "mcxent"), ("shared", (2, 5, 5), "mcxent")])
def test_conv_graph_finite_differences(builder, shape, loss):
    rng = np.random.default_rng(4)
    if builder == "residual":
        specs = residual_net()
    elif builder == "unet":
        specs = m.unet(size=shape[1], nc=shape[0], n_classes=3, nf=2, depth=2, loss=loss)
    else:
        specs = shared_source_net()
    net = o.net_from_specs(specs, shape)
    n = 3
    x = rng.standard_normal((n,) + shape)
    out = net.forward(x, True)
    y = onehot_map(rng, n, *out.shape[1:]) if loss == "mcxent" else rng.standard_normal(out.shape)
    fd_check(net, x, y, rng)


def test_unet_shapes_and_macs():
    specs = m.unet(size=16, nc=3, n_classes=4, nf=8, depth=2)
    net = o.net_from_specs(specs, (3, 16, 16))
    out = net.forward(np.zeros((2, 3, 16, 16)), False)
    assert out.shape == (2, 4, 16, 16)
    merges = [s for s in specs if s["type"] == "merge"]
    assert [s["inputs"] for s in merges] == [["unet_up1", "unet_enc1_act"], ["unet_up0", "unet_enc0_act"]]
    # the decoder convs read 2 * nf * 2^k channels: forward_macs follows the merges
    macs = m.forward_macs(specs, (3, 16, 16))
    enc = 16 * 16 * 8 * 3 * 9 + 8 * 8 * 16 * 8 * 9 + 4 * 4 * 32 * 16 * 9
    dec = 4 * 4 * 32 * 16 * 16 + 8 * 8 * 16 * 32 * 9 + 8 * 8 * 16 * 8 * 16 + 16 * 16 * 8 * 16 * 9 + 16 * 16 * 4 * 8
    assert macs == enc + dec


def every_op_net():
    """d1 -> d2 -> one vertex of each op on d1 (the input order alternating) -> merge with d1 -> d3 -> output(mse)."""
    specs = [dense("d1", 6), dense("d2", 6, "sigmoid")]
    prev = "d2"
    for k, op in enumerate(o.EW_OPS):
        specs += [m.elementwise(op, [prev, "d1"] if k % 2 == 0 else ["d1", prev], name=f"v{k}")]
        prev = f"v{k}"
    return specs + [m.merge(["d1", prev], name="mg"), dense("d3", 5),
                    {"type": "output", "name": "out", "n_out": 3, "loss": "mse", "activation": "identity", "updater": m.sgd(0.1)}]


def test_torch_autograd_agrees():
    """A dense graph with every op (and a merge) in float64: the oracle's gradients against torch.autograd's."""
    rng = np.random.default_rng(5)
    net = o.net_from_specs(every_op_net(), (4,))
    x, y = rng.standard_normal((5, 4)), rng.standard_normal((5, 3))
    net.compute_gradient_and_score(x, y)
    g = net.grads_flat()
    Ls = net.layers
    P = {l.name: {k: torch.tensor(v, requires_grad=True) for k, v in l.params.items()} for l in Ls if l.has_params}
    d = lambda h, nm: h @ P[nm]["W"] + P[nm]["b"]
    h1 = torch.tanh(d(torch.tensor(x), "d1")); h = torch.sigmoid(d(h1, "d2"))
    for k, op in enumerate(o.EW_OPS):
        a, b = (h, h1) if k % 2 == 0 else (h1, h)
        h = {"add": a + b, "subtract": a - b, "product": a * b, "average": (a + b) * 0.5, "max": torch.where(a >= b, a, b)}[op]
    h = torch.tanh(d(torch.cat([h1, h], 1), "d3"))
    z = d(h, "out")
    loss = ((z - torch.tensor(y)) ** 2).sum() / 3       # LossMSE: per example sum / nOut, summed over the batch
    loss.backward()
    want = np.concatenate([np.concatenate([P[l.name]["W"].grad.numpy().ravel(order="F"), P[l.name]["b"].grad.numpy()]) for l in Ls if l.has_params])
    assert np.allclose(g, want, rtol=1e-10, atol=1e-12)


def test_chain_nets_unchanged_by_the_walk():
    """On a net without vertices, the Net's backward walk computes bit for bit what a plain loop over the layers computes."""
    net = o.net_from_specs(m.dcgan_discriminator(16, 4, 3), (3, 16, 16))
    rng = np.random.default_rng(6)
    x, y = rng.standard_normal((4, 3, 16, 16)), rng.uniform(0, 1, (4, 1))
    score, _, _, eps_in = net.compute_gradient_and_score(x, y, collect=True)
    walked = net.grads_flat()
    loss_sum, eps = net.layers[-1].score_and_eps(y)      # the layers still hold the forward's inputs
    for l in reversed(net.layers[:-1]):
        eps = l.backward(eps)
    assert score == float(loss_sum) / x.shape[0] + net.l2_score()
    assert np.array_equal(walked, net.grads_flat()) and np.array_equal(eps_in, eps)


def test_residual_gan_step_on_the_oracle():
    """oracle.gan_step's backward walks (the discriminator's prefix and the generator) run through the vertices."""
    G = o.net_from_specs(m.dcgan_generator(16, 8, 4, 3, residual=True), (8,))
    D = o.net_from_specs(m.dcgan_discriminator(16, 4, 3, residual=True), (3, 16, 16))
    data = [a.astype(np.float64) for a in o.synthetic_batch(4, 16, 3, 8, seed=3)]
    p0 = G.params_flat().copy()
    r = o.gan_step(G, D, *data)
    assert np.isfinite([r["loss_d_real"], r["loss_d_fake"], r["loss_g"]]).all()
    assert not np.array_equal(G.params_flat(), p0)
    # the generator's residual conv weights moved: their gradient came through the Add
    g = G.layer("gen_res_1_conv_1")
    assert np.abs(g.grads["W"]).max() > 0


def test_default_dcgan_specs_unchanged():
    for f in (m.dcgan_generator, m.dcgan_discriminator):
        assert f() == f(residual=False)
        assert not any(s["type"] in E.VERTEX_TYPES for s in f())
    assert m.dcgan_discriminator(patch=True) == m.dcgan_discriminator(patch=True, residual=False)


def test_residual_specs():
    gs = m.dcgan_generator(32, 16, 8, 3, residual=True)
    adds = [s for s in gs if s["type"] == "elementwise"]
    assert [s["inputs"][1] for s in adds] == ["gen_act_1", "gen_act_2", "gen_act_3"]
    ds = m.dcgan_discriminator(32, 8, 3, residual=True, patch=True)
    assert [s["inputs"][1] for s in ds if s["type"] == "elementwise"] == ["dis_conv_1", "dis_act_2", "dis_act_3"]
    rb = m.residual_block("r", 8, "x")
    assert [s["type"] for s in rb] == ["conv2d", "batchnorm", "activation", "conv2d", "batchnorm", "elementwise", "activation"]
    assert rb[5]["op"] == "add" and rb[5]["inputs"] == ["r_bn_2", "x"]


def test_resolve_vertices():
    base = [dense("a", 4), dense("b", 4)]
    assert E.resolve_vertices(base + [m.elementwise("add", ["b", "a"], name="v")])[2] == (0, 0)
    assert E.resolve_vertices(base + [m.elementwise("add", ["a", "b"], name="v")])[2] == (0, 1)
    assert E.resolve_vertices(base + [m.merge(["b", "b"], name="v")])[2] == (1, 0)
    d = E.layer_desc(base[0] | {}, None)
    assert d.pre_h == 0 and d.pre_w == 0
    v = m.elementwise("max", ["a", "b"], name="v")
    d = E.layer_desc(v, E.resolve_vertices(base + [v])[2])
    assert (d.type, d.act, d.pre_h, d.pre_w) == (15, 4, 0, 1)


def test_oracle_resolves_vertices_as_the_library_does():
    """The oracle resolves every graph the tests build to the library's (j, order), and shifts j past the convolutionalFlat reshape."""
    from test_gpu_graph import _guard_net, _nets
    graphs = [residual_net(), shared_source_net(), every_op_net(), m.unet(size=8, nc=2, n_classes=3, nf=2, depth=2, loss="mcxent"),
              m.unet(size=16, nc=3, n_classes=4, nf=8, depth=2)]
    graphs += [ff_graph(v, order=order) for v in o.EW_OPS + ("merge",) for order in (0, 1)] + [ff_graph(v, src="d2") for v in o.EW_OPS]
    graphs += [_nets(kind)[0] for kind in ("residual", "unet", "shared", "ff_merge")] + [_guard_net(g)[0] for g in ("bn_act", "fold", "bwd")]
    for size, z, nf in ((16, 8, 4), (16, 12, 8), (32, 16, 8)):
        graphs += [m.dcgan_generator(size, z, nf, 3, residual=True)]
        graphs += [m.dcgan_discriminator(size, nf, 3, residual=True, patch=patch) for patch in (False, True)]
    for specs in graphs:
        want = E.resolve_vertices(specs)
        assert any(want)
        assert o.vertex_inputs(specs) == want
        assert o.vertex_inputs(specs, 1) == [None if r is None else (r[0] + 1, r[1]) for r in want]


@pytest.mark.parametrize("bad,msg", [
    ([dense("a", 4), dense("b", 4), dense("c", 4), m.elementwise("add", ["a", "b"], name="v")], "previous layer"),
    ([dense("a", 4), dense("b", 4), m.elementwise("add", ["b", "zz"], name="v")], "names 0"),
    ([dense("a", 4), dense("a", 4), dense("b", 4), m.elementwise("add", ["b", "a"], name="v")], "names 2"),
    ([m.elementwise("add", ["in", "in"], name="v")], "net input"),
    ([dense("a", 4), {"type": "elementwise", "name": "v", "op": "add", "inputs": ["a", "a", "a"]}], "exactly two"),
    ([dense("a", 4), {"type": "elementwise", "name": "v", "op": "mul", "inputs": ["a", "a"]}], "unknown op"),
])
def test_resolve_refusals(bad, msg):
    with pytest.raises(ValueError, match=msg):
        E.resolve_vertices(bad)


def test_builder_refusals():
    with pytest.raises(ValueError):
        m.elementwise("min", ["a", "b"])
    with pytest.raises(ValueError):
        m.merge(["a", "b", "c"])
    with pytest.raises(ValueError):
        m.unet(size=12, depth=3)


def test_forward_macs_resolves_merges_by_index():
    specs = m.unet(size=16, nc=3, n_classes=4, nf=8, depth=2)
    renamed = [dict(s, name=f"L{i}") for i, s in enumerate(specs)]
    for i, s in enumerate(renamed):           # the same graph under other names
        if s["type"] == "merge":
            s["inputs"] = [f"L{i - 1}", f"L{[x['name'] for x in specs].index(specs[i]['inputs'][1])}"]
    assert m.forward_macs(renamed, (3, 16, 16)) == m.forward_macs(specs, (3, 16, 16))
    ambiguous = [dict(s, name="") if s["type"] != "merge" else s for s in specs]
    with pytest.raises(ValueError):
        m.forward_macs(ambiguous, (3, 16, 16))
