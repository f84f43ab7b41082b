"""The benchmarked adversarial step at its full sizes: the BF16 step Gan.step_resident replays as a CUDA graph, with the nets, seeds and batch
sizes bench.py builds (its CONFIGS and build_specs are imported, so these tests follow the benchmark).  At these sizes the step overlaps work
across streams: G's train forward runs on a side stream under the D step, weight gradients run on side streams with split-K partials summed
by reduce-list launches, x_real arrives on a copy stream, and each updater reads the gradient buffer right after all of this.  An updater that
starts before a gradient is final, or a side-stream kernel racing a buffer, leaves parameters slightly wrong and different from run to run
while the losses still go down.  Three checks, each at C2, C4 and C5:

1. Replay determinism.  Three graph replays and then one ragged-batch step (which recaptures the graph) agree bit for bit with fresh nets of
   the same seeds and data, and with the eager step: losses, both nets' parameters, updater state, iteration counters and every bf16 weight
   operand.  Afterwards every bf16 operand equals its fp32 master rounded to nearest even.
2. Every update recomputed from the step's own gradients.  Before each replay both nets' parameters, updater state and iteration are
   snapshotted; after it the float64 oracle applies Net.apply_update to the snapshot with the gradient vector the step left (Net.gradients())
   and the device's parameters and state slots must match element by element within the bound below.  The same comparison must reject three
   perturbed references: t off by one, the previous replay's gradient vector, and one updater chunk (UPD_CHUNK elements) of one layer's
   gradient taken from the previous replay -- what an updater racing a side-stream reduction would have read.
3. G's gradient on the third replay against the oracle's backward on the activations of that replay (injected), with the thresholds of
   test_gpu_fullsize.test_bf16_whole_step_layer_by_layer.

D's gradient buffer after the step is still what D's updater read.  The G step's pass through D runs its forward with
FwdOpts.update_running = false, so no BatchNorm running-stat pseudo-gradient is written, and net_backward with want_wgrad = false, so no weight
or bias gradient is forked and the BatchNorm backward kernels get want_param_grads = 0.  Nothing writes D's gradients after D's updater.

The update bound (check 2).  Every net here is Adam on every parameter but the BatchNorm running statistics (NoOp).  u = 2^-24 is the fp32
unit roundoff.  m, v, p are an element's pre-step state and parameter and g its gradient divided by the minibatch (2N for D, N for G).  Both
are powers of two here, so the division is exact.  lr, b1, b2 and eps are the fp32 values the device holds; the oracle is given the same
values, so the comparison is of arithmetic only.  alpha_t = lr sqrt(1 - b2^t) / (1 - b1^t) with t = iteration + 1.  upd_elem (kernels_ew.cu)
computes
    m' = b1*m + (1-b1)*g,   v' = b2*v + ((1-b2)*g)*g,   p' = p - (alpha_t*m') / (sqrtf(v') + eps)
in fp32, and the build contracts with FMA (-fmad is on by default; no fast-math, so sqrtf and the division are correctly rounded and
subnormals are kept).  With S = |b1 m| + |(1-b1) g|, V = b2 v + (1-b2) g^2 and U = alpha_t S / (sqrt(V) + eps), the magnitude the update can
reach:
    |m'_gpu - m'| <= 2u S.   Two products and a sum.  With contraction one product is exact inside the FMA; without, both round.  The sum
                             can cancel (m' far below S), so the bound is in S and not in |m'|.
    |v'_gpu - v'| <= 3u V.   Three products and a sum.  Every term is >= 0, so V = v'.
    |p'_gpu - p'| <= ulp(p')/2 + (K(t) + 8) u U.
                             ulp(p')/2: the final subtraction.  8: m' (2, carried through alpha_t / (sqrt(v') + eps)), sqrtf of v' (1.5,
                             half of v's 3), the roundings of sqrtf, of + eps, of alpha_t*m' and of the division (1 each), rounded up.
    K(t) = 4/(1 - b2^t) + 16 b1^t/(1 - b1^t) + 4.  This is alpha_t's relative error in units of u.  powf is not correctly rounded; the bound
                             allows it 8 ulp.  powf(b2, t) lies in [1/2, 1), where an ulp is u, and 1 - powf(b2, t) is exact (Sterbenz).
                             So its relative error is 8u / (1 - b2^t), halved by sqrtf: the first term.  powf(b1, t) is off by 8 ulp
                             <= 16u b1^t: the second term.  The roundings of sqrtf, of 1 - powf(b1, t), of lr*sqrt and of the division: 4.
                             The powf term dominates.  At b2 = 0.999 and t = 1 .. 3, K is about 4000 .. 1300, so the bound is 2.4e-4 ..
                             8e-5 of U plus half an ulp of p'.  The net-level updater tests use 1e-3 of the parameter.
NoOp (running mean / var): p' = p - g in one fp32 subtraction, so |p'_gpu - p'| <= ulp(p')/2.  Their state slots are not touched (bit for
bit).  Every u-term is multiplied by 1 + 2^-20 for the second-order terms and the float64 reference's own rounding.  Every bound gets
8 * 2^-149 (the smallest subnormal, once per rounding) for underflow.
"""
import dataclasses

import numpy as np
import pytest

import bench
from helpers import (b200, bf16_weights, check_generator_step_grads, check_weight_operands, grads_by_tensor, push_state, state_flat,
                     w_internal, weight_operands)
from oracle import dl4j_oracle as o

pytestmark = pytest.mark.gpu

CASES = ("c2", "c4", "c5")
REPLAYS = 3
RAGGED = {"c2": 77, "c4": 19, "c5": 5001}       # the ragged step's batch (<= N, not a power of two)
UPD_CHUNK = 4096                                # kernels.h: elements per updater block, from the start of each parameter tensor
U = 2.0 ** -24
SLACK = 1 + 2.0 ** -20
FLOOR = 8 * 2.0 ** -149
POWF_ULP = 8


def bench_gan(b, ctx, cfg, graph):
    """G, D and their Gan as bench.make_gan builds them (BF16, BCE with logits, D on 2N rows in two BatchNorm groups, seeds 666 / 667,
    generator forward for the fakes in inference mode), replayed as a CUDA graph or eager."""
    gs, ds, gin, din = bench.build_specs(cfg)
    n = cfg["batch"]
    G = b.Net(ctx, gs, gin, max_batch=n, precision=b.BF16, xent_clip_eps=0.0, seed=666)
    D = b.Net(ctx, ds, din, max_batch=2 * n, precision=b.BF16, xent_clip_eps=0.0, bn_groups=2, seed=667)
    return G, D, b.Gan(G, D, fake_bn_train=False, use_cuda_graph=graph)


def bench_data(cfg):
    """Seeded synthetic inputs (x_real, z_d, z_g, y_real, y_fake, y_gen), fp32: synthetic_batch for the DCGANs, uniform samples for the MLP-GAN."""
    n = cfg["batch"]
    if cfg.get("mlp"):
        rng = np.random.default_rng(1)
        data = [rng.uniform(-1, 1, (n, cfg["d"])), rng.uniform(-1, 1, (n, cfg["z"])), rng.uniform(-1, 1, (n, cfg["z"])),
                1 + 0.05 * rng.standard_normal((n, 1)), 0.05 * rng.standard_normal((n, 1)), np.ones((n, 1))]
    else:
        data = o.synthetic_batch(n, cfg["size"], cfg["nc"], cfg["z"], seed=5)
    return [np.asarray(a, np.float32) for a in data]


def sized_specs(specs, input_shape):
    """specs with n_in on every GEMM layer (the MLP specs leave it to shape inference), as the weight-operand helpers read it."""
    net = o.net_from_specs(specs, input_shape, dtype=np.float32, flat_input=False)
    return [dict(s, n_in=s.get("n_in") or l.n_in) if s["type"] in ("dense", "output") else s for s, l in zip(specs, net.layers)]


def _same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def _snapshot(G, D, gs, ds, gan):
    out = {"losses": gan.losses()}
    for tag, net, specs in (("G", G, gs), ("D", D, ds)):
        out[f"{tag} params"], out[f"{tag} updater state"] = net.params(), net.updater_state()
        out[f"{tag} iteration"] = np.array([net.iteration()], np.int64)
        for (layer, which), v in weight_operands(net, specs).items():
            out[f"{tag} {layer} bf16 operand {which}"] = v
    return out


@pytest.mark.parametrize("name", CASES)
def test_replay_bit_for_bit(b200, name):
    """Check 1 of the module docstring."""
    b, ctx = b200
    cfg = bench.CONFIGS[name]
    n = cfg["batch"]
    gs, ds, gin, din = bench.build_specs(cfg)
    gs, ds = sized_specs(gs, gin), sized_specs(ds, din)
    data = bench_data(cfg)
    runs = {}
    for tag, graph in (("graph replay", True), ("graph replay, fresh nets", True), ("eager", False)):
        runs[tag] = bench_gan(b, ctx, cfg, graph)
        runs[tag][2].upload(*data)
    for k, batch in enumerate([n] * REPLAYS + [RAGGED[name]]):
        if batch != n:
            for _, _, gan in runs.values():
                gan.upload(*[a[:batch] for a in data])
        snaps = {}
        for tag, (G, D, gan) in runs.items():
            gan.step_resident(batch)
            snaps[tag] = _snapshot(G, D, gs, ds, gan)
        want = snaps["graph replay"]
        assert np.all(np.isfinite(want["losses"])), (name, k, want["losses"])
        for tag in ("graph replay, fresh nets", "eager"):
            for key, v in want.items():
                got = snaps[tag][key]
                if not _same_bits(got, v):
                    diff = np.count_nonzero(np.asarray(got).view(np.uint32) != np.asarray(v).view(np.uint32)) if v.dtype == np.float32 else None
                    raise AssertionError(f"{name}, step {k + 1} (batch {batch}): {key} of the {tag} run differs from the graph replay's "
                                         f"({diff} of {v.size} elements)")
    G, D, _ = runs["graph replay"]
    check_weight_operands(b, G, gs, f"{name} G"); check_weight_operands(b, D, ds, f"{name} D")
    for G, D, gan in runs.values():
        gan.close(); G.close(); D.close()


def oracle_net(specs, input_shape, seed):
    """The float64 oracle net of specs, holding the fp32 hyperparameters the device holds (b2g_layer_desc's lr, beta1, beta2, eps)."""
    net = o.net_from_specs(specs, input_shape, quirks=o.Quirks(xent_clip_eps=0.0), dtype=np.float64, seed=seed, flat_input=False)
    f32 = lambda x: float(np.float32(x))
    for l in net.layers:
        if getattr(l, "updater", None) is not None:
            u = l.updater
            l.updater = dataclasses.replace(u, lr=f32(u.lr), rms_decay=f32(u.rms_decay), beta1=f32(u.beta1), beta2=f32(u.beta2), eps=f32(u.eps))
    return net


def update_errors(onet, p0, s0, it, g, mb, p1, s1):
    """The oracle's update of (parameters p0, updater state s0, iteration it) by the gradient vector g on a minibatch of mb, against the
    device's (p1, s1), element by element within the bound of the module docstring.  Returns the failures: (layer, param, what, elements
    outside, elements, worst |d| / bound)."""
    n = p0.size
    slots = s0.size // n
    onet.set_params_flat(p0); push_state(onet, s0); onet.iteration = it
    onet.apply_update(mb, grads=grads_by_tensor(onet, g.astype(np.float64), shaped=True))
    p_ref, s_ref = onet.params_flat(), [state_flat(onet, j) for j in range(slots)]
    t = it + 1
    ulp = lambda x: np.spacing(np.abs(x).astype(np.float32)).astype(np.float64)
    out, off = [], 0
    for li, lname, pn, shape, _ in onet.param_table():
        k = int(np.prod(shape)); sl = slice(off, off + k)
        l = onet.layers[li]
        checks = []
        if pn in l.noop_names():
            checks.append(("params", p1[sl], p_ref[sl], 0.5 * ulp(p1[sl]) + FLOOR))
            for j in range(slots):
                if not _same_bits(s1[j * n:(j + 1) * n][sl], s0[j * n:(j + 1) * n][sl]):
                    out.append((lname, pn, f"state {j} changed", k, k, np.inf))
        else:
            u = l.updater
            assert u.kind == "adam", (lname, u.kind)
            b1, b2, lr, eps = u.beta1, u.beta2, u.lr, u.eps
            gg = g[sl].astype(np.float64) / mb
            m, v = s0[sl].astype(np.float64), s0[n:2 * n][sl].astype(np.float64)
            S = np.abs(b1 * m) + np.abs((1 - b1) * gg)
            V = b2 * v + (1 - b2) * gg * gg
            alpha_t = lr * np.sqrt(1 - b2 ** t) / (1 - b1 ** t)
            K = POWF_ULP / 2 / (1 - b2 ** t) + 2 * POWF_ULP * b1 ** t / (1 - b1 ** t) + 4
            checks += [("params", p1[sl], p_ref[sl], 0.5 * ulp(p1[sl]) + (K + 8) * U * SLACK * alpha_t * S / (np.sqrt(V) + eps) + FLOOR),
                       ("state 0 (m)", s1[sl], s_ref[0][sl], 2 * U * SLACK * S + FLOOR),
                       ("state 1 (v)", s1[n:2 * n][sl], s_ref[1][sl], 3 * U * SLACK * V + FLOOR)]
        for what, got, ref, bound in checks:
            d = np.abs(got.astype(np.float64) - ref)
            bad = ~(d <= bound)
            if bad.any():
                out.append((lname, pn, what, int(bad.sum()), k, float(np.max(np.where(np.isnan(d), np.inf, d) / bound))))
        off += k
    return out


def chunk_positions(onet, specs):
    """The positions, in the net's flat (DL4J-order) gradient vector, of the middle updater chunk of the net's largest weight tensor, and
    that layer's name.  The updater walks W in the engine's internal order ([A][taps][B] for a conv), UPD_CHUNK elements per block from the
    tensor's start."""
    off, best = 0, None
    for li, lname, pn, shape, _ in onet.param_table():
        k = int(np.prod(shape))
        if pn == "W" and (best is None or k > best[2]):
            best = (li, off, k)
        off += k
    li, off, k = best
    assert onet.layers[li].name == specs[li]["name"]
    perm = w_internal(specs[li], np.arange(k, dtype=np.float64)).astype(np.int64)       # internal element i is DL4J element perm[i]
    c = (k // UPD_CHUNK) // 2
    return off + perm[c * UPD_CHUNK:(c + 1) * UPD_CHUNK], specs[li]["name"]


@pytest.mark.parametrize("name", CASES)
def test_updates_recomputed_from_the_step_gradients(b200, name):
    """Check 2 of the module docstring, with its three sensitivity controls: each must be rejected on a weight tensor of each net, the
    chunk control exactly on the weight tensor whose chunk it swapped."""
    b, ctx = b200
    cfg = bench.CONFIGS[name]
    n = cfg["batch"]
    gs, ds, gin, din = bench.build_specs(cfg)
    G, D, gan = bench_gan(b, ctx, cfg, True)
    gan.upload(*bench_data(cfg))
    nets = (("G", G, oracle_net(gs, gin, 1), gs, n), ("D", D, oracle_net(ds, din, 2), ds, 2 * n))
    prev = {}
    for k in range(1, REPLAYS + 1):
        pre = {tag: (net.params(), net.updater_state(), net.iteration()) for tag, net, _, _, _ in nets}
        gan.step_resident(n)
        for tag, net, onet, specs, mb in nets:
            assert mb & (mb - 1) == 0, mb          # g / mb is exact: the bound has no term for it
            p0, s0, it0 = pre[tag]
            g, p1, s1 = net.gradients(), net.params(), net.updater_state()
            assert it0 == k - 1 and net.iteration() == k, (name, tag, it0, net.iteration())
            bad = update_errors(onet, p0, s0, it0, g, mb, p1, s1)
            assert not bad, f"{name} {tag}, replay {k}: the device's update differs from the one recomputed from its own gradients: {bad[:6]}"
            if k > 1:
                idx, layer = chunk_positions(onet, specs)
                g_chunk = g.copy(); g_chunk[idx] = prev[tag][idx]
                assert np.any(g_chunk != g)
                for what, it_ref, g_ref in (("t off by one", it0 + 1, g), ("the previous replay's gradient vector", it0, prev[tag]),
                                            (f"one updater chunk of {layer}.W from the previous replay", it0, g_chunk)):
                    bad = update_errors(onet, p0, s0, it_ref, g_ref, mb, p1, s1)
                    assert any(pn == "W" for _, pn, *_ in bad), f"{name} {tag}, replay {k}: the comparison accepts the update recomputed with {what}"
                    if it_ref == it0 and g_ref is g_chunk:
                        assert {(lname, pn) for lname, pn, *_ in bad} == {(layer, "W")}, (name, tag, k, bad)
            prev[tag] = g
    gan.close(); G.close(); D.close()


@pytest.mark.parametrize("name", CASES)
def test_generator_gradient_on_a_replayed_step(b200, name):
    """Check 3 of the module docstring.  G's parameters are the snapshot before the third replay; D's are those after it (the G step runs
    through the D the step has just updated and does not change it).  Both nets' activations are the G step's pass, each net's most recent
    forward.  Every G gradient but the running-stat pseudo-gradients: relative Frobenius error < 3e-2, cosine > 0.999."""
    b, ctx = b200
    cfg = bench.CONFIGS[name]
    n = cfg["batch"]
    gs, ds, gin, din = bench.build_specs(cfg)
    G, D, gan = bench_gan(b, ctx, cfg, True)
    data = bench_data(cfg)
    gan.upload(*data)
    for _ in range(REPLAYS - 1):
        gan.step_resident(n)
    pG = G.params()
    gan.step_resident(n)
    q = o.Quirks(xent_clip_eps=0.0)
    Go = o.net_from_specs(gs, gin, quirks=q, dtype=np.float32, seed=1)
    Do = o.net_from_specs(ds, din, quirks=q, dtype=np.float32, seed=2, flat_input=False)
    Go.set_params_flat(pG); Do.set_params_flat(D.params())
    bf16_weights(Go); bf16_weights(Do)
    check_generator_step_grads(Go, Do, G, D, gs, ds, data[2], data[5], f"{name}, replay {REPLAYS}: ")
    gan.close(); G.close(); D.close()
