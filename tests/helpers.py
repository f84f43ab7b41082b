"""Test-only utilities for comparing the oracle's nets (oracle.dl4j_oracle.net_from_specs) with the CUDA library's.

- b200: the module-scoped fixture (b, ctx), the library and a Context on device 0.  A test module imports it (from helpers import b200),
  which registers it in that module, so every module gets its own Context.
- Builders: mlp_convbn_specs (the small MLP and conv + BatchNorm nets), oracle_gan_pair / fp32_gan_pair (the 16x16 DCGAN pair of the
  oracle, and of the library with the oracle's parameters), bf16_gan (the BF16 pair of the launch-count tests).
- Comparisons: pclose, compare_params_and_state, assert_close_up_to_sign_flips, gan_step_parity, check_bf16, inject_forward and
  check_weight_operands; launches_per_step counts a GAN step's kernel launches; run_two_ranks runs a tools/ script on two GPUs.
- Flat vectors and the oracle: push_params / push_state load parameters into the library net and a library updater state into the oracle,
  state_flat flattens an oracle state slot, grads_by_tensor splits a library gradient vector per oracle tensor, flat_order flattens an oracle
  gradient like the library; weight_operands reads a BF16 net's bf16 weight copies."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import dl4j_oracle as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def b200():
    """(b, ctx): the library and a Context on device 0, closed when the module's tests are done."""
    import gan_deeplearning4j_b200 as b
    ctx = b.Context(0)
    yield b, ctx
    ctx.close()


def randomize(net, rng, scale=None):
    """Random (non-default) parameters incl. BN gamma/beta/mean/var and biases, so nothing hides behind 0/1 defaults."""
    for l in net.layers:
        if not l.has_params:
            continue
        for p, shape, _ in l.param_specs():
            if p == "W":
                continue
            if p == "var":
                l.params[p] = rng.uniform(0.5, 1.5, shape).astype(net.dtype)
            elif p == "gamma":
                l.params[p] = rng.uniform(0.7, 1.3, shape).astype(net.dtype)
            else:
                l.params[p] = (0.1 * rng.standard_normal(shape)).astype(net.dtype)


def push_params(onet, bnet):
    """Copy the oracle's parameters into the CUDA net through getParam/setParam-style calls (DL4J flattened order)."""
    bnet.set_params(onet.params_flat().astype(np.float32))


def push_state(onet, st):
    """Load a library net's updater state vector st (Net.updater_state(): [state0 | state1 (| state2)], each slot in DL4J flattened order)
    into the oracle's state slots: the inverse of state_flat.  A parameter the oracle keeps no state for must hold zeros in every slot."""
    n = onet.num_params()
    slots = st.size // n
    assert st.size == slots * n, (st.size, n)
    off = 0
    for li, name, p, shape, order in onet.param_table():
        k = int(np.prod(shape))
        have = onet.state.get((li, p), [])
        for j in range(slots):
            v = st[j * n + off:j * n + off + k]
            if j < len(have):
                have[j][...] = v.reshape(shape, order=order.upper())
            else:
                assert np.all(v == 0), (name, p, "slot", j)
        off += k


def grads_by_tensor(onet, flat, shaped=False):
    """A flat gradient vector (Net.gradients(), DL4J flattened order) per oracle tensor: {(layer index, param): the tensor's slice}, or with
    shaped the slice in the tensor's shape (dense W is 'f'-order), what Net.apply_update(grads=...) takes."""
    out, off = {}, 0
    for li, l in enumerate(onet.layers):
        if not l.has_params:
            continue
        for pname, shp, order in l.param_specs():
            n = int(np.prod(shp)); v = flat[off:off + n]; off += n
            out[(li, pname)] = v.reshape(shp, order=order.upper()) if shaped else v
    assert off == flat.size
    return out


def flat_order(l, pname):
    """oracle gradient tensor -> the element order of DL4J's flattened view (dense W is 'f'-order)."""
    g = np.asarray(l.grads[pname], np.float64)
    return g.ravel(order="F") if (isinstance(l, o.Dense) and pname == "W") else g.ravel()


def rel_fro(a, b):
    """Relative Frobenius error of a against b."""
    a = np.asarray(a, np.float64).ravel(); b = np.asarray(b, np.float64).ravel()
    return float(np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30))


def check_grads_against_oracle(onet, got_flat, specs, what):
    """A library gradient vector against the oracle's gradients after its backward, tensor by tensor (the running-stat pseudo-gradients
    excepted): relative Frobenius error < 3e-2 (about ten bf16-rounded epsilon tensors deep) and cosine > 0.999."""
    for (li, pname), gv in grads_by_tensor(onet, got_flat).items():
        if pname in ("mean", "var"):
            continue
        ref = flat_order(onet.layers[li], pname)
        fro = rel_fro(gv, ref); cos = float(np.dot(gv, ref) / (np.linalg.norm(gv) * np.linalg.norm(ref) + 1e-30))
        assert fro < 3e-2 and cos > 0.999, (f"{what} grad {specs[li].get('name')}.{pname}", fro, cos)


def bf16_weights(onet):
    """Every W of a float32 oracle net rounded to bf16 in place: the operands a BF16 library net's forward reads instead of its fp32 master."""
    for l in onet.layers:
        if l.has_params and "W" in l.params:
            l.params["W"] = bf16_round(l.params["W"]).astype(np.float32)


def check_generator_step_grads(G, D, bG, bD, gs, ds, z_g, y_gen, what=""):
    """After an adversarial step of the library nets bG, bD: G's gradient against the oracle's exact backward of the G step, on the activations
    of that step's pass injected layer by layer (inject_forward; the pass is each library net's most recent forward), by
    check_grads_against_oracle.  G, D: the oracle nets (float32) holding the parameters that pass ran with, W rounded to bf16.  what: a prefix
    of the messages."""
    n = z_g.shape[0]
    xg = inject_forward(G, bG, gs, bf16_round(z_g), n, f"{what}G (train, z_g)")
    inject_forward(D, bD, ds, xg, n, f"{what}D (G step)")
    _, eps = D.layers[-1].score_and_eps(np.asarray(y_gen, np.float32))
    if isinstance(D.layers[-1], o.Output):
        eps = D.layers[-1].backward(eps)
    eps_g = D.backward_from_prefix(eps).reshape(xg.shape)
    for l in reversed(G.layers):
        eps_g = l.backward(eps_g)
    check_grads_against_oracle(G, bG.gradients(), gs, f"{what}G")


def rel_err(a, b):
    a = np.asarray(a, np.float64).ravel(); b = np.asarray(b, np.float64).ravel()
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


def pclose(got, want, bound, tol=2e-3, step=0.0):
    """Every element within tol of the scale, max(want's largest magnitude, step); else every element within bound and at most 2% of them
    beyond tol.  step floors the scale: a parameter tensor that an update cancelled down to near zero (a one-element bias after one step) is
    measured against one update step, not against its own size."""
    d = np.abs(np.asarray(got, np.float64) - np.asarray(want, np.float64))
    scale = max(np.abs(want).max(), step)
    if d.max() < tol * scale:
        return True
    return d.max() <= bound and (d > tol * scale).mean() <= 0.02


def state_flat(onet, k):
    """The oracle's updater state slot k flattened like b2g_net_get_updater_state (zeros where a parameter has none)."""
    out = []
    for li, _, p, shape, order in onet.param_table():
        st = onet.state.get((li, p))
        out.append((st[k] if st is not None and k < len(st) else np.zeros(shape)).ravel(order=order.upper()))
    return np.concatenate(out)


def compare_params_and_state(onet, bnet, what, tol, bounds=None):
    """The library net's parameters and every updater state slot (2 or 3) against the oracle's, tensor by tensor, by pclose.  bounds: {layer
    name: the lr-step exemption bound of its updater}; a layer without one has none.  A slot the oracle holds at zero is zero on the device."""
    bounds = bounds or {}
    p_b, p_o = bnet.params(), onet.params_flat()
    st = bnet.updater_state(); n = bnet.num_params()
    slots = st.size // n
    assert slots in (2, 3)
    s_o = [state_flat(onet, k) for k in range(slots)]
    off = 0
    for li, name, pn, shape, _ in onet.param_table():
        k = int(np.prod(shape)); sl = slice(off, off + k)
        bound = bounds.get(name, 0.0)
        assert pclose(p_b[sl], p_o[sl], bound, tol, bound / 2), (what, name, pn, rel_err(p_b[sl], p_o[sl]))
        for j in range(slots):
            b_st, o_st = st[j * n:(j + 1) * n][sl], s_o[j][sl]
            if np.abs(o_st).max() > 0:
                assert pclose(b_st, o_st, np.inf if bound else 0.0, tol), (what, name, pn, "state", j, rel_err(b_st, o_st))
            else:
                assert np.all(b_st == 0), (what, name, pn, "state", j)
        off += k


def assert_close_up_to_sign_flips(got, want, lr, tol):
    """An update of lr * g / (|g| + eps) (Adam's first step; RmsProp with rmsDecay = eps = 1e-8 on every step) is about lr * sign(g): an
    element whose gradient is numerically zero may land one lr step apart.  Every difference within 2 lr (and a 1 % margin), and fewer than
    2 % of the elements beyond tol of want's largest magnitude."""
    d = np.abs(np.asarray(got, np.float64) - np.asarray(want, np.float64))
    assert d.max() <= 2.02 * lr, d.max()
    assert (d > tol * np.abs(want).max()).mean() < 2e-2, (d > tol * np.abs(want).max()).mean()


def mlp_convbn_specs(kind, updater):
    """(specs, input shape) of the 64 -> 256 -> 128 -> 1 MLP ("mlp": W of 8 chunks, every segment 16-byte aligned) or the conv + BatchNorm
    net ("convbn") on 3x8x8; updater() gives each layer with parameters its updater spec."""
    if kind == "mlp":
        return [{"type": "dense", "name": "d1", "n_out": 256, "activation": "tanh", "updater": updater(), "l2": 1e-3},
                {"type": "dense", "name": "d2", "n_out": 128, "activation": "lrelu", "alpha": 0.2, "updater": updater()},
                {"type": "output", "name": "out", "n_out": 1, "updater": updater()}], (64,)
    assert kind == "convbn", kind
    return ([{"type": "conv2d", "name": "c1", "n_out": 8, "kernel": (3, 3), "stride": (2, 2), "padding": (1, 1), "updater": updater()},
             {"type": "activation", "name": "a1", "activation": "lrelu", "alpha": 0.2},
             {"type": "conv2d", "name": "c2", "n_out": 12, "kernel": (3, 3), "stride": (1, 1), "padding": (1, 1), "has_bias": False, "updater": updater()},
             {"type": "batchnorm", "name": "bn2", "updater": updater()}, {"type": "activation", "name": "a2", "activation": "tanh"},
             {"type": "cnn_to_ff", "name": "flat"},
             {"type": "dense", "name": "fc", "n_out": 10, "activation": "tanh", "updater": updater()},
             {"type": "output", "name": "out", "n_out": 1, "updater": updater()}], (3, 8, 8))


def oracle_gan_pair(gs, ds, size=16, z=12, quirks=o.DEFAULT_QUIRKS, mask_seed=666):
    """The oracle's G (specs gs, seed 1, on a z-vector) and D (specs ds, seed 2, on 3 x size x size images), both randomized from
    default_rng(5), G first.  quirks: both nets'; mask_seed: D's dropout masks."""
    rng = np.random.default_rng(5)
    G = o.net_from_specs(gs, (z,), quirks=quirks, seed=1)
    D = o.net_from_specs(ds, (3, size, size), quirks=quirks, seed=2, mask_seed=mask_seed)
    randomize(G, rng); randomize(D, rng)
    return G, D


def fp32_gan_pair(b, ctx, gs, ds, n, size=16, z=12, quirks=o.DEFAULT_QUIRKS, mask_seed=666, g_kw=None, d_kw=None, **kw):
    """oracle_gan_pair, the library's G (batch n) and D (batch 2n, two BatchNorm groups) holding its parameters, and the float64
    synthetic_batch(n, size, 3, z, seed=3): (G, D, bG, bD, data).  kw: b.Net options of both library nets (precision, FP32 unless given;
    xent_clip_eps); g_kw / d_kw: of one of them (seed, gradient_normalization)."""
    G, D = oracle_gan_pair(gs, ds, size, z, quirks, mask_seed)
    kw.setdefault("precision", b.FP32)
    bG = b.Net(ctx, gs, (z,), max_batch=n, **kw, **(g_kw or {}))
    bD = b.Net(ctx, ds, (3, size, size), max_batch=2 * n, bn_groups=2, **kw, **(d_kw or {}))
    push_params(G, bG); push_params(D, bD)
    data = [a.astype(np.float64) for a in o.synthetic_batch(n, size, 3, z, seed=3)]
    return G, D, bG, bD, data


def bf16_gan(b, ctx, gs, ds, gin, din, n):
    """The BF16 G (input shape gin, batch n, seed 666) and D (din, batch 2n, two BatchNorm groups, seed 667) of the launch-count tests, on
    BCE-with-logits (xent_clip_eps 0) like bench.py."""
    G = b.Net(ctx, gs, gin, max_batch=n, precision=b.BF16, xent_clip_eps=0.0, seed=666)
    D = b.Net(ctx, ds, din, max_batch=2 * n, precision=b.BF16, xent_clip_eps=0.0, bn_groups=2, seed=667)
    return G, D


def launches_per_step(ctx, gan, n):
    """Kernel launches per resident GAN step of batch n on the uploaded data: the mean over three steps after two warm-up steps."""
    for _ in range(2):
        gan.step_resident(n)
    ctx.sync(); l0 = ctx.launch_count()
    for _ in range(3):
        gan.step_resident(n)
    ctx.sync()
    return (ctx.launch_count() - l0) / 3


def run_two_ranks(script, out_json, port, env=None, timeout=600, args=()):
    """tools/<script> out_json *args on two ranks of one node under torch.distributed.run (master 127.0.0.1:port); the JSON it wrote.  Skips the
    test on a machine with fewer than two GPUs."""
    try:
        import torch
        gpus = torch.cuda.device_count()
    except Exception:
        gpus = 0
    if gpus < 2:
        pytest.skip("needs two GPUs")
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                          "--master-port", str(port), os.path.join(ROOT, "tools", script), str(out_json), *args],
                         capture_output=True, text=True, timeout=timeout, env=env, cwd=ROOT)
    assert out.returncode == 0, out.stdout[-800:] + out.stderr[-1500:]
    with open(out_json) as f:
        return json.load(f)


def gan_step_parity(b, ctx, gs, ds, G, D, data, labels, lr, what, tol=1e-3):
    """The FP32 adversarial step of the library against the oracle's, on copies of the oracle nets G, D (specs gs, ds): over 3 steps on data
    (x_real, z_d, z_g and per-image labels), oracle gan_step with `labels` and Gan.step agree on the losses within tol and on both nets'
    parameters by pclose at 2 lr, once captured as a CUDA graph and once eager; the two runs agree bit for bit.  The discriminator has one
    output per label of an image."""
    import copy
    n, size, z = data[0].shape[0], data[0].shape[-1], data[1].shape[1]
    results = {}
    for graph in (True, False):
        Gc, Dc = copy.deepcopy(G), copy.deepcopy(D)
        bG = b.Net(ctx, gs, (z,), max_batch=n, precision=b.FP32)
        bD = b.Net(ctx, ds, (3, size, size), max_batch=2 * n, precision=b.FP32, bn_groups=2)
        assert bD.out_elems == labels[0][0].size
        push_params(Gc, bG); push_params(Dc, bD)
        gan = b.Gan(bG, bD, use_cuda_graph=graph)
        ls = []
        for it in range(3):
            r = o.gan_step(Gc, Dc, *data[:3], *labels)
            lo = gan.step(*data)
            ls.append(lo)
            want = np.array([r["loss_d_real"], r["loss_d_fake"], r["loss_g"]])
            assert np.all(np.abs(lo - want) < tol * np.maximum(1, np.abs(want))), (what, graph, it, lo, want)
            assert pclose(bD.params(), Dc.params_flat(), 2 * lr), (what, it, "D", rel_err(bD.params(), Dc.params_flat()))
            assert pclose(bG.params(), Gc.params_flat(), 2 * lr), (what, it, "G", rel_err(bG.params(), Gc.params_flat()))
        results[graph] = (np.array(ls), bG.params(), bD.params())
        gan.close(); bG.close(); bD.close()
    for u, v in zip(results[True], results[False]):
        assert np.array_equal(u, v), "graph replay == eager"


def bf16_round(a):
    """fp32 -> bf16 -> fp32 with round-to-nearest-even, the rounding of the kernels' __float2bfloat16_rn."""
    import torch
    return torch.tensor(np.asarray(a, np.float32)).to(torch.bfloat16).to(torch.float32).numpy()


def check_bf16(got, ref, what):
    """A bf16 tensor against its float64 reference: |got - ref| <= 2^-8 |ref| + 2e-3 rms(ref) elementwise (one bf16 rounding is 2^-9
    relative; the rms term absorbs fp32 accumulation order on elements that cancel).  A non-finite element of got fails."""
    got = np.asarray(got, np.float64); ref = np.asarray(ref, np.float64)
    tol = 2.0 ** -8 * np.abs(ref) + 2e-3 * np.sqrt(np.mean(ref ** 2)) + 1e-30
    d = np.abs(got - ref)
    bad = ~(d <= tol)          # NaN compares False: a NaN or inf in got (or ref) is an error, not a pass
    if bad.any():
        fin = np.isfinite(d)
        worst = d[fin].max() if fin.any() else float("nan")
        raise AssertionError(f"{what}: {bad.sum()} of {bad.size} elements outside 2^-8|ref| + 2e-3 rms ({(~np.isfinite(got)).sum()} non-finite); "
                             f"worst finite |d|={worst:.4g} rms={np.sqrt(np.mean(ref ** 2)):.4g}")


def inject_forward(onet, bnet, specs, x_in, batch, what):
    """Runs the oracle net layer by layer, each layer on the GPU's activation of the layer below; checks every produced tensor (check_bf16).
    The oracle's layer caches are left holding the injected activations, so its backward is the exact backward from the GPU's forward."""
    cur = np.asarray(x_in, np.float32)
    shape = cur.shape
    i = 0
    while i < len(specs):
        t = specs[i]["type"]; l = onet.layers[i]
        fused = t == "batchnorm" and i + 1 < len(specs) and specs[i + 1]["type"] == "activation"
        ref = l.forward(cur.reshape(shape), True)
        if fused:       # the engine stores BatchNorm+activation as one tensor
            ref = onet.layers[i + 1].forward(ref, True)
        shape = ref.shape
        if t in ("conv2d", "deconv2d", "dense", "batchnorm", "output"):
            got = bnet.activation(i, batch).reshape(shape)
            if t == "output":
                got_cmp, ref_cmp = got, l._z.reshape(shape)          # the engine keeps the logits; the oracle's forward returns sigmoid(z)
            else:
                got_cmp, ref_cmp = got, ref
            check_bf16(got_cmp, ref_cmp, f"{what} layer {i} ({specs[i].get('name', t)})")
            cur = got                                                 # inject the GPU's tensor into the next layer
            if t == "output":
                l._z = got.reshape(l._z.shape).astype(l._z.dtype)
        else:
            cur = ref
        i += 2 if fused else 1
    return cur.reshape(shape)


def w_internal(spec, w_dl4j):
    """A GEMM layer's W from DL4J's flattened view to the engine's internal order (o.internal_w; dense 'f'-order [nIn,nOut] already is
    [nOut][nIn])."""
    w = np.asarray(w_dl4j).ravel()
    if spec["type"] in ("dense", "output"):
        return w
    a, b = (spec["n_out"], spec["n_in"]) if spec["type"] == "conv2d" else (spec["n_in"], spec["n_out"])
    return o.internal_w(w.reshape((a, b) + tuple(spec.get("kernel", (1, 1)))))


def pack_deconv_ps(w):
    """The 4x4 stride-2 pad-1 transposed conv onto C <= 4 channels as a 3x3 conv over 2x2 output blocks.  w: [O][4][4][C] (O = input
    channels of the transposed conv).  Output pixel y = 2Y + py receives input row i = Y + dyr (dyr in -1..1) through filter row
    r = y + 1 - 2i = py + 1 - 2*dyr (no tap where r is outside [0, 4)); columns likewise.  Returns the flat operand
    [(py, px, c)][(dyr, dxc)][O] with c padded to 4 channels (zeros)."""
    w = np.asarray(w)
    O, C = w.shape[0], w.shape[3]
    assert w.shape[1:3] == (4, 4) and 1 <= C <= 4
    out = np.zeros((2, 2, 4, 3, 3, O), w.dtype)
    for py in range(2):
        for dyr in (-1, 0, 1):
            r = py + 1 - 2 * dyr
            if not 0 <= r < 4:
                continue
            for px in range(2):
                for dxc in (-1, 0, 1):
                    s = px + 1 - 2 * dxc
                    if 0 <= s < 4:
                        out[py, px, :C, dyr + 1, dxc + 1, :] = w[:, r, s, :].T
    return out.ravel()


def _ps_operand_O(spec):
    """O of the [O][4][4][C] weight when the layer's conv-equivalent is a 4x4 s2 p1 conv with C <= 4 image channels and O % 64 == 0 (the
    transposed conv onto the image, and the input gradient of the conv that reads it), else 0."""
    if tuple(spec.get("kernel", ())) != (4, 4) or tuple(spec.get("stride", ())) != (2, 2) or tuple(spec.get("padding", ())) != (1, 1):
        return 0
    O, C = (spec["n_in"], spec["n_out"]) if spec["type"] == "deconv2d" else (spec["n_out"], spec["n_in"])
    return O if C <= 4 and O % 64 == 0 else 0


def weight_operands(net, specs):
    """Every bf16 weight operand of a BF16 net, widened to fp32: {(layer name, which): operand}, which 0 the straight copy of W and 1 the
    packed pixel-shuffle operand of a layer that has one (Net.weight_operand)."""
    out = {}
    for li, s in enumerate(specs):
        if s["type"] not in ("conv2d", "deconv2d", "dense", "output"):
            continue
        k = s.get("kernel", (1, 1))
        out[(s["name"], 0)] = net.weight_operand(li, 0, s["n_in"] * s["n_out"] * k[0] * k[1])
        if _ps_operand_O(s):
            out[(s["name"], 1)] = net.weight_operand(li, 1, 144 * _ps_operand_O(s))
    return out


def check_weight_operands(b, net, specs, what):
    """The bf16 weight operands a BF16 net's forward reads instead of the fp32 master: every GEMM layer's straight copy of W, and the packed
    pixel-shuffle operand of a layer that has one, equal the master rounded to nearest even, bit for bit; a layer without one refuses the
    request with B2G_ERR_UNSUPPORTED (-6).  Returns how many packed operands were checked."""
    packed = 0
    for li, s in enumerate(specs):
        if s["type"] not in ("conv2d", "deconv2d", "dense", "output"):
            continue
        k = s.get("kernel", (1, 1)); size = s["n_in"] * s["n_out"] * k[0] * k[1]
        w = bf16_round(w_internal(s, net.get_param(s["name"], "W", size)))
        assert np.array_equal(net.weight_operand(li, 0, size), w), f"{what}: bf16 copy of {s['name']}.W differs from the rounded master"
        O = _ps_operand_O(s)
        if O:
            got = net.weight_operand(li, 1, 144 * O)
            assert np.array_equal(got, pack_deconv_ps(w.reshape(O, 4, 4, -1))), f"{what}: packed pixel-shuffle operand of {s['name']}"
            packed += 1
        else:
            with pytest.raises(b.B200GanError) as e:
                net.weight_operand(li, 1, 144)
            assert e.value.code == -6
    return packed
