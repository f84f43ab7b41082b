"""Test-only utilities for comparing the oracle's nets (oracle.dl4j_oracle.net_from_specs) with the CUDA library's."""
import numpy as np


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


def rel_err(a, b):
    a = np.asarray(a, np.float64).ravel(); b = np.asarray(b, np.float64).ravel()
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


def pclose(got, want, bound, tol=2e-3):
    """Every element within tol of want's largest magnitude; else every element within bound and at most 2% of them beyond tol."""
    d = np.abs(np.asarray(got, np.float64) - np.asarray(want, np.float64))
    if d.max() < tol * np.abs(want).max():
        return True
    return d.max() <= bound and (d > tol * np.abs(want).max()).mean() <= 0.02


def gan_step_parity(b, ctx, gs, ds, G, D, data, labels, lr, what, tol=1e-3):
    """The FP32 adversarial step of the library against the oracle's, on copies of the oracle nets G, D (specs gs, ds): over 3 steps on data
    (x_real, z_d, z_g and per-image labels), oracle gan_step with `labels` and Gan.step agree on the losses within tol and on both nets'
    parameters by pclose at 2 lr, once captured as a CUDA graph and once eager; the two runs agree bit for bit.  The discriminator has one
    output per label of an image."""
    import copy
    from oracle import dl4j_oracle as o
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
    """A GEMM layer's W from DL4J's flattened view to the engine's internal [A][taps][B] order (conv [nOut][kH*kW][nIn], transposed conv
    [nIn][kH*kW][nOut]; dense 'f'-order [nIn,nOut] already is [nOut][nIn])."""
    w = np.asarray(w_dl4j).ravel()
    k = spec.get("kernel", (1, 1))
    taps = k[0] * k[1]
    if spec["type"] in ("dense", "output") or taps == 1:
        return w
    a = spec["n_out"] if spec["type"] == "conv2d" else spec["n_in"]
    return w.reshape(a, -1, taps).transpose(0, 2, 1).ravel()


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
