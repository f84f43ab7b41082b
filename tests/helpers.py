"""Test-only glue: build the oracle's Net from the same layer specs the CUDA engine consumes."""
import numpy as np

from oracle import dl4j_oracle as o


def _upd(u):
    if u is None:
        return None
    if u["kind"] == "rmsprop":
        return o.RmsProp(u["lr"], u.get("rms_decay", 0.95), u.get("eps", 1e-8))
    if u["kind"] == "adam":
        return o.Adam(u["lr"], u.get("beta1", 0.9), u.get("beta2", 0.999), u.get("eps", 1e-8))
    if u["kind"] == "sgd":
        return o.Sgd(u["lr"])
    return o.UpdaterCfg("noop")


def oracle_from_specs(specs, input_shape, grad_clip=0.0, quirks=o.DEFAULT_QUIRKS, dtype=np.float64, seed=1, flat_input=True):
    """input_shape: (C,H,W) or (F,).  flat_input: prepend the convolutionalFlat reshape (index shift +1)."""
    layers = []
    shape = (1,) + tuple(input_shape)
    if len(input_shape) == 3 and flat_input:
        layers.append(o.Reshape(tuple(input_shape), name="in_reshape"))      # convolutionalFlat accepts [N,784] or [N,1,28,28]
    for s in specs:
        t, name = s["type"], s.get("name", "")
        u = _upd(s.get("updater"))
        if t == "conv2d":
            l = o.Conv2D(s.get("n_in") or shape[1], s["n_out"], s["kernel"], s.get("stride", (1, 1)), s.get("padding", (0, 0)), s.get("activation", "identity"), s.get("alpha", 0.01), u, s.get("l2", 0.0), name, s.get("has_bias", True))
        elif t == "deconv2d":
            l = o.Deconv2D(s.get("n_in") or shape[1], s["n_out"], s["kernel"], s.get("stride", (1, 1)), s.get("padding", (0, 0)), s.get("activation", "identity"), s.get("alpha", 0.01), u, s.get("l2", 0.0), name, s.get("has_bias", True))
        elif t == "dense":
            l = o.Dense(s.get("n_in") or shape[1], s["n_out"], s.get("activation", "identity"), s.get("alpha", 0.01), u, s.get("l2", 0.0), name, s.get("has_bias", True))
        elif t == "output":
            l = o.Output(s.get("n_in") or shape[1], s["n_out"], u, s.get("l2", 0.0), name, quirks)
        elif t == "batchnorm":
            l = o.BatchNorm(shape[1], s.get("decay", 0.9), s.get("eps", 1e-5), u, name)
        elif t == "activation":
            l = o.ActivationLayer(s["activation"], s.get("alpha", 0.01), name)
        elif t == "maxpool":
            l = o.MaxPool(s["kernel"], s.get("stride", (1, 1)), name)
        elif t == "upsample2d":
            l = o.Upsample2D(s.get("size", 2), name)
        elif t == "loss":
            l = o.LossLayer(name, quirks)
        elif t == "ff_to_cnn":
            h, w, c = s["to"]; l = o.Reshape((c, h, w), name)
        elif t == "cnn_to_ff":
            l = o.Reshape((int(np.prod(shape[1:])),), name)
        else:
            raise ValueError(t)
        layers.append(l)
        shape = l.out_shape(shape)
    return o.Net(layers, seed=seed, dtype=dtype, grad_clip=grad_clip, quirks=quirks)


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
