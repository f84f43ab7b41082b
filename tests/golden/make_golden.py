"""Generates tests/golden/*.npz from the oracle (oracle/dl4j_oracle.py).  Run from the repo root:  python tests/golden/make_golden.py

The reference holds no golden vectors and cannot run here (SURVEY.md 8c), so these fixtures do not pin the oracle to DL4J; they pin the oracle
-- and, through tests/test_gpu_parity.py, the CUDA path -- to FIXED BYTES across sessions (SURVEY.md 8c "substitute pins" item v):

  gan_step_dcgan16.npz   the adversarial step (oracle gan_step, J:408-471) on a 16x16x3 DCGAN (z=12, nf=8, batch 8; the configuration of
                         test_fp32_gan_step_matches_oracle): inputs, initial parameters, and losses + all parameters after each of 3 steps
  layer_cases.npz        forward / backward of ConvolutionLayer, Deconvolution2D, BatchNormalization (train), DenseLayer on tiny seeded inputs
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))

from helpers import randomize# noqa: E402
from oracle import dl4j_oracle as o  # noqa: E402

GAN_CFG = dict(size=16, z=12, nf=8, n=8, lr=2e-3, clip_eps=1e-5, seed_g=1, seed_d=2, seed_rand=5, seed_data=3, steps=3)


def gan_pair():
    from gan_deeplearning4j_b200 import models as m
    c = GAN_CFG
    gs, ds = m.dcgan_generator(c["size"], c["z"], c["nf"], 3, lr=c["lr"]), m.dcgan_discriminator(c["size"], c["nf"], 3, lr=c["lr"])
    q = o.Quirks(xent_clip_eps=c["clip_eps"]); rng = np.random.default_rng(c["seed_rand"])
    G = o.net_from_specs(gs, (c["z"],), quirks=q, seed=c["seed_g"]); D = o.net_from_specs(ds, (3, c["size"], c["size"]), quirks=q, seed=c["seed_d"])
    randomize(G, rng); randomize(D, rng)
    return gs, ds, G, D


def gan_step_vectors():
    c = GAN_CFG
    gs, ds, G, D = gan_pair()
    data = [a.astype(np.float64) for a in o.synthetic_batch(c["n"], c["size"], 3, c["z"], seed=c["seed_data"])]
    out = {"x_real": data[0], "z_d": data[1], "z_g": data[2], "y_real": data[3], "y_fake": data[4], "y_gen": data[5],
           "g_params0": G.params_flat(), "d_params0": D.params_flat()}
    for it in range(c["steps"]):
        r = o.gan_step(G, D, *data)
        out[f"losses{it + 1}"] = np.array([r["loss_d_real"], r["loss_d_fake"], r["loss_g"]])
        out[f"g_params{it + 1}"] = G.params_flat(); out[f"d_params{it + 1}"] = D.params_flat()
    return out


def layer_vectors():
    rng = np.random.default_rng(11); out = {}
    def run(tag, layer, x):
        layer.init(np.random.default_rng(7), np.float64)
        for p in layer.params:
            layer.params[p] = layer.params[p] + 0.1 * rng.standard_normal(layer.params[p].shape) if p != "var" else layer.params[p] * (1 + 0.3 * rng.random(layer.params[p].shape))
        y = layer.forward(x, True); eps = rng.standard_normal(y.shape); dx = layer.backward(eps)
        out.update({f"{tag}_x": x, f"{tag}_y": y, f"{tag}_eps": eps, f"{tag}_dx": dx})
        for p in layer.params:
            out[f"{tag}_param_{p}"] = layer.params[p]; out[f"{tag}_grad_{p}"] = layer.grads[p]
    run("conv", o.Conv2D(3, 4, (4, 4), (2, 2), (1, 1), activation="lrelu", alpha=0.2), rng.standard_normal((2, 3, 8, 8)))
    run("deconv", o.Deconv2D(4, 3, (4, 4), (2, 2), (1, 1), activation="tanh"), rng.standard_normal((2, 4, 4, 4)))
    run("bn", o.BatchNorm(5), rng.standard_normal((3, 5, 4, 4)))
    run("dense", o.Dense(6, 4, activation="sigmoid"), rng.standard_normal((5, 6)))
    return out


if __name__ == "__main__":
    np.savez_compressed(os.path.join(HERE, "gan_step_dcgan16.npz"), **gan_step_vectors())
    np.savez_compressed(os.path.join(HERE, "layer_cases.npz"), **layer_vectors())
    for f in ("gan_step_dcgan16.npz", "layer_cases.npz"):
        print(f, os.path.getsize(os.path.join(HERE, f)), "bytes")
