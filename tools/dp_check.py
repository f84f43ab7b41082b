"""Multi-GPU checks, run under torchrun on N GPUs:  python -m torch.distributed.run --nproc-per-node N tools/dp_check.py OUT.json [CHECK]
CHECK is one of CHECKS below (default core); each is a function that returns what rank 0 writes to OUT.json.  The GPU tests run them under
torchrun on two ranks when the machine has >= 2 GPUs: core from tests/test_gpu_dp.py, the others from the test file of their feature."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import torch.distributed as dist

import gan_deeplearning4j_b200 as b
from gan_deeplearning4j_b200 import models as m, parallel
from oracle.dl4j_oracle import dropout_mask  # noqa: E402  (the oracle's NumPy restatement of the mask)

rank, world, local = parallel.env_rank_world()


def replicated_data(n, z, d):
    """The same MLP-GAN data on every rank: x_real, z_d, z_g and the three label columns."""
    rng = np.random.default_rng(7)
    return [rng.uniform(-1, 1, (n, d)), rng.uniform(-1, 1, (n, z)), rng.uniform(-1, 1, (n, z)),
            1 + 0.05 * rng.standard_normal((n, 1)), 0.05 * rng.standard_normal((n, 1)), np.ones((n, 1))]


def gather(vec):
    """Every rank's vec, as a list of NumPy arrays in rank order."""
    t = torch.tensor(vec, device=f"cuda:{local}")
    allv = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(allv, t)
    return [v.cpu().numpy() for v in allv]


def core(ctx):
    """  1. NCCL all-reduce through the C-ABI communicator,
  2. replicated data on every rank  ==> the DP step equals the single-GPU step (gradient mean over ranks = the gradient),
  3. different data per rank        ==> all ranks hold bit-identical parameters after every step,
  4. the reference's parameter averaging (params + updater state) through b2g_net_average_parameters,
  5. sync_bn: W ranks x N/W images with pooled BatchNorm statistics == 1 GPU x N images (SURVEY.md 8e),
  6. the bf16 gradient payload and the overlapped two-bucket all-reduce (B2G_AR_OVERLAP=1 in the environment) keep ranks identical."""
    out = {"world": world}
    a = ctx.allreduce_test(np.full(1000, rank + 1.0, np.float32))
    assert np.allclose(a, world * (world + 1) / 2), a[:3]
    out["allreduce"] = "ok"

    def make(seed_shift, prec):
        n, size, z, nf = 16, 32, 16, 64
        gs, ds = m.dcgan_generator(size, z, nf, 3, lr=1e-3), m.dcgan_discriminator(size, nf, 3, lr=1e-3)
        G = b.Net(ctx, gs, (z,), max_batch=n, precision=prec, xent_clip_eps=0.0, seed=1)
        D = b.Net(ctx, ds, (3, size, size), max_batch=2 * n, precision=prec, xent_clip_eps=0.0, bn_groups=2, seed=2)
        if os.environ.get("B2G_P2P_AR", "1") != "0":        # collective: gradient all-reduce as one peer-memory kernel (CUDA IPC), else ncclAllReduce
            ok = [D.enable_p2p_allreduce(), G.enable_p2p_allreduce()]
            out["allreduce_transport"] = "peer-memory kernel" if all(ok) else "nccl (peer mapping unavailable)"
        else:
            out["allreduce_transport"] = "nccl"
        rng = np.random.default_rng(100 + seed_shift)
        data = [rng.uniform(-1, 1, (n, 3, size, size)), rng.uniform(-1, 1, (n, z)), rng.uniform(-1, 1, (n, z)),
                1 + 0.05 * rng.standard_normal((n, 1)), 0.05 * rng.standard_normal((n, 1)), np.ones((n, 1))]
        return G, D, b.Gan(G, D, use_cuda_graph=False), data

    for prec, name in ((b.FP32, "fp32"), (b.BF16, "bf16")):
        # (2) replicated data
        G, D, gan, data = make(0, prec)
        for _ in range(3):
            l_dp = gan.step(*data)
        pG, pD = G.params(), D.params()
        gan.close(); G.close(); D.close()
        ref_ctx = b.Context(local)            # no communicator: the single-GPU step
        Gs = b.Net(ref_ctx, m.dcgan_generator(32, 16, 64, 3, lr=1e-3), (16,), max_batch=16, precision=prec, xent_clip_eps=0.0, seed=1)
        Ds = b.Net(ref_ctx, m.dcgan_discriminator(32, 64, 3, lr=1e-3), (3, 32, 32), max_batch=32, precision=prec, xent_clip_eps=0.0, bn_groups=2, seed=2)
        gs_ = b.Gan(Gs, Ds, use_cuda_graph=False)
        for _ in range(3):
            l_1 = gs_.step(*data)
        tol = 2e-3 if prec == b.FP32 else 5e-2
        dG = np.abs(pG - Gs.params()).max(); dD = np.abs(pD - Ds.params()).max()
        out[f"replicated_{name}"] = {"max_abs_dG": float(dG), "max_abs_dD": float(dD), "loss_dp": l_dp.tolist(), "loss_1gpu": l_1.tolist()}
        assert np.allclose(l_dp, l_1, atol=tol), (l_dp, l_1)
        assert dG < 3.1e-3 and dD < 3.1e-3, (dG, dD)      # Adam steps are ~lr=1e-3 each: sign-level agreement after 3 steps
        gs_.close(); Gs.close(); Ds.close(); ref_ctx.close()
        # (3) different data per rank: parameters stay bit-identical across ranks
        G, D, gan, data = make(1 + rank, prec)
        for _ in range(3):
            gan.step(*data)
        for net, tag in ((G, "G"), (D, "D")):
            p = torch.from_numpy(net.params()).cuda()
            lo, hi = p.clone(), p.clone()
            dist.all_reduce(lo, op=dist.ReduceOp.MIN); dist.all_reduce(hi, op=dist.ReduceOp.MAX)
            out[f"sharded_{name}_{tag}_identical"] = bool(torch.equal(lo, hi))
            assert torch.equal(lo, hi), tag
        gan.close(); G.close(); D.close()
    # (4) the reference's own rule: local fits, then parameters AND updater state averaged over ranks (J:325-330)
    dspec = m.dcgan_discriminator(32, 64, 3, lr=1e-3)
    net = b.Net(ctx, dspec, (3, 32, 32), max_batch=16, precision=b.FP32, xent_clip_eps=0.0, seed=2)
    net.set_grad_allreduce(False)
    rng = np.random.default_rng(500 + rank)
    net.fit(rng.uniform(-1, 1, (16, 3, 32, 32)), rng.uniform(0, 1, (16, 1)))
    before = torch.from_numpy(np.concatenate([net.params(), net.updater_state()])).cuda()
    mean = before.clone(); dist.all_reduce(mean, op=dist.ReduceOp.SUM); mean /= world
    net.average_parameters()
    after = np.concatenate([net.params(), net.updater_state()])
    err = float(np.abs(after - mean.cpu().numpy()).max())
    out["parameter_averaging_max_abs_err"] = err
    assert err < 1e-6, err
    net.close()
    # (5) sync_bn: the global batch of W*n images, rank r holding slice r, must train like one GPU holding all of it (BF16: the fused BatchNorm path)
    n, size, z, nf = 16, 32, 16, 64
    gs, ds = m.dcgan_generator(size, z, nf, 3, lr=1e-3), m.dcgan_discriminator(size, nf, 3, lr=1e-3)
    rng = np.random.default_rng(900)
    NG = n * world
    full = [rng.uniform(-1, 1, (NG, 3, size, size)), rng.uniform(-1, 1, (NG, z)), rng.uniform(-1, 1, (NG, z)), 1 + 0.05 * rng.standard_normal((NG, 1)), 0.05 * rng.standard_normal((NG, 1)), np.ones((NG, 1))]
    mine = [a[rank * n:(rank + 1) * n] for a in full]
    G = b.Net(ctx, gs, (z,), max_batch=n, precision=b.BF16, xent_clip_eps=0.0, seed=1); D = b.Net(ctx, ds, (3, size, size), max_batch=2 * n, precision=b.BF16, xent_clip_eps=0.0, bn_groups=2, seed=2)
    G.set_sync_bn(True); D.set_sync_bn(True)
    gan = b.Gan(G, D, use_cuda_graph=False)
    for _ in range(2):
        l_sync = gan.step(*mine)
    pG, pD = G.params(), D.params()
    gan.close(); G.close(); D.close()
    one = b.Context(local)
    G1 = b.Net(one, gs, (z,), max_batch=NG, precision=b.BF16, xent_clip_eps=0.0, seed=1); D1 = b.Net(one, ds, (3, size, size), max_batch=2 * NG, precision=b.BF16, xent_clip_eps=0.0, bn_groups=2, seed=2)
    g1 = b.Gan(G1, D1, use_cuda_graph=False)
    for _ in range(2):
        l_one = g1.step(*full)
    dG = float(np.abs(pG - G1.params()).max()); dD = float(np.abs(pD - D1.params()).max())
    mG = float(np.abs(pG - G1.params()).mean()); mD = float(np.abs(pD - D1.params()).mean())
    lg = torch.tensor(np.asarray(l_sync, np.float64)).cuda(); dist.all_reduce(lg, op=dist.ReduceOp.SUM); lg = (lg / world).cpu().numpy()
    out["sync_bn"] = {"max_abs_dG": dG, "max_abs_dD": dD, "mean_abs_dG": mG, "mean_abs_dD": mD, "loss_mean_over_ranks": lg.tolist(), "loss_1gpu_full_batch": np.asarray(l_one).tolist()}
    # two Adam steps of lr 1e-3 (early Adam moves every weight by ~lr*sign(g)): an element whose gradient is numerically zero may flip sign in both
    # steps (2 x 2*lr); everything else agrees to round-off, so the MEAN difference is orders of magnitude below one step
    assert dG < 4.5e-3 and dD < 4.5e-3 and mG < 5e-5 and mD < 5e-5, (dG, dD, mG, mD)
    assert np.allclose(lg, l_one, atol=3e-2), (lg, l_one)
    g1.close(); G1.close(); D1.close(); one.close()
    # (6) bf16 gradient payload: ranks stay identical, result close to the fp32 payload
    G, D, gan, data = make(1 + rank, b.BF16)
    G.set_grad_payload_bf16(True); D.set_grad_payload_bf16(True)
    for _ in range(3):
        gan.step(*data)
    for net, tag in ((G, "G"), (D, "D")):
        p = torch.from_numpy(net.params()).cuda(); lo, hi = p.clone(), p.clone()
        dist.all_reduce(lo, op=dist.ReduceOp.MIN); dist.all_reduce(hi, op=dist.ReduceOp.MAX)
        out[f"bf16_payload_{tag}_identical"] = bool(torch.equal(lo, hi)); assert torch.equal(lo, hi), tag
    gan.close(); G.close(); D.close()
    out["ar_overlap_env"] = os.environ.get("B2G_AR_OVERLAP", "0")
    return out


def updater(ctx):
    """Parameter averaging of the three-slot updater state: every rank fits its own copy of an FP32 MLP whose layers use AMSGrad (three state
    slots), Nadam and AdaGrad on its own data with the gradient all-reduce switched off (ParameterAveragingTrainingMaster mode), then
    b2g_net_average_parameters averages the parameters and every state slot on the device.  Checked against the mean of what the ranks held
    before."""
    specs = [{"type": "dense", "name": "d1", "n_out": 96, "activation": "tanh", "updater": m.amsgrad(2e-3)},
             {"type": "dense", "name": "d2", "n_out": 64, "activation": "lrelu", "alpha": 0.2, "updater": m.nadam(1e-3)},
             {"type": "output", "name": "out", "n_out": 1, "updater": m.adagrad(0.02)}]
    net = b.Net(ctx, specs, (40,), max_batch=16, precision=b.FP32, seed=3)
    net.set_grad_allreduce(False)
    rng = np.random.default_rng(100 + rank)           # different data on every rank
    for _ in range(3):
        net.fit(rng.uniform(-1, 1, (16, 40)), rng.uniform(0, 1, (16, 1)))
    allv = gather(np.concatenate([net.params(), net.updater_state()]).astype(np.float64))
    want = sum(allv) / world
    net.average_parameters()
    after = np.concatenate([net.params(), net.updater_state()]).astype(np.float64)
    n = net.num_params()
    err = np.abs(after - want) / (np.abs(want) + 1e-30)
    res = {"world": world, "state_slots": int(net.updater_state_size() // n), "ranks_differed": bool(np.abs(allv[0] - allv[-1]).max() > 0),
           "max_rel_err_params": float(err[:n].max()), "max_rel_err_slot": [float(err[n * (k + 1):n * (k + 2)].max()) for k in range(3)]}
    net.close()
    return res


def dropout(ctx):
    """Every rank trains the same MLP-GAN with DropoutLayers in D on identical data (CUDA graph replay, gradient all-reduce).  The rank enters
    each mask's counter, so the ranks draw different masks, while the all-reduced gradients keep D's parameters identical across ranks."""
    n, z, hid, d = 128, 128, 256, 128
    G = b.Net(ctx, m.mlp_generator(z, hid, d, lr=1e-3), (z,), max_batch=n, precision=b.BF16, xent_clip_eps=0.0, seed=1)
    ds = m.mlp_discriminator(d, hid, lr=1e-3, dropout=0.5)
    D = b.Net(ctx, ds, (d,), max_batch=2 * n, precision=b.BF16, xent_clip_eps=0.0, bn_groups=2, seed=2)
    gan = b.Gan(G, D, use_cuda_graph=True)
    data = replicated_data(n, z, d)
    for _ in range(3):
        gan.step(*data)
    li = [i for i, s in enumerate(ds) if s["type"] == "dropout"][0]
    act = D.activation(li, n)                 # the generator step's D pass of step 3: pass 5
    mask_ok = bool(np.array_equal(act.reshape(n, hid) != 0, dropout_mask(2, rank, li, 5, n, 1, 1, hid, 0.5).reshape(n, hid)))
    allv = gather(np.concatenate([D.params(), act.ravel()]))
    npar = D.num_params()
    ok = torch.tensor([1.0 if mask_ok else 0.0], device=f"cuda:{local}")
    dist.all_reduce(ok, op=dist.ReduceOp.MIN)
    gan.close(); G.close(); D.close()
    return {"world": world, "d_params_identical": all(np.array_equal(allv[0][:npar], v[:npar]) for v in allv[1:]),
            "dropout_activations_differ": all(not np.array_equal(allv[0][npar:], v[npar:]) for v in allv[1:]), "masks_match_oracle": bool(ok.item() == 1.0)}


def replicated_matches_one_gpu(ctx, g_args, d_args):
    """Every rank trains the same FP32 MLP-GAN, its nets built with the extra Net arguments g_args / d_args, on identical data (gradient
    all-reduce, CUDA graph replay after the first step); this GPU also trains it alone, without a communicator.  The feature must act on the
    all-reduced gradient or update, so the ranks end with identical parameters equal to the single GPU's."""
    n, z, hid, d = 64, 32, 128, 48
    data = replicated_data(n, z, d)

    def train(c):
        G = b.Net(c, m.mlp_generator(z, hid, d, lr=1e-3), (z,), max_batch=n, precision=b.FP32, seed=1, **g_args)
        D = b.Net(c, m.mlp_discriminator(d, hid, lr=1e-3), (d,), max_batch=2 * n, precision=b.FP32, bn_groups=2, seed=2, **d_args)
        gan = b.Gan(G, D, use_cuda_graph=True)
        for _ in range(3):
            gan.step(*data)
        out = np.concatenate([G.params(), D.params()])
        gan.close(); G.close(); D.close()
        return out

    one = b.Context(local)
    single = train(one)
    one.close()
    mine = train(ctx)
    allv = gather(mine)
    return {"world": world, "params_identical_across_ranks": all(np.array_equal(allv[0], v) for v in allv[1:]),
            "max_rel_err_vs_one_gpu": float(np.abs(mine - single).max() / np.abs(single).max()), "moved": float(np.abs(mine).max())}


def gradnorm(ctx):
    """RenormalizeL2PerLayer on G and ClipL2PerParamType on D: the norms are taken on the all-reduced gradient, so the ranks derive the same
    multipliers."""
    return replicated_matches_one_gpu(ctx, dict(gradient_normalization="renormalize_l2_per_layer"),
                                      dict(gradient_normalization="clip_l2_per_param_type", gradient_normalization_threshold=0.05))


def constraint(ctx):
    """MaxNorm on every W: whole-tensor groups on G (one-pass and two-launch contiguous paths) and groups over nOut on D (dims {1}: strided
    groups, two launches).  The constraints act on the all-reduced update."""
    return replicated_matches_one_gpu(ctx, dict(constraints=[m.max_norm(2.0, ())]), dict(constraints=[m.max_norm(0.5, (1,))]))


def noise(ctx):
    """The dropout check with the other IDropout kinds: an Exponential-scheduled GaussianNoise on D's input and GaussianDropout and
    AlphaDropout after its hidden LeakyReLUs.  The ranks draw different noise (the rank enters the counter), the all-reduced gradients keep D's
    parameters identical, and every rank evaluates the same scheduled value."""
    n, z, hid, d = 128, 128, 256, 128
    G = b.Net(ctx, m.mlp_generator(z, hid, d, lr=1e-3), (z,), max_batch=n, precision=b.BF16, xent_clip_eps=0.0, seed=1)
    ds = m.mlp_discriminator(d, hid, lr=1e-3, instance_noise=m.exponential_schedule(0.2, 0.9))
    ds = ds[:2] + [m.gaussian_dropout(0.3, "gd")] + ds[2:3] + [m.alpha_dropout(0.9, "ad")] + ds[3:]
    D = b.Net(ctx, ds, (d,), max_batch=2 * n, precision=b.BF16, xent_clip_eps=0.0, bn_groups=2, seed=2)
    gan = b.Gan(G, D, use_cuda_graph=True)
    data = replicated_data(n, z, d)
    for _ in range(3):
        gan.step(*data)
    acts = np.concatenate([D.activation(i, n).ravel() for i, s in enumerate(ds) if s["type"] == "dropout"])
    allv = gather(np.concatenate([D.params(), [D.dropout_value("dis_instance_noise")], acts]))
    npar = D.num_params()
    gan.close(); G.close(); D.close()
    return {"world": world, "d_params_identical": all(np.array_equal(allv[0][:npar + 1], v[:npar + 1]) for v in allv[1:]),
            "noise_differs": all(not np.array_equal(allv[0][npar + 1:], v[npar + 1:]) for v in allv[1:]),
            "scheduled_value": float(allv[0][npar])}


def regularization(ctx):
    """l1, l2, l1Bias and l2Bias on every layer of G and D (the global builder's): the terms act on the all-reduced update, on parameters the
    ranks hold identically."""
    reg = dict(regularization={"l1": 1e-3, "l2": 1e-2, "l1_bias": 5e-4, "l2_bias": 5e-3})
    return replicated_matches_one_gpu(ctx, reg, reg)


CHECKS = {"core": core, "updater": updater, "dropout": dropout, "noise": noise, "gradnorm": gradnorm, "constraint": constraint,
          "regularization": regularization}


def main():
    out_json, check = sys.argv[1], sys.argv[2] if len(sys.argv) > 2 else "core"
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    ctx = b.Context(local)
    parallel.attach_communicator(ctx, dist, rank, world)
    res = CHECKS[check](ctx)
    if rank == 0:
        with open(out_json, "w") as f:
            json.dump(res, f, indent=1)
        print(f"dp_check {check} ok", json.dumps(res)[:600])
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
