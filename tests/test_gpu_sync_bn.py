"""Cross-replica (sync) BatchNorm on one GPU: the 128-bit accumulator kernels with replicas = R > 1, as R data-parallel ranks run them
(b2g_test_bn_ex): each replica's statistics kernel on its own rows, the replicas' accumulator words summed as uint64 modulo 2^64 (what the
ncclUint64 sum all-reduce does), every replica's apply kernel on the sum with replicas = R, and the backward the same way.
  - against float64: oracle.dl4j_oracle.BatchNorm over each group's R x rows rows (the replicas concatenated) with the fused activation after
    it (test_gpu_batchnorm._reference), on paths 1 and 2; gamma / beta gradients = the initial value + (global sum) / R, which the gradient
    all-reduce sums back to the global gradient.  Edges: one row per replica (each rank's own variance is 0, the global one is not), channels
    whose replicas' sums cancel exactly (the all-reduced words wrap through zero), and row counts ragged against the statistics kernels' chunks.
  - bit for bit, forward: R replicas of `rows` rows == one replica of the R x rows rows.  On the grid x = k * 2^-6, |k| <= 2^8, every
    per-thread double sum of x and x^2 is exact, and so is each sacc_add split of a partial (r a multiple of 2^-12, lo a multiple of 2^48 with
    |lo| <= 2^49), so sacc_read returns the exact sums however the rows are partitioned, up to 2^20 rows.  The backward's per-thread sums
    are fp32 (bn_bwd_stats_acc_kernel), so the backward is held to the float64 bounds only.
  - every replica holds the same coefficient and parameter-gradient bits, and replicas = 1 equals b2g_test_bn bit for bit.
Tolerances are test_gpu_batchnorm's: y / eps_in by helpers.check_bf16, mean / invstd / the four parameter gradients within 1e-5 relative;
gamma / beta gradients also within the rounding bound of the backward's fp32 per-lane sums (_param_grad_rounding).
"""
import numpy as np
import pytest

import test_gpu_batchnorm as bn
from helpers import b200, bf16_round, check_bf16

pytestmark = pytest.mark.gpu

ALPHA = bn.ALPHA
EPS, DECAY = 1e-5, 0.9
U = 2.0 ** -24          # fp32 unit roundoff

# (C, rows per replica, groups, replicas R, activation, |mean|/std, zero-mean).  zero-mean: replicas R/2..R-1 hold the negation of replicas
# 0..R/2-1, so every channel's global sum is exactly 0 and the replicas' partial sums have opposite signs.
CASES = [
    (8, 64, 2, 2, "relu", 100, False), (8, 1, 1, 8, "identity", 10, False), (8, 4096, 2, 4, "lrelu", 100, False), (8, 5, 2, 4, "sigmoid", 0, True),
    (64, 5, 2, 3, "tanh", 100, False), (64, 1, 2, 4, "relu", 0, False), (64, 3000, 1, 8, "sigmoid", 10, False), (64, 64, 2, 2, "identity", 0, True),
    (512, 64, 2, 8, "identity", 100, False), (512, 5, 1, 2, "lrelu", 10, False), (512, 1, 2, 3, "tanh", 10, False), (512, 3, 1, 8, "relu", 0, True),
    (2048, 5, 2, 4, "relu", 10, False), (2048, 64, 1, 3, "lrelu", 100, False), (2048, 1, 2, 2, "sigmoid", 0, False), (2048, 5, 2, 2, "tanh", 0, True),
]
RUNS = [(c, p) for c in CASES for p in (1, 2)]


def _replica_inputs(C, rows, groups, R, ratio, zero_mean, seed):
    """test_gpu_batchnorm._inputs over the R x rows rows of each group, bf16-rounded, split into replicas: x, e [R, groups, rows, C]"""
    if zero_mean:
        x, e, par, g0 = bn._inputs(C, R // 2 * rows, groups, ratio, seed)
        x = np.concatenate([x, -x], axis=1)
        e = np.concatenate([e, bn._inputs(C, R // 2 * rows, groups, ratio, seed + 1)[1]], axis=1)
    else:
        x, e, par, g0 = bn._inputs(C, R * rows, groups, ratio, seed)
    split = lambda a: np.ascontiguousarray(bf16_round(a).reshape(groups, R, rows, C).transpose(1, 0, 2, 3))
    return split(x), split(e), par, g0


def _concat(a):
    """[R, groups, rows, ...] -> [groups, R * rows, ...]: each group's rows, replica after replica"""
    R, groups, rows = a.shape[:3]
    return a.transpose(1, 0, 2, *range(3, a.ndim)).reshape(groups, R * rows, *a.shape[3:])


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _premul(x, e, par, act):
    """path 2's eps_out: dy' = eps * act'(z) from the float64 pre-activation over the global batch, rounded like the GEMM output"""
    xc = _concat(x).astype(np.float64)
    zr = (xc - xc.mean(1, keepdims=True)) / np.sqrt(xc.var(1, keepdims=True) + EPS) * par["gamma"] + par["beta"]
    ec = bf16_round(_concat(e) * bn.act_grad(act, zr, bn.act_fwd(act, zr)))
    R, groups, rows, C = x.shape
    return np.ascontiguousarray(ec.reshape(groups, R, rows, C).transpose(1, 0, 2, 3))


@pytest.mark.parametrize("case,path", RUNS, ids=[f"C{c[0]}-rows{c[1]}-g{c[2]}-R{c[3]}-{c[4]}-off{c[5]}{'-zero' if c[6] else ''}-path{p}" for c, p in RUNS])
def test_sync_batchnorm_matches_float64_over_all_replicas(b200, case, path):
    b, ctx = b200
    C, rows, groups, R, act, ratio, zero_mean = case
    x, e, par, g0 = _replica_inputs(C, rows, groups, R, ratio, zero_mean, seed=C * 1000 + rows * 10 + R)
    if path == 2:
        e = _premul(x, e, par, act)
    got = b.test_bn(ctx, b.BF16, path, x, e, par["gamma"], par["beta"], par["run_mean"], par["run_var"], act=act, alpha=ALPHA, eps=EPS, decay=DECAY,
                    g_gamma=g0["g_gamma"], g_beta=g0["g_beta"], replicas=R)
    what = f"C={C} rows={rows} groups={groups} R={R} {act} |m|/s={ratio}{' zero-mean' if zero_mean else ''} path {path}"
    # every replica derives its coefficients and parameter gradients from the same summed words: the same bits on every replica
    for k in ("mean", "invstd", "g_gamma", "g_beta", "g_mean", "g_var"):
        for r in range(1, R):
            assert np.array_equal(_bits(got[k][r]), _bits(got[k][0])), f"{what}: replica {r}'s {k} differs from replica 0's"
    zero = {k: np.zeros(C, np.float32) for k in g0}
    ref = bn._reference(_concat(x).astype(np.float64), _concat(e).astype(np.float64), par, zero, act, EPS, DECAY, path == 2, _concat(got["y"]))
    for k in ("y", "eps_in"):
        check_bf16(_concat(got[k]), ref[k], f"{what}: {k}")
    rel = np.abs(got["invstd"][0] - ref["invstd"]) / ref["invstd"]
    assert rel.max() <= 1e-5, f"{what}: invstd relative error {rel.max():.3g} (channel {np.unravel_index(rel.argmax(), rel.shape)})"
    # the batch mean relative to the largest mean, or to the largest std where the means cancel to 0 (zero-mean: float64 leaves ~1e-17 there)
    err = np.abs(got["mean"][0] - ref["mean"]).max() / max(np.abs(ref["mean"]).max(), (1.0 / ref["invstd"]).max())
    assert err <= 1e-5, f"{what}: mean error {err:.3g}"
    if zero_mean:
        assert np.all(got["mean"][0] == 0.0), f"{what}: the replicas' sums cancel exactly, the mean is {np.abs(got['mean'][0]).max():.3g}"
    # each rank keeps (global sum) / R; the gradient all-reduce adds the R copies back to the global gradient
    ref["g_gamma"] = g0["g_gamma"] + ref["g_gamma"] / R
    ref["g_beta"] = g0["g_beta"] + ref["g_beta"] / R
    for k in ("g_mean", "g_var"):
        err = np.abs(got[k][0] - ref[k]).max() / (np.abs(ref[k]).max() + 1e-30)
        assert err <= 1e-5, f"{what}: {k} relative error {err:.3g}"
    bound = _param_grad_rounding(x, e, ref["mean"], ref["invstd"], path)
    for k in ("g_gamma", "g_beta"):
        d = np.abs(got[k][0] - ref[k])
        tol = 1e-5 * np.abs(ref[k]).max() + bound[k] / R
        assert (d <= tol).all(), f"{what}: {k} error {d.max():.3g} (relative {d.max() / np.abs(ref[k]).max():.3g}), {np.max(d / tol):.3g} x the bound"


def _param_grad_rounding(x, e, mean, invstd, path):
    """Per channel, the rounding bound of the backward's fp32 per-lane sums (bn_bwd_stats_acc_kernel) on the global gamma / beta gradient sums.
    A lane adds L = ceil(chunk / TY) terms in fp32 (chunk = ceil(rows / S), S = clamp(rows / (4 TY), 1, min(256, 2^20 / C)), TY = 256 / (C/8)
    row lanes), so it is off by at most gamma_L times the sum of the terms' magnitudes (gamma_L = L u / (1 - L u); Higham, Accuracy and Stability,
    eq. 4.4); the lanes fold in double.  |dy'| <= |eps_out| for all five activations.  Path 1 sums dy' * xhat.  Path 2 sums dy' and dy' * z with
    z the raw input, and k_bn_bwd_apply_acc forms invstd (sum dy' z - mean sum dy'): at |mean| / std = 100 that cancels about two digits, so
    the fp32 lane sums, not the 1e-5, bound the gamma gradient (the kernel's arithmetic emulated in numpy at C = 8, 4 x 4096 rows, lrelu
    reproduces the GPU's gamma gradient bit for bit, 3.5e-5 from float64)."""
    R, groups, rows, C = x.shape
    TY = 256 // (C // 8)
    S = max(1, min(rows // (4 * TY), min(256, (1 << 20) // C)))
    L = -(-(-(-rows // S)) // TY)
    gam = L * U / (1 - L * U)
    xc, ec = _concat(x).astype(np.float64), np.abs(_concat(e).astype(np.float64))
    if path == 2:
        mag = invstd * (ec * (np.abs(xc) + np.abs(mean)[:, None, :])).sum(1)
    else:
        mag = (ec * np.abs((xc - mean[:, None, :]) * invstd[:, None, :])).sum(1)
    return {"g_gamma": gam * mag.sum(0), "g_beta": gam * ec.sum(1).sum(0)}


# (C, rows per replica, groups, R, activation).  The statistics kernels split a group's rows into S = clamp(rows / (4 TY), 1, 256) chunks of
# ceil(rows / S) rows (TY = 256 / (C/8) row lanes): in each case the concatenated rows' chunk boundaries are not the replicas' boundaries.
BIT_CASES = [(8, 1000, 2, 3, "lrelu"), (8, 1, 1, 8, "identity"), (64, 300, 1, 8, "tanh"), (64, 4099, 2, 4, "relu"), (512, 37, 2, 4, "sigmoid"),
             (2048, 7, 2, 2, "relu"), (2048, 97, 1, 3, "tanh")]


def _grid_inputs(C, rows, groups, R, seed):
    """x = k * 2^-6 with |k| <= 2^8 (exact in bf16), per-channel centres of both signs up to |k| = 200 so that |mean| >> std on some channels"""
    rng = np.random.default_rng(seed)
    centre = rng.integers(-200, 201, C)
    k = np.clip(centre + rng.integers(-40, 41, (R, groups, rows, C)), -256, 256)
    x = (k * 2.0 ** -6).astype(np.float32)
    assert np.array_equal(bf16_round(x), x)
    e = bf16_round(rng.standard_normal((R, groups, rows, C)))
    s = rng.uniform(0.5, 2.0, C)
    par = dict(gamma=rng.uniform(0.5, 1.5, C), beta=0.3 * rng.standard_normal(C), run_mean=centre * 2.0 ** -6 + 0.1 * rng.standard_normal(C),
               run_var=s * s)
    return x, e, {k: v.astype(np.float32) for k, v in par.items()}


@pytest.mark.parametrize("case", BIT_CASES, ids=[f"C{c[0]}-rows{c[1]}-g{c[2]}-R{c[3]}-{c[4]}" for c in BIT_CASES])
def test_sync_batchnorm_forward_equals_one_replica_bit_for_bit(b200, case):
    """dp_check's W x N/W == 1 x N at kernel level: R replicas of `rows` rows give the bits of one replica over the R x rows rows."""
    b, ctx = b200
    C, rows, groups, R, act = case
    x, e, par = _grid_inputs(C, rows, groups, R, seed=C + rows + R)
    kw = dict(act=act, alpha=ALPHA, eps=EPS, decay=DECAY)
    many = b.test_bn(ctx, b.BF16, 1, x, e, par["gamma"], par["beta"], par["run_mean"], par["run_var"], replicas=R, **kw)
    one = b.test_bn(ctx, b.BF16, 1, _concat(x), _concat(e), par["gamma"], par["beta"], par["run_mean"], par["run_var"], **kw)
    what = f"C={C} rows={rows} groups={groups} R={R} {act}"
    assert np.array_equal(_bits(_concat(many["y"])), _bits(one["y"])), f"{what}: y"
    for r in range(R):
        for k in ("mean", "invstd"):
            assert np.array_equal(_bits(many[k][r]), _bits(one[k])), f"{what}: replica {r}'s {k}"
        for k in ("g_mean", "g_var"):
            assert np.array_equal(_bits(many[k][r]), _bits(one[k])), f"{what}: replica {r}'s {k}"
    # the backward's fp32 per-thread sums depend on the partition (its float64 parity is the test above): R x (global sum / R) against the
    # single replica's sum within the float64 bound
    for k in ("g_gamma", "g_beta"):
        err = np.abs(R * many[k][0].astype(np.float64) - one[k]).max() / (np.abs(one[k]).max() + 1e-30)
        assert err <= 1e-5, f"{what}: R x {k} against one replica's, relative error {err:.3g}"


@pytest.mark.parametrize("path", [1, 2])
@pytest.mark.parametrize("case", [(8, 64, 2, "lrelu", 100), (64, 5, 1, "tanh", 10), (512, 1, 2, "relu", 0), (2048, 37, 2, "sigmoid", 100)],
                         ids=lambda c: f"C{c[0]}-rows{c[1]}-g{c[2]}-{c[3]}-off{c[4]}")
def test_one_replica_equals_b2g_test_bn(b200, case, path):
    """replicas = 1 through the cross-replica hook runs b2g_test_bn's launches: every output the same bits, with and without parameter gradients."""
    b, ctx = b200
    C, rows, groups, act, ratio = case
    x, e, par, g0 = bn._inputs(C, rows, groups, ratio, seed=C + rows)
    x, e = bf16_round(x), bf16_round(e)
    for want in (True, False):
        kw = dict(act=act, alpha=ALPHA, eps=EPS, decay=DECAY, g_gamma=g0["g_gamma"], g_beta=g0["g_beta"], want_param_grads=want)
        ex = b.test_bn(ctx, b.BF16, path, x[None], e[None], par["gamma"], par["beta"], par["run_mean"], par["run_var"], replicas=1, **kw)
        old = b.test_bn(ctx, b.BF16, path, x, e, par["gamma"], par["beta"], par["run_mean"], par["run_var"], **kw)
        for k, v in old.items():
            assert np.array_equal(_bits(ex[k][0]), _bits(v)), f"C={C} rows={rows} path {path} want={want}: {k}"
        if not want:
            assert np.array_equal(ex["g_gamma"][0], g0["g_gamma"]) and np.array_equal(ex["g_beta"][0], g0["g_beta"])


def test_sync_batchnorm_refuses_unsupported_channels(b200):
    """The accumulator kernels exist for C % 8 == 0 and 256 % (C/8) == 0 only: the cross-replica hook refuses anything else (B2G_ERR_UNSUPPORTED)."""
    b, ctx = b200
    for C in (24, 4096):
        x, e, par, _ = _replica_inputs(C, 4, 1, 2, 0, False, seed=5)
        with pytest.raises(b.B200GanError) as err:
            b.test_bn(ctx, b.BF16, 1, x, e, par["gamma"], par["beta"], par["run_mean"], par["run_var"], replicas=2)
        assert err.value.code == -6, C
