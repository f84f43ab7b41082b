"""BatchNorm(+activation) kernels of the training step against a float64 reference, one kernel chain at a time (b2g_test_bn):
    path 0  the two-stage kernels (k_bn_stats -> k_bn_apply -> k_bn_bwd), fp32 and bf16, scalar kernels (bf16 apply 16-byte vectorised where C allows);
    path 1  the 128-bit accumulator kernels (k_bn_stats_acc -> k_bn_apply_acc -> k_bn_bwd_stats_acc -> k_bn_bwd_apply_acc);
    path 2  the accumulator kernels fed the way the fused BatchNorm-backward GEMM epilogue feeds them: eps already multiplied by act',
            backward statistics (sum dy', sum dy'*z) converted to (sum dy', sum dy'*xhat) in k_bn_bwd_apply_acc.
The reference is oracle.dl4j_oracle.BatchNorm in float64 on the same (bf16-rounded) inputs, one statistics group at a time, with the fused
activation applied after it; running-statistic pseudo-gradients averaged over groups, gamma / beta gradients summed over groups and added to
the values already in the gradient buffer.  Inputs are offset per channel (x = m + s*N(0,1), |m|/s up to 100, both signs) and one channel is
constant, so a one-pass variance that cancels catastrophically, or a variance clamp that misfires, fails here.
Tolerances: bf16 tensors (y, eps_in) within one bf16 rounding (helpers.check_bf16); fp32 tensors of fp32 nets within 1e-4 rms; mean / invstd /
the four parameter gradients within 1e-5 relative (invstd elementwise, the others relative to the largest element; gamma / beta gradients
of fp32 inputs at |m|/s = 100 within 2e-5, the measured bound of an fp32 batch mean).
"""
import numpy as np
import pytest

from helpers import b200, bf16_round, check_bf16
from oracle import dl4j_oracle as o

pytestmark = pytest.mark.gpu

ALPHA = 0.2


def act_fwd(act, z):
    return {"identity": lambda: z, "relu": lambda: np.maximum(z, 0.0), "lrelu": lambda: np.where(z > 0, z, ALPHA * z),
            "tanh": lambda: np.tanh(z), "sigmoid": lambda: 1.0 / (1.0 + np.exp(-z))}[act]()


def act_grad(act, z, y_gpu):
    """f'(z).  For the piecewise-linear activations the branch is read from the kernel's own output y (same sign as its z): an element whose
    pre-activation lies within fp32 rounding of the kink would otherwise take different branches here and on the GPU."""
    if act == "relu":
        return (y_gpu > 0).astype(np.float64)
    if act == "lrelu":
        return np.where(y_gpu > 0, 1.0, ALPHA)
    if act == "tanh":
        return 1.0 - np.tanh(z) ** 2
    if act == "sigmoid":
        s = 1.0 / (1.0 + np.exp(-z)); return s * (1.0 - s)
    return np.ones_like(z)


# (C, rows per group, groups, activation, |mean|/std).  C = 8 and 2048 are the vector-kernel extremes (256 row lanes / 1 row lane per block);
# C = 3 and 24 are not vector-eligible.  Rows: 1 (fewer rows than lanes), 5 (ragged last chunk), 64, 32768 (the C2 size of D2's BatchNorm).
CASES = [
    (8, 64, 2, "relu", 0), (8, 32768, 2, "lrelu", 100), (8, 5, 1, "sigmoid", 10),
    (64, 32768, 2, "relu", 10), (64, 1, 2, "identity", 0), (64, 5, 2, "tanh", 100),
    (512, 64, 2, "lrelu", 100), (512, 5, 1, "relu", 10),
    (2048, 64, 2, "sigmoid", 100), (2048, 1, 1, "tanh", 10), (2048, 5, 2, "identity", 0),
    (3, 32768, 2, "tanh", 100), (3, 1, 2, "relu", 10), (24, 64, 2, "lrelu", 100), (24, 5, 1, "sigmoid", 0),
]


def _runs():
    out = []
    for case in CASES:
        vec = case[0] % 8 == 0 and 256 % (case[0] // 8) == 0
        out += [(case, "fp32", 0), (case, "bf16", 0)] + ([(case, "bf16", 1), (case, "bf16", 2)] if vec else [])
    return out


RUNS = _runs()


def _inputs(C, rows, groups, ratio, seed):
    rng = np.random.default_rng(seed)
    s = rng.uniform(0.5, 2.0, C)
    m = ratio * s * np.where(np.arange(C) % 2 == 0, 1.0, -1.0)               # offsets of both signs
    x = m + s * rng.standard_normal((groups, rows, C))
    x[:, :, 1 % C] = m[1 % C] + (0.3 if ratio == 0 else 0.0)                  # a constant channel: batch variance 0
    e = rng.standard_normal((groups, rows, C))
    par = dict(gamma=rng.uniform(0.5, 1.5, C), beta=0.3 * rng.standard_normal(C), run_mean=m + 0.5 * s * rng.standard_normal(C),
               run_var=s * s * rng.uniform(0.5, 2.0, C))
    g0 = dict(g_gamma=0.1 * rng.standard_normal(C), g_beta=0.1 * rng.standard_normal(C))
    return x, e, {k: v.astype(np.float32) for k, v in par.items()}, {k: v.astype(np.float32) for k, v in g0.items()}


def _reference(x, e, par, g0, act, eps, decay, premul, y_gpu):
    groups, rows, C = x.shape
    ref = {k: [] for k in ("y", "eps_in", "mean", "invstd")}
    gsum = {k: np.zeros(C) for k in ("gamma", "beta", "mean", "var")}
    for g in range(groups):
        l = o.BatchNorm(C, decay, eps); l.init(np.random.default_rng(0), np.float64)
        for k, pk in (("gamma", "gamma"), ("beta", "beta"), ("mean", "run_mean"), ("var", "run_var")):
            l.params[k] = par[pk].astype(np.float64)
        z = l.forward(x[g], True)
        ref["y"].append(act_fwd(act, z)); ref["mean"].append(l._mu); ref["invstd"].append(1.0 / np.sqrt(l._var + eps))
        dy = e[g] if premul else e[g] * act_grad(act, z, y_gpu[g])
        ref["eps_in"].append(l.backward(dy))
        for k in gsum:
            gsum[k] += l.grads[k]
    ref = {k: np.stack(v) for k, v in ref.items()}
    ref["g_gamma"] = g0["g_gamma"] + gsum["gamma"]; ref["g_beta"] = g0["g_beta"] + gsum["beta"]
    ref["g_mean"] = gsum["mean"] / groups; ref["g_var"] = gsum["var"] / groups
    return ref


@pytest.mark.parametrize("case,prec,path", RUNS, ids=[f"C{c[0]}-rows{c[1]}-g{c[2]}-{c[3]}-off{c[4]}-{p}-path{k}" for c, p, k in RUNS])
def test_batchnorm_kernels_match_float64(b200, case, prec, path):
    b, ctx = b200
    C, rows, groups, act, ratio = case
    eps, decay = 1e-5, 0.9
    x, e, par, g0 = _inputs(C, rows, groups, ratio, seed=C * 1000 + rows + 7 * ratio)
    rnd = bf16_round if prec == "bf16" else (lambda a: np.asarray(a, np.float32))
    x = rnd(x); e = rnd(e)
    if path == 2:
        # the epilogue hands the BatchNorm backward dy' = eps * act'(z): form it from the float64 pre-activation, round like the GEMM output
        zr = np.stack([(x[g] - x[g].astype(np.float64).mean(0)) / np.sqrt(x[g].astype(np.float64).var(0) + eps) * par["gamma"] + par["beta"] for g in range(groups)])
        e = bf16_round(e * act_grad(act, zr, act_fwd(act, zr)))
    P = b.BF16 if prec == "bf16" else b.FP32
    got = b.test_bn(ctx, P, path, x, e, par["gamma"], par["beta"], par["run_mean"], par["run_var"], act=act, alpha=ALPHA, eps=eps, decay=decay,
                    g_gamma=g0["g_gamma"], g_beta=g0["g_beta"])
    ref = _reference(x.astype(np.float64), e.astype(np.float64), par, g0, act, eps, decay, path == 2, got["y"])
    what = f"C={C} rows={rows} groups={groups} {act} |m|/s={ratio} {prec} path {path}"
    if rows == 1:
        # one row per group: batch variance 0 and eps_in exactly 0 in float64; fp32 leaves gamma * invstd * (dy' - mean dy') at the rounding
        # of dy' (invstd = 1/sqrt(eps) ~ 316 amplifies it), so the bound is that rounding, not a relative one
        scale = np.abs(par["gamma"].astype(np.float64) * ref["invstd"][:, None, :] * e).max()
        assert np.abs(got["eps_in"]).max() <= 2.0 ** -22 * scale, f"{what}: eps_in {np.abs(got['eps_in']).max():.3g} for a one-row batch"
    for k in ("y", "eps_in") if rows > 1 else ("y",):
        if prec == "bf16":
            check_bf16(got[k], ref[k], f"{what}: {k}")
        else:
            d = np.abs(got[k] - ref[k]); tol = 1e-4 * np.sqrt(np.mean(ref[k] ** 2)) + 1e-5 * np.abs(ref[k])
            assert (d <= tol).all(), f"{what}: {k} worst |d| = {d.max():.3g}, rms = {np.sqrt(np.mean(ref[k] ** 2)):.3g}"
    rel = np.abs(got["invstd"] - ref["invstd"]) / ref["invstd"]
    assert rel.max() <= 1e-5, f"{what}: invstd relative error {rel.max():.3g} (channel {np.unravel_index(rel.argmax(), rel.shape)})"
    # fp32 nets carry the batch mean in fp32, so xhat = (x - mean) * invstd inherits |mean| * 2^-24 * invstd ~ (|m|/s) * 6e-8.  Measured on an
    # H100 80GB HBM3: the largest gamma / beta gradient error of the fp32 |m|/s = 100 cases is 1.31e-5 (C = 3, 32768 rows, tanh; the others
    # <= 5.7e-6), so those two gradients of fp32 inputs at |m|/s = 100 are held to 2e-5.  bf16 inputs and smaller offsets are held to 1e-5.
    tol_pg = 2e-5 if (prec == "fp32" and ratio >= 100) else 1e-5
    for k in ("mean", "g_gamma", "g_beta", "g_mean", "g_var"):
        err = np.abs(got[k] - ref[k]).max() / (np.abs(ref[k]).max() + 1e-30)
        assert err <= (tol_pg if k in ("g_gamma", "g_beta") else 1e-5), f"{what}: {k} relative error {err:.3g}"


def test_batchnorm_param_grads_untouched_when_not_wanted(b200):
    """want_param_grads = 0 (a frozen-below / no-weight-gradient pass): gamma / beta gradient buffers keep their contents, on every path."""
    b, ctx = b200
    x, e, par, g0 = _inputs(64, 64, 2, 10, seed=3)
    x, e = bf16_round(x), bf16_round(e)
    for P, path in ((b.FP32, 0), (b.BF16, 0), (b.BF16, 1), (b.BF16, 2)):
        got = b.test_bn(ctx, P, path, x, e, par["gamma"], par["beta"], par["run_mean"], par["run_var"], act="relu", g_gamma=g0["g_gamma"], g_beta=g0["g_beta"],
                        want_param_grads=False)
        assert np.array_equal(got["g_gamma"], g0["g_gamma"]) and np.array_equal(got["g_beta"], g0["g_beta"]), (P, path)


def test_batchnorm_accumulator_paths_refuse_unsupported_channels(b200):
    """The accumulator kernels exist for bf16 with C % 8 == 0 and 256 % (C/8) == 0 only: anything else is refused, never approximated."""
    b, ctx = b200
    for C, P in ((24, b.BF16), (3, b.BF16), (4096, b.BF16), (64, b.FP32)):
        x, e, par, _ = _inputs(C, 8, 1, 0, seed=4)
        for path in (1, 2):
            with pytest.raises(b.B200GanError) as err:
                b.test_bn(ctx, P, path, x, e, par["gamma"], par["beta"], par["run_mean"], par["run_var"])
            assert err.value.code == -6, (C, P, path)
