"""The reduction, loss and element-wise kernels that finish each gradient, one production wrapper at a time (b2g_test_ew), against float64 or
exact references (tests/ew_ref.py): split-K sums bit for bit against their documented orders, bias column sums exactly on integers and within
a derived bound on random data, binary and multi-class cross-entropy, activation derivatives on the vector and scalar paths, max-pool ties and
upsampling exactly.  Every test asserts the kernel the wrapper dispatched, so each path is provably reached."""
import math

import numpy as np
import pytest

import ew_ref as er
from helpers import b200, bf16_round

pytestmark = pytest.mark.gpu
PRECS = ["fp32", "bf16"]
U = 2.0 ** -24          # fp32 unit roundoff


def _P(b, prec):
    return b.BF16 if prec == "bf16" else b.FP32


def _rnd(prec, a):
    """the values a T tensor holds on the device"""
    return bf16_round(a) if prec == "bf16" else np.asarray(a, np.float32)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _finite(*arrs):
    for a in arrs:
        assert np.isfinite(a).all(), f"{(~np.isfinite(a)).sum()} non-finite elements"


# ---------------------------------------------------------------- split-K reductions ---------------------------------------------------------
@pytest.mark.parametrize("splits,n,kernel", [
    (63, 4096, "reduce_splits_kernel"), (64, 4096, "reduce_splits_wide_kernel"),           # splits threshold
    (64, 65536, "reduce_splits_wide_kernel"), (64, 65537, "reduce_splits_kernel"),         # output-count threshold
    (300, 3072, "reduce_splits_wide_kernel"), (96, 1, "reduce_splits_wide_kernel"), (3, 100003, "reduce_splits_kernel")])
@pytest.mark.parametrize("accumulate", [False, True])
def test_reduce_splits_bit_exact(b200, splits, n, kernel, accumulate):
    b, ctx = b200
    rng = np.random.default_rng(splits * 7 + n)
    stride = n + 5
    src = (rng.standard_normal((splits, stride)) * np.exp(rng.uniform(-6, 6, (splits, stride)))).astype(np.float32)
    init = rng.standard_normal(n).astype(np.float32)
    (got, _, _), info = b.test_ew(ctx, b.FP32, "reduce_splits", src, init if accumulate else None, (n, 0, 0), n=n, splits=splits, stride=stride,
                                  accumulate=accumulate, poison=not accumulate)
    assert info["kernel"] == kernel
    part = src[:, :n]
    want = (er.reduce_wide if kernel.endswith("wide_kernel") else er.reduce_narrow)(part, init if accumulate else None)
    assert np.array_equal(_bits(got), _bits(want))
    # the emulation of the other order differs: bit equality above does pin the order
    other = (er.reduce_narrow if kernel.endswith("wide_kernel") else er.reduce_wide)(part, init if accumulate else None)
    assert splits < 32 or n < 1000 or not np.array_equal(_bits(other), _bits(want))


def _job_list(specs, gap=3):
    """specs: (n, splits, stride, src_misalign, dst_misalign) -> jobs laid out one after another in one buffer, sources first"""
    jobs, off = [], 0
    for n, splits, stride, sm, _ in specs:
        off += sm
        jobs.append(dict(n=n, splits=splits, stride=stride, src_off=off, dst_off=0))
        off += (splits - 1) * stride + n + gap
        off = (off + 3) // 4 * 4
    for j, (n, _, _, _, dm) in zip(jobs, specs):
        off += dm
        j["dst_off"] = off
        off += n + gap
        off = (off + 3) // 4 * 4
    return jobs, off + 16


REDUCE_LISTS = {
    # both modes in one launch, the scalar branch (n % 4, stride % 4, misaligned source / destination) beside the float4 one
    "mixed": [(3072, 300, 3072, 0, 0), (4096, 7, 4096, 0, 0), (1001, 3, 1004, 0, 0), (1024, 4, 1027, 0, 0), (512, 2, 512, 1, 0),
              (512, 5, 512, 0, 2), (64, 96, 64, 0, 0), (70000, 64, 70000, 0, 0)],
    "one": [(5000, 9, 5000, 0, 0)],
    # 24 jobs (the list's capacity) whose block counts (n / 1024 rounded up, or n / 8 warps) put job boundaries inside every block walk
    "full": [(n, sp, n + (i % 3), i % 2, (i // 2) % 2) for i, (n, sp) in enumerate(
        [(1, 1), (1025, 2), (3, 70), (2047, 3), (4097, 1), (17, 64), (9, 65), (8, 64), (2500, 5), (1023, 4), (7, 100), (4096, 6),
         (333, 2), (1024, 3), (1030, 64), (5, 7), (12345, 2), (640, 80), (1, 64), (2049, 1), (96, 200), (3000, 4), (1, 2), (8193, 3)])],
}


@pytest.mark.parametrize("case", sorted(REDUCE_LISTS))
@pytest.mark.parametrize("offset", [0, 1])
def test_reduce_multi_bit_exact(b200, case, offset):
    b, ctx = b200
    specs = REDUCE_LISTS[case]
    jobs, size = _job_list(specs)
    rng = np.random.default_rng(len(specs) + offset)
    buf = (rng.standard_normal(size) * np.exp(rng.uniform(-6, 6, size))).astype(np.float32)
    (got, _, _), info = b.test_ew(ctx, b.FP32, "reduce_multi", buf, None, (size, 0, 0), n=size, jobs=jobs, poison=True, offset=offset)
    assert info["kernel"] == "reduce_multi_kernel"
    assert info["wide"] == [int(sp >= 64 and n <= 65536) for n, sp, _, _, _ in specs]      # the warp-per-output rule of reduce_list_push
    if case == "mixed":
        assert set(info["wide"]) == {0, 1}
    want = er.reduce_multi(buf, jobs, info["wide"])
    assert np.array_equal(_bits(got), _bits(want))


# deferred (one reduce-list launch after the kernel, as in a backward pass) == immediate, bit for bit, at the C2 shapes
WGRAD_DEFER = [("D2 wgrad (2N)", 1, 256, 32, 64, 128), ("G2 wgrad (N)", 1, 128, 8, 256, 512),
               ("D1 edge wgrad (2N)", 3, 256, 64, 3, 64), ("G-last edge wgrad (N)", 3, 128, 64, 3, 64)]


@pytest.mark.parametrize("case", WGRAD_DEFER, ids=[c[0] for c in WGRAD_DEFER])
def test_deferred_wgrad_reduction_equals_immediate(b200, case):
    b, ctx = b200
    name, impl, n, h, c, oc = case
    rng = np.random.default_rng(n + c)
    x = bf16_round(rng.standard_normal((n, h, h, c))); dy = bf16_round(rng.standard_normal((n, h // 2, h // 2, oc)))
    geom = dict(n=n, h=h, w=h, c=c, oh=h // 2, ow=h // 2, o=oc, kh=4, kw=4, sh=2, sw=2, ph=1, pw=1)
    res = []
    for defer in (False, True):
        db = np.full(oc, np.nan, np.float32) if impl == 3 else None
        dw, _, kernel, _ = b.test_conv_ex(ctx, 2, geom, x, dy, oc * 16 * c, impl=impl, defer=defer, db=db)
        assert kernel == ("tc_edge_wgrad_kernel" if impl == 3 else "tc_wgrad_kernel<128,4>"), (name, kernel)
        _finite(dw)
        res.append((dw, db))
    assert np.array_equal(_bits(res[0][0]), _bits(res[1][0])), name
    if impl == 3:
        assert np.array_equal(_bits(res[0][1]), _bits(res[1][1])), name
        ref = dy.reshape(-1, oc).astype(np.float64).sum(0)              # the conv bias gradient: column sums of dy
        _finite(res[0][1])
        assert np.abs(res[0][1] - ref).max() <= 1e-4 * np.abs(dy).reshape(-1, oc).sum(0).max(), name      # a lost split or pixel is off by O(1)


# ---------------------------------------------------------------- bias column sums -----------------------------------------------------------
SMALL_C = "colsum_small_c_kernel<{}>"
COLSUM_CASES = [
    # prec, rows, C, offset, kernel the wrapper must dispatch
    ("bf16", 128 * 64 * 64, 3, 0, SMALL_C.format(3)),          # C2 G-last bias gradient
    ("bf16", 4096, 1, 0, SMALL_C.format(1)), ("bf16", 4096, 2, 0, SMALL_C.format(2)), ("bf16", 8192, 4, 0, SMALL_C.format(4)),
    ("bf16", 4095, 3, 0, "colsum_partial_kernel"),              # rows < 4096 (and rows % 8 != 0)
    ("bf16", 4088, 3, 0, "colsum_partial_kernel"),              # rows % 8 == 0 but < 4096
    ("bf16", 4100, 3, 0, "colsum_partial_kernel"),              # rows >= 4096, rows % 8 != 0
    ("bf16", 8192, 3, 1, "colsum_partial_kernel"),              # misaligned x
    ("bf16", 5000, 64, 0, "colsum_partial_bf16x8_kernel"), ("bf16", 777, 2048, 0, "colsum_partial_bf16x8_kernel"),
    ("bf16", 3001, 256, 0, "colsum_partial_bf16x8_kernel"),
    ("bf16", 5000, 24, 0, "colsum_partial_kernel"),             # 256 % (C/8) != 0
    ("bf16", 5000, 64, 1, "colsum_partial_kernel"),             # misaligned x: no 16-byte loads
    ("fp32", 128 * 64 * 64, 3, 0, "colsum_partial_kernel"), ("fp32", 5000, 64, 1, "colsum_partial_kernel"), ("fp32", 3, 1000, 0, "colsum_partial_kernel"),
]


def _colsum(b, ctx, prec, x, C, offset, init=None):
    rows = x.shape[0]
    (got, _, _), info = b.test_ew(ctx, _P(b, prec), "colsum", x, init, (C, 0, 0), rows=rows, cols=C, offset=offset, accumulate=init is not None,
                                  poison=init is None)
    return got, info["kernel"]


@pytest.mark.parametrize("case", COLSUM_CASES, ids=[f"{c[0]}-{c[1]}x{c[2]}-off{c[3]}" for c in COLSUM_CASES])
def test_colsum_exact_on_integers(b200, case):
    """Small integers with column sums below 2^24: every partial sum is exact in any order, so a dropped, duplicated or mis-channelled row
    changes the result.  With accumulate the initial value is added once."""
    b, ctx = b200
    prec, rows, C, offset, kernel = case
    rng = np.random.default_rng(rows + C)
    x = rng.integers(-4, 5, (rows, C)).astype(np.float32)
    x[rng.integers(0, rows, 5), rng.integers(0, C, 5)] = 7.0           # a few marked elements in random rows and channels
    want = x.astype(np.float64).sum(0)
    got, k = _colsum(b, ctx, prec, x, C, offset)
    assert k == kernel
    assert np.array_equal(got, want)
    init = rng.integers(-100, 101, C).astype(np.float32)
    got, k = _colsum(b, ctx, prec, x, C, offset, init)
    assert k == kernel
    assert np.array_equal(got, want + init)


def _colsum_chain(kernel, rows, C):
    """Longest chain of fp32 additions any column sum goes through on this path's launch geometry (kernels_ew.cu); the final stage sums the
    partials in double and rounds once.
      colsum_partial_kernel: S = clamp(rows / 8, 1, min(2048, 2^20 / C)) slices; a thread sums rows s, s+S, ... : ceil(rows / S) terms.
      colsum_partial_bf16x8_kernel: TY = 256 / (C/8) row lanes, S = clamp(rows / (4 TY), 1, min(256, 2^20 / C)) blocks of ceil(rows / S)
        rows; a lane sums ceil(chunk / TY) rows, then the block folds its TY lanes in order: ceil(chunk / TY) + TY terms.
      colsum_small_c_kernel<C>: groups of 8 pixels, S = min(256, ceil(rows / 8 / 256)) blocks of 256 threads striding over the groups; a thread
        adds the 8 elements of each channel in every group it visits, then a 5-level shuffle tree and the fold of 8 warps: + 5 + 8 terms."""
    if kernel.startswith("colsum_small_c_kernel"):
        g8 = rows // 8; S = min(256, -(-g8 // 256))
        return -(-g8 // (S * 256)) * 8 + 5 + 8
    if kernel == "colsum_partial_bf16x8_kernel":
        TY = 256 // (C // 8); S = max(1, min(rows // (4 * TY), min(256, (1 << 20) // C)))
        chunk = -(-rows // S)
        return -(-chunk // TY) + TY
    S = max(1, min(rows // 8, min(2048, (1 << 20) // C)))
    return -(-rows // S)


@pytest.mark.parametrize("case", COLSUM_CASES, ids=[f"{c[0]}-{c[1]}x{c[2]}-off{c[3]}" for c in COLSUM_CASES])
def test_colsum_random_within_derived_bound(b200, case):
    """Random data against float64 on the stored values: a sum through a chain of L fp32 additions is off by at most
    gamma_L * sum|x| (gamma_L = L u / (1 - L u), u = 2^-24; Higham, Accuracy and Stability, eq. 4.4), then rounded to fp32 once (u |s|)."""
    b, ctx = b200
    prec, rows, C, offset, kernel = case
    rng = np.random.default_rng(rows * 3 + C)
    x = _rnd(prec, rng.standard_normal((rows, C)) + 0.5)
    got, k = _colsum(b, ctx, prec, x, C, offset)
    assert k == kernel
    _finite(got)
    L = _colsum_chain(kernel, rows, C)
    ref = x.astype(np.float64).sum(0)
    bound = L * U / (1 - L * U) * np.abs(x).astype(np.float64).sum(0) + U * np.abs(ref)
    assert (np.abs(got - ref) <= bound).all(), (kernel, L, np.max(np.abs(got - ref) / bound))


# ---------------------------------------------------------------- LossBinaryXENT ----------------------------------------------------------
# Worst errors over the cases below, measured on an H100 80GB HBM3 (power limit 400 W), keyed by (precision, clip): max |dz - ref| (dz is
# O(1); a bf16 dz rounds to 2^-9 relative) and the largest relative error of a per-group loss sum.  Bounds = 2x the measurement.
# The clipped mode is the least accurate by construction: sigmoid'(z) = sg (1 - sg) loses 1 - sg to fp32 cancellation for z >~ 10, and p is
# clipped to the fp32 value of 1 - 1e-5 (1 - p = 1.0013e-5); a missing or wrong factor is off by O(1) or by up to 1e5.
XENT_DZ_MEASURED = {("fp32", 1e-5): 6.33e-3, ("fp32", 0.0): 1.17e-7, ("bf16", 1e-5): 7.55e-3, ("bf16", 0.0): 3.91e-3}
XENT_DZ_TOL = {k: 2 * v for k, v in XENT_DZ_MEASURED.items()}
XENT_LOSS_MEASURED = {("fp32", 1e-5): 5.91e-5, ("fp32", 0.0): 3.29e-8, ("bf16", 1e-5): 5.90e-5, ("bf16", 0.0): 3.47e-8}
XENT_LOSS_TOL = {k: 2 * v for k, v in XENT_LOSS_MEASURED.items()}


def _logits(rng, n, lim):
    """logits across the saturating range: uniform magnitude 0..lim with random sign, plus fixed points where expf(-z) overflows (z < -88.7)
    and where sigmoid rounds to 0 or 1 in fp32"""
    z = rng.uniform(0, lim, n) * rng.choice([-1.0, 1.0], n)
    fixed = np.array([0.0, 1e-3, -1e-3, 11.5, -11.5, 16.0, -16.0, 17.5, -17.5, 40.0, -40.0, 88.0, -88.0, 88.8, -88.8, 89.0, -89.0, 90.0, -90.0])
    k = min(n, fixed.size)
    z[rng.choice(n, k, replace=False)] = fixed[:k]
    return z


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("clip", [1e-5, 0.0])
@pytest.mark.parametrize("groups", [1, 2])
@pytest.mark.parametrize("rows", [77, 3001])
def test_xent_against_float64(b200, prec, clip, groups, rows):
    b, ctx = b200
    rng = np.random.default_rng(rows * 10 + groups)
    z = _rnd(prec, _logits(rng, groups * rows, 90.0)).reshape(groups, rows)
    real = rng.random((groups, rows)) < 0.5                          # the reference's noisy labels: 1 + 0.05 N(0,1) (real), 0.05 N(0,1) (fake)
    y = (np.where(real, 1.0, 0.0) + 0.05 * rng.standard_normal((groups, rows))).astype(np.float32)
    (dz, loss, _), info = b.test_ew(ctx, _P(b, prec), "xent", z, y, (groups * rows, groups, 0), rows=rows, groups=groups, clip_eps=clip, poison=True)
    assert info["kernel"] == "xent_kernel"
    _finite(dz, loss)
    ref_loss, ref_dz = er.xent(z, y, clip)
    e_dz = float(np.abs(dz.reshape(groups, rows) - ref_dz).max())
    e_loss = float((np.abs(loss - ref_loss) / np.abs(ref_loss)).max())
    print(f"xent {prec} clip={clip} groups={groups} rows={rows}: max |dz - ref| {e_dz:.3e}, loss rel {e_loss:.3e}")
    assert e_dz <= XENT_DZ_TOL[(prec, clip)] and e_loss <= XENT_LOSS_TOL[(prec, clip)]


# ---------------------------------------------------------------- LossMCXENT + softmax --------------------------------------------------------
# Measured on the same H100: max |dz - ref| and |p - ref| (both in [-1, 1]; bf16 stores round to 2^-9 relative) and the loss sum's relative
# error (accumulated in double from fp32 probabilities in either precision).  Bounds = 2x the measurement.
MCXENT_DZ_MEASURED = {"fp32": 1.46e-7, "bf16": 1.95e-3}
MCXENT_DZ_TOL = {k: 2 * v for k, v in MCXENT_DZ_MEASURED.items()}
MCXENT_LOSS_MEASURED = {"fp32": 3.01e-8, "bf16": 1.41e-8}
MCXENT_LOSS_TOL = {k: 2 * v for k, v in MCXENT_LOSS_MEASURED.items()}


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("K", [10, 7])
@pytest.mark.parametrize("labels", ["one-hot", "soft"])
def test_softmax_xent_against_float64(b200, prec, K, labels):
    b, ctx = b200
    rows = 1500
    rng = np.random.default_rng(K * 3 + len(labels))
    z = rng.uniform(-80, 80, (rows, K)) * (rng.random((rows, 1)) < 0.5) + rng.standard_normal((rows, K))     # half the rows +-80, half O(1)
    z = _rnd(prec, z)
    if labels == "one-hot":
        y = np.eye(K, dtype=np.float32)[rng.integers(0, K, rows)]
    else:
        y = rng.random((rows, K)); y = (y / y.sum(1, keepdims=True)).astype(np.float32)
    (dz, loss, p), info = b.test_ew(ctx, _P(b, prec), "softmax_xent", z, y, (rows * K, 1, rows * K), rows=rows, cols=K, poison=True)
    assert info["kernel"] == "softmax_xent_kernel"
    _finite(dz, loss, p)
    ref_loss, ref_dz, ref_p = er.mcxent(z, y)
    e_dz = float(np.abs(dz.reshape(rows, K) - ref_dz).max()); e_p = float(np.abs(p.reshape(rows, K) - ref_p).max())
    e_loss = abs(float(loss[0]) - ref_loss) / abs(ref_loss)
    print(f"mcxent {prec} K={K} {labels}: max |dz - ref| {e_dz:.3e}, max |p - ref| {e_p:.3e}, loss rel {e_loss:.3e}")
    assert e_dz <= MCXENT_DZ_TOL[prec] and e_p <= MCXENT_DZ_TOL[prec] and e_loss <= MCXENT_LOSS_TOL[prec]
    # the inference call: no labels, no dz, no loss -- the probabilities and nothing else
    (dz2, loss2, p2), info = b.test_ew(ctx, _P(b, prec), "softmax_xent", z, None, (rows * K, 1, rows * K), rows=rows, cols=K, poison=True)
    assert info["kernel"] == "softmax_xent_kernel"
    assert np.array_equal(_bits(p2), _bits(p))
    assert np.isnan(dz2).all() and np.isnan(loss2).all()


# ---------------------------------------------------------------- activations -----------------------------------------------------------------
ACTS = ["identity", "tanh", "sigmoid", "relu", "lrelu"]


def _act_inputs(rng, n):
    """exact zeros, the saturated tails of tanh and sigmoid (sigmoid(-200) == 0 and tanh(+-20) == +-1 in fp32), and O(1) values"""
    x = rng.standard_normal(n) * 3
    k = n // 8
    idx = rng.permutation(n)
    x[idx[:k]] = 0.0
    x[idx[k:2 * k]] = rng.choice([-200.0, -100.0, -20.0, 20.0, 100.0, 200.0], k)
    return x


def _check_act_fwd(prec, got, x, act):
    ref = er.act_fwd(x, act, 0.2)
    tol = (2.0 ** -8 if prec == "bf16" else 8 * U) * np.abs(ref) + 1e-30       # bf16: one rounding; fp32: tanhf / expf within a few ulp
    assert (np.abs(got - ref) <= tol).all(), (prec, act, float(np.max(np.abs(got - ref) / tol)))


def _check_act_bwd(prec, got, a, eo, act):
    g = er.act_grad_from_out(a, act, 0.2)
    ref = eo.astype(np.float64) * g
    # f'(a) in fp32 (1 - a a, a (1 - a)): 2 roundings of O(1) values; the product: one more; bf16: the store rounds to 2^-9 relative
    tol = 4 * U * np.abs(eo) * (1 + np.abs(g)) + (2.0 ** -8 if prec == "bf16" else 2 * U) * np.abs(ref) + 1e-30
    assert (np.abs(got - ref) <= tol).all(), (prec, act, float(np.max(np.abs(got - ref) / tol)))


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("act", ACTS)
def test_activation_forward_and_backward(b200, prec, act):
    b, ctx = b200
    P = _P(b, prec)
    n = 8 * 12345
    rng = np.random.default_rng(ACTS.index(act) + 10 * len(prec))
    x = _rnd(prec, _act_inputs(rng, n))
    (a, _, _), info = b.test_ew(ctx, P, "act_fwd", x, None, (n, 0, 0), act=act, alpha=0.2, n=n, poison=True)
    assert info["kernel"] == "act_fwd_kernel"
    _finite(a)
    _check_act_fwd(prec, a, x, act)
    if act in ("tanh", "relu", "lrelu"):
        assert (a == 0).sum() >= n // 8              # a == 0 exactly wherever x == 0: the kink of relu / leaky relu is exercised
    if act in ("tanh", "sigmoid"):
        assert (np.abs(a) == 1).any() and (act != "sigmoid" or (a == 0).any())      # saturated outputs: f'(a) == 0 exactly there
    eo = _rnd(prec, rng.standard_normal(n))
    vec = prec == "bf16"
    res = {}
    for offset in (0, 1):                            # offset 1: misaligned operands, the scalar kernel on the same data
        for in_place in (False, True):
            (ei, _, _), info = b.test_ew(ctx, P, "act_bwd", a, eo, (n, 0, 0), act=act, alpha=0.2, n=n, in_place=in_place, offset=offset,
                                         poison=not in_place)
            assert info["kernel"] == ("act_bwd_out_bf16x8_kernel" if vec and offset == 0 else "act_bwd_out_kernel"), (offset, info["kernel"])
            _finite(ei)
            _check_act_bwd(prec, ei, a, eo, act)
            res[(offset, in_place)] = ei
    for k, v in res.items():                         # vector and scalar path, in place or not: the same bits
        assert np.array_equal(_bits(v), _bits(res[(0, False)])), k
    # n % 8 != 0: the scalar path also without misalignment
    m = n - 3
    (ei, _, _), info = b.test_ew(ctx, P, "act_bwd", a[:m], eo[:m], (m, 0, 0), act=act, alpha=0.2, n=m, poison=True)
    assert info["kernel"] == "act_bwd_out_kernel"
    assert np.array_equal(_bits(ei), _bits(res[(0, False)][:m]))


# ---------------------------------------------------------------- max-pool and upsampling ---------------------------------------------------
POOL_CASES = [
    # N, H, W, C, KH, KW, SH, SW
    (2, 9, 11, 5, 3, 3, 2, 2),       # overlapping windows
    (2, 7, 6, 5, 2, 2, 1, 1),        # overlapping, stride 1
    (2, 8, 8, 5, 2, 2, 2, 2),        # windows tile the input
    (2, 10, 12, 3, 3, 3, 2, 2),      # truncating: the last input row and column are in no window
    (3, 9, 9, 4, 2, 2, 2, 2),        # truncating by one
    (2, 16, 17, 3, 15, 15, 1, 1),    # 15x15 windows: the argmax exceeds 127
]


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("case", POOL_CASES, ids=[f"{c[1]}x{c[2]}k{c[4]}s{c[6]}" for c in POOL_CASES])
def test_maxpool_first_max_wins_and_gather_backward_exact(b200, prec, case):
    b, ctx = b200
    N, H, W, C, KH, KW, SH, SW = case
    OH, OW = (H - KH) // SH + 1, (W - KW) // SW + 1
    rng = np.random.default_rng(H * W + KH)
    x = rng.integers(0, 3, (N, H, W, C)).astype(np.float32)           # values in {0, 1, 2}: ties in nearly every window
    if KH * KW > 128:         # the maxima (still tied) sit in the window's last rows: the first of them has an argmax above 127
        x[:, :H - 4] = np.minimum(x[:, :H - 4], 1.0)
    eo = rng.integers(-3, 4, (N, OH, OW, C)).astype(np.float32)       # integer eps: the gather sums are exact in any order
    (y, ei, arg), info = b.test_ew(ctx, _P(b, prec), "maxpool", x, eo, (eo.size, x.size, eo.size), N=N, H=H, W=W, C=C, KH=KH, KW=KW, SH=SH, SW=SW,
                                   poison=True)
    assert info["kernel"] == "maxpool_fwd_kernel,maxpool_bwd_kernel"
    ry, rarg, rei = er.maxpool(x, eo, (KH, KW), (SH, SW))
    assert np.array_equal(y.reshape(ry.shape), ry)
    assert np.array_equal(arg.reshape(rarg.shape), rarg)
    assert np.array_equal(ei.reshape(rei.shape), rei)
    if KH * KW > 128:
        assert arg.max() > 127
    ties = (np.sort(np.lib.stride_tricks.sliding_window_view(x, (KH, KW), (1, 2))[:, ::SH, ::SW].reshape(N, OH, OW, C, -1), -1)[..., -2:] == ry[..., None]).all(-1)
    assert ties.mean() > 0.3                        # most windows hold their maximum twice or more


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("f", [2, 3])
def test_upsample_forward_and_backward_exact(b200, prec, f):
    b, ctx = b200
    N, H, W, C = 3, 5, 7, 6
    rng = np.random.default_rng(f)
    x = _rnd(prec, rng.standard_normal((N, H, W, C)))
    eo = rng.integers(-8, 9, (N, H * f, W * f, C)).astype(np.float32)
    (y, ei, _), info = b.test_ew(ctx, _P(b, prec), "upsample", x, eo, (eo.size, x.size, 0), N=N, H=H, W=W, C=C, KH=f, poison=True)
    assert info["kernel"] == "upsample_fwd_kernel,upsample_bwd_kernel"
    ry, rei = er.upsample(x, eo, f)
    assert np.array_equal(y.reshape(ry.shape), ry)
    assert np.array_equal(ei.reshape(rei.shape), rei)


# ---------------------------------------------------------------- l2 score ------------------------------------------------------------------
def test_sumsq_segments_against_float64(b200):
    b, ctx = b200
    n = 1_000_003
    rng = np.random.default_rng(9)
    p = (rng.standard_normal(n) * np.exp(rng.uniform(-5, 5, n))).astype(np.float32)
    off = np.array([1, 1001, 5003, 5003, 77777, 300001, 999_001], np.int64)
    ln = np.array([999, 4001, 0, 70001, 200003, 600000, 1001], np.int64)        # one empty segment; all start at odd offsets
    coef = np.array([0.5, 1e-4, 3.0, 0.0, 2.5e-3, 1.0, 7.0], np.float32)       # a zero coefficient
    _, info = b.test_ew(ctx, b.FP32, "sumsq", p, None, (0, 0, 0), n=n, segments=(off, ln, coef), poison=True)
    assert info["kernel"] == "sumsq_segments_kernel"
    ref = math.fsum(float(c) * math.fsum((p[o:o + k].astype(np.float64) ** 2).tolist()) for o, k, c in zip(off, ln, coef))
    assert abs(info["sumsq"] - ref) <= 1e-12 * abs(ref), (info["sumsq"], ref)


# ---------------------------------------------------------------- layout conversion and the bf16 cast ---------------------------------------
def _pass_elems(ctx):
    """Elements one grid-stride pass of the layout and cast kernels covers: ew_blocks caps their grid at 16 blocks of 256 threads per SM."""
    return 16 * ctx.device_info()["sm_count"] * 256


LAYOUT_SHAPES = [
    # N, C, H, W (HW = H * W), offset
    (1, 1, 1, 1, 0), (1, 5, 1, 1, 0), (3, 1, 7, 5, 0), (1, 7, 3, 3, 1), (2, 3, 5, 7, 3), (4, 64, 8, 8, 0),
    (7, 131, 43, 47, 0), (7, 131, 43, 47, 1),      # 1.85M elements: more than three grid-stride passes on an H100
]


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("shape", LAYOUT_SHAPES, ids=[f"{s[0]}x{s[1]}x{s[2]}x{s[3]}-off{s[4]}" for s in LAYOUT_SHAPES])
def test_layout_kernels_exact(b200, prec, shape):
    """NCHW fp32 -> NHWC T (input staging), NHWC T -> NCHW fp32 (output read-back) and the T -> T permutes of the FF <-> CNN preprocessors: numpy's
    transpose of the stored values, bit for bit, every element written (NaN-poisoned outputs)."""
    b, ctx = b200
    N, C, H, W, offset = shape
    HW, n = H * W, N * C * H * W
    if n > 1_000_000:
        assert n > 3 * _pass_elems(ctx)
    rng = np.random.default_rng(n + offset)
    x = (rng.standard_normal(n) * np.exp(rng.uniform(-8, 8, n))).astype(np.float32)        # many binades: a misplaced element shows
    nchw, nhwc = x.reshape(N, C, HW), x.reshape(N, HW, C)
    geom = dict(N=N, C=C, H=H, W=W, offset=offset, poison=True)
    P = _P(b, prec)
    (got, _, _), info = b.test_ew(ctx, P, "nchw_to_nhwc", x, None, (n, 0, 0), **geom)
    assert info["kernel"] == "nchw_f32_to_nhwc_kernel"
    assert np.array_equal(_bits(got), _bits(_rnd(prec, nchw.transpose(0, 2, 1)).ravel()))
    (got, _, _), info = b.test_ew(ctx, P, "nhwc_to_nchw", x, None, (n, 0, 0), **geom)
    assert info["kernel"] == "nhwc_to_nchw_f32_kernel"
    assert np.array_equal(_bits(got), _bits(_rnd(prec, nhwc).transpose(0, 2, 1).ravel()))
    for to_nhwc, want in ((1, _rnd(prec, nchw).transpose(0, 2, 1)), (0, _rnd(prec, nhwc).transpose(0, 2, 1))):
        (got, _, _), info = b.test_ew(ctx, P, "permute", x, None, (n, 0, 0), groups=to_nhwc, **geom)
        assert info["kernel"] == "permute_kernel"
        assert np.array_equal(_bits(got), _bits(want.ravel())), f"permute to_nhwc={to_nhwc}"


def _cast_specials():
    """fp32 bit patterns where a bf16 rounding can go wrong: exact ties between bf16 neighbours (even and odd upper halves, both signs), one ulp
    either side of a tie, +-0, subnormals (the largest rounds up to the smallest normal), the largest finite values (round to inf), +-inf and NaNs
    (quiet, and signalling ones whose payload is only in the low 16 bits)"""
    hi = np.array([0x3F80, 0x3F81, 0x4049, 0x404A, 0x7F7E, 0x0080, 0x0001, 0x4B00], np.uint32)
    ties = [(h << 16) | lo for h in hi for lo in (0x8000, 0x7FFF, 0x8001, 0x0000, 0xFFFF)]
    bits = ties + [0x00000000, 0x00000001, 0x00008000, 0x00018000, 0x007FFFFF, 0x00800000, 0x7F7FFFFF, 0x7F7F7FFF, 0x7F800000,
                   0x7FC00000, 0x7F800001, 0x7F808000, 0x7FFFFFFF]
    bits = np.array(bits, np.uint32)
    return np.concatenate([bits, bits | np.uint32(0x80000000)]).view(np.float32)


def _bf16_rne(x):
    """fp32 -> bf16 -> fp32, round to nearest even, in integer arithmetic on the bits (NaNs excepted): helpers.bf16_round's rounding, without
    depending on which conversion the host CPU's torch build uses for subnormals"""
    u = _bits(x).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return r.astype(np.uint32).view(np.float32)


def _check_cast(x, got, round_trip):
    want = _bf16_rne(x)
    nan = np.isnan(x)
    normal = (np.abs(x) >= 2.0 ** -126) & (np.abs(x) < 1e38)          # the same rounding as helpers.bf16_round where no host can differ
    assert np.array_equal(_bits(bf16_round(x[normal])), _bits(want[normal]))
    assert np.isnan(got[nan]).all(), "a NaN must stay NaN"
    assert np.array_equal(_bits(got[~nan]), _bits(want[~nan])), f"{int((_bits(got[~nan]) != _bits(want[~nan])).sum())} elements not rounded to nearest even"
    assert np.array_equal(_bits(round_trip), _bits(got)), "the device widen of the bf16 payload differs from its bits"


@pytest.mark.parametrize("case", ["specials", "random-bits", "wrap"])
@pytest.mark.parametrize("offset", [0, 1])
def test_cast_f32_to_bf16_rounds_to_nearest_even(b200, case, offset):
    """k_cast_f32_to_bf16 (the bf16 gradient payload, the hooks' bf16 uploads) against round-to-nearest-even, and the payload's widen back to fp32
    through nhwc_to_nchw_f32_kernel at 1 x 1 x n: the cast's bits, NaN-poisoned outputs, n not a multiple of 4 or 8."""
    b, ctx = b200
    rng = np.random.default_rng(len(case) + offset)
    if case == "specials":
        x = _cast_specials()
    elif case == "random-bits":        # every binade, subnormals, infinities and NaNs in proportion to their bit patterns
        x = rng.integers(0, 2 ** 32, 12347, dtype=np.uint64).astype(np.uint32).view(np.float32)
    else:                              # more than two grid-stride passes, the specials spread through every pass
        n = 2 * _pass_elems(ctx) + 4099
        x = (rng.standard_normal(n) * np.exp(rng.uniform(-30, 30, n))).astype(np.float32)
        sp = _cast_specials()
        x[rng.choice(n, 40 * sp.size, replace=False)] = np.tile(sp, 40)
    n = x.size
    assert n % 4 != 0
    (got, rt, _), info = b.test_ew(ctx, b.BF16, "cast_bf16", x, None, (n, n, 0), n=n, offset=offset, poison=True)
    assert info["kernel"] == "cast_f32_to_bf16_kernel,nhwc_to_nchw_f32_kernel"
    _check_cast(x, got, rt)
