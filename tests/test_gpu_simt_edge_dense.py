"""GPU: the SIMT implicit-GEMM kernel (kernels_simt.cu), the skinny-layer kernels and the dense 1x1-geometry kernels (kernels_edge.cu) against
float64, element by element, through the kernel-level hook b2g_test_conv_ex with the epilogue (bias, folded BatchNorm scale, activation) their
production wrappers take, parameter offsets, and the geometry edges where GEMM kernels go wrong.

Every case runs on an output poisoned with NaN (kind 2: the fp32 dw and the split-K partials too), asserts the kernel its wrapper dispatched
and, for the split-K weight gradients, the number of splits, mirrored here from kernels_simt.cu wgrad_splits, kernels_edge.cu
edge_wgrad_ctas and dense_wgrad_splits.  Each case is checked two ways:

* exact: integer operands in [-3, 3], integer bias, power-of-two scale, identity / relu / lrelu(0.25).  Every partial sum is an integer
  below 2^24, so each fp32 FMA chain, split-K sum and epilogue is exact: fp32 outputs equal the float64 reference bit for bit, bf16 outputs
  equal its one round-to-nearest-even rounding.
* random: per element |got - ref| <= gamma_K' * sum|a*b| * |scale| + u * |bias| on the pre-activation, u = 2^-24,
  gamma_K' = K'u / (1 - K'u), K' = the reduction length K + 64 (the at most 64 split-K partials, or the 5 + 2 levels of a block
  reduction, are summed in fp32 after the chains) + 4 (the scale product, the bias sum and one spare rounding).  The activations are
  1-Lipschitz and tanhf / expf add a few ulps of the result: + 8u |act(ref)|.  A bf16 output adds its own round-to-nearest: bf16 has 8
  significant bits, so its unit roundoff is 2^-8 and the bound grows by 2^-8 (|ref| + e) (measured on an H100: up to 1.97 x 2^-9 |ref|, so
  2^-9 would be too tight).  bf16 operands are rounded first and the reference runs on the rounded values.
"""
import math
import zlib

import numpy as np
import pytest

import conv_ref
from gan_deeplearning4j_b200 import models as m
from helpers import assert_close_up_to_sign_flips, b200, bf16_round, push_params, randomize, rel_err
from oracle import dl4j_oracle as o

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
TOL = 1e-3          # the FP32 DL4J-parity bar of tests/test_gpu_parity.py


def geom(n, h, w, c, oc, k=(1, 1), s=(1, 1), p=(0, 0)):
    return dict(n=n, h=h, w=w, c=c, oh=conv_ref.out_size(h, k[0], s[0], p[0]), ow=conv_ref.out_size(w, k[1], s[1], p[1]), o=oc,
                kh=k[0], kw=k[1], sh=s[0], sw=s[1], ph=p[0], pw=p[1])


def act_ref(name, z, alpha):
    if name == "tanh":
        return np.tanh(z)
    if name == "sigmoid":
        return 1.0 / (1.0 + np.exp(-z))
    if name == "relu":
        return np.maximum(z, 0.0)
    if name == "lrelu":
        return np.where(z > 0, z, alpha * z)
    return z


def reference(kind, g, a, b):
    """float64 result of kind 0 (y, NHWC), 1 (dx, NHWC) or 2 (dw, [O][KH][KW][C]) on flat operands a, b."""
    n, h, w, c, oh, ow, oc = (g[k] for k in ("n", "h", "w", "c", "oh", "ow", "o"))
    k, s, p = (g["kh"], g["kw"]), (g["sh"], g["sw"]), (g["ph"], g["pw"])
    if kind == 0:
        return conv_ref.conv2d(a.reshape(n, h, w, c), b.reshape(oc, k[0], k[1], c), s, p)
    if kind == 1:
        return conv_ref.conv2d_input_grad(a.reshape(n, oh, ow, oc), b.reshape(oc, k[0], k[1], c), (h, w), s, p)
    return conv_ref.conv2d_weight_grad(a.reshape(n, h, w, c), b.reshape(n, oh, ow, oc), k[0], k[1], s, p)


def reduction_length(kind, g):
    return (g["kh"] * g["kw"] * g["c"], g["kh"] * g["kw"] * g["o"], g["n"] * g["oh"] * g["ow"])[kind]


def run_case(b, ctx, kind, impl, prec, g, rng, *, exact, bias=False, scale=False, act="identity", param_offset=0):
    """One launch through the hook against float64.  Returns (kernel name, split count)."""
    P = b.BF16 if prec == "bf16" else b.FP32
    nx, ny, nw = g["n"] * g["h"] * g["w"] * g["c"], g["n"] * g["oh"] * g["ow"] * g["o"], g["o"] * g["kh"] * g["kw"] * g["c"]
    na, nb = (nx, ny, nx)[kind], (nw, nw, ny)[kind]
    oc = g["o"] if kind == 0 else g["c"]
    alpha = 0.25
    if exact:
        a = rng.integers(-3, 4, na).astype(np.float32); bb = rng.integers(-3, 4, nb).astype(np.float32)
        bv = rng.integers(-3, 4, oc).astype(np.float32) if bias else None
        sv = rng.choice([0.5, 2.0], oc).astype(np.float32) if scale else None
    else:
        rnd = bf16_round if prec == "bf16" else (lambda v: np.asarray(v, np.float32))
        a = rnd(rng.standard_normal(na)); bb = rnd(rng.standard_normal(nb) / math.sqrt(max(1, reduction_length(kind, g) // max(1, g["n"]))))
        bv = rng.standard_normal(oc).astype(np.float32) if bias else None
        sv = rng.uniform(0.5, 1.5, oc).astype(np.float32) if scale else None
    size = (ny, nx, nw)[kind]
    info = {}
    got, _, kern, _ = b.test_conv_ex(ctx, kind, g, a, bb, size, impl=impl, precision=P, poison=True, info=info, bias=bv, scale=sv,
                                     act=act, alpha=alpha, param_offset=param_offset)
    got = got.astype(np.float64).ravel()
    ref = reference(kind, g, a, bb).ravel()
    mag = reference(kind, g, np.abs(a), np.abs(bb)).ravel()
    if kind != 2:
        ch = np.arange(ref.size) % oc
        s64 = sv.astype(np.float64)[ch] if sv is not None else 1.0
        b64 = bv.astype(np.float64)[ch] if bv is not None else 0.0
        z = ref * s64 + b64
        mag = mag * np.abs(s64)
        babs = np.abs(b64)
    else:
        z, babs = ref, 0.0
    want = act_ref(act, z, alpha)
    what = f"{kern} kind {kind} impl {impl} {prec} {g} act={act} bias={bias} scale={scale} offset={param_offset}"
    if exact:
        want32 = want.astype(np.float32)
        if prec == "bf16" and kind != 2:
            want32 = bf16_round(want32)
        bad = ~(got == want32.astype(np.float64))
        assert not bad.any(), f"{what}: {bad.sum()} of {bad.size} elements differ from the exact result (first at {np.flatnonzero(bad)[:5]}: " \
                              f"got {got[bad][:5]}, want {want32[bad][:5]})"
    else:
        kp = reduction_length(kind, g) + 68
        e = kp * U / (1 - kp * U) * mag + U * babs
        if act in ("tanh", "sigmoid"):
            e = e + 8 * U * np.abs(want)
        if prec == "bf16" and kind != 2:
            e = e + 2.0 ** -8 * (np.abs(want) + e)
        d = np.abs(got - want)
        bad = ~(d <= e)
        assert not bad.any(), f"{what}: {bad.sum()} of {bad.size} elements outside the bound (worst d/bound {np.nanmax(d / (e + 1e-300)):.3g}, " \
                              f"non-finite {(~np.isfinite(got)).sum()})"
    return kern, info["splits"]


# ------------------------------------------------------------------ split counts, mirrored from the host wrappers ---------------------------
def simt_wgrad_splits(g):
    tiles = -(-g["o"] // 64) * -(-(g["kh"] * g["kw"] * g["c"]) // 64)
    P = g["n"] * g["oh"] * g["ow"]
    return max(1, min(-(-296 // tiles), 64, max(P // 256, 1)))


def edge_wgrad_ctas(g, sms):
    P = g["n"] * g["oh"] * g["ow"]
    return max(1, min(2 * sms, -(-P // 64)))


def dense_wgrad_splits(g):
    return max(1, min(-(-g["n"] // 8), 32))


SIMT_NAMES = ("simt_gemm_kernel<FpropProb>", "simt_gemm_kernel<DgradProb>", "simt_gemm_kernel<WgradProb>")


# ------------------------------------------------------------------ (1) the SIMT kernel (impl 0) ------------------------------------------
# n, h, w, c, o, (kh, kw), (sh, sw), (ph, pw)
SIMT_GEOMS = {
    "c1_dis_conv2": (8, 28, 28, 1, 64, (5, 5), (2, 2), (0, 0)),      # C1's layers (reference_discriminator / reference_generator), batch 8
    "c1_dis_conv4": (8, 11, 11, 64, 128, (5, 5), (2, 2), (0, 0)),
    "c1_gen_conv6": (8, 14, 14, 128, 64, (5, 5), (1, 1), (2, 2)),
    "c1_gen_conv8": (8, 28, 28, 64, 1, (5, 5), (1, 1), (2, 2)),
    "asym": (2, 9, 11, 4, 6, (3, 5), (1, 2), (0, 2)),                # KH != KW, SH != SW, PH != PW
    "truncate": (2, 10, 10, 3, 5, (3, 3), (2, 2), (0, 0)),           # the last input row / column is read by no tap: its dgrad is 0 + bias
    "stride_gt_k_1x1": (2, 7, 9, 5, 6, (1, 1), (2, 2), (0, 0)),       # dgrad has holes
    "stride_gt_k_2x2": (2, 11, 8, 3, 4, (2, 2), (3, 3), (0, 0)),
    "pad_ge_k": (2, 5, 6, 3, 4, (2, 2), (1, 1), (2, 3)),             # border outputs see only padding
    "k_5x5x256": (2, 5, 5, 256, 8, (5, 5), (1, 1), (0, 0)),          # K = 6400: the rounding bound at a long reduction
}


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("name", list(SIMT_GEOMS))
def test_simt_kernel_geometries(b200, name, prec):
    b, ctx = b200
    g = geom(*SIMT_GEOMS[name])
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    for exact in (True, False):
        for kind in (0, 1):
            kw = dict(bias=True, scale=True, act="lrelu") if exact else dict(bias=True, scale=True, act="tanh")
            kern, sp = run_case(b, ctx, kind, 0, prec, g, rng, exact=exact, param_offset=0 if exact else 5, **kw)
            assert (kern, sp) == (SIMT_NAMES[kind], 1)
        kern, sp = run_case(b, ctx, 2, 0, prec, g, rng, exact=exact, param_offset=0 if exact else 3)
        assert (kern, sp) == (SIMT_NAMES[2], simt_wgrad_splits(g))


EPILOGUES = [(a, True, True) for a in ("identity", "tanh", "sigmoid", "relu", "lrelu")] + \
    [("identity", True, False), ("identity", False, True), ("relu", True, False), ("lrelu", False, True), ("sigmoid", False, False)]


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("epi", EPILOGUES, ids=[f"{a}{'_bias' if bb else ''}{'_scale' if s else ''}" for a, bb, s in EPILOGUES])
def test_simt_kernel_epilogues(b200, epi, prec):
    """act(acc * scale + bias), every activation with and without bias and scale, on fprop and dgrad (the (acc + bias) * scale order fails)."""
    b, ctx = b200
    act, bias, scale = epi
    g = geom(*SIMT_GEOMS["asym"])
    rng = np.random.default_rng(3)
    for kind in (0, 1):
        if act in ("identity", "relu", "lrelu"):
            run_case(b, ctx, kind, 0, prec, g, rng, exact=True, bias=bias, scale=scale, act=act)
        kern, _ = run_case(b, ctx, kind, 0, prec, g, rng, exact=False, bias=bias, scale=scale, act=act)
        assert kern == SIMT_NAMES[kind]


# 1x1 dense shapes at the 64 x 64 x 16 tile remainders: C, O and the pixel count N each cycle through their sets
TILE_C, TILE_O, TILE_N = (1, 3, 17, 63, 64, 65, 129), (1, 3, 17, 63, 64, 65, 129), (1, 63, 64, 65, 130)
TILE_CASES = [(TILE_N[(i + j) % 5], c, TILE_O[(i + j) % 7]) for i, c in enumerate(TILE_C) for j in (0, 3)]


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("case", TILE_CASES, ids=[f"n{n}_c{c}_o{oc}" for n, c, oc in TILE_CASES])
def test_simt_kernel_tile_remainders(b200, case, prec):
    b, ctx = b200
    n, c, oc = case
    g = geom(n, 1, 1, c, oc)
    rng = np.random.default_rng(n * 1000 + c * 10 + oc)
    for kind in (0, 1):
        assert run_case(b, ctx, kind, 0, prec, g, rng, exact=True, bias=True, act="relu", param_offset=1)[0] == SIMT_NAMES[kind]
    assert run_case(b, ctx, 2, 0, prec, g, rng, exact=True, param_offset=1) == (SIMT_NAMES[2], simt_wgrad_splits(g))


# the wgrad_splits regimes: (geometry, expected split count, what it covers)
WGRAD_REGIMES = {
    "direct_store": ((2, 9, 11, 4, 6, (3, 5), (1, 2), (0, 2)), 1),            # P = 108 < 512: one split, stored straight into dw
    "tiles_ge_296": ((1, 24, 25, 9472, 128, (1, 1)), 1),                       # 2 x 148 = 296 tiles: one split although P = 600
    "capped_by_p": ((1290, 1, 1, 16, 8), 5),                                   # one tile, P = 1290: P / 256 = 5 splits
    "64_empty_tail": ((5, 32, 116, 4, 1, (4, 4)), 64),                         # P = 16385: 64 splits of 272 pixels, the last three empty
}


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("name", list(WGRAD_REGIMES))
def test_simt_wgrad_split_regimes(b200, name, prec):
    b, ctx = b200
    args, want = WGRAD_REGIMES[name]
    g = geom(*args)
    assert simt_wgrad_splits(g) == want
    rng = np.random.default_rng(11)
    assert run_case(b, ctx, 2, 0, prec, g, rng, exact=True) == (SIMT_NAMES[2], want)
    assert run_case(b, ctx, 2, 0, prec, g, rng, exact=False, param_offset=7) == (SIMT_NAMES[2], want)


# ------------------------------------------------------------------ (2) the skinny-layer kernels (impl 2), 4x4 s2 p1 ----------------------
def edge_geom(n, oh, ow, c, oc):
    return geom(n, 2 * oh, 2 * ow, c, oc, (4, 4), (2, 2), (1, 1))


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("c", [1, 2, 3, 4])
def test_edge_deconv_small_c(b200, c, prec):
    """G-last's forward: transposed conv onto C <= 4 channels, bias + tanh; H != W, N = 1, and a batch whose grid-stride loop takes two passes."""
    b, ctx = b200
    sms = ctx.device_info()["sm_count"]
    rng = np.random.default_rng(20 + c)
    passes = 8 * sms * 128                                 # positions one pass of the capped grid covers
    for oc in (8, 24, 128):
        for n, oh, ow in ((1, 3, 5), (2, 5, 3)):
            g = edge_geom(n, oh, ow, c, oc)
            assert run_case(b, ctx, 1, 2, prec, g, rng, exact=True, bias=True, act="lrelu", param_offset=1)[0] == "edge_deconv_small_c_kernel"
            assert run_case(b, ctx, 1, 2, prec, g, rng, exact=False, bias=True, act="tanh", param_offset=3)[0] == "edge_deconv_small_c_kernel"
    n = passes // (32 * 16) + 2
    g = edge_geom(n, 32, 16, c, 8)
    assert n * 32 * 16 > passes
    assert run_case(b, ctx, 1, 2, prec, g, rng, exact=True, bias=True, act="relu")[0] == "edge_deconv_small_c_kernel"


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("c", [1, 2, 3, 4])
def test_edge_conv_small_cin(b200, c, prec):
    """D1's forward: conv from C <= 4 channels, bias + lrelu; O = 192 at C = 4 is exactly the 48 KB shared-memory predicate."""
    b, ctx = b200
    sms = ctx.device_info()["sm_count"]
    rng = np.random.default_rng(30 + c)
    for oc in (16, 48) + ((192,) if c == 4 else ()):
        for n, oh, ow in ((1, 3, 4), (2, 5, 8)):
            g = edge_geom(n, oh, ow, c, oc)
            assert run_case(b, ctx, 0, 2, prec, g, rng, exact=True, bias=True, act="lrelu", param_offset=1)[0] == "edge_conv_small_cin_kernel"
            assert run_case(b, ctx, 0, 2, prec, g, rng, exact=False, bias=True, act="lrelu", param_offset=2)[0] == "edge_conv_small_cin_kernel"
    per_img = 16 * (16 // 4) * (16 // 16)                  # output rows x pixel quads x 16-channel groups of one 32 x 32 image
    n = 8 * sms * 128 // per_img + 2
    assert run_case(b, ctx, 0, 2, prec, edge_geom(n, 16, 16, c, 16), rng, exact=True, bias=True, act="relu")[0] == "edge_conv_small_cin_kernel"


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("oc", [8, 24, 128, 136, 256])
def test_edge_wgrad_small_cin(b200, oc, prec):
    """D1 / G-last weight gradient at every C <= 4: one CTA with a 15-pixel tail, and a multi-CTA batch.  O = 136 and 256 need more than
    48 KB of dynamic shared memory."""
    b, ctx = b200
    sms = ctx.device_info()["sm_count"]
    rng = np.random.default_rng(40 + oc)
    for c in (1, 2, 3, 4):
        for n, oh, ow in ((1, 3, 5), (4, 8, 12)):
            g = edge_geom(n, oh, ow, c, oc)
            for exact, off in ((True, 1), (False, 0)):
                kern, sp = run_case(b, ctx, 2, 2, prec, g, rng, exact=exact, param_offset=off)
                assert (kern, sp) == ("edge_wgrad_small_cin_kernel", edge_wgrad_ctas(g, sms))
    assert edge_wgrad_ctas(edge_geom(1, 3, 5, 4, oc), sms) == 1


# ------------------------------------------------------------------ (3) the dense kernels (impl 4) ----------------------------------------
SMALL_O_N = (1, 7, 8, 9, 257)
SMALL_O_CASES = [(SMALL_O_N[(oc + ci + j) % 5], c, oc) for oc in (1, 2, 3, 4) for ci, c in enumerate((8, 24, 1032)) for j in (0, 2)]


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("case", SMALL_O_CASES, ids=[f"n{n}_c{c}_o{oc}" for n, c, oc in SMALL_O_CASES])
def test_dense_small_o(b200, case, prec):
    """<= 4 output units: forward with bias + activation, input gradient, split weight gradient; W / dW at an odd offset (load8_any's
    scalar path) and aligned."""
    b, ctx = b200
    n, c, oc = case
    g = geom(n, 1, 1, c, oc)
    rng = np.random.default_rng(n * 7 + c + oc)
    for off in (0, 3):
        assert run_case(b, ctx, 0, 4, prec, g, rng, exact=True, bias=True, act="lrelu", param_offset=off)[0] == "dense_small_o_fwd_kernel"
        assert run_case(b, ctx, 0, 4, prec, g, rng, exact=False, bias=True, act="sigmoid", param_offset=off)[0] == "dense_small_o_fwd_kernel"
        for exact in (True, False):
            assert run_case(b, ctx, 1, 4, prec, g, rng, exact=exact, param_offset=off)[0] == "dense_small_o_dgrad_kernel"
            assert run_case(b, ctx, 2, 4, prec, g, rng, exact=exact, param_offset=off) == ("dense_small_o_wgrad_kernel", dense_wgrad_splits(g))


SMALL_K_N = (1, 7, 8, 9, 63, 64, 65, 129)
SMALL_K_CASES = [(SMALL_K_N[(3 * i + ci) % 8], c, oc) for i, oc in enumerate((1, 5, 15, 16, 17, 100, 128)) for ci, c in enumerate((256, 768, 8192))]


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("case", SMALL_K_CASES, ids=[f"n{n}_c{c}_o{oc}" for n, c, oc in SMALL_K_CASES])
def test_dense_small_k(b200, case, prec):
    """Reduction of <= 128 (G-first): the input-gradient form with bias + activation and the weight gradient.  dW at an odd element offset
    is not 8-byte aligned: the SIMT kernel then stores scalars, and BF16 takes it instead of the mma.sync kernel."""
    b, ctx = b200
    n, c, oc = case
    g = geom(n, 1, 1, c, oc)
    rng = np.random.default_rng(n * 13 + c + oc)
    dgrad = "dense_small_k_dgrad_kernel" if prec == "fp32" else "dense_k_fwd_mma_kernel"
    for off in (0, 1, 2, 5):
        assert run_case(b, ctx, 1, 4, prec, g, rng, exact=True, bias=True, act="relu", param_offset=off)[0] == dgrad
        assert run_case(b, ctx, 1, 4, prec, g, rng, exact=False, bias=True, act="tanh", param_offset=off)[0] == dgrad
        if oc <= 4:          # gemm_wgrad takes the <= 4 output-unit kernel first
            wgrad = ("dense_small_o_wgrad_kernel", dense_wgrad_splits(g))
        elif off % 2:
            wgrad = ("dense_small_k_wgrad_kernel<st1>", 1)
        else:
            wgrad = ("dense_small_k_wgrad_kernel<st2>" if prec == "fp32" else "dense_k_wgrad_mma_kernel", 1)
        for exact in (True, False):
            assert run_case(b, ctx, 2, 4, prec, g, rng, exact=exact, param_offset=off) == wgrad


def test_hook_refuses_epilogues_the_wrappers_lack(b200):
    b, ctx = b200
    x = np.ones(8 * 24, np.float32); w = np.ones(24, np.float32); dy = np.ones(8, np.float32)
    g = geom(8, 1, 1, 24, 1)
    for kind, a, bb, size, kw in ((1, dy, w, 8 * 24, dict(bias=np.ones(24))), (1, dy, w, 8 * 24, dict(act="tanh")), (2, x, dy, 24, dict(act="relu")),
                                  (0, x, w, 8, dict(scale=np.ones(1))), (0, x, w, 8, dict(epi=b.EPI_STATS))):
        with pytest.raises(b.B200GanError) as e:
            b.test_conv_ex(ctx, kind, g, a, bb, size, impl=4, precision=b.FP32, **kw)
        assert e.value.code == -6, (kind, kw, str(e.value))          # B2G_ERR_UNSUPPORTED


# ------------------------------------------------------------------ (4) through the engine --------------------------------------------------
def _fp32_grads_and_fit(b, ctx, specs, in_shape, x, y, prec):
    rng = np.random.default_rng(2)
    onet = o.net_from_specs(specs, in_shape, quirks=o.Quirks(xent_clip_eps=0.0)); randomize(onet, rng)
    bnet = b.Net(ctx, specs, in_shape, max_batch=x.shape[0], precision=prec, xent_clip_eps=0.0)
    push_params(onet, bnet)
    s_o = onet.compute_gradient_and_score(x, y); s_b = bnet.compute_gradient_and_score(x, y)
    tol = TOL if prec == b.FP32 else 4e-2
    assert abs(s_b - s_o) < tol * max(1.0, abs(s_o)), (s_b, s_o)
    g_b, g_o = bnet.gradients(), onet.grads_flat(); off = 0
    for li, name, p, shape, _ in onet.param_table():
        k = int(np.prod(shape))
        if prec == b.FP32:
            assert rel_err(g_b[off:off + k], g_o[off:off + k]) < TOL, (name, p)
        else:
            d = np.linalg.norm(g_b[off:off + k] - g_o[off:off + k]) / (np.linalg.norm(g_o[off:off + k]) + 1e-30)
            assert d < 0.1, (name, p, d)
        off += k
    onet.fit(x, y); bnet.fit(x, y)
    if prec == b.FP32:
        assert rel_err(bnet.params(), onet.params_flat()) < TOL
    else:
        assert np.linalg.norm(bnet.params() - onet.params_flat()) / np.linalg.norm(onet.params_flat()) < 4e-2
    bnet.close()


def _bug1_nets():
    u = m.sgd(0.1)
    head = [{"type": "conv2d", "name": "c", "n_out": 5, "kernel": (4, 4), "stride": (1, 1), "padding": (0, 0), "activation": "tanh", "updater": u},
            {"type": "cnn_to_ff", "name": "flat"}, {"type": "output", "name": "out", "n_out": 1, "updater": u}]
    onexone = [{"type": "conv2d", "name": "c", "n_out": 1, "kernel": (1, 1), "activation": "tanh", "updater": u},
               {"type": "cnn_to_ff", "name": "flat"}, {"type": "dense", "name": "fc", "n_out": 10, "activation": "tanh", "updater": u},
               {"type": "output", "name": "out", "n_out": 1, "updater": u}]
    # full-window conv head: [b(5) | W(1280)], W at offset 5, the 1x1 geometry C = 256, O = 5;  1x1 conv (5 parameters) -> dense 256 -> 10:
    # the dense layer's W at offset 5, C = 256, O = 10.  Both weight gradients are dense_small_k_wgrad at an odd dW offset.
    return {"full_window_conv_head": (head, (16, 4, 4), 1), "dense_after_1x1_conv": (onexone, (4, 16, 16), 1)}


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("net", ["full_window_conv_head", "dense_after_1x1_conv"])
def test_dense_small_k_wgrad_at_odd_parameter_offset_through_the_engine(b200, net, prec):
    b, ctx = b200
    specs, in_shape, n_out = _bug1_nets()[net]
    rng = np.random.default_rng(9)
    x = rng.uniform(-1, 1, (8,) + in_shape); y = rng.uniform(0, 1, (8, n_out))
    _fp32_grads_and_fit(b, ctx, specs, in_shape, x, y, b.FP32 if prec == "fp32" else b.BF16)


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_dcgan_with_192_filters_steps(b200, prec):
    """D1 with 192 filters and G-last from 192 channels: edge_wgrad_small_cin at O = 192 needs 64 KB of dynamic shared memory."""
    b, ctx = b200
    P = b.BF16 if prec == "bf16" else b.FP32
    size, z, nf, n = 16, 12, 192, 8
    gs, ds = m.dcgan_generator(size, z, nf, 3, lr=1e-3), m.dcgan_discriminator(size, nf, 3, lr=1e-3)
    q = o.Quirks(xent_clip_eps=0.0)
    rng = np.random.default_rng(13)
    G = o.net_from_specs(gs, (z,), quirks=q, seed=1); D = o.net_from_specs(ds, (3, size, size), quirks=q, seed=2)
    randomize(G, rng); randomize(D, rng)
    bG = b.Net(ctx, gs, (z,), max_batch=n, precision=P, xent_clip_eps=0.0)
    bD = b.Net(ctx, ds, (3, size, size), max_batch=2 * n, precision=P, xent_clip_eps=0.0, bn_groups=2)
    push_params(G, bG); push_params(D, bD)
    x, z_d, z_g, y_r, y_f, y_g = [a.astype(np.float64) for a in o.synthetic_batch(n, size, 3, z, seed=5)]
    s_o = D.compute_gradient_and_score(x, y_r); s_b = bD.compute_gradient_and_score(x, y_r)
    tol = TOL if prec == "fp32" else 4e-2
    assert abs(s_b - s_o) < tol * max(1.0, abs(s_o))
    g_b, g_o = bD.gradients(), D.grads_flat(); off = 0
    for li, name, p, shape, _ in D.param_table():
        k = int(np.prod(shape))
        if p not in ("mean", "var"):
            if prec == "fp32":
                assert rel_err(g_b[off:off + k], g_o[off:off + k]) < tol, (name, p)
            else:
                d = np.linalg.norm(g_b[off:off + k] - g_o[off:off + k]) / (np.linalg.norm(g_o[off:off + k]) + 1e-30)
                assert d < 0.1, (name, p, d)
        off += k
    gan = b.Gan(bG, bD, use_cuda_graph=False)
    r = o.gan_step(G, D, x, z_d, z_g, y_r, y_f, y_g)
    losses = gan.step(x, z_d, z_g, y_r, y_f, y_g)
    want = np.array([r["loss_d_real"], r["loss_d_fake"], r["loss_g"]])
    assert np.all(np.abs(losses - want) < (tol if prec == "fp32" else 0.1) * np.maximum(1.0, np.abs(want))), (losses, want)
    if prec == "fp32":
        for onet, bnet in ((D, bD), (G, bG)):
            p_b, p_o = bnet.params(), onet.params_flat(); off = 0
            for li, name, p, shape, _ in onet.param_table():
                k = int(np.prod(shape))
                if p in ("mean", "var"):
                    assert rel_err(p_b[off:off + k], p_o[off:off + k]) < 2 * TOL, (name, p)
                else:
                    assert_close_up_to_sign_flips(p_b[off:off + k], p_o[off:off + k], 1e-3, TOL)
                off += k
    gan.close(); bG.close(); bD.close()
