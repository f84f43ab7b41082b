"""The persistent tensor-core conv kernel (kernels_tc.cu tc_conv_kernel) at multi-tile schedules.

A CTA walks the work items b, b + grid, ...: one TMA ring position runs on across its tiles, the consumers alternate between the
accumulator park slots (two for 64-column tiles and the pixel-shuffle tile, one for 128-column tiles), and the epilogue of one tile
overlaps the MMAs of the next.  The kernel's claim is that results do not depend on the grid.  Here every shape of CASES runs, at each
tile width its channels allow and with every epilogue the step uses, at grids of 1, 2, 3 and 5 CTAs, one CTA per tile and the production
grid (min(tiles, SMs)), each on an output poisoned with bf16 NaN:
  - every output element is finite (no tile left unwritten), and the production grid's output matches the float64 reference of
    tests/conv_ref.py under check_bf16, with the epilogue applied in float64 to the same bf16 operands;
  - outputs and fused BatchNorm statistics are bit-identical across all grids (per-tile arithmetic does not depend on the grid, and the
    statistics are added as integers);
  - the statistics match float64 sums of the stored output per group;
  - the hook reports the forced kernel instantiation.
test_schedule_table_reaches_every_corner (CPU) checks, with the schedule mirror of tests/tc_schedule.py, that the table exercises the
corners of the schedule: CTAs that reuse every park slot, every ring slot at the start of a CTA's second and later tiles, even and ragged
grids, and phase-form work items over several column tiles.
"""
import collections
import zlib

import numpy as np
import pytest

import conv_ref
import tc_schedule as ts
from helpers import b200, bf16_round, check_bf16

Case = collections.namedtuple("Case", "name kind n h w c o k s p groups tiles num_kb")
# kind: fprop (conv forward, 1x1 dense included), dgrad (4x4 s2 p1 input gradient in phase form: c = dx channels, o = dy channels), ps (the
# same onto c <= 4 channels, pixel-shuffle tile), wmn (dense input gradient: reduction c = the layer's nOut, o = its nIn, weight [c][o]).
# tiles / num_kb: work items at BN = 64 (16 for ps) and K-blocks per tile -- test_schedule_table_reaches_every_corner recomputes them.
CASES = [
    Case("dense 1x1 N4096 64-128 g2", "fprop", 4096, 1, 1, 64, 128, 1, 1, 0, 2, 64, 1),           # num_kb < STAGES: ring slot moves by 1 a tile
    Case("1x1 8x8 N16 64-192", "fprop", 16, 8, 8, 64, 192, 1, 1, 0, 1, 24, 1),                     # odd tiles_n (3), two images a tile
    Case("3x3 s1p1 16x16 N6 64-128 g3", "fprop", 6, 16, 16, 64, 128, 3, 1, 1, 3, 24, 9),           # Nt = 1, tiles_y = 2, odd num_kb
    Case("4x4 s2p1 16x16 N12 128-256 g2", "fprop", 12, 16, 16, 128, 256, 4, 2, 1, 2, 24, 32),      # D3-like, four column tiles
    Case("4x4 s2p1 16x16 N12 128-256 g3", "fprop", 12, 16, 16, 128, 256, 4, 2, 1, 3, 24, 32),
    Case("5x5 s2p2 16x16 N8 64-64", "fprop", 8, 16, 16, 64, 64, 5, 2, 2, 1, 4, 25),               # many taps, odd num_kb
    Case("2x2 s2p0 32x32 N4 192-128", "fprop", 4, 32, 32, 192, 128, 2, 2, 0, 1, 16, 12),           # three channel chunks
    Case("4x4 s2p1 8x32 N4 64-128", "fprop", 4, 8, 32, 64, 128, 4, 2, 1, 1, 4, 16),                # non-square: H / W not swapped
    Case("dgrad 16x16 N2 c64 o64", "dgrad", 2, 16, 16, 64, 64, 4, 2, 1, 1, 4, 4),                  # num_kb = STAGES; phases only
    Case("dgrad 32x32 N3 c192 o128", "dgrad", 3, 32, 32, 192, 128, 4, 2, 1, 1, 72, 8),             # tiles_n = 3 x 4 phases
    Case("dgrad 8x8 N24 c128 o320 g3", "dgrad", 24, 8, 8, 128, 320, 4, 2, 1, 3, 24, 20),           # Nt = 8
    Case("dgrad 8x32 N4 c64 o64", "dgrad", 4, 8, 32, 64, 64, 4, 2, 1, 1, 8, 4),                    # non-square (dgrad)
    Case("ps 64x64 N4 c3 o64", "ps", 4, 64, 64, 3, 64, 4, 2, 1, 1, 32, 9),                         # C = 3: packed 32-bit stores
    Case("ps 16x16 N8 c1 o192", "ps", 8, 16, 16, 1, 192, 4, 2, 1, 1, 4, 27),
    Case("ps 16x16 N8 c4 o192", "ps", 8, 16, 16, 4, 192, 4, 2, 1, 1, 4, 27),
    Case("wmn N256 1024-1024", "wmn", 256, 1, 1, 1024, 1024, 1, 1, 0, 1, 32, 16),                  # the C5 hidden-layer input gradient
    Case("wmn N1024 64-64", "wmn", 1024, 1, 1, 64, 64, 1, 1, 0, 1, 8, 1),
]

EPIS = {
    "fprop": ["plain", "bias_lrelu", "affine_relu", "stats", "bnbwd_relu", "bnbwd_lrelu", "actbwd_lrelu", "actbwd_tanh"],
    "ps": ["bias_tanh", "actbwd_tanh"],
    "wmn": ["plain", "bnbwd_relu", "actbwd_lrelu"],
}
EPIS["dgrad"] = EPIS["fprop"]


def tile_widths(case):
    if case.kind == "ps":
        return [16]
    oc = case.c if case.kind == "dgrad" else case.o
    return [bn for bn in (64, 128) if oc % bn == 0]


def geometry(case, bn):
    return ts.geometry(case.kind, case.n, case.h, case.w, case.c, case.o, case.k, case.s, case.p, None if case.kind == "ps" else bn)


def grids(tiles):
    """The max_ctas values each run is launched with: 0 = production (min(tiles, SMs)), a few small grids, one CTA per tile."""
    return sorted({0, 1, 2, 3, 5, tiles})


RUNS = [(case, bn, epi) for case in CASES for bn in tile_widths(case) for epi in EPIS[case.kind]]


# ------------------------------------------------------------------------------------------------ CPU: what the table reaches
def test_schedule_table_reaches_every_corner():
    long_cta = {1: False, 2: False}          # park count -> some CTA runs >= 2 * PARKS + 1 tiles (every slot reused, parity flipped twice)
    slots = set()                            # ring slots at the start of a CTA's tile with local index >= 1
    even = uneven = phases_x_cols = False
    for case in CASES:
        for bn in tile_widths(case):
            geo = geometry(case, bn)
            assert geo is not None, case.name
            if bn in (16, 64):
                assert (geo["tiles"], geo["num_kb"]) == (case.tiles, case.num_kb), (case.name, geo)
            if case.kind != "ps":
                assert case.n // case.groups % geo["Nt"] == 0, f"{case.name}: a statistics group must hold whole tiles"
            for mc in grids(geo["tiles"]):
                grid = ts.grid_size(geo["tiles"], mc)
                even |= geo["tiles"] % grid == 0
                uneven |= geo["tiles"] % grid != 0
                for cta in range(grid):
                    local = ts.cta_tiles(geo["tiles"], grid, cta)
                    if len(local) >= 2 * ts.parks(bn) + 1:
                        long_cta[ts.parks(bn)] = True
                    slots |= {ts.ring_slot_at_tile_start(i, geo["num_kb"]) for i in range(1, len(local))}
            phases_x_cols |= geo["phases"] == 4 and geo["tiles_n"] > 1
    assert long_cta == {1: True, 2: True}, long_cta
    assert slots == set(range(ts.STAGES)), slots
    assert even and uneven
    assert phases_x_cols


# ------------------------------------------------------------------------------------------------ GPU
_OPERANDS = {}


def operands(case):
    """(hook geometry, a, b, output shape, float64 GEMM result) of a case; a / b bf16-rounded, shared by all its runs."""
    if case.name in _OPERANDS:
        return _OPERANDS[case.name]
    rng = np.random.default_rng(1000 + CASES.index(case))
    n, h, w, c, o, k, s, p = case.n, case.h, case.w, case.c, case.o, case.k, case.s, case.p
    if case.kind in ("fprop", "wmn"):
        oh, ow = conv_ref.out_size(h, k, s, p), conv_ref.out_size(w, k, s, p)
        geom = dict(n=n, h=h, w=w, c=c, oh=oh, ow=ow, o=o, kh=k, kw=k, sh=s, sw=s, ph=p, pw=p)
        a = bf16_round(rng.standard_normal((n, h, w, c)))
        if case.kind == "wmn":
            wt = bf16_round(rng.standard_normal((c, o)) / np.sqrt(c))
            gemm, oshape = conv_ref.dense(a.reshape(n, c), wt, w_mn=True), (n, o)
        else:
            wt = bf16_round(rng.standard_normal((o, k, k, c)) / np.sqrt(k * k * c))
            gemm = conv_ref.conv2d(a, wt, s, p); oshape = gemm.shape
    else:
        geom = dict(n=n, h=h, w=w, c=c, oh=h // 2, ow=w // 2, o=o, kh=4, kw=4, sh=2, sw=2, ph=1, pw=1)
        a = bf16_round(rng.standard_normal((n, h // 2, w // 2, o)))
        wt = bf16_round(rng.standard_normal((o, 4, 4, c)) / np.sqrt(4 * o))
        gemm = conv_ref.conv2d_input_grad(a, wt, (h, w), 2, 1); oshape = gemm.shape
    _OPERANDS[case.name] = (geom, a, wt, oshape, gemm)
    return _OPERANDS[case.name]


def epilogue(b, name, gemm, oshape, groups, rng):
    """Hook keyword arguments of an epilogue and its float64 result on the GEMM output (aux operands bf16-rounded, as the kernel reads them)."""
    oc = oshape[-1]
    lrelu_grad = lambda v: np.where(v > 0, 1.0, 0.2)
    if name == "plain":
        return {}, gemm
    if name in ("bias_lrelu", "bias_tanh"):
        bias = (0.1 * rng.standard_normal(oc)).astype(np.float32)
        z = gemm + bias.astype(np.float64)
        if name == "bias_tanh":
            return dict(act="tanh", bias=bias), np.tanh(z)
        return dict(act="lrelu", alpha=0.2, bias=bias), np.where(z > 0, z, 0.2 * z)
    if name == "affine_relu":
        scale = rng.uniform(0.5, 1.5, oc).astype(np.float32); shift = (0.2 * rng.standard_normal(oc)).astype(np.float32)
        return dict(act="relu", bias=shift, scale=scale), np.maximum(gemm * scale.astype(np.float64) + shift.astype(np.float64), 0)
    if name == "stats":
        return dict(epi=b.EPI_STATS, groups=groups), gemm
    if name.startswith("bnbwd"):
        z = bf16_round(rng.standard_normal(oshape))
        u = z * rng.uniform(0.5, 1.5, oc) + 0.3 * rng.standard_normal(oc)
        if name == "bnbwd_relu":
            y = bf16_round(np.maximum(u, 0))
            return dict(epi=b.EPI_BNBWD, act="relu", groups=groups, aux=y, aux2=z), gemm * (y > 0)
        y = bf16_round(np.where(u > 0, u, 0.2 * u))
        return dict(epi=b.EPI_BNBWD, act="lrelu", alpha=0.2, groups=groups, aux=y, aux2=z), gemm * lrelu_grad(y)
    if name == "actbwd_lrelu":
        a = bf16_round(rng.standard_normal(oshape))
        return dict(epi=b.EPI_ACTBWD, act="lrelu", alpha=0.2, aux=a), gemm * lrelu_grad(a)
    if name == "actbwd_tanh":
        a = bf16_round(np.tanh(rng.standard_normal(oshape)))
        return dict(epi=b.EPI_ACTBWD, act="tanh", aux=a), gemm * (1.0 - a.astype(np.float64) ** 2)
    raise ValueError(name)


@pytest.mark.gpu
@pytest.mark.parametrize("case,bn,epi", RUNS, ids=[f"{c.name}-bn{bn}-{e}" for c, bn, e in RUNS])
def test_tc_conv_results_do_not_depend_on_the_grid(b200, case, bn, epi):
    b, ctx = b200
    geom, a, wt, oshape, gemm = operands(case)
    geo = geometry(case, bn)
    kw, ref = epilogue(b, epi, gemm, oshape, case.groups, np.random.default_rng(zlib.crc32(f"{case.name}/{epi}".encode())))
    kind = 0 if case.kind in ("fprop", "wmn") else 1
    impl, force_bn = (3, 0) if case.kind == "ps" else (1, bn)
    kernel = "tc_conv_kernel<16,4,PS>" if case.kind == "ps" else f"tc_conv_kernel<{bn},4>"
    size = int(np.prod(oshape))
    what = f"{case.name} BN {bn} {epi}"
    runs = {}
    for mc in grids(geo["tiles"]):
        out, stats, k, _ = b.test_conv_ex(ctx, kind, geom, a, wt, size, impl=impl, bn=force_bn, max_ctas=mc, poison=True, w_mn=case.kind == "wmn", **kw)
        assert k == kernel, f"{what}: max_ctas={mc} ran {k}"
        bad = ~np.isfinite(out)
        assert not bad.any(), f"{what}: max_ctas={mc}: {bad.sum()} of {out.size} output elements non-finite (first at flat index {np.argmax(bad)})"
        runs[mc] = (out, stats)
    out, stats = runs[0]
    check_bf16(out.reshape(oshape), ref, f"{what} (production grid)")
    for mc, (o2, s2) in runs.items():
        diff = o2.view(np.uint32) != out.view(np.uint32)
        assert not diff.any(), f"{what}: max_ctas={mc}: {diff.sum()} elements differ from the production grid (first at flat index {np.argmax(diff)})"
        if stats is not None:
            assert np.array_equal(s2, stats), f"{what}: max_ctas={mc}: BatchNorm statistics differ from the production grid's"
    if stats is not None:
        og = out.reshape(case.groups, -1, oshape[-1]).astype(np.float64)
        second = og ** 2 if epi == "stats" else og * np.asarray(kw["aux2"], np.float64).reshape(og.shape)
        np.testing.assert_allclose(stats[:, 0, :], og.sum(1), rtol=2e-5, atol=2e-3, err_msg=what)
        np.testing.assert_allclose(stats[:, 1, :], second.sum(1), rtol=2e-5, atol=5e-3 if epi != "stats" else 2e-3, err_msg=what)
