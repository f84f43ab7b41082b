"""The slab path of the tensor-core conv kernel (kernels_tc.cu tc_conv_kernel<..., SLAB>).

In a 4x4 stride-2 pad-1 conv forward the 16 taps fall into four (ky mod 2, kx mod 2) classes, and in the phase-form input gradient each
sub-pixel phase has 2x2 taps; inside a class the taps of one column read the same activations one row of the row grid apart.  Where the
tile's row grid allows it (64-column tiles; Wt % 8 == 0; one image of at least two rows per tile, or two images, one per MMA warpgroup; at
most 144 slab rows) the producer loads one slab box of Nt x (Ht+1) x Wt rows per (row pair, column tap, channel chunk) and the MMA warpgroups run the two
taps from descriptors Wt rows apart.  Other shapes keep one activation box per tap.

CPU: a model of the slab schedule, independent of the kernel's code, checks that
  - the two taps of every K unit read exactly the slab's rows (the slab covers the footprint of its taps, no more), that the slab element
    each tap reads at each output pixel is the input element the convolution needs, with the halo rows at the top and bottom of the image
    and the columns left / right of it outside the tensor (TMA zero fill) exactly where the padding is;
  - the table below reaches every (ring slot, phase parity) a slab schedule can start a CTA's second or later tile in.
GPU: every case runs at each tile width its channels allow, with every epilogue the step uses, at grids of 1, 2, 3 and 5 CTAs, one CTA per
tile and the production grid, on outputs poisoned with bf16 NaN: every element against the float64 reference of tests/conv_ref.py,
outputs and BatchNorm statistics bit-identical across grids, the kernel label and the activation path (slab or per tap) as the model
predicts.  The production grid is also run on the per-tap path, which must match the same reference.
"""
import collections
import zlib

import numpy as np
import pytest

import conv_ref
import test_gpu_tc_conv_schedule as sched
from helpers import b200, bf16_round, check_bf16

SLAB_ROWS = 144
SMS = 132
Case = collections.namedtuple("Case", "name kind n h w c o groups")
# kind fprop: x [n, h, w, c] -> y [n, h/2, w/2, o]; dgrad: dy [n, h/2, w/2, o] -> dx [n, h, w, c].  All 4x4 s2 p1.
CASES = [
    Case("fprop 32x32 N2 64-128 g2", "fprop", 2, 32, 32, 64, 128, 2),          # 16x16 grid: Nt 1, Ht 8, Wt 16
    Case("fprop 64x64 N1 64-64", "fprop", 1, 64, 64, 64, 64, 1),               # 32x32 grid: per tap (a 160-row slab)
    Case("fprop 16x16 N4 128-128 g2", "fprop", 4, 16, 16, 128, 128, 2),        # 8x8 grid: two images a tile
    Case("fprop 16x64 N2 64-128", "fprop", 2, 16, 64, 64, 128, 1),             # 8x32 grid: per tap (two images of 3 x 32 rows)
    Case("fprop 8x8 N16 64-128 g2", "fprop", 16, 8, 8, 64, 128, 2),            # 4x4 grid: per tap (Wt 4)
    Case("dgrad 32x32 N2 c64 o128 g2", "dgrad", 2, 32, 32, 64, 128, 2),        # 16x16 phase grid
    Case("dgrad 64x64 N1 c128 o64", "dgrad", 1, 64, 64, 128, 64, 1),           # 32x32 phase grid: per tap
    Case("dgrad 16x16 N4 c128 o128 g2", "dgrad", 4, 16, 16, 128, 128, 2),      # 8x8 phase grid, two images a tile
    Case("dgrad 16x32 N2 c64 o64", "dgrad", 2, 16, 32, 64, 64, 1),             # 8x16 phase grid: non-square, one tile an image
    Case("dgrad 8x8 N16 c128 o64 g2", "dgrad", 16, 8, 8, 128, 64, 2),          # 4x4 phase grid: per tap
]


# ------------------------------------------------------------------------------------------------ the schedule model
def row_tile(n, gh, gw, rows=128):
    p = gh * gw
    if gw > rows or rows % gw:
        return None
    if p >= rows:
        ht = rows // gw
        return (1, ht, gw) if p % rows == 0 and gh % ht == 0 else None
    if rows % p or n % (rows // p):
        return None
    return rows // p, gh, gw


def slab_applies(nt, ht, wt, bn):
    return bn == 64 and wt % 8 == 0 and ((nt == 1 and ht >= 2) or (nt == 2 and ht * wt == 64)) and nt * (ht + 1) * wt <= SLAB_ROWS


def grid_of(case):
    return case.h // 2, case.w // 2


def schedule(case, bn):
    """Work items, K units per work item and ring depth of a case at tile width bn."""
    gh, gw = grid_of(case)
    nt, ht, wt = row_tile(case.n, gh, gw)
    tiles_m = case.n * gh * gw // 128
    slab = slab_applies(nt, ht, wt, bn)
    if case.kind == "fprop":
        items, chunks = tiles_m * (case.o // bn), case.c // 64
        units = (2 * 4 if slab else 16) * chunks
    else:
        items, chunks = tiles_m * (case.c // bn) * 4, case.o // 64
        units = (2 if slab else 4) * chunks
    return dict(Nt=nt, Ht=ht, Wt=wt, slab=slab, tiles=items, units=units, stages=4)


def unit_taps(kind, pair, tb, py=0, px=0):
    """The (row offset, column offset, filter row, filter column) of the lower and upper tap of a K unit.  Offsets are in the row grid
    (fprop: input rows / columns 2 y + off; dgrad: dy rows / columns q + off)."""
    if kind == "fprop":
        return [(-1 + ky, -1 + tb, ky, tb) for ky in (pair, pair + 2)]      # input row 2 oy - 1 + ky
    # dgrad phase (py, px): output row 2 q + py takes dy row q + d through filter row r with 2 (q + d) - 1 + r = 2 q + py
    taps = []
    for d in ((-1, 0) if py == 0 else (0, 1)):
        dc = (-1, 0) if px == 0 else (0, 1)
        e = dc[tb]
        taps.append((d, e, py + 1 - 2 * d, px + 1 - 2 * e))
    return taps


def slab_box(kind, case, y0, n0, nt, ht, wt, taps):
    """Rows of the slab box the producer loads for a unit: (image, grid row, grid column) per slab row, in load order, and whether each
    lies inside the tensor.  The box starts at the lower tap's offsets; fprop samples every second input row / column."""
    lo = taps[0]
    out = []
    for i in range(nt):
        for r in range(ht + 1):
            for cc in range(wt):
                if kind == "fprop":
                    iy, ix = 2 * (y0 + r) + lo[0], 2 * cc + lo[1]
                    inside = 0 <= iy < case.h and 0 <= ix < case.w
                else:
                    iy, ix = y0 + r + lo[0], cc + lo[1]
                    inside = 0 <= iy < case.h // 2 and 0 <= ix < case.w // 2
                out.append((n0 + i, iy, ix, inside))
    return out


def test_slab_boxes_cover_exactly_the_taps_footprint():
    seen_top_halo = seen_bottom_halo = seen_left = seen_right = False
    for case in CASES:
        gh, gw = grid_of(case)
        nt, ht, wt = row_tile(case.n, gh, gw)
        if not slab_applies(nt, ht, wt, 64):
            continue
        wg_rows = 64 if nt == 1 else (ht + 1) * wt
        phases = [(0, 0)] if case.kind == "fprop" else [(0, 0), (0, 1), (1, 0), (1, 1)]
        for y0 in range(0, gh if nt == 1 else 1, ht):
            for (py, px) in phases:
                for pair in ((0, 1) if case.kind == "fprop" else (0,)):
                    for tb in range(4 if case.kind == "fprop" else 2):
                        taps = unit_taps(case.kind, pair, tb, py, px)
                        assert taps[1][0] == taps[0][0] + (2 if case.kind == "fprop" else 1) and taps[1][1] == taps[0][1]
                        box = slab_box(case.kind, case, y0, 0, nt, ht, wt, taps)
                        used = set()
                        for row in range(128):                       # accumulator row -> (image, grid row, grid column) of the tile
                            img, yy, xx = row // (ht * wt), row % (ht * wt) // wt, row % wt
                            wg, r_in = row // 64, row % 64
                            for t, (dy, dx, fr, fc) in enumerate(taps):
                                # descriptor: warpgroup base + t * Wt rows, then the warpgroup's row r_in
                                srow = wg * wg_rows + t * wt + r_in
                                n_, iy, ix, inside = box[srow]
                                if case.kind == "fprop":
                                    want = (img, 2 * (y0 + yy) - 1 + fr, 2 * xx - 1 + fc)
                                    need_inside = 0 <= want[1] < case.h and 0 <= want[2] < case.w
                                else:
                                    want = (img, y0 + yy + dy, xx + dx)
                                    need_inside = 0 <= want[1] < gh and 0 <= want[2] < gw
                                    assert 0 <= fr < 4 and 0 <= fc < 4
                                assert (n_, iy, ix) == want, (case.name, y0, py, px, pair, tb, row, t)
                                assert inside == need_inside
                                used.add(srow)
                        assert used == set(range(len(box))), f"{case.name}: slab rows no tap reads"
                        seen_top_halo |= not box[0][3] and box[0][1] < 0
                        seen_bottom_halo |= any(not r[3] and r[1] >= (case.h if case.kind == "fprop" else gh) for r in box)
                        seen_left |= any(r[2] < 0 for r in box)
                        seen_right |= any(r[2] >= (case.w if case.kind == "fprop" else gw) for r in box)
    assert seen_top_halo and seen_bottom_halo and seen_left and seen_right


def test_slab_table_reaches_every_ring_slot():
    """(ring slot, phase parity) at the start of every tile a CTA runs after its first.  A tile has 2 or 8 K units per channel chunk, so on
    the 4-deep ring a tile starts in slot 0 or 2; the table must reach both, each with both parities."""
    slots = set()
    for case in CASES:
        for bn in tile_widths(case):
            s = schedule(case, bn)
            assert case.n // case.groups % s["Nt"] == 0, f"{case.name}: a statistics group must hold whole tiles"
            if not s["slab"]:
                continue
            for mc in sched.grids(s["tiles"]):
                grid = min(s["tiles"], mc if mc > 0 else SMS)
                for cta in range(grid):
                    local = list(range(cta, s["tiles"], grid))
                    st = s["stages"]
                    slots |= {(i * s["units"] % st, i * s["units"] // st % 2) for i in range(1, len(local))}
    assert slots == {(0, 0), (0, 1), (2, 0), (2, 1)}, slots


def tile_widths(case):
    oc = case.o if case.kind == "fprop" else case.c
    return [bn for bn in (64, 128) if oc % bn == 0]


# ------------------------------------------------------------------------------------------------ GPU
RUNS = [(case, bn, epi) for case in CASES for bn in tile_widths(case) for epi in sched.EPIS[case.kind]]
_OPERANDS = {}


def operands(case):
    if case.name in _OPERANDS:
        return _OPERANDS[case.name]
    rng = np.random.default_rng(2000 + CASES.index(case))
    n, h, w, c, o = case.n, case.h, case.w, case.c, case.o
    geom = dict(n=n, h=h, w=w, c=c, oh=h // 2, ow=w // 2, o=o, kh=4, kw=4, sh=2, sw=2, ph=1, pw=1)
    if case.kind == "fprop":
        a = bf16_round(rng.standard_normal((n, h, w, c)))
        wt = bf16_round(rng.standard_normal((o, 4, 4, c)) / np.sqrt(16 * c))
        gemm = conv_ref.conv2d(a, wt, 2, 1)
    else:
        a = bf16_round(rng.standard_normal((n, h // 2, w // 2, o)))
        wt = bf16_round(rng.standard_normal((o, 4, 4, c)) / np.sqrt(4 * o))
        gemm = conv_ref.conv2d_input_grad(a, wt, (h, w), 2, 1)
    _OPERANDS[case.name] = (geom, a, wt, gemm.shape, gemm)
    return _OPERANDS[case.name]


@pytest.mark.gpu
@pytest.mark.parametrize("case,bn,epi", RUNS, ids=[f"{c.name}-bn{bn}-{e}" for c, bn, e in RUNS])
def test_slab_path_results(b200, case, bn, epi):
    b, ctx = b200
    geom, a, wt, oshape, gemm = operands(case)
    s = schedule(case, bn)
    kw, ref = sched.epilogue(b, epi, gemm, oshape, case.groups, np.random.default_rng(zlib.crc32(f"{case.name}/{epi}".encode())))
    kind = 0 if case.kind == "fprop" else 1
    size = int(np.prod(oshape))
    what = f"{case.name} BN {bn} {epi}"
    runs = {}
    for mc in sched.grids(s["tiles"]):
        info = {}
        out, stats, k, _ = b.test_conv_ex(ctx, kind, geom, a, wt, size, bn=bn, max_ctas=mc, poison=True, info=info, **kw)
        assert k == f"tc_conv_kernel<{bn},4>", f"{what}: max_ctas={mc} ran {k}"
        assert info["slab"] == s["slab"], f"{what}: slab path {info['slab']}, expected {s['slab']}"
        check_bf16(out.reshape(oshape), ref, f"{what} max_ctas={mc}")
        runs[mc] = (out, stats)
    out, stats = runs[0]
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
    info = {}
    pt, _, k, _ = b.test_conv_ex(ctx, kind, geom, a, wt, size, bn=bn, poison=True, per_tap=True, info=info, **kw)
    assert k == f"tc_conv_kernel<{bn},4>" and not info["slab"]
    check_bf16(pt.reshape(oshape), ref, f"{what} (per-tap path)")
