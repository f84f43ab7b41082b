"""The tensor-core weight gradients and the skinny-layer conv forward (kernels_tc.cu) at every split schedule, bit for bit on integer operands.

tc_wgrad_kernel<BNW,4> splits the reduction over pixels into 64-pixel K-blocks (Nt images x Ht rows x Wt columns of the dy grid):
split b runs K-blocks [b * kb_per_split, min(kb_total, (b + 1) * kb_per_split)), kb_per_split = ceil(kb_total / splits), so the last
split can be ragged or empty, and a split can start in the middle of an image.  Each CTA writes one fp32 partial per split, and the
partials are summed in fixed order, right away or in the backward pass's one reduce-list launch (defer).  tc_edge_wgrad_kernel (D1 and
G-last, <= 4 image channels) walks tiles_per_cta consecutive 128-pixel tiles per CTA, prefetching the next tile's slab, builds the im2col
rows in shared memory (odd C: a funnel-shift row builder) and, for C < 4, adds a ones column that makes the MMA produce the bias gradient
too.  tc_edge_conv_kernel is the D1 forward with its bias and activation fused in.

The hook b2g_test_conv_ex forces the split count (splits) and the edge conv's CTA target (max_ctas), poisons dw, db, the partials and
the output with NaN before every launch, and can put dw / db a few elements past an aligned address (param_offset).  Each case runs at the
production split (asserted against the mirror below, at the card's SM count), at 1, 2 and 3 splits, at counts that leave a split ragged
or empty, and at one K-block (or tile) per split and beyond:

* integer operands: x and dy from {-3, -2, -1, 1, 2, 3} (no zeros, so a padding / data mix-up or a dropped or doubled pixel changes a
  sum) with N * OH * OW <= 2^18.  Products are exact in bf16 and every partial and total is an integer below 2^22, exact in fp32 in any
  order: dw (and db = sum dy) must equal float64 conv_ref.conv2d_weight_grad bit for bit, immediate and deferred.  The edge conv takes x
  from {-2, -1, 1, 2}, w from {-1, 1} and an integer bias in [-8, 8]: |acc + bias| <= 136 is exact in fp32 and in bf16, so identity,
  relu and lrelu(0.2) outputs equal bf16_rn(float32(act(float32(acc + bias)))) bit for bit, tanh lies within one bf16 ulp of float64,
  and every output is bit-identical across CTA targets.
* normal operands, bf16-rounded: at the production schedule, max|err| <= 1e-4 max|ref| for the weight gradients, check_bf16 for the
  edge conv with each epilogue, and every element finite.

test_table_reaches_every_corner (CPU) checks with the mirror that the tables reach the corners of both schedules.
"""
import collections
import zlib

import numpy as np
import pytest

import conv_ref
import tc_schedule as ts
from helpers import b200, bf16_round, check_bf16, rel_err

SMS = ts.SMS                 # H100 SXM
STAGES = 4                   # TMA ring depth of tc_wgrad_kernel<BNW, 4>
EDGE_SLAB_BYTES = 6144       # kernels_tc.cu EDGE_SLAB_BYTES


# ------------------------------------------------------------------------------------------------ mirror of the host-side schedule
def out_hw(h, w, k, s, p):
    return conv_ref.out_size(h, k, s, p), conv_ref.out_size(w, k, s, p)


def wgrad_bnw(c, k):
    """Columns of the (tap, c) axis per CTA: 128 where the k*k*c columns split into 128-column blocks, else 64; 0 when C % 64 != 0."""
    if c % 64:
        return 0
    return 128 if (k * k * c) % 128 == 0 else 64


def wgrad_tile(n, h, w, c, o, k, s, p):
    """(Nt, Ht, Wt) of a 64-pixel K-block, or None where tc_wgrad_supported is false."""
    oh, ow = out_hw(h, w, k, s, p)
    t = ts.row_tile(n, oh, ow, 64)
    if o % 128 or not wgrad_bnw(c, k) or not 1 <= s <= 2 or (n * oh * ow) % 64 or t is None or t[2] * s > 256 or t[1] * s > 256:
        return None
    return t


def wgrad_splits_for(n, h, w, c, o, k, s, p, sms=SMS):
    """Production split count: the whole grid (o tiles x column blocks x splits) is at most 2 * SMs / 3 CTAs, at most kb_total / 8 splits."""
    oh, ow = out_hw(h, w, k, s, p)
    tiles = (o // 128) * (k * k * c // wgrad_bnw(c, k))
    kbt = n * oh * ow // 64
    return max(1, min((2 * sms) // 3 // tiles, max(1, kbt // 8)))


def split_ranges(kb_total, splits):
    """[(kb_beg, num_kb)] of every split, as tc_wgrad_kernel computes them."""
    per = -(-kb_total // splits)
    return [(b * per, max(0, min(kb_total, b * per + per) - b * per)) for b in range(splits)]


def edge_tile(n, h, w, c):
    """Ht (output rows per 128-pixel tile) of the 4x4 s2 p1 skinny-layer kernels, or None where they do not apply."""
    oh, ow = h // 2, w // 2
    if not 1 <= c <= 4 or ow > 128 or 128 % ow:
        return None
    ht = 128 // ow
    if oh % ht or (w * c) % 8 or (2 * ht + 2) * w * c * 2 > EDGE_SLAB_BYTES:
        return None
    return ht


def edge_ctas(tiles, target):
    """(CTAs, tiles per CTA) of the edge kernels: tiles_per_cta = ceil(tiles / target).  Production targets: 2 x SMs for the weight
    gradient, 8 x SMs for the conv forward; the hook's splits / max_ctas replace them."""
    tpc = max(1, -(-tiles // target))
    return -(-tiles // tpc), tpc


# ------------------------------------------------------------------------------------------------ the tables
WCase = collections.namedtuple("WCase", "name n h w c o k s p extra offsets")
# extra: split counts besides production, 1, 2, 3, kb_total and kb_total + 2 (ragged / empty last splits); offsets: param_offset runs
WGRAD_CASES = [
    WCase("C5 hidden 1x1 N256 1024-1024", 256, 1, 1, 1024, 1024, 1, 1, 0, (), True),     # Nt = 64, kb_total 4, 8 o-tiles
    WCase("1x1 N4096 64-128", 4096, 1, 1, 64, 128, 1, 1, 0, (7,), False),                # BNW 64, Nt = 64, production 8 splits
    WCase("4x4s2p1 16x16 N81 64-128", 81, 16, 16, 64, 128, 4, 2, 1, (10,), True),        # kb_total 81: 10 splits leave the tenth empty
    WCase("3x3s1p1 16x16 N4 64-128", 4, 16, 16, 64, 128, 3, 1, 1, (5,), False),          # tiles_y 4: 3 splits start mid-image; BNW 64
    WCase("4x4s2p1 32x32 N2 192-128", 2, 32, 32, 192, 128, 4, 2, 1, (5,), True),         # 128-column blocks straddle two taps
    WCase("5x5s2p2 16x16 N8 64-128", 8, 16, 16, 64, 128, 5, 2, 2, (5,), False),          # 25 taps, BNW 64
    WCase("2x2s2p0 32x32 N4 128-256", 4, 32, 32, 128, 256, 2, 2, 0, (5,), False),        # two o-tiles, no padding
    WCase("4x4s2p1 8x32 N4 64-128", 4, 8, 32, 64, 128, 4, 2, 1, (), False),              # non-square
    WCase("4x4s2p1 4x4 N32 256-512", 32, 4, 4, 256, 512, 4, 2, 1, (), False),            # 2x2 grid, Nt = 16, four o-tiles
    WCase("4x4s1p0 4x4 N128 256-128", 128, 4, 4, 256, 128, 4, 1, 0, (), False),          # full-window conv, Nt = 64
    WCase("3x3s1p1 64x64 N2 64-128", 2, 64, 64, 64, 128, 3, 1, 1, (), True),             # Wt = 64, stride 1, tiles_y 64
    WCase("C4 D2 4x4s2p1 128x128 N2 64-128", 2, 128, 128, 64, 128, 4, 2, 1, (), False),  # Wt * SW = 128
    WCase("4x4s2p1 16x16 N4 64-128", 4, 16, 16, 64, 128, 4, 2, 1, (), False),            # one image per K-block
    WCase("4x4s2p1 32x32 N2 128-128", 2, 32, 32, 128, 128, 4, 2, 1, (), False),          # four rows per K-block
    WCase("4x4s2p1 8x8 N16 256-256", 16, 8, 8, 256, 256, 4, 2, 1, (), False),            # four images per K-block, two o-tiles
]

ECase = collections.namedtuple("ECase", "name n h w")
# 4x4 s2 p1 from C <= 4 image channels; OW = w / 2 output columns, 128 / OW output rows per tile
EDGE_GEOMS = [
    ECase("ow4 64x8 N270", 270, 64, 8),         # 270 tiles: several tiles per CTA at the production target (2 x SMs)
    ECase("ow8 32x16 N5", 5, 32, 16),
    ECase("ow16 32x32 N5", 5, 32, 32),          # two tiles per image
    ECase("ow32 32x64 N5", 5, 32, 64),          # non-square
    ECase("ow64 64x128 N1", 1, 64, 128),        # C = 4: the slab holds exactly 6144 bytes
    ECase("ow128 16x256 N1", 1, 16, 256),       # C = 3: the slab holds exactly 6144 bytes; C = 4 does not fit
]
EDGE_CASES = [(c, g) for c in (1, 2, 3, 4) for g in EDGE_GEOMS if edge_tile(g.n, g.h, g.w, c)]
EDGE_OUT = (64, 128, 192)
EDGE_EPIS = ["plain", "bias_identity", "bias_relu", "bias_lrelu", "bias_tanh"]


def wgrad_counts(case):
    """Forced split counts of a case (it also runs at the production count)."""
    oh, ow = out_hw(case.h, case.w, case.k, case.s, case.p)
    kbt = case.n * oh * ow // 64
    return sorted({1, 2, 3, kbt, kbt + 2, *case.extra})


def edge_tiles(g):
    """128-pixel tiles of an edge geometry (the tile height does not depend on C)."""
    return g.n * (g.h // 2) // edge_tile(g.n, g.h, g.w, 1)


def conv_geom(g):
    """The forward's batch: at most 9 images (the forward's production target, 8 x SMs, gives one tile per CTA at any of these sizes)."""
    return g._replace(n=min(g.n, 9))


CONV_TARGETS = [0, 1, 3, 7]       # the edge conv's max_ctas: production, everything in one CTA, and two forced targets


def edge_counts(tiles):
    """Forced CTA targets (0: production): one CTA for everything, 3 and 7 (ragged last CTAs), one tile each."""
    return [0] + sorted({1, 3, 7, tiles})


# ------------------------------------------------------------------------------------------------ CPU: what the tables reach
def test_table_reaches_every_corner():
    seen = collections.Counter()
    for case in WGRAD_CASES:
        n, h, w, c, o, k, s, p = case[1:9]
        t = wgrad_tile(n, h, w, c, o, k, s, p)
        assert t is not None, case.name
        nt, ht, wt = t
        oh, ow = out_hw(h, w, k, s, p)
        assert n * oh * ow <= 2 ** 18, f"{case.name}: integer sums must stay below 2^22"
        tiles_y, kbt, bnw = oh // ht, n * oh * ow // 64, wgrad_bnw(c, k)
        seen["bnw%d" % bnw] += 1
        seen["Nt>1"] += nt > 1
        seen["Nt=64"] += nt == 64
        seen["o-tiles>1"] += o // 128 > 1
        seen["straddle"] += any((col0 // c) != ((col0 + 64) // c) for col0 in range(0, k * k * c, bnw) if bnw == 128)
        seen["pad top/left"] += p > 0
        seen["pad bottom/right"] += (oh - 1) * s - p + k - 1 >= h
        for sp in [wgrad_splits_for(n, h, w, c, o, k, s, p)] + wgrad_counts(case):
            r = split_ranges(kbt, sp)
            full = [x for x in r if x[1]]
            per = -(-kbt // sp)
            assert sum(m for _, m in r) == kbt and full[0][0] == 0
            seen["empty"] += any(m == 0 for _, m in r)
            seen["ragged"] += full[-1][1] < per
            seen["one kb"] += any(m == 1 for _, m in r)
            seen["mid-image"] += nt == 1 and tiles_y > 1 and any(b % tiles_y for b, m in full)
            seen["num_kb<4"] += any(0 < m < STAGES for _, m in r)
            seen["num_kb>=9"] += any(m > 2 * STAGES for _, m in r)
    for what in ("bnw64", "bnw128", "Nt>1", "Nt=64", "o-tiles>1", "straddle", "pad top/left", "pad bottom/right", "empty", "ragged", "one kb",
                 "mid-image", "num_kb<4", "num_kb>=9"):
        assert seen[what], f"no tc_wgrad case reaches: {what}"
    # the example of an SM-count-dependent empty split: on 132 SMs the N81 layer's production count leaves the tenth split empty, on 114 not
    n81 = WGRAD_CASES[2]
    assert [m for _, m in split_ranges(81, wgrad_splits_for(*n81[1:9], sms=132))][-1] == 0
    assert all(m for _, m in split_ranges(81, wgrad_splits_for(*n81[1:9], sms=114)))

    edge = collections.defaultdict(set)
    for c, g in EDGE_CASES:
        ht = edge_tile(g.n, g.h, g.w, c)
        tiles = edge_tiles(g)
        if (2 * ht + 2) * g.w * c * 2 == EDGE_SLAB_BYTES:
            edge["capacity"].add((c, g.w))
        for target in [2 * SMS] + edge_counts(tiles)[1:]:
            ctas, tpc = edge_ctas(tiles, target)
            if tpc > 1:
                edge["multi"].add(c)
            if tiles % tpc:
                edge["ragged"].add(c)
        edge["production multi"].add(edge_ctas(tiles, 2 * SMS)[1] > 1)
        conv_tiles = edge_tiles(conv_geom(g))
        for target in [8 * SMS] + CONV_TARGETS[1:]:
            ctas, tpc = edge_ctas(conv_tiles, target)
            if tpc > 1:
                edge["conv multi"].add(c)
            if conv_tiles % tpc:
                edge["conv ragged"].add(c)
    assert {c for c, _ in EDGE_CASES} == {1, 2, 3, 4}
    for what in ("multi", "ragged", "conv multi", "conv ragged"):
        assert edge[what] == {1, 2, 3, 4}, (what, dict(edge))
    assert edge["capacity"] == {(4, 128), (3, 256)}, edge["capacity"]
    assert True in edge["production multi"]
    assert not edge_tile(1, 16, 256, 4)


# ------------------------------------------------------------------------------------------------ GPU
def ints(rng, values, shape):
    return rng.choice(np.array(values, np.float32), shape)


def assert_exact(got, want, what):
    got = np.asarray(got, np.float64).ravel(); want = np.asarray(want, np.float64).ravel()
    bad = ~(got == want)
    assert not bad.any(), f"{what}: {bad.sum()} of {bad.size} elements differ from the exact result (first at {np.flatnonzero(bad)[:5]}: " \
                          f"got {got[bad][:5]}, want {want[bad][:5]})"


def wgrad_geom(case):
    oh, ow = out_hw(case.h, case.w, case.k, case.s, case.p)
    return dict(n=case.n, h=case.h, w=case.w, c=case.c, oh=oh, ow=ow, o=case.o, kh=case.k, kw=case.k, sh=case.s, sw=case.s, ph=case.p, pw=case.p)


@pytest.mark.gpu
@pytest.mark.parametrize("case", WGRAD_CASES, ids=[c.name for c in WGRAD_CASES])
def test_tc_wgrad_exact_at_every_split(b200, case):
    b, ctx = b200
    sms = ctx.device_info()["sm_count"]
    g = wgrad_geom(case)
    rng = np.random.default_rng(zlib.crc32(case.name.encode()))
    x = ints(rng, [-3, -2, -1, 1, 2, 3], (case.n, case.h, case.w, case.c))
    dy = ints(rng, [-3, -2, -1, 1, 2, 3], (case.n, g["oh"], g["ow"], case.o))
    want = conv_ref.conv2d_weight_grad(x, dy, case.k, case.k, case.s, case.p)
    kernel = f"tc_wgrad_kernel<{wgrad_bnw(case.c, case.k)},4>"
    runs = [(sp, defer, 0) for sp in [0] + wgrad_counts(case) for defer in (False, True)]
    if case.offsets:
        runs += [(3, False, 1), (3, True, 3)]
    for sp, defer, off in runs:
        info = {}
        got, _, k, _ = b.test_conv_ex(ctx, 2, g, x, dy, want.size, impl=1, poison=True, info=info, defer=defer, param_offset=off, splits=sp)
        splits = sp or wgrad_splits_for(*case[1:9], sms=sms)
        what = f"{case.name}: {splits} splits{'' if sp else ' (production)'} defer={defer} offset={off}"
        assert (k, info["splits"]) == (kernel, splits), f"{what}: ran {k} at {info['splits']} splits"
        assert_exact(got, want, what)
    # normal operands at the production split: fp32 accumulation, only the summation order differs from float64
    x = bf16_round(rng.standard_normal(x.shape)); dy = bf16_round(rng.standard_normal(dy.shape))
    got, _, k, _ = b.test_conv_ex(ctx, 2, g, x, dy, want.size, impl=1, poison=True)
    assert np.isfinite(got).all(), f"{case.name}: {(~np.isfinite(got)).sum()} non-finite elements"
    assert rel_err(got, conv_ref.conv2d_weight_grad(x, dy, case.k, case.k, case.s, case.p)) <= 1e-4, case.name


def edge_geom(c, g, o=64):
    return dict(n=g.n, h=g.h, w=g.w, c=c, oh=g.h // 2, ow=g.w // 2, o=o, kh=4, kw=4, sh=2, sw=2, ph=1, pw=1)


@pytest.mark.gpu
@pytest.mark.parametrize("c,g", EDGE_CASES, ids=[f"C{c}-{g.name}" for c, g in EDGE_CASES])
def test_tc_edge_wgrad_exact_at_every_cta_count(b200, c, g):
    b, ctx = b200
    sms = ctx.device_info()["sm_count"]
    geom = edge_geom(c, g)
    rng = np.random.default_rng(zlib.crc32(f"wgrad C{c} {g.name}".encode()))
    x = ints(rng, [-3, -2, -1, 1, 2, 3], (g.n, g.h, g.w, c))
    dy = ints(rng, [-3, -2, -1, 1, 2, 3], (g.n, g.h // 2, g.w // 2, 64))
    want = conv_ref.conv2d_weight_grad(x, dy, 4, 4, 2, 1)
    want_db = dy.astype(np.float64).sum((0, 1, 2))
    tiles = edge_tiles(g)
    if c == 4:        # no spare column for the bias gradient: the hook refuses db
        with pytest.raises(b._lib.B200GanError, match="no bias column"):
            b.test_conv_ex(ctx, 2, geom, x, dy, want.size, impl=3, db=np.empty(64, np.float32))
    runs = [(t, defer, 0) for t in edge_counts(tiles) for defer in (False, True)] + [(3, False, 1), (3, True, 3)]
    for target, defer, off in runs:
        info = {}
        db = np.empty(64, np.float32) if c < 4 else None
        got, _, k, _ = b.test_conv_ex(ctx, 2, geom, x, dy, want.size, impl=3, poison=True, info=info, defer=defer, param_offset=off,
                                      splits=target, db=db)
        ctas = edge_ctas(tiles, target or 2 * sms)[0]
        what = f"C{c} {g.name}: CTA target {target or 'production'} ({ctas} CTAs) defer={defer} offset={off}"
        assert (k, info["splits"]) == ("tc_edge_wgrad_kernel", ctas), f"{what}: ran {k} with {info['splits']} CTAs"
        assert_exact(got, want, what)
        if db is not None:
            assert_exact(db, want_db, what + " db")
    x = bf16_round(rng.standard_normal(x.shape)); dy = bf16_round(rng.standard_normal(dy.shape))
    db = np.empty(64, np.float32) if c < 4 else None
    got, _, _, _ = b.test_conv_ex(ctx, 2, geom, x, dy, want.size, impl=3, poison=True, db=db)
    assert np.isfinite(got).all()
    assert rel_err(got, conv_ref.conv2d_weight_grad(x, dy, 4, 4, 2, 1)) <= 1e-4
    if db is not None:
        assert rel_err(db, dy.astype(np.float64).sum((0, 1, 2))) <= 1e-4


def edge_epilogue(name, rng, o, exact):
    """Hook keyword arguments of an epilogue."""
    if name == "plain":
        return {}
    bias = rng.integers(-8, 9, o).astype(np.float32) if exact else (0.1 * rng.standard_normal(o)).astype(np.float32)
    act = name[len("bias_"):]
    return dict(bias=bias, act=act, alpha=0.2 if act == "lrelu" else 0.0)


def edge_act64(kw, acc):
    z = acc + (kw["bias"].astype(np.float64) if "bias" in kw else 0.0)
    act = kw.get("act", "identity")
    if act == "relu":
        return np.maximum(z, 0.0)
    if act == "lrelu":
        return np.where(z > 0, z, 0.2 * z)
    if act == "tanh":
        return np.tanh(z)
    return z


def edge_act_emulated(kw, acc):
    """bf16_rn(float32(act(float32(acc + bias)))), alpha as float32: the kernel's epilogue on exact integer accumulators."""
    z = (acc + (kw["bias"].astype(np.float64) if "bias" in kw else 0.0)).astype(np.float32)
    act = kw.get("act", "identity")
    if act == "relu":
        z = np.maximum(z, np.float32(0))
    elif act == "lrelu":
        z = np.where(z > 0, z, np.float32(kw["alpha"]) * z)
    return bf16_round(z)


@pytest.mark.gpu
@pytest.mark.parametrize("c,g", EDGE_CASES, ids=[f"C{c}-{g.name}" for c, g in EDGE_CASES])
def test_tc_edge_conv_epilogues_at_every_cta_count(b200, c, g):
    b, ctx = b200
    sms = ctx.device_info()["sm_count"]
    rng = np.random.default_rng(zlib.crc32(f"conv C{c} {g.name}".encode()))
    g = conv_geom(g)
    for o in EDGE_OUT:
        geom = edge_geom(c, g, o)
        x = ints(rng, [-2, -1, 1, 2], (g.n, g.h, g.w, c))
        wt = ints(rng, [-1, 1], (o, 4, 4, c))
        acc = conv_ref.conv2d(x, wt, 2, 1)
        for epi in EDGE_EPIS:
            kw = edge_epilogue(epi, rng, o, exact=True)
            if epi == "bias_tanh":
                ref = edge_act64(kw, acc).ravel()
                ulp = 2.0 ** (np.frexp(np.abs(ref))[1] - 8)           # one bf16 ulp of |ref|: 8 significant bits
            else:
                want = edge_act_emulated(kw, acc)
            outs = {}
            for mc in CONV_TARGETS:
                got, _, k, _ = b.test_conv_ex(ctx, 0, geom, x, wt, acc.size, impl=3, poison=True, max_ctas=mc, **kw)
                what = f"C{c} {g.name} O{o} {epi}: max_ctas {mc or 'production'}"
                assert k == "tc_edge_conv_kernel", f"{what}: ran {k}"
                outs[mc] = got
                if epi == "bias_tanh":
                    d = np.abs(got.astype(np.float64) - ref)
                    assert (d <= ulp).all(), f"{what}: {(~(d <= ulp)).sum()} elements more than one bf16 ulp from float64 tanh"
                else:
                    assert_exact(got, want, what)
            for mc, got in outs.items():
                diff = got.view(np.uint32) != outs[0].view(np.uint32)
                assert not diff.any(), f"C{c} {g.name} O{o} {epi}: max_ctas {mc}: {diff.sum()} elements differ from the production grid"
        # normal operands, bf16-rounded, at the production CTA target
        x = bf16_round(rng.standard_normal(x.shape)); wt = bf16_round(rng.standard_normal(wt.shape) / np.sqrt(16 * c))
        acc = conv_ref.conv2d(x, wt, 2, 1)
        for epi in EDGE_EPIS:
            kw = edge_epilogue(epi, rng, o, exact=False)
            got, _, _, _ = b.test_conv_ex(ctx, 0, geom, x, wt, acc.size, impl=3, poison=True, **kw)
            check_bf16(got.reshape(acc.shape), edge_act64(kw, acc), f"C{c} {g.name} O{o} {epi} (normal operands)")
