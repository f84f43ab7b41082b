"""The weighted / masked instantiations of the five loss kernels through b2g_test_loss, in both precisions, against an emulation of the order
stated at b2g_loss, bit for bit: dz and the loss sums, with weights only, a per-row mask only, both, and a per-output mask; on one block and
many, one group and two, the 16-byte and the scalar path of cnn_xent_kernel, aligned and misaligned operands, outputs poisoned with NaN.

The emulation takes what does not depend on the weights from the unweighted FP32 kernels on the same (bf16-rounded) logits -- XENT's
per-element fp32 score and dz (one element per group), the softmax probabilities (the inference call) -- and forms everything else on the host
in the stated order: s = w_j * m_rj in fp32, the score term (double)l * (double)s, dz * s, each thread's double sum in its slice order, the
warp's xor butterfly, the warps in order, the last block's fold of the per-block partials in slice order.  Codes 2-8 run on the identity, so
their double scores are formed on the host exactly."""
import numpy as np
import pytest

from helpers import b200, bf16_round

pytestmark = pytest.mark.gpu

LOSS_THREADS = 256


def _butterfly(v):
    v = np.array(v, np.float64)
    idx = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[idx ^ o]
    return float(v[0])


def _block_sum(acc):
    """block_sum / the xent kernels' reduction: each warp's xor butterfly, the warps added in order to 0."""
    t = 0.0
    for w in range(len(acc) // 32):
        t += _butterfly(acc[32 * w:32 * w + 32])
    return t


def _thread_sums(terms, owner, order, nthreads):
    """Each thread's double sum of its terms in its order (owner: thread index per term; order: position within that thread's sequence)."""
    acc = [0.0] * nthreads
    for i in np.lexsort((order, owner)):
        acc[owner[i]] += float(terms[i])
    return acc


def _fold(partial, groups, bpg):
    out = []
    for g in range(groups):
        lanes = [0.0] * 32
        for k in range(bpg):
            lanes[k % 32] += partial[g * bpg + k]
        out.append(_butterfly(lanes))
    return out


def _loss_blocks(n_per_group, groups):
    return int(min(max((n_per_group + 1023) // 1024, 1), max(1, 1024 // groups)))


def _scale(w, m, mw, rows_idx, cols_idx):
    """s = w_j * m_rj in fp32 (what is absent is 1)."""
    s = np.ones(rows_idx.shape, np.float32) if w is None else np.asarray(w, np.float32)[cols_idx]
    if m is not None:
        mv = np.asarray(m, np.float32).ravel()
        s = (s * mv[rows_idx * mw + (cols_idx if mw > 1 else 0)]).astype(np.float32)
    return s


def _store(v, P, b):
    v = np.asarray(v, np.float32)
    return bf16_round(v) if P == b.BF16 else v


def _xent_parts(b, ctx, op, z, y, clip):
    """Per-element fp32 score and dz of the unweighted FP32 kernel: one element per group, so each group's sum is its element's score."""
    n = z.size
    kw = dict(rows=1, groups=n, clip_eps=clip) if op == "xent" else dict(rows=1, cols=1, groups=n, clip_eps=clip)
    (g, l, _), _ = b.test_ew(ctx, b.FP32, op, z, y, (n, n, 0), **kw)
    return l.astype(np.float32), g.astype(np.float32)


def _cases_wm(rng, rows_total, cols, per_output=True):
    w = rng.uniform(0.2, 2.5, cols).astype(np.float32)
    m1 = np.where(rng.uniform(0, 1, (rows_total, 1)) < 0.3, 0.0, rng.uniform(0.1, 1.0, (rows_total, 1))).astype(np.float32)
    out = [("weights", w, None), ("row mask", None, m1), ("weights + row mask", w, m1)]
    if per_output and cols > 1:
        out.append(("weights + per-output mask", w, rng.uniform(0, 1, (rows_total, cols)).astype(np.float32)))
    return out


def _check(got_dz, want_dz, got_ls, want_ls, what):
    assert np.isfinite(got_dz).all() and np.isfinite(got_ls).all(), (what, "an output left unwritten reads back as NaN")
    bad = got_dz.view(np.uint32) != np.asarray(want_dz, np.float32).view(np.uint32)
    assert not bad.any(), (what, "dz", int(bad.sum()), got_dz[bad][:4], np.asarray(want_dz)[bad][:4])
    assert np.array_equal(got_ls.view(np.uint32), np.asarray(want_ls, np.float32).view(np.uint32)), (what, "loss sums", got_ls, want_ls)


PRECS = ["fp32", "bf16"]


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("clip", [1e-5, 0.0])
def test_xent_kernel_wm(b200, clip, offset, prec):
    b, ctx = b200
    P = b.FP32 if prec == "fp32" else b.BF16
    rows, groups = 1500, 2
    rng = np.random.default_rng(1)
    n = rows * groups
    z = _store(rng.uniform(-6, 6, n), P, b); y = rng.uniform(0, 1, n).astype(np.float32)
    l, g = _xent_parts(b, ctx, "xent", z, y, clip)
    i = np.arange(n)
    for name, w, m in _cases_wm(rng, n, 1):
        s = _scale(w, m, 1, i, np.zeros(n, np.int64))
        terms = l.astype(np.float64) * s.astype(np.float64)
        want = []
        for gg in range(groups):
            r = np.arange(rows)
            acc = _thread_sums(terms[gg * rows + r], r % 1024, r // 1024, 1024)
            want.append(_block_sum(acc))
        dz, ls, kern = b.test_loss(ctx, P, "xent", z, y, w, m, rows=rows, cols=1, groups=groups, clip_eps=clip, offset=offset, poison=True)
        assert kern == "xent_kernel<wm>"
        _check(dz, _store(g * s, P, b), ls, want, (name, clip, offset, prec))


def _softmax_parts(b, ctx, op, z, rows, cols, groups=1):
    if op == "softmax_xent":
        (_, _, p), _ = b.test_ew(ctx, b.FP32, op, z, None, (0, 0, z.size), rows=rows, cols=cols)
    else:
        (_, _, p), _ = b.test_ew(ctx, b.FP32, op, z, None, (0, 0, z.size), rows=rows, cols=cols, groups=groups)
    return p.astype(np.float32).reshape(-1, cols)


def _softmax_rows(p, y, w, mr):
    """dz and the double score terms of every (row, class) in the kernels' fp32 / double order."""
    R, C = p.shape
    f = np.float32
    wy = (np.asarray(w, f)[None, :] * y).astype(f) if w is not None else y
    if w is not None:
        sy = np.zeros(R, f)
        for c in range(C):
            sy = (sy + (np.asarray(w, f)[c] * y[:, c]).astype(f)).astype(f)
        d = ((p * sy[:, None]).astype(f) - wy).astype(f)
    else:
        d = (p - y).astype(f)
    dz = (mr[:, None] * d).astype(f)
    clamp = np.minimum(np.maximum(p, f(1e-10)), f(1) - f(1e-10)).astype(np.float64)
    terms = -((mr[:, None] * wy).astype(f).astype(np.float64) * np.log(clamp))
    return dz, terms


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("offset", [0, 1])
def test_softmax_xent_kernel_wm(b200, offset, prec):
    b, ctx = b200
    P = b.FP32 if prec == "fp32" else b.BF16
    rows, cols = 1300, 5
    rng = np.random.default_rng(2)
    z = _store(rng.uniform(-4, 4, (rows, cols)), P, b)
    y = rng.uniform(0, 1, (rows, cols)).astype(np.float32); y = (y / y.sum(1, keepdims=True)).astype(np.float32)
    p = _softmax_parts(b, ctx, "softmax_xent", z, rows, cols)
    for name, w, m in _cases_wm(rng, rows, cols, per_output=False):
        mr = np.ones(rows, np.float32) if m is None else m[:, 0]
        d, terms = _softmax_rows(p, y, w, mr)
        r = np.repeat(np.arange(rows), cols); c = np.tile(np.arange(cols), rows)
        want = [_block_sum(_thread_sums(terms.ravel(), r % 1024, (r // 1024) * cols + c, 1024))]
        dz, ls, kern = b.test_loss(ctx, P, "softmax_xent", z, y, w, m, rows=rows, cols=cols, offset=offset, poison=True)
        assert kern == "softmax_xent_kernel<wm>"
        _check(dz, _store(d, P, b).ravel(), ls, want, (name, offset, prec))


def _codes_elem(loss, a, y, nf):
    """loss_kernel's double score and fp32 dL/da of each element on the identity (a = z)."""
    f = np.float32
    a64, y64 = a.astype(np.float64), y.astype(np.float64)
    e, m = a64 - y64, 1.0 - y64 * a64
    sgn = ((a > y).astype(f) - (a < y).astype(f)).astype(f)
    l = {"mse": e * e, "l2": e * e, "l1": np.abs(e), "mae": np.abs(e), "hinge": np.maximum(m, 0.0), "squared_hinge": np.where(m > 0, m * m, 0.0),
         "wasserstein": y64 * a64}[loss]
    d = (a - y).astype(f)
    ga = {"mse": ((f(2) * d).astype(f) / f(nf)).astype(f), "l2": (f(2) * d).astype(f), "l1": sgn, "mae": (sgn / f(nf)).astype(f),
          "hinge": np.where(m > 0, -y, f(0)).astype(f),
          "squared_hinge": np.where(m > 0, ((f(-2) * y).astype(f) * m.astype(f)).astype(f), f(0)).astype(f),
          "wasserstein": (y / f(nf)).astype(f)}[loss]
    return l, ga


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("loss", ["mse", "l1", "l2", "mae", "hinge", "squared_hinge", "wasserstein"])
def test_loss_kernel_wm(b200, loss, offset, prec):
    b, ctx = b200
    P = b.FP32 if prec == "fp32" else b.BF16
    rows, cols, groups = 1500, 3, 2
    per = rows * cols; n = per * groups
    rng = np.random.default_rng(3)
    z = _store(rng.uniform(-2, 2, n), P, b)
    y = (rng.choice([-1.0, 1.0], n) if "hinge" in loss else rng.uniform(-1, 1, n)).astype(np.float32)
    l, ga = _codes_elem(loss, z.astype(np.float32), y, cols)
    bpg = _loss_blocks(per, groups)
    i = np.arange(n); j = i % per; gidx = i // per
    blk = gidx * bpg + (j // LOSS_THREADS) % bpg
    owner = blk * LOSS_THREADS + j % LOSS_THREADS
    order = j // (bpg * LOSS_THREADS)
    per_out = loss in ("mse", "mae", "wasserstein")
    for name, w, m in _cases_wm(rng, rows * groups, cols):
        s = _scale(w, m, 1 if m is None else m.shape[1], i // cols, i % cols)
        acc = _thread_sums(l * s.astype(np.float64), owner, order, groups * bpg * LOSS_THREADS)
        partial = [_block_sum(acc[k * LOSS_THREADS:(k + 1) * LOSS_THREADS]) for k in range(groups * bpg)]
        want = [v / cols if per_out else v for v in _fold(partial, groups, bpg)]
        dz, ls, kern = b.test_loss(ctx, P, "codes", z, y, w, m, rows=rows, cols=cols, groups=groups, loss=loss, offset=offset, poison=True)
        assert kern == "loss_kernel<wm>"
        _check(dz, _store(((ga * np.float32(1)).astype(np.float32) * s).astype(np.float32), P, b), ls, want, (loss, name, offset, prec))


CNN_SHAPES = [(2, 301, 3), (2, 400, 4), (1, 5000, 3)]      # (groups, pixels per group, C): scalar (groups not chunk-aligned), vector, many blocks


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("clip", [1e-5, 0.0])
@pytest.mark.parametrize("shape", CNN_SHAPES)
def test_cnn_xent_kernel_wm(b200, shape, clip, offset, prec):
    b, ctx = b200
    P = b.FP32 if prec == "fp32" else b.BF16
    groups, rows, cols = shape
    per = rows * cols; n = per * groups
    V = 4 if P == b.FP32 else 8
    rng = np.random.default_rng(rows + cols)
    z = _store(rng.uniform(-6, 6, n), P, b); y = rng.uniform(0, 1, n).astype(np.float32)
    l, g = _xent_parts(b, ctx, "cnn_xent", z, y, clip)
    bpg = _loss_blocks(per, groups)
    i = np.arange(n); e = i % per; gidx = i // per; chunk = e // V
    blk = gidx * bpg + (chunk // LOSS_THREADS) % bpg
    owner = blk * LOSS_THREADS + chunk % LOSS_THREADS
    order = (chunk // (bpg * LOSS_THREADS)) * V + e % V
    vec = offset == 0 and (groups == 1 or per % V == 0)
    for name, w, m in _cases_wm(rng, rows * groups, cols):
        s = _scale(w, m, 1 if m is None else m.shape[1], i // cols, i % cols)
        acc = _thread_sums(l.astype(np.float64) * s.astype(np.float64), owner, order, groups * bpg * LOSS_THREADS)
        partial = [_block_sum(acc[k * LOSS_THREADS:(k + 1) * LOSS_THREADS]) for k in range(groups * bpg)]
        dz, ls, kern = b.test_loss(ctx, P, "cnn_xent", z, y, w, m, rows=rows, cols=cols, groups=groups, clip_eps=clip, offset=offset, poison=True)
        assert kern == ("cnn_xent_kernel<vec,wm>" if vec else "cnn_xent_kernel<scalar,wm>"), (kern, shape, offset)
        _check(dz, _store((g * s).astype(np.float32), P, b), ls, _fold(partial, groups, bpg), (shape, name, clip, offset, prec))


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("shape", [(2, 700, 5), (1, 3000, 21)])
def test_cnn_softmax_xent_kernel_wm(b200, shape, offset, prec):
    b, ctx = b200
    P = b.FP32 if prec == "fp32" else b.BF16
    groups, rows, cols = shape
    rng = np.random.default_rng(rows)
    z = _store(rng.uniform(-4, 4, (groups * rows, cols)), P, b)
    k = rng.integers(0, cols, groups * rows); y = np.eye(cols, dtype=np.float32)[k]
    p = _softmax_parts(b, ctx, "cnn_softmax_xent", z, rows, cols, groups)
    bpg = _loss_blocks(rows * 4, groups)
    for name, w, m in _cases_wm(rng, rows * groups, cols, per_output=False):
        mr = np.ones(rows * groups, np.float32) if m is None else m[:, 0]
        d, terms = _softmax_rows(p, y, w, mr)
        px = np.repeat(np.arange(groups * rows), cols); c = np.tile(np.arange(cols), groups * rows)
        r, gidx = px % rows, px // rows
        blk = gidx * bpg + (r // LOSS_THREADS) % bpg
        owner = blk * LOSS_THREADS + r % LOSS_THREADS
        order = (r // (bpg * LOSS_THREADS)) * cols + c
        acc = _thread_sums(terms.ravel(), owner, order, groups * bpg * LOSS_THREADS)
        partial = [_block_sum(acc[q * LOSS_THREADS:(q + 1) * LOSS_THREADS]) for q in range(groups * bpg)]
        dz, ls, kern = b.test_loss(ctx, P, "cnn_softmax_xent", z, y, w, m, rows=rows, cols=cols, groups=groups, offset=offset, poison=True)
        assert kern == "cnn_softmax_xent_kernel<wm>"
        _check(dz, _store(d, P, b).ravel(), ls, _fold(partial, groups, bpg), (shape, name, offset, prec))


def test_loss_hook_refusals(b200):
    b, ctx = b200
    z = np.zeros(12, np.float32)
    for kw in (dict(kernel="xent", rows=6, cols=2, groups=1), dict(kernel="softmax_xent", rows=3, cols=2, groups=2),
               dict(kernel="codes", rows=4, cols=3, groups=1, loss="xent")):
        k = kw.pop("kernel")
        with pytest.raises(b.B200GanError):
            b.test_loss(ctx, b.FP32, k, z, z, **kw)
    with pytest.raises(b.B200GanError):
        b.test_loss(ctx, b.FP32, "cnn_xent", z, z, None, np.ones((4, 2), np.float32), rows=4, cols=3, groups=1)      # width neither 1 nor C
