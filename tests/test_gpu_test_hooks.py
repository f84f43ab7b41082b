"""GPU: the argument checks and the device memory of the kernel-level conv hook b2g_test_conv_ex.

Each option of the hook applies to some (impl, kind) pairs only.  Every other pairing, a shape or precision no kernel of that impl runs,
and a fused epilogue without its operands is refused before any conv kernel launches: B2G_ERR_UNSUPPORTED (-6), or B2G_ERR_ARG (-1) for
a missing aux / aux2 and for a kind or impl outside the table.  A refusal after the operands are on the device gives their memory back.
"""
import numpy as np
import pytest

import conv_ref
from helpers import b200, bf16_round, rel_err

pytestmark = pytest.mark.gpu

UNSUPPORTED, ARG = -6, -1


def geom(n, h, w, c, o, k=4, s=2, p=1):
    return dict(n=n, h=h, w=w, c=c, oh=conv_ref.out_size(h, k, s, p), ow=conv_ref.out_size(w, k, s, p), o=o, kh=k, kw=k, sh=s, sw=s, ph=p, pw=p)


def sizes(kind, g):
    """(a, b, result) element counts of kind 0 fprop / 1 dgrad / 2 wgrad."""
    nx, ny, nw = g["n"] * g["h"] * g["w"] * g["c"], g["n"] * g["oh"] * g["ow"] * g["o"], g["o"] * g["kh"] * g["kw"] * g["c"]
    return (nx, nw, ny) if kind == 0 else (ny, nw, nx) if kind == 1 else (nx, ny, nw)


def conv_ex(b, ctx, kind, impl, g, prec, **kw):
    na, nb, no = sizes(min(max(kind, 0), 2), g)
    ch = max(g["o"], g["c"])
    for name in ("bias", "scale"):
        if kw.get(name) is True:
            kw[name] = np.ones(ch, np.float32)
    for name in ("aux", "aux2"):
        if kw.get(name) is True:
            kw[name] = np.ones(no, np.float32)
    if kw.get("db") is True:
        kw["db"] = np.empty(g["o"], np.float32)
    P = b.BF16 if prec == "bf16" else b.FP32
    return b.test_conv_ex(ctx, kind, g, np.ones(na, np.float32), np.ones(nb, np.float32), no, impl=impl, precision=P, **kw)


TC = geom(4, 16, 16, 64, 128)                  # the tensor-core fprop, dgrad (64 result channels) and wgrad (impl 1)
TC3 = geom(2, 8, 8, 64, 128, k=3, s=1, p=1)
EDGE = geom(2, 32, 32, 3, 64)                  # the skinny-layer kernels from 3 image channels (impl 2 / 3)
EDGE8 = geom(2, 32, 32, 8, 64)
DENSE = geom(8, 1, 1, 24, 1, k=1, s=1, p=0)    # <= 4 output units; C = 24: no short-reduction kernel (impl 4)
HEAD = geom(1, 5, 5, 16, 1, k=3, s=1, p=1)     # the few-output conv (impl 5)
HEAD12 = geom(1, 5, 5, 12, 1, k=3, s=1, p=1)

# (what, kind, impl, geometry, precision, options, code)
REFUSALS = [
    # epilogues
    ("epi on impl 4 kind 1", 1, 4, DENSE, "fp32", dict(epi=1), UNSUPPORTED),
    ("epi on impl 4 kind 2", 2, 4, DENSE, "fp32", dict(epi=1), UNSUPPORTED),
    ("bias on impl 4 kind 1 off the short-reduction kernel", 1, 4, DENSE, "fp32", dict(bias=True), UNSUPPORTED),
    ("act on impl 4 kind 2", 2, 4, DENSE, "fp32", dict(act="relu"), UNSUPPORTED),
    ("bias on impl 0 kind 2", 2, 0, TC, "fp32", dict(bias=True), UNSUPPORTED),
    ("bias on impl 1 kind 2", 2, 1, TC, "bf16", dict(bias=True), UNSUPPORTED),
    ("epi on a weight gradient", 2, 1, TC, "bf16", dict(epi=1), UNSUPPORTED),
    ("act on impl 3 kind 2", 2, 3, EDGE, "bf16", dict(act="relu"), UNSUPPORTED),
    ("epi on impl 3 kind 0", 0, 3, EDGE, "bf16", dict(epi=1), UNSUPPORTED),
    ("EPI_STATS on the pixel-shuffle deconv", 1, 3, EDGE, "bf16", dict(epi=1), UNSUPPORTED),
    ("EPI_BNBWD on the pixel-shuffle deconv", 1, 3, EDGE, "bf16", dict(epi=2, aux=True, aux2=True), UNSUPPORTED),
    ("scale on impl 2", 0, 2, EDGE, "fp32", dict(scale=True), UNSUPPORTED),
    ("scale on impl 4", 0, 4, DENSE, "fp32", dict(scale=True), UNSUPPORTED),
    ("scale on impl 5", 0, 5, HEAD, "bf16", dict(scale=True), UNSUPPORTED),
    ("scale on impl 3 kind 0", 0, 3, EDGE, "bf16", dict(scale=True), UNSUPPORTED),
    ("scale on the pixel-shuffle deconv", 1, 3, EDGE, "bf16", dict(scale=True), UNSUPPORTED),
    # parameter offsets and schedule controls
    ("param_offset < 0", 0, 0, TC, "fp32", dict(param_offset=-1), UNSUPPORTED),
    ("param_offset on impl 1 kind 0", 0, 1, TC, "bf16", dict(param_offset=3), UNSUPPORTED),
    ("param_offset on impl 3 kind 1", 1, 3, EDGE, "bf16", dict(param_offset=3), UNSUPPORTED),
    ("bn 96", 0, 1, TC, "bf16", dict(bn=96), UNSUPPORTED),
    ("bn 128 not dividing 64 output channels", 1, 1, TC, "bf16", dict(bn=128), UNSUPPORTED),
    ("bn on impl 0", 0, 0, TC, "fp32", dict(bn=64), UNSUPPORTED),
    ("bn on impl 1 kind 2", 2, 1, TC, "bf16", dict(bn=64), UNSUPPORTED),
    ("per_tap on impl 0", 0, 0, TC, "fp32", dict(per_tap=True), UNSUPPORTED),
    ("per_tap on impl 3", 0, 3, EDGE, "bf16", dict(per_tap=True), UNSUPPORTED),
    ("max_ctas on impl 2", 0, 2, EDGE, "fp32", dict(max_ctas=4), UNSUPPORTED),
    ("max_ctas on impl 1 kind 2", 2, 1, TC, "bf16", dict(max_ctas=4), UNSUPPORTED),
    ("max_ctas < 0", 0, 1, TC, "bf16", dict(max_ctas=-1), UNSUPPORTED),
    ("splits on a forward", 0, 1, TC, "bf16", dict(splits=2), UNSUPPORTED),
    ("splits on impl 0 kind 2", 2, 0, TC, "fp32", dict(splits=2), UNSUPPORTED),
    ("splits < 0", 2, 1, TC, "bf16", dict(splits=-1), UNSUPPORTED),
    ("w_mn on a 3x3", 0, 1, TC3, "bf16", dict(w_mn=True), UNSUPPORTED),
    ("w_mn on kind 1", 1, 1, TC, "bf16", dict(w_mn=True), UNSUPPORTED),
    ("defer on impl 0", 2, 0, TC, "fp32", dict(defer=True), UNSUPPORTED),
    ("defer on impl 5", 2, 5, HEAD, "bf16", dict(defer=True), UNSUPPORTED),
    ("db on impl 1", 2, 1, TC, "bf16", dict(db=True), UNSUPPORTED),
    ("db on impl 3 kind 0", 0, 3, EDGE, "bf16", dict(db=True), UNSUPPORTED),
    # precisions and shapes without a kernel
    ("impl 1 in FP32", 0, 1, TC, "fp32", {}, UNSUPPORTED),
    ("impl 1 from 3 channels", 0, 1, EDGE, "bf16", {}, UNSUPPORTED),
    ("impl 2 from 8 image channels", 0, 2, EDGE8, "fp32", {}, UNSUPPORTED),
    ("impl 3 from 8 image channels", 0, 3, EDGE8, "bf16", {}, UNSUPPORTED),
    ("impl 4 on a 3x3", 0, 4, HEAD, "fp32", {}, UNSUPPORTED),
    ("impl 5 in FP32", 0, 5, HEAD, "fp32", {}, UNSUPPORTED),
    ("impl 5 from 12 channels", 0, 5, HEAD12, "bf16", {}, UNSUPPORTED),
    # the operands of the backward epilogues
    ("EPI_BNBWD without aux", 0, 1, TC, "bf16", dict(epi=2, aux2=True), ARG),
    ("EPI_BNBWD without aux2", 0, 1, TC, "bf16", dict(epi=2, aux=True), ARG),
    ("EPI_ACTBWD without aux", 1, 1, TC, "bf16", dict(epi=3), ARG),
]


@pytest.mark.parametrize("what,kind,impl,g,prec,kw,code", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_conv_hook_refusal(b200, what, kind, impl, g, prec, kw, code):
    b, ctx = b200
    with pytest.raises(b.B200GanError) as e:
        conv_ex(b, ctx, kind, impl, g, prec, **kw)
    assert e.value.code == code, str(e.value)


@pytest.mark.parametrize("kind,impl", [(3, 0), (0, 6), (0, -1)])
def test_conv_hook_refuses_kind_and_impl_outside_the_table(b200, kind, impl):
    b, ctx = b200
    with pytest.raises(b.B200GanError) as e:
        conv_ex(b, ctx, kind, impl, TC, "bf16")
    assert e.value.code == ARG, str(e.value)


def test_conv_hook_refusal_frees_the_operands(b200):
    """EPI_BNBWD without aux is refused after the operands are on the device: here about 576 MiB of them.  Eight such calls leave the
    device's free memory where it was (within 1 GiB: the reading covers every process on the device), and the context still runs a conv."""
    import torch
    b, ctx = b200
    g = geom(64, 64, 64, 256, 512)
    na, nb, no = sizes(0, g)
    x, w = np.zeros(na, np.float32), np.zeros(nb, np.float32)
    free0, _ = torch.cuda.mem_get_info()
    for _ in range(8):
        with pytest.raises(b.B200GanError) as e:
            b.test_conv_ex(ctx, 0, g, x, w, no, epi=b.EPI_BNBWD)
        assert e.value.code == ARG, str(e.value)
    free1, _ = torch.cuda.mem_get_info()
    assert free0 - free1 <= 1 << 30, f"free device memory fell by {(free0 - free1) / 2 ** 20:.0f} MiB"
    rng = np.random.default_rng(3)
    x = bf16_round(rng.standard_normal((4, 16, 16, 64))); w = bf16_round(rng.standard_normal((128, 4, 4, 64)) / 32)
    got, _, kernel, _ = b.test_conv_ex(ctx, 0, TC, x, w, sizes(0, TC)[2])
    assert kernel and rel_err(got, conv_ref.conv2d(x, w, 2, 1)) < 1e-2, kernel
