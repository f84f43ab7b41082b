"""CPU checks of the summation-order emulations in tests/ew_ref.py: on integer-valued inputs (every partial sum exact in fp32) each order
equals math.fsum, and the vectorised warp emulation equals a direct lane-by-lane simulation of the kernel on random floats."""
import math

import numpy as np
import pytest

import ew_ref as er


def _ints(rng, shape, lo=-50, hi=50):
    return rng.integers(lo, hi + 1, shape).astype(np.float32)


@pytest.mark.parametrize("splits,n", [(1, 5), (7, 33), (63, 100), (64, 100), (300, 17)])
@pytest.mark.parametrize("with_init", [False, True])
def test_every_order_equals_fsum_on_integers(splits, n, with_init):
    rng = np.random.default_rng(splits * 1000 + n)
    src = _ints(rng, (splits, n))
    init = _ints(rng, n) if with_init else None
    want = np.array([math.fsum(list(src[:, i]) + ([init[i]] if with_init else [])) for i in range(n)], np.float32)
    for got in (er.reduce_narrow(src, init), er.reduce_wide(src, init)):
        assert got.dtype == np.float32 and np.array_equal(got, want)


def test_reduce_multi_equals_fsum_on_integers_in_both_modes():
    rng = np.random.default_rng(7)
    buf = _ints(rng, 20000)
    jobs = [dict(n=37, splits=70, stride=37, src_off=0, dst_off=2600), dict(n=101, splits=5, stride=104, src_off=3000, dst_off=9000),
            dict(n=8, splits=1, stride=8, src_off=10000, dst_off=10100)]
    for wide in ([True, False, False], [False, True, True]):
        out = er.reduce_multi(buf, jobs, wide)
        touched = np.zeros(buf.size, bool)
        for j in jobs:
            part = er.splits_view(buf, j["src_off"], j["splits"], j["stride"], j["n"])
            want = np.array([math.fsum(part[:, i]) for i in range(j["n"])], np.float32)
            assert np.array_equal(out[j["dst_off"]: j["dst_off"] + j["n"]], want)
            touched[j["dst_off"]: j["dst_off"] + j["n"]] = True
        assert np.array_equal(out[~touched], buf[~touched])


def _warp_direct(col, init):
    """One output of reduce_splits_wide_kernel, simulated lane by lane: 32 registers, the strided loop, then five rounds of
    a += __shfl_xor_sync(a, m) in which every lane reads its partner's value from before the round."""
    reg = [np.float32(0)] * 32
    for lane in range(32):
        for k in range(lane, len(col), 32):
            reg[lane] = np.float32(reg[lane] + col[k])
    for m in (16, 8, 4, 2, 1):
        reg = [np.float32(reg[lane] + reg[lane ^ m]) for lane in range(32)]
    return np.float32((np.float32(0) if init is None else init) + reg[0])


@pytest.mark.parametrize("splits", [1, 31, 64, 65, 300])
def test_wide_emulation_equals_lane_by_lane_simulation(splits):
    rng = np.random.default_rng(splits)
    n = 9
    src = (rng.standard_normal((splits, n)) * np.exp(rng.uniform(-8, 8, (splits, n)))).astype(np.float32)
    init = rng.standard_normal(n).astype(np.float32)
    for ini in (None, init):
        got = er.reduce_wide(src, ini)
        want = np.array([_warp_direct(src[:, i], None if ini is None else ini[i]) for i in range(n)], np.float32)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    # on these magnitudes the orders differ: the emulations are not all the same sum
    assert splits < 2 or not np.array_equal(er.reduce_wide(src), er.reduce_narrow(src))
