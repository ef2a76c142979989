"""The plain references of the var data kernels (tests/var_data_ref.py) checked without a GPU: the reduction's restated order
against math.fsum, exact sums and a lane-by-lane restatement; the checksum's additivity; the key layout against synth.hash_field."""
import math

import numpy as np
import pytest

from tests.var_data_ref import (BLOCK, KEYS, U, checksum_ref, checksum_terms, fsum_check, grid_for, index_keys, reduce_ref,
                                reduce_step)
from yask_b200.synth import _splitmix64, hash_field

SIZES = [1, 31, 32, 33, 255, 256, 257, 606207, 606208, 606209, 3_000_001]


def _lane_sim(x):
    """Scalar, lane-by-lane restatement of box_reduce_kernel + reduce_final_kernel (shfl_down: lane i reads lane i + d when
    i + d < 32, else its own value)."""
    init = [0.0, 0.0, 1.0, -math.inf, math.inf]

    def merge(a, b):
        return [a[0] + b[0], a[1] + b[1], a[2] * b[2], float(np.fmax(a[3], b[3])), float(np.fmin(a[4], b[4]))]

    def shfl_tree(lanes, deltas):
        lanes = [list(v) for v in lanes]
        for d in deltas:
            lanes = [merge(lanes[i], lanes[i + d] if i + d < 32 else lanes[i]) for i in range(32)]
        return lanes[0]

    def block(thr):
        w = [shfl_tree(thr[32 * k:32 * k + 32], (16, 8, 4, 2, 1)) for k in range(BLOCK // 32)]
        return shfl_tree(w + [init] * (32 - len(w)), (4, 2, 1))

    n = len(x)
    g = grid_for(n)
    T = g * BLOCK
    parts = []
    for b in range(g):
        thr = []
        for t in range(BLOCK):
            r = list(init)
            for i in range(b * BLOCK + t, n, T):
                v = float(x[i])
                r = [r[0] + v, r[1] + v * v, r[2] * v, float(np.fmax(r[3], v)), float(np.fmin(r[4], v))]
            thr.append(r)
        parts.append(block(thr))
    thr = []
    for t in range(BLOCK):
        r = list(init)
        for i in range(t, g, BLOCK):
            r = merge(r, parts[i])
        thr.append(r)
    return tuple(block(thr))


def _same(a, b):
    return all((x == y) or (math.isnan(x) and math.isnan(y)) for x, y in zip(a, b))


@pytest.mark.parametrize("n", [1, 31, 33, 257, 513, 2900])
def test_reduce_ref_matches_a_lane_by_lane_restatement(n):
    x = np.random.default_rng(n).uniform(-1, 1, n).astype(np.float32).astype(np.float64)
    assert _same(reduce_step(x), _lane_sim(x))


@pytest.mark.parametrize("n", SIZES)
def test_reduce_ref_within_its_bound_of_fsum(n):
    rng = np.random.default_rng(n)
    for dt in (np.float32, np.float64):
        x = rng.uniform(-1, 1, n).astype(dt)
        r = reduce_ref(x)
        assert r["num"] == n
        ok, err, bound = fsum_check(r["sum"], x)
        assert ok, (n, dt, err, bound)
        ok, err, bound = fsum_check(r["sum_squares"], x, square=True)
        assert ok, (n, dt, err, bound)
        assert r["max"] == x.max() and r["min"] == x.min()


def test_reduce_ref_bound_over_steps():
    x = np.random.default_rng(5).uniform(-3, 1, (3, 700_001)).astype(np.float32)
    r = reduce_ref(x, 3)
    assert r["num"] == x.size
    assert fsum_check(r["sum"], x)[0] and fsum_check(r["sum_squares"], x, square=True)[0]
    assert r["max"] == x.max() and r["min"] == x.min()


@pytest.mark.parametrize("n", SIZES)
def test_reduce_ref_exact_on_power_of_two_values(n):
    """Values +-2^e, e in [-4, 4]: every partial sum (and sum of squares) is a multiple of 2^-8 below 2^53, so any order is
    exact.  Products of +-2^e, e in {-1, 0, 1}, are exact too."""
    rng = np.random.default_rng(n + 1)
    x = np.ldexp(rng.choice([-1.0, 1.0], n), rng.integers(-4, 5, n))
    r = reduce_ref(x)
    assert r["sum"] == math.fsum(x.tolist()) and r["sum_squares"] == math.fsum((x * x).tolist())
    e = np.where(rng.random(n) < 1e-3, rng.choice([-1, 1], n), 0)
    y = np.ldexp(rng.choice([-1.0, 1.0], n), e)
    sign = -1.0 if np.count_nonzero(y < 0) % 2 else 1.0
    assert reduce_ref(y)["product"] == math.ldexp(sign, int(e.sum()))


def test_reduce_ref_special_values():
    x = np.random.default_rng(3).uniform(-1, 1, 1000)
    x[417] = np.nan
    r = reduce_ref(x)
    assert math.isnan(r["sum"]) and math.isnan(r["sum_squares"]) and math.isnan(r["product"])
    assert r["max"] == np.nanmax(x) and r["min"] == np.nanmin(x)
    y = -np.abs(x[:400]) - 0.5
    r = reduce_ref(y)
    assert r["max"] < 0 and r["max"] == y.max() and r["sum_squares"] != r["sum"]
    r = reduce_ref(np.array([0.5, 0.0, 3.0]))
    assert r["product"] == 0.0
    r = reduce_ref(np.array([1.0, np.inf, -2.0]))
    assert r["sum"] == np.inf and r["max"] == np.inf and r["product"] == -np.inf
    assert set(KEYS) <= set(r)


@pytest.mark.parametrize("shape,first", [((37,), (-4,)), ((9, 13), (-2, 5)), ((5, 6, 7), (-8, 3, 1000))])
def test_checksum_ref_additive_over_a_split_box(shape, first):
    rng = np.random.default_rng(len(shape))
    a = rng.uniform(-1, 1, shape).astype(np.float32)
    whole = checksum_ref(a, first)
    for ax in range(len(shape)):
        k = shape[ax] // 3 + 1
        lo, hi = np.split(a, [k], axis=ax)
        f2 = list(first)
        f2[ax] += k
        assert (checksum_ref(lo, first) + checksum_ref(hi, f2)) % (1 << 64) == whole
    # each term depends on the element's value and position
    b = a.copy()
    b.flat[7] = np.float32(2.0)
    assert checksum_ref(b, first) != whole
    assert checksum_ref(a.astype(np.float64), first) != whole
    assert (int(checksum_terms(a, first).ravel()[7]) - int(checksum_terms(b, first).ravel()[7])) % (1 << 64) == \
        (whole - checksum_ref(b, first)) % (1 << 64)


def _field_from_keys(seed, salt, keys, lo, hi, dt):
    with np.errstate(over="ignore"):
        h = _splitmix64(keys ^ (np.uint64(seed) << np.uint64(32) | np.uint64(salt)) * np.uint64(0xD6E8FEB86659FD93))
    return (lo + (hi - lo) * ((h >> np.uint64(40)).astype(np.float64) * (1.0 / 16777216.0))).astype(dt)


@pytest.mark.parametrize("first,shape", [((-3,), (11,)), ((4, -6), (5, 9)), ((-8, 0, 7), (3, 4, 5)), ((2, -1, 5, 9), (3, 2, 4, 6))])
def test_key_layout_agrees_with_hash_field(first, shape):
    seed, salt = 17, 0xDEADBEEF
    for dt in (np.float32, np.float64):
        ref = hash_field(seed, salt, first, shape, -1.0, 1.0, dt)
        if len(shape) == 4:      # the leading index perturbs the salt; the rest is a 3-D field
            got = np.stack([_field_from_keys(seed, (salt + (first[0] + m) * 0x9E3779B1) & 0xFFFFFFFF,
                                             index_keys(first[1:], shape[1:]), -1.0, 1.0, dt) for m in range(shape[0])])
        else:
            got = _field_from_keys(seed, salt, index_keys(first, shape), -1.0, 1.0, dt)
        assert got.shape == ref.shape and np.array_equal(got, ref)


def test_bound_constants():
    assert U == 2.0 ** -53 and grid_for(606208) == 2368 and grid_for(606209) == 2368 and grid_for(1) == 1
