"""Plain references of the var data kernels of yask_b200/csrc/yb_fill.cu (numpy only).

`reduce_ref` restates the device reduction (`yb_var_reduce_slice`) in its exact order, so a test can compare sum, product, max,
min and the fp32 sum of squares bit for bit:

* The grid is g = min(ceil(N / 256), 2368) blocks of 256 threads (`grid_for`, `MAX_GRID`).  Thread k of the grid accumulates the
  dense elements k, k + 256 g, k + 512 g, ... (innermost box dim fastest) onto (sum 0, sumsq 0, prod 1, max -inf, min +inf): sum
  += v, sumsq = fma(v, v, sumsq) (a DFMA in the SASS), prod *= v, max = fmax(max, v), min = fmin(min, v).
* Each warp combines its lanes with shfl_down at d = 16, 8, 4, 2, 1; warp 0 then combines the 8 warp results at d = 4, 2, 1, and
  that is the block's partial.  Combining adds sums, multiplies products and takes fmax / fmin.
* One final block of 256 threads: thread k combines partial k, k + 256, ... onto the initial values, then the same two trees.
* The host combines the steps of a box in order onto the initial values, with std::max / std::min (`yb_core.cu`).

For an fp32 var v * v is exact in double, so the fused and unfused sums of squares are the same bits.  For an fp64 var the fused
chain is not restated: `reduce_bound` bounds every sum against math.fsum instead.

`checksum_ref` restates `checksum_kernel`: the sum mod 2^64 of splitmix64(key(g) ^ (bits * 0x9E3779B97F4A7C15)) over the box,
keyed by the global index g of each element with the key layout of `synth.hash_field`.
"""
from __future__ import annotations

import math

import numpy as np

from yask_b200.synth import _M, _OFF, _splitmix64

BLOCK = 256
MAX_GRID = 2368
U = 2.0 ** -53
_INIT = (0.0, 0.0, 1.0, -np.inf, np.inf)
KEYS = ("sum", "sum_squares", "product", "max", "min")


def grid_for(n: int) -> int:
    return int(min(max(-(-n // BLOCK), 1), MAX_GRID))


def _merge(a, b):
    """red_merge: a combined with b, field by field (arrays of any shape)."""
    return (a[0] + b[0], a[1] + b[1], a[2] * b[2], np.fmax(a[3], b[3]), np.fmin(a[4], b[4]))


def _tree(r, deltas):
    """shfl_down tree over the last axis; returns lane 0."""
    r = [np.array(x, dtype=np.float64, copy=True) for x in r]
    for d in deltas:
        m = _merge([x[..., :d] for x in r], [x[..., d:2 * d] for x in r])
        for x, y in zip(r, m):
            x[..., :d] = y
    return [x[..., 0] for x in r]


def _red_block(r):
    """red_block over the last axis of 256 thread values: per-warp trees, then warp 0 over the 8 warp results."""
    lead = r[0].shape[:-1]
    warps = _tree([x.reshape(lead + (BLOCK // 32, 32)) for x in r], (16, 8, 4, 2, 1))
    return _tree(warps, (4, 2, 1))


def _chains(x, nthreads):
    """Grid-stride accumulation of dense elements x by `nthreads` threads: per-thread (sum, sumsq, prod, max, min)."""
    n = x.size
    L = -(-n // nthreads)
    r = [np.full(nthreads, v, dtype=np.float64) for v in _INIT]
    for j in range(L):
        seg = x[j * nthreads:(j + 1) * nthreads]
        k = seg.size
        s, q, p, mx, mn = (a[:k] for a in r)
        s += seg
        q += seg * seg      # fma(v, v, q) on the device: the same bits when v * v is exact
        p *= seg
        np.fmax(mx, seg, out=mx)
        np.fmin(mn, seg, out=mn)
    return r


def _chains_of_partials(parts, nthreads):
    """reduce_final_kernel's loop: thread k merges partials k, k + 256, ... onto the initial values."""
    g = parts[0].size
    r = [np.full(nthreads, v, dtype=np.float64) for v in _INIT]
    for j0 in range(0, g, nthreads):
        k = min(nthreads, g - j0)
        m = _merge([a[:k] for a in r], [p[j0:j0 + k] for p in parts])
        for a, b in zip(r, m):
            a[:k] = b
    return r


def reduce_step(values):
    """Device reduction of one step's dense box (float64 array): (sum, sumsq, prod, max, min) as the device forms them."""
    x = np.ascontiguousarray(values, dtype=np.float64).ravel()
    g = grid_for(x.size)
    with np.errstate(all="ignore"):      # overflow, inf * 0 and NaN behave as on the device
        thr = _chains(x, g * BLOCK)
        parts = _red_block([a.reshape(g, BLOCK) for a in thr])
        fin = _red_block(_chains_of_partials(parts, BLOCK))
    return tuple(float(a) for a in fin)


def reduce_ref(values, nsteps: int = 1) -> dict:
    """The reduction of a box of `nsteps` steps (values: dense, step outermost, any float dtype) in the device's exact order.
    Keys as capi.Var.reduce_elements_in_slice; "sum_squares" is exact only for values that square exactly in double."""
    x = np.ascontiguousarray(values).astype(np.float64).reshape(nsteps, -1)
    tot = list(_INIT)
    for t in range(nsteps):
        r = reduce_step(x[t])
        tot[0] += r[0]
        tot[1] += r[1]
        with np.errstate(all="ignore"):
            tot[2] = float(np.float64(tot[2]) * r[2])
        tot[3] = r[3] if tot[3] < r[3] else tot[3]     # std::max(tot, r)
        tot[4] = r[4] if r[4] < tot[4] else tot[4]     # std::min(tot, r)
    out = dict(zip(KEYS, tot))
    out["num"] = x.size
    return out


def chain_length(n_per_step: int) -> int:
    """L: the longest per-thread grid-stride chain of a step of n elements."""
    return -(-n_per_step // (grid_for(n_per_step) * BLOCK))


def reduce_bound(n_per_step: int, nsteps: int, abs_sum: float) -> float:
    """Bound on |device sum - exact sum| in any order of the same tree shape: every value passes through at most
    L + ceil(g/256) + 16 + S roundings (chain, 5 + 3 tree levels twice, final chain, host steps), each at most 2^-53 relative."""
    g = grid_for(n_per_step)
    return (chain_length(n_per_step) + -(-g // BLOCK) + 16 + nsteps) * U * abs_sum


def fsum_check(got: float, values, square: bool = False) -> tuple[bool, float, float]:
    """(within the bound, |got - fsum|, bound) of a device sum (or sum of squares) of `values` (nsteps, n_per_step)."""
    x = np.asarray(values, dtype=np.float64)
    x = x.reshape(1, -1) if x.ndim == 1 else x.reshape(x.shape[0], -1)
    terms = (x * x if square else x).ravel()
    exact = math.fsum(terms.tolist())
    bound = reduce_bound(x.shape[1], x.shape[0], float(np.abs(terms).sum()))
    if square:
        bound += U * float(terms.sum())        # fsum of the rounded squares (fp64 values) vs the exact squares
    err = abs(got - exact)
    return err <= bound, err, bound


# ---- checksum -------------------------------------------------------------------------------------------------------------
def index_keys(first, shape) -> np.ndarray:
    """Keys of a box of global indices (<= 3 dims, right-aligned into the triple, left-padded with index 0), as synth.hash_field
    and the device's index_key form them; shape `shape`."""
    first, shape = list(first), list(shape)
    nd = len(shape)
    assert nd <= 3 and len(first) == nd
    first = [0] * (3 - nd) + first
    shp = [1] * (3 - nd) + shape
    idx = []
    for d in range(3):
        a = (np.arange(shp[d], dtype=np.int64) + np.int64(first[d])).astype(np.uint64)
        with np.errstate(over="ignore"):
            idx.append((a + _OFF) & _M)
    key = (idx[0][:, None, None] << np.uint64(40)) | (idx[1][None, :, None] << np.uint64(20)) | idx[2][None, None, :]
    return key.reshape(shape)


def element_bits(arr) -> np.ndarray:
    a = np.ascontiguousarray(arr)
    return (a.view(np.uint32) if a.dtype == np.float32 else a.view(np.uint64)).astype(np.uint64)


def checksum_terms(arr, first) -> np.ndarray:
    """Per-element checksum terms of the box `arr` whose origin has global index `first`."""
    with np.errstate(over="ignore"):
        return _splitmix64(index_keys(first, np.shape(arr)) ^ (element_bits(arr) * np.uint64(0x9E3779B97F4A7C15)))


def checksum_ref(arr, first) -> int:
    """Sum mod 2^64 of the box's checksum terms: what yb_var_checksum returns for that box."""
    t = checksum_terms(arr, first).ravel()
    with np.errstate(over="ignore"):
        return int(np.add.reduce(t, dtype=np.uint64)) if t.size else 0
