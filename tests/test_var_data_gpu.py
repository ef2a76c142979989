"""GPU: the var data kernels of yask_b200/csrc/yb_fill.cu against numpy and the plain references of tests/var_data_ref.py.

The strided box copies behind get/set_elements_in_slice (host staging and device buffers), the same-value fills, fill_hash, the
checksum and the reduction, on every kind of var: 1-D, 2-D and 3-D, with and without a step dim, a misc dim innermost or
outermost, fp32 and fp64, spare temporal-tile slots; on boxes of every shape and at the element counts where the kernels' grid
and chains change; on rank grids; past 2^31 elements per slot.  Bit for bit wherever the operation is; max and min with ==.
"""
import ctypes as C
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.large_domain import TWO31, bits, crossing_index, elem_offset, storage_bytes
from tests.var_data_ref import checksum_ref, checksum_terms, fsum_check, reduce_ref
from yask_b200 import capi, multi
from yask_b200.synth import hash_field, var_salt

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STEP, DOMAIN, MISC = 0, 1, 2


# ---- vars under test ----------------------------------------------------------------------------------------------------------
def _solution(stencil, n, eb=4, radius=0, opts=None, user=None):
    s = capi.Solution(stencil, radius=radius, elem_bytes=eb)
    s.set_overall_domain_size_vec(n)
    for k, v in (opts or {}).items():
        s.set_option(k, v)
    if user:
        s.new_fixed_size_var(*user)
    s.prepare_solution(0)
    return s


# name -> (stencil, domain size, elem_bytes, radius, options, var, user var to create)
CASES = {
    "iso-p-f32": ("iso3dfd", (24, 20, 70), 4, 0, None, "p", None),
    "iso-v-f32": ("iso3dfd", (24, 20, 70), 4, 0, None, "v", None),
    "iso-p-f64": ("iso3dfd", (24, 20, 70), 8, 0, None, "p", None),
    "iso-v-f64": ("iso3dfd", (24, 20, 70), 8, 0, None, "v", None),
    "test_1d": ("test_1d", (1000,), 0, 0, None, "A", None),
    "wave2d": ("wave2d", (60, 70), 0, 0, None, "u", None),
    "ssg2-v": ("ssg2", (16, 12, 20), 0, 0, None, "v", None),
    "ssg2-coef": ("ssg2", (16, 12, 20), 0, 0, None, "coef", None),
    "user-mxyz": ("iso3dfd", (24, 20, 70), 4, 0, None, "w", ("w", ["m", "x", "y", "z"], [3, 10, 9, 12])),
    "iso-r2-bt2": ("iso3dfd", (24, 20, 70), 4, 2, {"block_steps": 2}, "p", None),
}


def _case(name):
    stencil, n, eb, radius, opts, var, user = CASES[name]
    s = _solution(stencil, n, eb, radius, opts, user)
    return s, s.get_var(var)


class Geo:
    """Index ranges of a var, step dim included: the valid steps, the allocation and the rank's halo box."""

    def __init__(self, var):
        vi = var.info
        self.vi = vi
        self.dt = np.float32 if vi.elem_bytes == 4 else np.float64
        self.kind, self.alo, self.ahi, self.hlo, self.hhi = [], [], [], [], []
        for i in range(vi.num_dims):
            d = vi.dims[i]
            self.kind.append(d.kind)
            if d.kind == STEP:
                a = h = (vi.first_valid_step, vi.last_valid_step)
            elif d.kind == MISC:
                a = h = (d.first_misc_index, d.first_misc_index + d.domain_size - 1)
            else:
                a = (d.rank_offset - d.left_pad, d.rank_offset + d.domain_size + d.right_pad - 1)
                h = (d.rank_offset - d.left_halo, d.rank_offset + d.domain_size + d.right_halo - 1)
            self.alo.append(a[0]); self.ahi.append(a[1]); self.hlo.append(h[0]); self.hhi.append(h[1])
        self.has_step = bool(vi.has_step)

    def at_step(self, lo, hi, t):
        lo, hi = list(lo), list(hi)
        if self.has_step:
            lo[0] = hi[0] = t
        return lo, hi

    def boxes(self):
        """Single elements, an extent-1 dim in each position, the halo box, the whole allocation, a range of steps."""
        t = self.vi.last_valid_step if self.has_step else 0
        hb = self.at_step(self.hlo, self.hhi, t)
        mid = [(a + b) // 2 for a, b in zip(self.hlo, self.hhi)]
        out = [self.at_step(self.alo, self.alo, t), self.at_step(mid, mid, t), self.at_step(self.ahi, self.ahi, t)]
        for k in range(len(self.kind)):
            if self.kind[k] != STEP:
                f, l = list(hb[0]), list(hb[1])
                f[k] = l[k] = mid[k]
                out.append((f, l))
        out += [hb, self.at_step(self.alo, self.ahi, t)]
        if self.has_step and self.vi.step_alloc >= 2:
            f, l = list(self.hlo), list(self.hhi)
            f[0], l[0] = self.vi.first_valid_step, self.vi.first_valid_step + 1
            out.append((f, l))
        return out

    def whole(self):
        return list(self.alo), list(self.ahi)

    def region(self, first, last):
        """Slices of a box within the array of `whole()`."""
        return tuple(slice(f - a, l - a + 1) for f, l, a in zip(first, last, self.alo))


def _shape(first, last):
    return [int(l - f + 1) for f, l in zip(first, last)]


def get(var, first, last):
    return var.get_elements_in_slice(first, last).reshape(_shape(first, last))


def nonstep(g, first, last):
    """First index and shape of the non-step dims of a box."""
    k = 1 if g.has_step else 0
    return list(first[k:]), _shape(first[k:], last[k:])


def load_random(var, g, rng, lo=-1.0, hi=1.0):
    f, l = g.whole()
    a = rng.uniform(lo, hi, _shape(f, l)).astype(g.dt)
    var.set_elements_in_slice(a, f, l)
    return a


def _set_dev(var, t, first, last):
    n = C.c_int64(0)
    capi._chk(capi.lib().yb_var_set_slice_device(var.soln._h, var.index, C.c_void_p(t.data_ptr()), capi._arr(first), capi._arr(last),
                                                 C.byref(n)))
    return n.value


def _get_dev(var, t, first, last):
    n = C.c_int64(0)
    capi._chk(capi.lib().yb_var_get_slice_device(var.soln._h, var.index, C.c_void_p(t.data_ptr()), capi._arr(first), capi._arr(last),
                                                 C.byref(n)))
    return n.value


def check_reduction(r, vals, nsteps, dt, where=None):
    """Device reduction r of `vals` (dense, step outermost) against reduce_ref: sum, product, max, min and the fp32 sum of squares
    bit for bit, both sums within the fsum bound."""
    ref = reduce_ref(vals, nsteps)
    x = np.asarray(vals, np.float64).reshape(nsteps, -1)
    assert r["num"] == ref["num"], where
    for k in ("sum", "product", "max", "min") + (("sum_squares",) if dt == np.float32 else ()):
        assert r[k] == ref[k] or (math.isnan(r[k]) and math.isnan(ref[k])), (where, k, r[k], ref[k])
    if np.isfinite(x).all():
        ok, err, bound = fsum_check(r["sum"], x)
        assert ok, (where, "sum", err, bound)
        ok, err, bound = fsum_check(r["sum_squares"], x, square=True)
        assert ok, (where, "sum_squares", err, bound)


# ---- A. copies --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(CASES))
def test_copy_round_trips_touch_only_the_box(case):
    import torch
    s, v = _case(case)
    g = Geo(v)
    rng = np.random.default_rng(1)
    whole = load_random(v, g, rng)
    assert np.array_equal(bits(get(v, *g.whole())), bits(whole))
    for i, (f, l) in enumerate(g.boxes()):
        new = rng.uniform(-2, 2, _shape(f, l)).astype(g.dt)
        if i % 2:       # device-buffer forms
            assert _set_dev(v, torch.from_numpy(new).cuda(), f, l) == new.size
            back = torch.empty(new.shape, dtype=torch.float32 if g.dt == np.float32 else torch.float64, device="cuda")
            assert _get_dev(v, back, f, l) == new.size
            torch.cuda.synchronize()
            assert np.array_equal(bits(back.cpu().numpy()), bits(new)), (case, f, l)
        else:
            assert v.set_elements_in_slice(new, f, l) == new.size
            assert np.array_equal(bits(get(v, f, l)), bits(new)), (case, f, l)
        whole[g.region(f, l)] = new
        assert np.array_equal(bits(get(v, *g.whole())), bits(whole)), (case, f, l)
    s.close()


def test_host_staging_chunks_of_a_long_1d_box():
    """More than 64M fp32 elements: several 256 MiB staging chunks and a short last one."""
    n = (64 << 20) + 3_000_017
    s = _solution("test_1d", (n,))
    v = s.get_var("A")
    g = Geo(v)
    f, l = g.at_step(g.hlo, g.hhi, 0)
    a = np.random.default_rng(2).uniform(-1, 1, _shape(f, l)).astype(np.float32)
    assert a.nbytes > (256 << 20) and a.nbytes % (256 << 20)
    assert v.set_elements_in_slice(a, f, l) == a.size
    assert np.array_equal(bits(get(v, f, l)), bits(a))
    s.close()


def test_host_staging_one_row_per_chunk():
    """A 3-D box whose single outer row is larger than the 256 MiB staging buffer: one row per chunk."""
    s = capi.Solution("iso3dfd", radius=1)
    s.set_overall_domain_size_vec((2, 8200, 8200))
    need = storage_bytes(s)
    import torch
    if torch.cuda.mem_get_info()[0] < need + (2 << 30):
        s.close()
        pytest.skip(f"needs {need / 1e9:.1f} GB of device memory plus a 2 GB margin")
    s.prepare_solution(0)
    v = s.get_var("p")
    g = Geo(v)
    f, l = g.at_step([g.hlo[0], 0, -1, -1], [g.hhi[0], 3, 8200, 8200], 1)
    f[1], l[1] = 0, 1       # two rows of x
    a = np.random.default_rng(3).uniform(-1, 1, _shape(f, l)).astype(np.float32)
    assert a[0].nbytes > (256 << 20)
    assert v.set_elements_in_slice(a, f, l) == a.size
    assert np.array_equal(bits(get(v, f, l)), bits(a))
    s.close()


# ---- B. fills ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(CASES))
def test_set_elements_in_slice_same_writes_exactly_the_box(case):
    s, v = _case(case)
    g = Geo(v)
    whole = load_random(v, g, np.random.default_rng(4))
    for i, (f, l) in enumerate(g.boxes()):
        val = 0.1 + 0.37 * i      # not an fp32 value: rounds to the element type
        assert v.set_elements_in_slice_same(val, f, l) == int(np.prod(_shape(f, l)))
        whole[g.region(f, l)] = g.dt(val)
        assert np.array_equal(bits(get(v, *g.whole())), bits(whole)), (case, f, l)
    s.close()


@pytest.mark.parametrize("case", ["iso-p-f32", "test_1d", "ssg2-v", "iso-r2-bt2"])
def test_set_elements_in_slice_same_moves_the_valid_steps(case):
    windows = []
    for same in (True, False):
        s, v = _case(case)
        g = Geo(v)
        t = v.get_last_valid_step_index() + 1
        f, l = g.at_step(g.hlo, g.hhi, t)
        if same:
            v.set_elements_in_slice_same(0.5, f, l)
        else:
            v.set_elements_in_slice(np.full(_shape(f, l), 0.5, g.dt), f, l)
        windows.append((v.get_first_valid_step_index(), v.get_last_valid_step_index(), t))
        assert np.all(get(v, f, l) == g.dt(0.5))
        s.close()
    assert windows[0] == windows[1] and windows[0][1] == windows[0][2], windows


@pytest.mark.parametrize("case", list(CASES))
def test_set_all_elements_same_fills_every_slot(case):
    s, v = _case(case)
    g = Geo(v)
    load_random(v, g, np.random.default_rng(5))
    v.set_all_elements_same(-0.7)
    vi = v.info
    slot_bytes = vi.slot_elems * vi.elem_bytes
    nslots = vi.storage_bytes // slot_bytes
    assert nslots * slot_bytes == vi.storage_bytes and nslots >= (vi.step_alloc if vi.has_step else 1)
    if case == "iso-r2-bt2":
        assert nslots > vi.step_alloc, "the temporal tile's spare slots are part of the storage"
    base = v.device_ptr(0)
    buf = np.empty(vi.slot_elems, g.dt)
    for k in range(nslots):
        capi._chk(capi.lib().yb_copy_to_host(buf.ctypes.data, C.c_void_p(base + k * slot_bytes), slot_bytes))
        assert np.all(buf == g.dt(-0.7)), (case, k)
    s.close()


# ---- C. fill_hash -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(CASES))
def test_fill_hash_equals_hash_field(case):
    s, v = _case(case)
    g = Geo(v)
    ndd = len(s.get_domain_dim_names())
    shift = [3, -2, 5][:ndd]
    steps = range(v.info.step_alloc) if g.has_step else [0]
    for t in steps:
        f, l = g.at_step(g.hlo, g.hhi, t)
        first, shape = nonstep(g, f, l)
        salt = var_salt(v.get_name(), t)
        v.fill_hash(t, 23, salt, -1.0, 1.0)
        assert np.array_equal(bits(get(v, f, l).reshape(shape)), bits(hash_field(23, salt, first, shape, -1.0, 1.0, g.dt))), (case, t)
        v.fill_hash(t, 29, salt, 0.25, 0.75, shift=shift)
        sh = list(first)
        k = 0
        for i in range(v.info.num_dims):
            d = v.info.dims[i]
            if d.kind == STEP:
                continue
            if d.kind == DOMAIN:
                sh[k] += shift[d.domain_index]
            k += 1
        assert np.array_equal(bits(get(v, f, l).reshape(shape)), bits(hash_field(29, salt, sh, shape, 0.25, 0.75, g.dt))), (case, t)
    s.close()


# ---- D. reductions ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(CASES))
def test_reductions_match_the_restated_order(case):
    s, v = _case(case)
    g = Geo(v)
    rng = np.random.default_rng(6)
    for lo, hi in ((-1.0, 1.0), (0.97, 1.03)):     # the second keeps products of large boxes informative
        load_random(v, g, rng, lo, hi)
        for f, l in g.boxes():
            nsteps = l[0] - f[0] + 1 if g.has_step else 1
            check_reduction(v.reduce_elements_in_slice(f, l), get(v, f, l), nsteps, g.dt, (case, f, l))
    s.close()


COUNTS = [1, 31, 32, 33, 255, 256, 257, 606207, 606208, 606209, 3_000_001]


@pytest.mark.parametrize("eb", [4, 8])
def test_reductions_at_the_kernel_boundaries(eb):
    """Element counts around a warp, a block, the capped grid (2368 x 256) and chains of five."""
    rng = np.random.default_rng(7)
    if eb == 4:         # test_1d is generated for fp32 only
        s = _solution("test_1d", (3_100_000,))
        v = s.get_var("A")
        g = Geo(v)
        load_random(v, g, rng)
        for n in COUNTS:
            f, l = g.at_step([0], [n - 1], 0)
            check_reduction(v.reduce_elements_in_slice(f, l), get(v, f, l), 1, g.dt, n)
        f, l = [0, 0], [1, 606208]      # two steps of 606209
        check_reduction(v.reduce_elements_in_slice(f, l), get(v, f, l), 2, g.dt, "steps")
        s.close()
    s = _solution("iso3dfd", (48, 256, 256), eb)
    v = s.get_var("p")
    g = Geo(v)
    load_random(v, g, rng)
    for box in ([1, 0, 0, 0], [1, 36, 63, 255]), ([1, 0, 0, 0], [1, 45, 255, 255]), ([0, 5, 7, 9], [1, 5, 7, 265]):
        check_reduction(v.reduce_elements_in_slice(*box), get(v, *box), box[1][0] - box[0][0] + 1, g.dt, box)
    s.close()


@pytest.mark.parametrize("eb", [4, 8])
def test_reduction_special_values(eb):
    s = _solution("iso3dfd", (24, 20, 70), eb)
    v = s.get_var("p")
    g = Geo(v)
    rng = np.random.default_rng(8)
    box = ([1, 2, 3, 4], [1, 20, 17, 60])
    load_random(v, g, rng)
    pt = [1, 7, 9, 33]
    for planted in (np.nan, np.inf, -np.inf, 0.0):
        old = get(v, pt, pt)
        v.set_elements_in_slice(np.full((1, 1, 1, 1), planted, g.dt), pt, pt)
        r = v.reduce_elements_in_slice(*box)
        vals = get(v, *box)
        check_reduction(r, vals, 1, g.dt, planted)
        x = vals.astype(np.float64)
        if np.isnan(planted):
            assert math.isnan(r["sum"]) and math.isnan(r["sum_squares"]) and math.isnan(r["product"])
            assert r["max"] == np.nanmax(x) and r["min"] == np.nanmin(x)
        elif np.isinf(planted):
            assert r["sum"] == planted and r["sum_squares"] == np.inf and (r["max"] if planted > 0 else r["min"]) == planted
        else:
            assert r["product"] == 0.0
        v.set_elements_in_slice(old, pt, pt)
    # an all-negative box has a negative max; the sum of squares is not the sum
    neg = -rng.uniform(0.5, 1.5, _shape(*box)).astype(g.dt)
    v.set_elements_in_slice(neg, *box)
    r = v.reduce_elements_in_slice(*box)
    assert r["max"] == neg.max() < 0 and r["min"] == neg.min()
    assert r["sum"] < 0 < r["sum_squares"]
    check_reduction(r, neg, 1, g.dt, "negative")
    s.close()


_CLIP_SCRIPT = r'''
import json, math
import yask_kernel as yk
fac = yk.yk_factory()
s = fac.new_solution(fac.new_env())
for d, n in zip(s.get_domain_dim_names(), (24, 20, 70)):
    s.set_overall_domain_size(d, n)
s.prepare_solution()
p = s.get_var("p")
p.set_all_elements_same(0.25)
p.set_elements_in_slice_same(-3.0, [1, 10, 0, 0], [1, 30, 5, 5], False)
lo, hi = p.get_first_local_index_vec(), p.get_last_local_index_vec()
m = sum(getattr(yk.yk_var, k) for k in ("yk_sum_reduction", "yk_sum_squares_reduction", "yk_product_reduction",
                                        "yk_max_reduction", "yk_min_reduction"))
def red(f, l, strict):
    r = p.reduce_elements_in_slice(m, f, l, strict)
    return [r.get_num_elements_reduced(), r.get_sum(), r.get_sum_squares(), r.get_product(), r.get_max(), r.get_min()]
out = {"lo": lo, "hi": hi}
f, l = [0, -100, 3, -50], [5, 15, 400, 30]
out["clip"] = red(f, l, False)
out["explicit"] = red([max(a, b) for a, b in zip(f, lo)], [min(a, b) for a, b in zip(l, hi)], True)
out["outside"] = red([1, 1000, 0, 0], [1, 1100, 5, 5], False)
try:
    red(f, l, True)
    out["strict"] = "no error"
except Exception as e:
    out["strict"] = str(e)
out["same_clip"] = p.set_elements_in_slice_same(0.5, [1, -100, 3, -50], [1, 15, 400, 30], False)
out["same_outside"] = p.set_elements_in_slice_same(0.5, [1, 1000, 0, 0], [1, 1100, 5, 5], False)
print(json.dumps(out))
'''


def test_non_strict_reduction_and_fill_clip_to_the_allocation():
    """reduce_elements_in_slice and set_elements_in_slice_same with strict_indices false, through the C++ API module: a box
    partly outside the allocation is clipped to it, one wholly outside reduces nothing and writes nothing."""
    env = dict(os.environ, PYTHONPATH=os.path.join(ROOT, "yask_b200", "lib", "python", "iso3dfd"))
    r = subprocess.run([sys.executable, "-c", _CLIP_SCRIPT], capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    lo, hi = out["lo"], out["hi"]
    f, l = [0, -100, 3, -50], [5, 15, 400, 30]
    cf = [max(a, b) for a, b in zip(f, lo)]
    cl = [min(a, b) for a, b in zip(l, hi)]
    count = int(np.prod(_shape(cf, cl)))
    assert out["clip"] == out["explicit"] and out["clip"][0] == count
    assert out["outside"] == [0, 0.0, 0.0, 1.0, -math.inf, math.inf]
    assert "not" in out["strict"] or "outside" in out["strict"], out["strict"]
    assert out["same_clip"] == int(np.prod(_shape(cf[1:], cl[1:]))) and out["same_outside"] == 0


# ---- E. checksum ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["iso-p-f32", "iso-v-f32", "iso-p-f64", "iso-v-f64", "test_1d", "wave2d", "iso-r2-bt2"])
def test_checksum_equals_checksum_ref(case):
    s, v = _case(case)
    g = Geo(v)
    load_random(v, g, np.random.default_rng(9))
    for t in (range(v.info.step_alloc) if g.has_step else [0]):
        f, l = v.domain_box(t)
        first, shape = nonstep(g, f, l)
        assert v.checksum(t) == checksum_ref(get(v, f, l).reshape(shape), first), (case, t)
    s.close()


@pytest.mark.parametrize("case", ["ssg2-v", "ssg2-coef", "user-mxyz"])
def test_checksum_refuses_four_non_step_dims(case):
    s, v = _case(case)
    with pytest.raises(capi.YaskError) as e:
        v.checksum(0)
    assert e.value.code == -6 and "at most 3 non-step dims" in str(e.value)     # YB_EUNSUPPORTED
    s.close()


# ---- F. rank grids ----------------------------------------------------------------------------------------------------------
GRIDS = [("iso3dfd", (48, 40, 64), (2, 1, 1), ("p", "v")), ("iso3dfd", (40, 48, 64), (1, 2, 1), ("p", "v")),
         ("wave2d", (60, 70), (2, 2), ("u", "v", "e"))]


def _ranks(stencil, n, grid):
    solns = []
    for r in range(int(np.prod(grid))):
        s = capi.Solution(stencil)
        s.set_overall_domain_size_vec(n)
        s.set_num_ranks_vec(grid)
        s.set_rank_index_vec(multi.grid_coords(r, grid))
        s.prepare_solution(0)
        solns.append(s)
    multi.connect_local(solns)
    return solns


def _fill(s, names, seed):
    for name in names:
        v = s.get_var(name)
        for t in (range(v.info.step_alloc) if v.info.has_step else [0]):
            v.fill_hash(t, seed, var_salt(name, t), -1.0, 1.0)


def _box_in(var, f, l):
    """Part of box [f, l] (every dim but the step) inside the rank's domain, or None."""
    df, dl = var.domain_box(f[0])
    cf = [f[0]] + [max(a, b) for a, b in zip(f[1:], df[1:])]
    cl = [l[0]] + [min(a, b) for a, b in zip(l[1:], dl[1:])]
    return (cf, cl) if all(a <= b for a, b in zip(cf, cl)) else None


@pytest.mark.parametrize("stencil,n,grid,names", GRIDS, ids=["iso-2x1x1", "iso-1x2x1", "wave2d-2x2"])
def test_rank_grid_fill_hash_reductions_and_checksums(stencil, n, grid, names):
    one = _solution(stencil, n)
    _fill(one, names, 31)
    ranks = _ranks(stencil, n, grid)
    for s in ranks:
        _fill(s, names, 31)
    for name in names:
        ref = one.get_var(name)
        dt = ref.dtype
        for t in (0, 1):
            f, l = ref.domain_box(t)
            whole = get(ref, f, l).astype(np.float64)
            r1 = ref.reduce_elements_in_slice(f, l)
            parts = []
            csum = 0
            for s in ranks:
                v = s.get_var(name)
                hf, hl = v.halo_box(t)
                first, shape = nonstep(Geo(v), hf, hl)
                assert np.array_equal(bits(get(v, hf, hl).reshape(shape)),
                                      bits(hash_field(31, var_salt(name, t if ref.info.has_step else 0), first, shape, -1.0, 1.0,
                                                      dt))), (name, t)
                parts.append(v.reduce_elements_in_slice(*v.domain_box(t)))
                csum += v.checksum(t)
            assert csum % (1 << 64) == ref.checksum(t), (name, t)
            assert sum(p["num"] for p in parts) == r1["num"] == whole.size
            assert max(p["max"] for p in parts) == r1["max"] and min(p["min"] for p in parts) == r1["min"]
            for k, sq in (("sum", False), ("sum_squares", True)):
                ok, err, bound = fsum_check(sum(p[k] for p in parts), whole, square=sq)
                assert ok and fsum_check(r1[k], whole, square=sq)[0], (name, t, k, err, bound)
    for s in ranks + [one]:
        s.close()


@pytest.mark.parametrize("stencil,n,grid,names", GRIDS, ids=["iso-2x1x1", "iso-1x2x1", "wave2d-2x2"])
def test_rank_grid_fills_reach_the_neighbours(stencil, n, grid, names):
    """set_elements_in_slice_same of a box straddling the rank boundaries, and set_all_elements_same, between runs: the
    neighbours must see the writes (the fills mark the halos dirty), so the ranks give the single-rank result bit for bit."""
    nd = len(n)
    box_f = [n[d] // 2 - 3 for d in range(nd)]
    box_l = [n[d] // 2 + 2 for d in range(nd)]
    target = names[0]

    def run(solns, clip):
        for s in solns:
            _fill(s, names, 37)
        for s in solns:
            s.run_solution(0, 1)
        for s in solns:
            v = s.get_var(target)
            t = v.get_last_valid_step_index()
            b = _box_in(v, [t] + box_f, [t] + box_l) if clip else ([t] + box_f, [t] + box_l)
            if b:
                v.set_elements_in_slice_same(1.75, *b)
        for s in solns:
            s.run_solution(2, 3)
        for s in solns:
            s.get_var(names[1]).set_all_elements_same(0.125)
        for s in solns:
            s.run_solution(4, 5)
        out = {}
        for s in solns:
            for name in names:
                v = s.get_var(name)
                if not v.info.has_step:
                    continue
                t = v.get_last_valid_step_index()
                f, l = v.domain_box(t)
                out.setdefault(name, []).append((f, get(v, f, l)))
        return out

    one = _solution(stencil, n)
    ref = run([one], False)
    ranks = _ranks(stencil, n, grid)
    got = run(ranks, True)
    for name, pieces in got.items():
        (rf, whole), = ref[name]
        for f, a in pieces:
            sl = tuple(slice(x - y, x - y + m) for x, y, m in zip(f[1:], rf[1:], a.shape[1:]))
            assert np.array_equal(bits(a[0]), bits(whole[0][sl])), (name, f)
    for s in ranks + [one]:
        s.close()


# ---- G. past 2^31 elements per slot -----------------------------------------------------------------------------------------
def test_var_data_past_2_31():
    import torch
    s = capi.Solution("iso3dfd")
    n = (1300, 1300, 1300)
    s.set_overall_domain_size_vec(n)
    need = storage_bytes(s)
    free = torch.cuda.mem_get_info()[0]
    if free < need + (2 << 30):
        s.close()
        pytest.skip(f"needs {need / 1e9:.1f} GB of device memory plus a 2 GB margin, {free / 1e9:.1f} GB free")
    try:
        s.prepare_solution(0)
        p = s.get_var("p")
        vi = p.info
        assert vi.slot_elems > TWO31
        g = Geo(p)
        dims = [vi.dims[i] for i in range(1, 4)]
        xc = crossing_index(vi)

        def point_of(off):
            """Global index of the element at offset `off` of a slot (inside the allocation)."""
            idx = []
            for d in dims:
                c, off = divmod(off, d.stride)
                idx.append(c + d.rank_offset - d.left_pad)
            return idx

        # fill_hash: windows straddling element offset 2^31 (the x plane where it crosses, and the row inside that plane)
        p.fill_hash(0, 41, var_salt("p", 0), -1.0, 1.0)
        c = point_of(TWO31)
        wins = [([0, xc - 2, 300, 500], [0, xc + 1, 340, 560]), ([0] + c[:2] + [c[2] - 40], [0] + c[:2] + [c[2] + 40])]
        for f, l in wins:
            first, shape = f[1:], _shape(f[1:], l[1:])
            assert elem_offset(vi, first) < TWO31 <= elem_offset(vi, l[1:])
            assert np.array_equal(bits(get(p, f, l).reshape(shape)), bits(hash_field(41, var_salt("p", 0), first, shape, -1.0, 1.0)))
        # get / set / set_elements_in_slice_same of the same windows
        rng = np.random.default_rng(11)
        for f, l in wins:
            f1, l1 = [1] + f[1:], [1] + l[1:]
            a = rng.uniform(-1, 1, _shape(f1, l1)).astype(np.float32)
            p.set_elements_in_slice(a, f1, l1)
            assert np.array_equal(bits(get(p, f1, l1)), bits(a))
            assert p.set_elements_in_slice_same(0.3, f1, l1) == a.size
            assert np.all(get(p, f1, l1) == np.float32(0.3))
        # reduction over the whole slot: 0.5 everywhere but four planted values; every partial sum is exact
        p.set_all_elements_same(0.5)
        last_off = elem_offset(vi, g.ahi[1:])
        planted = {0: 3.0, TWO31 - 1: -2.5, TWO31: 7.5, last_off: -4.0}
        for off, val in planted.items():
            pt = [0] + point_of(off)
            assert elem_offset(vi, pt[1:]) == off
            p.set_elements_in_slice(np.full((1, 1, 1, 1), val, np.float32), pt, pt)
        f, l = g.at_step(g.alo, g.ahi, 0)
        num = int(np.prod(_shape(f, l)))
        assert num == last_off + 1
        r = p.reduce_elements_in_slice(f, l)
        assert r["num"] == num
        assert r["sum"] == 0.5 * (num - 4) + sum(planted.values())
        assert r["max"] == 7.5 and r["min"] == -4.0
        # checksum: changing one element past 2^31 changes it by exactly term(new) - term(old)
        p.fill_hash(1, 43, var_salt("p", 1), -1.0, 1.0)
        before = p.checksum(1)
        pt = [c[0] + 1, 650, 650]
        assert elem_offset(vi, pt) >= TWO31
        old = get(p, [1] + pt, [1] + pt).reshape(1, 1, 1)
        new = np.full((1, 1, 1), 0.8125, np.float32)
        p.set_elements_in_slice(new.reshape(1, 1, 1, 1), [1] + pt, [1] + pt)
        diff = int(checksum_terms(new, pt).ravel()[0]) - int(checksum_terms(old, pt).ravel()[0])
        assert (p.checksum(1) - before) % (1 << 64) == diff % (1 << 64)
    finally:
        s.close()
