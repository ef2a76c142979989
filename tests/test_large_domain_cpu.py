"""CPU: domains past 2^31 elements per var slot.

  * plan_geometry() plans them for the generated and the hand-written solutions without refusing, with 64-bit slot sizes and
    storage byte counts through the C ABI;
  * the size limits the generated kernels keep (32-bit neighbour offsets: (x halo + 1) x-planes below 2^31 elements; 32-bit
    coordinates: a dimension below 2^31 elements) are refused by plan_geometry(), before anything is allocated, with a message
    that names them;
  * the window method of tests/test_large_domain_gpu.py: on a domain small enough for the CPU oracle to run whole, the points
    the cone rule keeps in a window run on its own are bit-identical to the same points of the full run.
"""
import ctypes

import numpy as np
import pytest

from tests.large_domain import TWO31, Window, bits, gen_reach, gen_window_ref, iso_window_ref
from yask_b200 import capi

# (solution, radius, elem_bytes, overall size): each just past 2^31 elements in the slot of its largest var
PLANS = [
    ("3axis", 0, 0, (1300, 1300, 1300)),
    ("iso3dfd_sponge", 8, 4, (1300, 1300, 1300)),     # generated (radius 8 fp32)
    ("test_2d", 0, 0, (47000, 47000)),
    ("iso3dfd", 8, 8, (1300, 1300, 1300)),            # generated (fp64 radius 8)
    ("iso3dfd", 8, 4, (1300, 1300, 1300)),            # hand-written
]


def test_var_info_sizes_are_64_bit():
    fields = dict(capi.VarInfo._fields_)
    assert fields["slot_elems"] is ctypes.c_int64 and fields["storage_bytes"] is ctypes.c_int64


@pytest.mark.parametrize("stencil,radius,eb,n", PLANS, ids=[f"{p[0]}-r{p[1]}-eb{p[2]}" for p in PLANS])
def test_plan_geometry_past_2_31(stencil, radius, eb, n):
    s = capi.Solution(stencil, radius=radius, elem_bytes=eb)
    s.set_overall_domain_size_vec(n)
    s.plan_geometry()
    ebytes = s.get_element_bytes()
    biggest = 0
    for var in s.get_vars():
        vi = var.info
        slots = vi.step_alloc if vi.has_step else 1
        assert vi.storage_bytes == slots * vi.slot_elems * ebytes, (vi.name, vi.storage_bytes, vi.slot_elems)
        biggest = max(biggest, vi.slot_elems)
    assert biggest > TWO31
    s.close()


def test_generated_neighbour_offset_limit_is_refused_by_plan_geometry():
    """A thin slab with a huge y*z plane: 5 x-planes (3axis: x halo 4) of about 5.8e8 elements pass 2^31."""
    s = capi.Solution("3axis", elem_bytes=0)
    s.set_overall_domain_size_vec((8, 24000, 24000))
    with pytest.raises(capi.YaskError) as e:
        s.plan_geometry()
    msg = str(e.value)
    assert "2^31" in msg and "24000 x 24000" in msg, msg
    s.close()
    # the same plane count with a smaller plane is fine, whatever the x extent
    s = capi.Solution("3axis", elem_bytes=0)
    s.set_overall_domain_size_vec((20000, 2000, 2000))
    s.plan_geometry()
    assert s.get_var("A").info.slot_elems > TWO31
    s.close()


@pytest.mark.parametrize("stencil,n", [("test_1d", ((1 << 31) + 1000,)), ("test_2d", (3, (1 << 31) + 1000))])
def test_generated_dimension_limit_is_refused_by_plan_geometry(stencil, n):
    """Launch boxes and point coordinates of the generated kernels are int: a dimension of 2^31 elements or more (1-D, or the
    unit-stride dim of a 2-D solution with few rows, both within one card's memory) is refused, naming the limit and the size."""
    s = capi.Solution(stencil, elem_bytes=0)
    s.set_overall_domain_size_vec(n)
    with pytest.raises(capi.YaskError) as e:
        s.plan_geometry()
    msg = str(e.value)
    assert "2^31 - 1" in msg and f"domain {n[-1]}" in msg, msg
    s.close()
    # just below the limit, pads included, it plans
    s = capi.Solution(stencil, elem_bytes=0)
    s.set_overall_domain_size_vec(n[:-1] + ((1 << 31) - 1000,))
    s.plan_geometry()
    s.close()


def _windows(n, size, m):
    nd = len(n)
    mid = [a // 2 - s // 2 for a, s in zip(n, size)]
    return [Window(n, [0] * nd, size, m), Window(n, mid, size, m), Window(n, [a - s for a, s in zip(n, size)], size, m)]


@pytest.mark.parametrize("stencil,n,size", [("3axis", (48, 40, 72), (24, 22, 26)), ("iso3dfd_sponge", (70, 66, 80), (40, 42, 44)),
                                            ("test_2d", (90, 110), (30, 34))])
def test_window_method_on_generated_solutions(stencil, n, size):
    seed, steps = 23, 2
    m = steps * gen_reach(stencil)
    full = Window(n, [0] * len(n), n, m)
    whole = gen_window_ref(stencil, full, seed, steps, 1)
    for w in _windows(n, size, m):
        got = gen_window_ref(stencil, w, seed, steps, 1)
        assert got.keys() == whole.keys()
        for name, (tl, arr) in got.items():
            ref = whole[name][1][tuple(slice(a, b) for a, b in zip(w.kept_lo, w.kept_hi))]
            assert tl == whole[name][0] and np.array_equal(bits(arr), bits(ref)), (stencil, name, w.lo)
    # and the trimming is needed: the middle window, untrimmed, differs from the full run next to its faces
    w = _windows(n, size, 0)[1]
    name, (_, arr) = next(iter(gen_window_ref(stencil, w, seed, steps, 1).items()))
    ref = whole[name][1][tuple(slice(a, a + s) for a, s in zip(w.lo, w.size))]
    assert not np.array_equal(bits(arr), bits(ref))


@pytest.mark.parametrize("R,eb,steps", [(8, 4, 2), (4, 8, 2), (2, 4, 4)])
def test_window_method_on_iso3dfd(R, eb, steps):
    seed, n, size = 31, (76, 70, 84), (44, 40, 50)
    dt = np.float32 if eb == 4 else np.float64
    m = steps * R
    whole = iso_window_ref(Window(n, [0, 0, 0], n, m), seed, R, R, steps, 2, dt)
    for w in _windows(n, size, m):
        got = iso_window_ref(w, seed, R, R, steps, 2, dt)
        ref = whole[tuple(slice(a, b) for a, b in zip(w.kept_lo, w.kept_hi))]
        assert np.array_equal(bits(got), bits(ref)), w.lo
    # and the trimming is needed: the middle window, untrimmed, differs from the full run next to its faces
    w = _windows(n, size, 0)[1]
    untrimmed = iso_window_ref(w, seed, R, R, steps, 2, dt)
    ref = whole[tuple(slice(a, a + s) for a, s in zip(w.lo, w.size))]
    assert not np.array_equal(bits(untrimmed), bits(ref))
