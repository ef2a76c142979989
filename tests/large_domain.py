"""Windows of a large domain checked against the CPU oracle (test infrastructure of tests/test_large_domain_*.py).

A domain past 2^31 elements per var slot is too large for the CPU oracle, but the engine fills it with a hash of GLOBAL indices
(fill_hash), so any window of it can be refilled on the host.  The oracle runs `steps` steps over the window alone; the window's
halo cells then hold initial values where the full run had evolving ones, and the error this makes moves inwards by at most
`reach` points per step.  The cone rule keeps the points at least steps * reach from every window face that lies inside the
global domain; faces on the global domain's boundary keep everything, because there the window's halo is the real halo, which
no step writes.
"""
import numpy as np

from oracle import oracle as O
from tests.golden.ranges import RANGES
from tests.helpers import range_of
from yask_b200.synth import hash_field, var_salt

TWO31 = 1 << 31

# (below, at) sizes of the generated kernels' switch to 64-bit positions (GenEngine::prepare), for the switch-point cases of
# tests/test_generated_wide_gpu.py: the largest var slot lies under 2^31 elements by less than one x plane, then at or above
# 2^31 by less than one x plane.  At the "at" size 2^31 falls inside the last x pad plane, so only the high corner's x
# neighbours read past it.  tests/test_generated_wide_cpu.py checks both from plan_geometry().
SWITCH_SIZES = {
    "3axis": ((1416, 1200, 1200), (1417, 1200, 1200)),
    "test_2d": ((45644, 47000), (45645, 47000)),
}


class Window:
    """Oracle window [lo, lo + size) of a global domain of size n, trimmed by the cone rule to the kept box [kept_lo, kept_hi)."""

    def __init__(self, n, lo, size, margin):
        self.n, self.lo, self.size = list(n), [int(a) for a in lo], [int(a) for a in size]
        assert all(0 <= a and a + s <= m for a, s, m in zip(self.lo, self.size, self.n)), (lo, size, n)
        self.kept_lo = [a + (margin if a > 0 else 0) for a in self.lo]
        self.kept_hi = [a + s - (margin if a + s < m else 0) for a, s, m in zip(self.lo, self.size, self.n)]
        assert all(a < b for a, b in zip(self.kept_lo, self.kept_hi)), "window too small for its margin"

    def kept_slices(self):
        """Slices of the kept box within an array over the window's domain."""
        return tuple(slice(k - a, h - a) for k, h, a in zip(self.kept_lo, self.kept_hi, self.lo))

    def kept_box(self, step):
        """(first, last) of the kept box at API step `step`, for get_elements_in_slice."""
        return [step] + self.kept_lo, [step] + [h - 1 for h in self.kept_hi]


def elem_offset(info, point):
    """Element offset, within its step slot, of the global domain point `point` of a var (VarInfo from the C ABI)."""
    off, k = 0, 0
    for i in range(info.num_dims):
        d = info.dims[i]
        if d.kind != 1:       # domain dims only
            continue
        off += (point[k] - d.rank_offset + d.left_pad) * d.stride
        k += 1
    return off


def crossing_index(info):
    """Smallest index of the first domain dim whose plane (at the low corner of the other dims) starts at element offset
    2^31 or more."""
    d0 = [info.dims[i] for i in range(info.num_dims) if info.dims[i].kind == 1][0]
    nd = sum(1 for i in range(info.num_dims) if info.dims[i].kind == 1)
    base = elem_offset(info, [0] * nd)
    return -(-(TWO31 - base) // d0.stride)


def three_windows(info, n, size, margin):
    """The windows a large-domain case checks: at the low corner, straddling the plane of the first domain dim where the element
    offset crosses 2^31 (the other dims centred), and at the high corner.  Asserts that the last two lie past 2^31 elements."""
    nd = len(n)
    xc = crossing_index(info)
    mid = [max(0, min(m - s, m // 2 - s // 2)) for m, s in zip(n, size)]
    wins = [Window(n, [0] * nd, size, margin),
            Window(n, [xc - size[0] // 2] + mid[1:], size, margin),
            Window(n, [m - s for m, s in zip(n, size)], size, margin)]
    first = [elem_offset(info, w.kept_lo) for w in wins]
    last = [elem_offset(info, [h - 1 for h in w.kept_hi]) for w in wins]
    assert last[0] < TWO31, "the low corner window should lie below 2^31 elements"
    assert first[1] < TWO31 <= last[1], ("the middle window should straddle 2^31 elements", first[1], last[1])
    assert first[2] >= TWO31, ("the high corner window should lie past 2^31 elements", first[2])
    return wins


# ---- emitter-generated solutions (oracle.gen_run) -----------------------------------------------------------------------------
def gen_reach(stencil):
    """Points of dependence per step of a generated solution: its largest halo."""
    ir = O.gen_ir(stencil)
    return max([h for v in ir["vars"] for hs in v["halo"].values() for h in hs] + [0])


def gen_window_inputs(stencil, w, seed):
    """Oracle inputs over window w (its domain plus each var's halo), from the same hash of global indices as fill_hash."""
    ir = O.gen_ir(stencil)
    dt = np.float32 if ir["elem_bytes"] == 4 else np.float64
    dd = ir["domain_dims"]
    ins = {}
    for v in ir["vars"]:
        if v.get("scratch"):
            continue
        vlo, vhi = range_of(RANGES[stencil], v["name"])
        vd = [d for d in v["dims"] if d != ir["step_dim"]]
        first = [w.lo[dd.index(d)] - v["halo"][d][0] for d in vd]
        shp = [w.size[dd.index(d)] + sum(v["halo"][d]) for d in vd]
        has_step = bool(v["dims"]) and v["dims"][0] == ir["step_dim"]
        for t in range(v["alloc_t"] if has_step else 1):
            ins[(v["name"], t)] = hash_field(seed, var_salt(v["name"], t), first, shp, vlo, vhi, dt)
    return ins


def gen_window_ref(stencil, w, seed, steps, contract):
    """{var: (last valid step, kept box)} of every written var of a generated solution, run by the oracle over window w."""
    ir = O.gen_ir(stencil)
    dd = ir["domain_dims"]
    out = O.gen_run(stencil, w.size, steps, gen_window_inputs(stencil, w, seed), contract=contract)
    res = {}
    for name, (tl, arr) in out.items():
        v = [x for x in ir["vars"] if x["name"] == name][0]
        dom = arr[tuple(slice(v["halo"][d][0], v["halo"][d][0] + w.size[i]) for i, d in enumerate(dd))]
        res[name] = (tl, np.ascontiguousarray(dom[w.kept_slices()]))
    return res


def fill_gen(s, stencil, seed):
    """fill_hash every var of a prepared generated solution, every step slot, with the ranges its oracle inputs use."""
    for var in s.get_vars():
        vi = var.info
        lo, hi = range_of(RANGES[stencil], vi.name.decode())
        for t in (range(vi.step_alloc) if vi.has_step else [0]):
            var.fill_hash(t, seed, var_salt(vi.name.decode(), t), lo, hi)


# ---- hand-written iso3dfd (oracle.iso3dfd_run) --------------------------------------------------------------------------------
def iso_window_ref(w, seed, R, h, steps, mode, dt):
    """Kept box of p after `steps` steps of iso3dfd radius R (p's halo h), run by the oracle over window w."""
    p = [hash_field(seed, var_salt("p", t), [a - h for a in w.lo], [s + 2 * h for s in w.size], -1, 1, dt) for t in (0, 1)]
    v = hash_field(seed, var_salt("v", 0), w.lo, w.size, 0.05, 0.3, dt)
    out = O.iso3dfd_run(p[0], p[1], v, R, steps, mode)[h:-h, h:-h, h:-h]
    return np.ascontiguousarray(out[w.kept_slices()])


def fill_iso(s, seed):
    p = s.get_var("p")
    for t in (0, 1):
        p.fill_hash(t, seed, var_salt("p", t), -1.0, 1.0)
    s.get_var("v").fill_hash(0, seed, var_salt("v", 0), 0.05, 0.3)


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def storage_bytes(s):
    """Device memory the vars of a solution need, from plan_geometry() (no device involved)."""
    s.plan_geometry()
    return sum(v.info.storage_bytes for v in s.get_vars())
