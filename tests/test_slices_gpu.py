"""Slice recorders on the device, bit for bit against the reference API loop on the same hash-filled inputs:

    for t in steps: run_solution(t, t); [sources; receivers]; frame[(u - t0) // every] = get_elements_in_slice(var, u, box)[::stride]

(u = t + 1, or t - 1 for a reverse solution; a frame only when u - t0 is a multiple of `every` and its row is below nrows).  Every
frame, every written var at its valid steps and the exact number of recording launches are compared."""
import numpy as np
import pytest

from tests.test_points_gpu import amp_table, calls, fill, make, outputs, same
from yask_b200 import capi, multi

pytestmark = pytest.mark.gpu


class Rec:
    """A recorder: var, inclusive global box, stride, t0, every, nrows."""

    def __init__(self, var, first, last, stride=None, t0=1, every=1, nrows=None):
        self.var, self.first, self.last = var, list(first), list(last)
        self.stride = list(stride) if stride else [1] * len(first)
        self.t0, self.every, self.nrows = t0, every, nrows

    def row(self, u):
        k = u - self.t0
        return k // self.every if k >= 0 and k % self.every == 0 and k // self.every < self.nrows else None

    def shape(self):
        return tuple((b - a) // k + 1 for a, b, k in zip(self.first, self.last, self.stride))

    def add(self, s):
        return s.add_slice(self.var, self.first, self.last, self.t0, self.nrows, stride=self.stride, every=self.every)

    def read(self, s, u):
        box = s.get_var(self.var).get_elements_in_slice([u] + self.first, [u] + self.last)
        return box[tuple(slice(None, None, k) for k in self.stride)]


def slice_loop(s, first, last, off, recs, src=None, frames=None):
    """The reference API loop: one step per call, sources through one-element slices, then each due frame read back."""
    dt = np.float32 if s.get_element_bytes() == 4 else np.float64
    if frames is None:
        frames = [np.zeros((r.nrows,) + r.shape(), dt) for r in recs]
    step = 1 if last >= first else -1
    for t in range(first, last + step, step):
        s.run_solution(t, t)
        u = t + off
        if src and 0 <= u - src[2] < len(src[3]):
            var = s.get_var(src[0])
            for i, p in enumerate(src[1]):
                idx = [u] + list(p)
                cur = var.get_elements_in_slice(idx, idx).reshape(-1)[0]
                var.set_elements_in_slice(np.array([dt(cur) + dt(src[3][u - src[2]][i])], dt), idx, idx)
        for r, f in zip(recs, frames):
            if r.row(u) is not None:
                f[r.row(u)] = r.read(s, u)
    return frames


def due_steps(first, last, off, recs):
    step = 1 if last >= first else -1
    return sum(1 for t in range(first, last + step, step) if any(r.row(t + off) is not None for r in recs))


def single_case(stencil, n, steps, recs, radius=0, eb=4, opts=(), reverse=False, splits=None, src=None, fill_steps=None):
    first, last, off = (steps, 1, -1) if reverse else (0, steps - 1, 1)
    fill_steps = fill_steps or (list(range(steps, steps + 4)) if reverse else [0, 1, 2, 3])
    s = make(stencil, n, radius, eb, opts)
    fill(s, stencil, fill_steps)
    if src:
        s.set_sources(*src)
    ids = [r.add(s) for r in recs]
    assert ids == list(range(len(recs)))
    for a, b in calls(first, last, splits):
        s.run_solution(a, b)
    got = [s.get_slice_frames(i) for i in ids]
    fields = outputs(s)
    launches = int(s.get_option("slice_launches"))
    tt = s.get_option("tt_launches") if ("block_steps", 2) in opts else "0"
    s.close()
    o = make(stencil, n, radius, eb, opts)
    fill(o, stencil, fill_steps)
    ref = slice_loop(o, first, last, off, recs, src)
    ref_fields = outputs(o)
    o.close()
    for (f, owned), rf in zip(got, ref):
        assert owned.all()
        assert same(f, rf), np.argwhere(f != rf)[:5]
    assert fields.keys() == ref_fields.keys()
    for k in ref_fields:
        assert same(fields[k], ref_fields[k]), k
    assert tt == "0"                                       # no pair runs while a recorder is set
    assert launches == due_steps(first, last, off, recs), launches


N8 = (40, 36, 64)
ISO_R8 = {
    "x-plane": [Rec("p", [17, 0, 0], [17, 35, 63], nrows=6)],
    "y-plane": [Rec("p", [0, 20, 0], [39, 20, 63], nrows=6)],
    "z-plane": [Rec("p", [0, 0, 31], [39, 35, 31], nrows=6)],
    "decimated-odd-first": [Rec("p", [1, 1, 1], [39, 35, 63], stride=[2, 3, 4], nrows=6)],
    "every-3-mid-run-short": [Rec("p", [0, 3, 0], [39, 3, 63], t0=3, every=3, nrows=2)],
    "two-on-one-var": [Rec("p", [0, 0, 5], [39, 35, 5], nrows=6), Rec("p", [2, 1, 0], [38, 34, 63], stride=[4, 3, 2], t0=2, every=2, nrows=3)],
}


@pytest.mark.parametrize("case", list(ISO_R8))
def test_iso3dfd_r8(case):
    """The resident radius-8 sweep: planes in each dim, a decimated full box, an interval, two recorders at once."""
    steps = 9 if case == "every-3-mid-run-short" else 6
    single_case("iso3dfd", N8, steps, ISO_R8[case], radius=8)


def test_iso3dfd_r8_split_calls():
    """A run split over two run_solution() calls fills the rows one call does."""
    single_case("iso3dfd", N8, 7, [Rec("p", [1, 0, 2], [39, 35, 62], stride=[2, 5, 3], t0=2, every=2, nrows=3)], radius=8, splits=[3, 4])


def test_block_steps_fall_back_and_resume():
    """iso3dfd radius 2, block_steps=2: while recording every step is one launch; after clear_slices() pairs come back."""
    n, opts = (40, 24, 160), (("block_steps", 2), ("tt_variant", 0))
    rec = Rec("p", [0, 5, 0], [39, 5, 159], nrows=4)
    single_case("iso3dfd", n, 4, [rec], radius=2, opts=opts)
    s = make("iso3dfd", n, 2, 4, opts)
    fill(s, "iso3dfd", [0, 1])
    rec.add(s)
    s.run_solution(0, 3)
    assert s.get_option("tt_launches") == "0" and s.get_option("slice_launches") == "4"
    frames, _ = s.get_slice_frames(0)
    s.clear_slices()
    s.run_solution(4, 7)
    assert int(s.get_option("tt_launches")) == 2 and s.get_option("slice_launches") == "4"
    got = outputs(s)
    s.close()
    o = make("iso3dfd", n, 2, 4, opts)
    fill(o, "iso3dfd", [0, 1])
    ref_frames = slice_loop(o, 0, 3, 1, [rec])[0]
    slice_loop(o, 4, 7, 1, [])
    ref = outputs(o)
    o.close()
    assert same(frames, ref_frames)
    for k in ref:
        assert same(got[k], ref[k]), k


def out_vars(stencil, eb):
    s = capi.Solution(stencil, elem_bytes=eb)
    names = [v.get_name() for v in s.get_vars() if v.info.is_output]
    s.close()
    return names


def whole_box(n):
    return [0] * len(n), [m - 1 for m in n]


@pytest.mark.parametrize("stencil,n,steps,radius,eb,opts,reverse", [
    ("iso3dfd", (32, 28, 48), 5, 4, 8, (), False),
    ("iso3dfd_sponge", (30, 26, 48), 5, 4, 4, (), False),
    ("3axis", (30, 20, 64), 5, 1, 8, (("block_steps", 2),), False),
    ("awp_elastic", (21, 19, 40), 4, 0, 0, (), False),
    ("ssg", (21, 19, 40), 4, 0, 8, (), False),
    ("wave2d", (37, 50), 5, 0, 0, (), False),
    ("test_1d", (70,), 5, 0, 0, (), False),
    ("test_reverse_2d", (37, 50), 5, 0, 0, (), True),
], ids=["iso-fp64-r4", "sponge-r4", "3axis-fp64-r1-bt2", "awp_elastic", "ssg-fp64", "wave2d", "test_1d", "reverse-2d"])
def test_other_stencils(stencil, n, steps, radius, eb, opts, reverse):
    """A decimated whole box of the first written var and a plane of the last (awp_elastic: a velocity and a stress, written
    in place by two stages)."""
    names = out_vars(stencil, eb)
    if stencil == "awp_elastic":
        names = ["vel_x", "stress_xx"]
    lo, hi = whole_box(n)
    mid, plane_hi = list(lo), list(hi)
    mid[0] = plane_hi[0] = n[0] // 2
    # A reverse run computes u = steps - 1 down to 0, and rows still count upwards in u from t0.  Its interval recorder starts
    # at t0 = -1, a step the run never computes: row 0 must stay 0, and only u = 1 and 3 are due.  A row taken from a u that is
    # not a multiple of `every` away from t0 (u = 0 -> row 0, u = 4 -> row 2) would either land on row 0 or reach a row before
    # its right step does, so the run could not end with the right frames by overwriting them.
    recs = [Rec(names[0], lo, hi, stride=[2] + [3] * (len(n) - 1), t0=1, nrows=steps),
            Rec(names[-1], mid, plane_hi, t0=-1, every=2, nrows=3) if reverse else Rec(names[-1], mid, plane_hi, t0=3, nrows=steps)]
    single_case(stencil, n, steps, recs, radius=radius, eb=eb, opts=opts, reverse=reverse)


def test_points_and_slices_together():
    """A source inside a recorded box: the frame sees it, as the loop's read after the add does."""
    n, steps = N8, 5
    src_pts = [[20, 18, 31], [20, 18, 31], [3, 4, 5]]
    src = ("p", src_pts, 1, amp_table(steps, len(src_pts), np.float32))
    recs = [Rec("p", [0, 0, 31], [39, 35, 31], nrows=steps), Rec("p", [19, 17, 30], [21, 19, 32], nrows=steps)]
    single_case("iso3dfd", n, steps, recs, radius=8, src=src)


def test_in_run_tuner():
    """The tuner times each step with its recording launch inside."""
    single_case("iso3dfd", N8, 6, [Rec("p", [0, 0, 17], [39, 35, 17], nrows=6)], radius=8, opts=(("auto_tune", 1),))


def test_past_2_31_elements_per_slot():
    """64-bit offsets: a plane past element 2^31 of a slot, near its far end (iso3dfd fp32 radius 8)."""
    from tests.large_domain import crossing_index
    n, steps = (1100, 1024, 1984), 2
    s = make("iso3dfd", n)
    p = s.get_var("p")
    xc = int(crossing_index(p.info))
    assert p.info.slot_elems > 1 << 31 and xc < n[0] - 2
    recs = [Rec("p", [n[0] - 3, 0, 0], [n[0] - 3, n[1] - 1, n[2] - 1], stride=[1, 1, 3], nrows=steps),
            Rec("p", [xc - 2, 1000, 0], [n[0] - 1, 1000, n[2] - 1], stride=[5, 1, 7], nrows=steps)]
    fill(s, "iso3dfd", [0, 1])
    for r in recs:
        r.add(s)
    s.run_solution(0, steps - 1)
    got = [s.get_slice_frames(i)[0] for i in range(len(recs))]
    assert s.get_option("slice_launches") == str(steps)
    s.close()
    o = make("iso3dfd", n)
    fill(o, "iso3dfd", [0, 1])
    ref = slice_loop(o, 0, steps - 1, 1, recs)
    o.close()
    for a, b in zip(got, ref):
        assert same(a, b)


def test_fuse_vars_after_add_slice():
    """fuse_vars on a prepared solution replaces a var's storage (and frees the old one when nothing else holds it): a recorder
    set before the fuse must read the new storage."""
    rec = Rec("p", [0, 0, 31], [39, 35, 31], stride=[1, 2, 1], nrows=4)
    a = make("iso3dfd", N8, 8)
    rec.add(a)
    b = make("iso3dfd", N8, 8)
    a.get_var("p").fuse_vars(b.get_var("p"))
    assert a.get_var("p").device_ptr(0) == b.get_var("p").device_ptr(0)
    fill(a, "iso3dfd", [0, 1])                        # p's inputs land in b's allocation, which a now uses
    a.run_solution(0, 3)
    frames, owned = a.get_slice_frames(0)
    launches = a.get_option("slice_launches")
    a.close()
    b.close()
    o = make("iso3dfd", N8, 8)
    fill(o, "iso3dfd", [0, 1])
    ref = slice_loop(o, 0, 3, 1, [rec])[0]
    o.close()
    assert owned.all() and launches == "4"
    assert same(frames, ref), np.argwhere(frames != ref)[:5]


# rank grids in one process, each rank's frames merged by its owned mask, against the loop on one rank over the global domain
def grid_case(stencil, n, grid, recs, steps, radius=0, eb=4, opts=()):
    world = int(np.prod(grid))
    solns = [make(stencil, n, radius, eb, opts, grid, r) for r in range(world)]
    multi.connect_local(solns)
    for s in solns:
        fill(s, stencil, [0, 1, 2, 3])
        for r in recs:
            r.add(s)
    for s in solns:             # enqueue every rank first: ranks wait for each other on the device
        s.run_solution(0, steps - 1)
    for s in solns:
        s.sync()
    dt = np.float32 if solns[0].get_element_bytes() == 4 else np.float64
    frames = [np.zeros((r.nrows,) + r.shape(), dt) for r in recs]
    cover = [np.zeros(r.shape(), int) for r in recs]
    for s in solns:
        for i, r in enumerate(recs):
            f, owned = s.get_slice_frames(i)
            frames[i][:, owned] = f[:, owned]
            assert not f[:, ~owned].any()
            cover[i] += owned
        want = due_steps(0, steps - 1, 1, [r for i, r in enumerate(recs) if s.get_slice_frames(i)[1].any()])
        assert int(s.get_option("slice_launches")) == want
        s.close()
    o = make(stencil, n, radius, eb, opts)
    fill(o, stencil, [0, 1, 2, 3])
    ref = slice_loop(o, 0, steps - 1, 1, recs)
    o.close()
    for c, f, rf in zip(cover, frames, ref):
        assert (c == 1).all()
        assert same(f, rf), np.argwhere(f != rf)[:5]


def crossing_recs(n, grid, var="p"):
    """A plane across every interface, a decimated box whose phase differs between ranks, and a box around an interface."""
    ifs = [(m + g - 1) // g for m, g in zip(n, grid)]
    hi = [m - 1 for m in n]
    return [Rec(var, [0, 0, n[2] // 2], [hi[0], hi[1], n[2] // 2], nrows=4),
            Rec(var, [1, 2, 3], hi, stride=[3, 2, 5], t0=2, every=2, nrows=2),
            Rec(var, [max(0, i - 3) for i in ifs], [min(m - 1, i + 2) for i, m in zip(ifs, n)], nrows=4)]


GRIDS = [("2x1x1-fused", (2, 1, 1), (75, 40, 64), ()),
         ("2x1x1-split", (2, 1, 1), (75, 40, 64), (("fused_halo", 0),)),
         ("2x1x1-whole", (2, 1, 1), (75, 40, 64), (("overlap_comms", 0),)),
         ("1x2x1", (1, 2, 1), (40, 75, 64), ()),
         ("2x2x2", (2, 2, 2), (61, 59, 72), ())]


@pytest.mark.parametrize("radius", [8, 2])
@pytest.mark.parametrize("name,grid,n,opts", GRIDS, ids=[g[0] for g in GRIDS])
def test_rank_grid_matches_single_rank_loop(name, grid, n, opts, radius):
    """Every form a last stage takes: the fused x launch (default), the split form (fused_halo=0) and the whole box
    (overlap_comms=0); uneven splits; boxes across interfaces."""
    grid_case("iso3dfd", n, grid, crossing_recs(n, grid), 4, radius=radius, opts=opts)


def test_awp_elastic_split_form_in_place():
    """awp_elastic on 2x1x1 in the split form: its vars are updated in place (alloc_t = 1), so a frame must be recorded after
    the interior launch of the last stage and before the next step's first stage."""
    n, grid = (41, 19, 40), (2, 1, 1)
    recs = crossing_recs(n, grid, "stress_xx") + crossing_recs(n, grid, "vel_x")[:1]
    grid_case("awp_elastic", n, grid, recs, 4, eb=0, opts=(("fused_halo", 0),))
