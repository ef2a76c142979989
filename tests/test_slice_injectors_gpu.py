"""Slice injectors on the device, bit for bit against the reference API loop on the same hash-filled inputs:

    for t in steps:
        run_solution(t, t)
        for each injector with row r due at u, in id order:
            box = get_elements_in_slice(var, u, first, last)
            box[::stride] = frame[r]                 (set)   or   box[::stride] = box[::stride] + frame[r] in T   (add)
            set_elements_in_slice(box)
        then the sources, the receivers and the recorders

(u = t + 1, or t - 1 for a reverse solution; row r = (u - t0) / every when u - t0 is a multiple of `every` and r < nrows).  Every
written var at every valid step, every trace and frame, and on one rank the exact number of injecting launches are compared."""
import glob
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from tests.test_points_gpu import amp_table, calls, fill, make, outputs, same
from tests.test_points_weighted_gpu import receiver_sums
from tests.test_slices_gpu import Rec, out_vars
from yask_b200 import capi, multi

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class Inj:
    """An injector: var, inclusive global box, stride, window, mode, and frames (float64, rounded to the element type by the
    engine and by the loop alike)."""

    def __init__(self, var, first, last, stride=None, t0=1, every=1, nrows=4, mode="add", seed=0):
        self.var, self.first, self.last = var, list(first), list(last)
        self.stride = list(stride) if stride else [1] * len(first)
        self.t0, self.every, self.nrows, self.mode = t0, every, nrows, mode
        self.frames = np.random.default_rng(100 + seed).uniform(-0.75, 0.75, (nrows,) + self.shape())

    def shape(self):
        return tuple((b - a) // k + 1 for a, b, k in zip(self.first, self.last, self.stride))

    def row(self, u):
        k = u - self.t0
        return k // self.every if k >= 0 and k % self.every == 0 and k // self.every < self.nrows else None

    def bbox(self):
        return [(a, a + (n - 1) * k) for a, n, k in zip(self.first, self.shape(), self.stride)]

    def add(self, s):
        return s.add_slice_injector(self.var, self.first, self.last, self.t0, self.frames, stride=self.stride, every=self.every,
                                    mode=self.mode)

    def apply(self, s, u):
        r = self.row(u)
        if r is None:
            return
        var = s.get_var(self.var)
        dt = np.float32 if s.get_element_bytes() == 4 else np.float64
        box = var.get_elements_in_slice([u] + self.first, [u] + self.last)
        sl = tuple(slice(None, None, k) for k in self.stride)
        fr = self.frames[r].astype(dt)
        box[sl] = fr if self.mode == "set" else box[sl] + fr
        var.set_elements_in_slice(np.ascontiguousarray(box), [u] + self.first, [u] + self.last)


def groups(injs):
    """The launch groups by the documented rule: a new group where a box meets an earlier member's on the same var."""
    out = [[]]
    for j, b in enumerate(injs):
        if any(a.var == b.var and all(x0 <= y1 and y0 <= x1 for (x0, x1), (y0, y1) in zip(a.bbox(), b.bbox())) for a in
               (injs[m] for m in out[-1])):
            out.append([])
        out[-1].append(j)
    return out if injs else []


def expected_launches(first, last, off, injs):
    step = 1 if last >= first else -1
    return sum(1 for t in range(first, last + step, step) for g in groups(injs) if any(injs[j].row(t + off) is not None for j in g))


def inject_loop(s, first, last, off, injs, src=None, wsrc=None, rcv=None, wrcv=None, recs=()):
    """The reference API loop: injectors, then (weighted or on-grid) sources, (on-grid or weighted) receivers and recorders."""
    dt = np.float32 if s.get_element_bytes() == 4 else np.float64
    step = 1 if last >= first else -1
    trace = np.zeros((rcv[3], len(rcv[1])), dt) if rcv else np.zeros((wrcv[4], len(wrcv[1])), dt) if wrcv else None
    frames = [np.zeros((r.nrows,) + r.shape(), dt) for r in recs]
    for t in range(first, last + step, step):
        s.run_solution(t, t)
        u = t + off
        for j in injs:
            j.apply(s, u)
        if wsrc and 0 <= u - wsrc[3] < len(wsrc[4]):
            var, idx, w = s.get_var(wsrc[0]), wsrc[1], wsrc[2]
            for i in range(len(idx)):
                for q in range(idx.shape[1]):
                    if w[i, q] == 0:
                        continue
                    at = [u] + idx[i, q].tolist()
                    cur = var.get_elements_in_slice(at, at).reshape(-1)[0]
                    var.set_elements_in_slice(np.array([dt(cur) + dt(float(w[i, q]) * float(wsrc[4][u - wsrc[3]][i]))], dt), at, at)
        if src and 0 <= u - src[2] < len(src[3]):
            var = s.get_var(src[0])
            for i, p in enumerate(src[1]):
                at = [u] + list(p)
                cur = var.get_elements_in_slice(at, at).reshape(-1)[0]
                var.set_elements_in_slice(np.array([dt(cur) + dt(src[3][u - src[2]][i])], dt), at, at)
        if rcv and 0 <= u - rcv[2] < rcv[3]:
            var = s.get_var(rcv[0])
            for j, p in enumerate(rcv[1]):
                at = [u] + list(p)
                trace[u - rcv[2], j] = var.get_elements_in_slice(at, at).reshape(-1)[0]
        if wrcv and 0 <= u - wrcv[3] < wrcv[4]:
            var = s.get_var(wrcv[0])
            trace[u - wrcv[3]] = receiver_sums(var.get_elements_in_slice(*var.domain_box(u)), wrcv[1], wrcv[2], dt)
        for r, f in zip(recs, frames):
            if r.row(u) is not None:
                f[r.row(u)] = r.read(s, u)
    return trace, frames


def single_case(stencil, n, steps, injs, radius=0, eb=4, opts=(), reverse=False, splits=None, src=None, wsrc=None, rcv=None,
                wrcv=None, recs=()):
    first, last, off = (steps, 1, -1) if reverse else (0, steps - 1, 1)
    fill_steps = list(range(steps, steps + 4)) if reverse else [0, 1, 2, 3]
    s = make(stencil, n, radius, eb, opts)
    fill(s, stencil, fill_steps)
    if src:
        s.set_sources(*src)
    if wsrc:
        s.set_sources_weighted(*wsrc)
    if rcv:
        s.set_receivers(*rcv)
    if wrcv:
        s.set_receivers_weighted(*wrcv)
    assert [j.add(s) for j in injs] == list(range(len(injs)))
    for r in recs:
        r.add(s)
    want_groups = ";".join(",".join(map(str, g)) for g in groups(injs))
    assert s.get_option("slice_injector_groups") == want_groups
    for a, b in calls(first, last, splits):
        s.run_solution(a, b)
    fields = outputs(s)
    launches = int(s.get_option("slice_injector_launches"))
    tt = s.get_option("tt_launches") if ("block_steps", 2) in opts else "0"
    trace = s.get_traces()[0] if (rcv or wrcv) else None
    frames = [s.get_slice_frames(i)[0] for i in range(len(recs))]
    s.close()
    o = make(stencil, n, radius, eb, opts)
    fill(o, stencil, fill_steps)
    ref_trace, ref_frames = inject_loop(o, first, last, off, injs, src, wsrc, rcv, wrcv, recs)
    ref_fields = outputs(o)
    o.close()
    assert fields.keys() == ref_fields.keys()
    for k in ref_fields:
        assert same(fields[k], ref_fields[k]), (k, np.argwhere(fields[k] != ref_fields[k])[:5])
    if trace is not None:
        assert same(trace, ref_trace), np.argwhere(trace != ref_trace)[:5]
    for f, rf in zip(frames, ref_frames):
        assert same(f, rf), np.argwhere(f != rf)[:5]
    assert tt == "0"                                       # no pair runs while an injector is set
    assert launches == expected_launches(first, last, off, injs), launches


N8 = (40, 36, 64)
ISO_R8 = {
    "x-plane-add": [Inj("p", [17, 0, 0], [17, 35, 63])],
    "y-plane-add": [Inj("p", [0, 20, 0], [39, 20, 63])],
    "z-plane-add": [Inj("p", [0, 0, 31], [39, 35, 31])],
    "decimated-odd-first-set": [Inj("p", [1, 1, 1], [39, 35, 63], stride=[2, 3, 4], mode="set")],
    "every-3-mid-run-short": [Inj("p", [0, 3, 0], [39, 3, 63], t0=3, every=3, nrows=2)],
    "overlap-add-then-set": [Inj("p", [5, 5, 5], [30, 30, 40], seed=1), Inj("p", [0, 0, 20], [39, 35, 20], mode="set", seed=2)],
    "overlap-set-then-add": [Inj("p", [0, 0, 20], [39, 35, 20], mode="set", seed=2), Inj("p", [5, 5, 5], [30, 30, 40], seed=1)],
    "disjoint-share-a-launch": [Inj("p", [0, 0, 0], [39, 35, 0]), Inj("p", [0, 0, 63], [39, 35, 63], mode="set", seed=3),
                                Inj("p", [0, 0, 63], [39, 35, 63], seed=4)],
}


@pytest.mark.parametrize("case", list(ISO_R8))
def test_iso3dfd_r8(case):
    """The resident radius-8 sweep: planes in each dim, a decimated box with an odd first, an interval that ends mid-run, and
    overlapping injectors in both orders (launch groups keep id order)."""
    steps = 9 if case == "every-3-mid-run-short" else 6
    single_case("iso3dfd", N8, steps, ISO_R8[case], radius=8)


def faces(n, R, var, mode="set"):
    """The outer R planes of each face of the domain (boundary replay, Dirichlet data)."""
    hi = [m - 1 for m in n]
    out = []
    for d in range(len(n)):
        for lo_side in (True, False):
            f, l = [0] * len(n), list(hi)
            if lo_side:
                l[d] = R - 1
            else:
                f[d] = n[d] - R
            out.append(Inj(var, f, l, mode=mode, nrows=6, seed=10 + len(out)))
    return out


@pytest.mark.parametrize("stencil,n,steps,radius,eb,opts,reverse", [
    ("iso3dfd", (32, 28, 48), 5, 4, 8, (), False),
    ("iso3dfd_sponge", (30, 26, 48), 5, 4, 4, (), False),
    ("awp_elastic", (21, 19, 40), 4, 0, 0, (), False),
    ("wave2d", (37, 50), 5, 0, 0, (), False),
    ("test_1d", (70,), 5, 0, 0, (), False),
    ("test_reverse_2d", (37, 50), 5, 0, 0, (), True),
], ids=["iso-fp64-r4", "sponge-r4", "awp_elastic", "wave2d", "test_1d", "reverse-2d"])
def test_other_stencils(stencil, n, steps, radius, eb, opts, reverse):
    """A decimated box with an odd first in `add` and a plane in `set` (awp_elastic: a stress and a velocity, vars updated in
    place, alloc_t = 1)."""
    names = out_vars(stencil, eb)
    if stencil == "awp_elastic":
        names = ["stress_xx", "vel_x"]
    hi = [m - 1 for m in n]
    mid, plane_hi = [0] * len(n), list(hi)
    mid[0] = plane_hi[0] = n[0] // 2
    # a reverse run computes u = steps - 1 down to 0; the window starts at t0 = -1, a step it never computes
    injs = [Inj(names[0], [1] * len(n), hi, stride=[2] + [3] * (len(n) - 1), t0=1, nrows=steps),
            Inj(names[-1], mid, plane_hi, t0=-1 if reverse else 2, every=2, nrows=3, mode="set", seed=5)]
    single_case(stencil, n, steps, injs, radius=radius, eb=eb, opts=opts, reverse=reverse)


@pytest.mark.parametrize("radius,eb", [(0, 4), (2, 8)], ids=["generated-fp32", "hand-written-fp64-r2"])
def test_3axis_dirichlet_faces(radius, eb):
    """3axis with `set` on all six faces as time-varying Dirichlet data: the generated kernel (fp32 at its default radius) and
    the hand-written sweep (fp64, radius 2)."""
    n = (30, 20, 64)
    single_case("3axis", n, 5, faces(n, max(radius, 1), "A"), radius=radius, eb=eb)


def test_split_calls():
    injs = [Inj("p", [1, 0, 2], [39, 35, 62], stride=[2, 5, 3], t0=2, every=2, nrows=3), Inj("p", [0, 0, 31], [39, 35, 31], nrows=7)]
    single_case("iso3dfd", N8, 7, injs, radius=8, splits=[3, 1, 3])


def test_in_run_tuner():
    """The tuner times each step with its injecting launch inside."""
    single_case("iso3dfd", N8, 6, [Inj("p", [0, 0, 17], [39, 35, 17], nrows=6)], radius=8, opts=(("auto_tune", 1),))


def test_block_steps_fall_back_and_resume():
    """iso3dfd radius 2, block_steps=2: while injecting every step is one launch; after clear_slice_injectors() pairs come back."""
    n, opts = (40, 24, 160), (("block_steps", 2), ("tt_variant", 0))
    inj = Inj("p", [0, 5, 0], [39, 5, 159], nrows=4)
    single_case("iso3dfd", n, 4, [inj], radius=2, opts=opts)
    s = make("iso3dfd", n, 2, 4, opts)
    fill(s, "iso3dfd", [0, 1])
    inj.add(s)
    s.run_solution(0, 3)
    assert s.get_option("tt_launches") == "0" and s.get_option("slice_injector_launches") == "4"
    s.clear_slice_injectors()
    s.run_solution(4, 7)
    assert int(s.get_option("tt_launches")) == 2 and s.get_option("slice_injector_launches") == "4"
    got = outputs(s)
    s.close()
    o = make("iso3dfd", n, 2, 4, opts)
    fill(o, "iso3dfd", [0, 1])
    inject_loop(o, 0, 3, 1, [inj])
    inject_loop(o, 4, 7, 1, [])
    ref = outputs(o)
    o.close()
    for k in ref:
        assert same(got[k], ref[k]), k


@pytest.mark.parametrize("weighted", [False, True], ids=["on-grid", "weighted"])
def test_order_within_a_step(weighted):
    """Injectors, sources, receivers and a recorder on the same points: the sources add onto the injected values and the
    receivers and the recorder see both."""
    n, steps = N8, 5
    pts = [[20, 18, 31], [20, 18, 31], [3, 4, 31], [20, 19, 31]]
    amp = amp_table(steps, len(pts), np.float32)
    injs = [Inj("p", [0, 0, 31], [39, 35, 31], mode="set", nrows=steps), Inj("p", [19, 17, 30], [21, 19, 32], nrows=steps, seed=7)]
    recs = [Rec("p", [0, 0, 31], [39, 35, 31], nrows=steps), Rec("p", [19, 17, 30], [21, 19, 32], nrows=steps)]
    if not weighted:
        single_case("iso3dfd", n, steps, injs, radius=8, src=("p", pts, 1, amp), rcv=("p", pts, 1, steps), recs=recs)
        return
    pos = np.array([[20.25, 18.5, 31.0], [3.0, 4.0, 31.0], [19.5, 18.75, 30.5]])
    idx, w = capi.trilinear(pos)
    amp = amp_table(steps, len(pos), np.float32)
    single_case("iso3dfd", n, steps, injs, radius=8, wsrc=("p", idx, w, 1, amp), wrcv=("p", idx, w, 1, steps), recs=recs)


def test_fuse_vars_after_add_slice_injector():
    """fuse_vars on a prepared solution replaces a var's storage: an injector set before the fuse must write the new storage."""
    inj = Inj("p", [0, 0, 31], [39, 35, 31], stride=[1, 2, 1], nrows=4)
    a = make("iso3dfd", N8, 8)
    inj.add(a)
    b = make("iso3dfd", N8, 8)
    a.get_var("p").fuse_vars(b.get_var("p"))
    fill(a, "iso3dfd", [0, 1])
    a.run_solution(0, 3)
    got = outputs(a)
    launches = a.get_option("slice_injector_launches")
    a.close()
    b.close()
    o = make("iso3dfd", N8, 8)
    fill(o, "iso3dfd", [0, 1])
    inject_loop(o, 0, 3, 1, [inj])
    ref = outputs(o)
    o.close()
    assert launches == "4"
    for k in ref:
        assert same(got[k], ref[k]), k


def test_past_2_31_elements_per_slot():
    """64-bit offsets: an x-plane near the far end of a slot past element 2^31, and a decimated box across the crossing."""
    from tests.large_domain import crossing_index
    n, steps = (1100, 1024, 1984), 2
    s = make("iso3dfd", n)
    p = s.get_var("p")
    xc = int(crossing_index(p.info))
    assert p.info.slot_elems > 1 << 31 and xc < n[0] - 2
    injs = [Inj("p", [n[0] - 3, 0, 0], [n[0] - 3, n[1] - 1, n[2] - 1], nrows=steps),
            Inj("p", [xc - 2, 1000, 0], [n[0] - 1, 1000, n[2] - 1], stride=[5, 1, 7], nrows=steps, mode="set", seed=1)]
    fill(s, "iso3dfd", [0, 1])
    for j in injs:
        j.add(s)
    s.run_solution(0, steps - 1)
    boxes = [(j.first, j.last) for j in injs]
    got = [p.get_elements_in_slice([steps] + f, [steps] + l) for f, l in boxes]
    assert s.get_option("slice_injector_launches") == str(expected_launches(0, steps - 1, 1, injs))   # two groups: the boxes meet
    s.close()
    o = make("iso3dfd", n)
    fill(o, "iso3dfd", [0, 1])
    inject_loop(o, 0, steps - 1, 1, injs)
    q = o.get_var("p")
    ref = [q.get_elements_in_slice([steps] + f, [steps] + l) for f, l in boxes]
    o.close()
    for a, b in zip(got, ref):
        assert same(a, b)


MOD = glob.glob(os.path.join(ROOT, "yask_b200", "lib", "python", "iso3dfd", "yask_kernel*.so"))
SCRIPT = textwrap.dedent("""
    import struct
    import numpy as np
    import yask_kernel as yk

    steps, n = 5, (40, 36, 64)
    fac, env = yk.yk_factory(), None

    def solution():
        global env
        env = env or fac.new_env()
        s = fac.new_solution(env)
        s.set_overall_domain_size_vec(list(n))
        s.prepare_solution()
        s.get_var("v").set_all_elements_same(0.1)
        p = s.get_var("p")
        p.set_all_elements_same(0.0)
        p.set_element(0.25, [0, 20, 18, 32])
        p.set_element(-0.5, [1, 21, 17, 30])
        return s

    first, last, stride = [20, 0, 1], [20, 35, 63], [1, 2, 3]
    frames = np.random.default_rng(5).uniform(-1, 1, (2, 1, 18, 21))        # doubles: rounded once to float
    a = solution()
    assert yk.yk_add_slice_injector(a, "p", first, last, 2, 2, frames.reshape(-1).tolist(), stride, 2, True) == 0   # set p(2), p(4)
    a.run_solution(0, steps - 1)
    assert yk.yk_get_slice_injector_launches(a) == 2, yk.yk_get_slice_injector_launches(a)
    got = np.zeros((1, 40, 36, 64), np.float32)
    a.get_var("p").get_elements_in_slice(got, [steps, 0, 0, 0], [steps, 39, 35, 63])

    b = solution()
    p = b.get_var("p")
    for t in range(steps):
        b.run_solution(t)
        if t + 1 in (2, 4):
            buf = np.zeros((1, 36, 63), np.float32)
            p.get_elements_in_slice(buf, [t + 1] + first, [t + 1] + last)
            buf[:, ::2, ::3] = frames[(t + 1 - 2) // 2, 0].astype(np.float32)
            p.set_elements_in_slice(buf, [t + 1] + first, [t + 1] + last)
    ref = np.zeros_like(got)
    p.get_elements_in_slice(ref, [steps, 0, 0, 0], [steps, 39, 35, 63])
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))
    try:
        yk.yk_add_slice_injector(a, "p", first, last, 0, 2, [0.0] * 5)
        raise SystemExit("a wrong frame count was accepted")
    except RuntimeError as e:
        assert "frame values" in str(e), e
    yk.yk_clear_slice_injectors(a)
    a.run_solution(steps, steps)
    assert yk.yk_get_slice_injector_launches(a) == 2
    print("injectors api ok")
""")


@pytest.mark.skipif(not MOD, reason="python module not built")
def test_yask_kernel_module_injectors_match_reference_loop():
    """The C++ mirror through the yask_kernel module, against the module's own get/set_elements_in_slice loop."""
    env = dict(os.environ, PYTHONPATH=os.path.dirname(MOD[0]))
    r = subprocess.run([sys.executable, "-c", SCRIPT], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "injectors api ok" in r.stdout


# rank grids in one process, every rank's fields merged by its domain box, against the loop on one rank over the global domain
def grid_case(stencil, n, grid, injs, steps, radius=0, eb=4, opts=()):
    world = int(np.prod(grid))
    solns = [make(stencil, n, radius, eb, opts, grid, r) for r in range(world)]
    multi.connect_local(solns)
    for s in solns:
        fill(s, stencil, [0, 1, 2, 3])
        for j in injs:
            j.add(s)
    for s in solns:             # enqueue every rank first: ranks wait for each other on the device
        s.run_solution(0, steps - 1)
    for s in solns:
        s.sync()
    merged = {}
    for s in solns:
        for v in s.get_vars():
            vi = v.info
            if not vi.is_output:
                continue
            for t in range(vi.first_valid_step, vi.last_valid_step + 1):
                f, l = v.domain_box(t)
                key = (vi.name.decode(), t)
                if key not in merged:
                    merged[key] = np.zeros(n, v.get_elements_in_slice(f, f).dtype)
                merged[key][tuple(slice(a, b + 1) for a, b in zip(f[1:], l[1:]))] = v.get_elements_in_slice(f, l)
        assert int(s.get_option("slice_injector_launches")) <= 2 * steps * len(groups(injs))
        s.close()
    o = make(stencil, n, radius, eb, opts)
    fill(o, stencil, [0, 1, 2, 3])
    inject_loop(o, 0, steps - 1, 1, injs)
    ref = outputs(o)
    o.close()
    assert merged.keys() == ref.keys()
    for k in ref:
        assert same(merged[k], ref[k]), (k, np.argwhere(merged[k] != ref[k])[:5])


def near_far(n, radius, near):
    """A y-z box on each side of the x interface of 2x1x1, within the x halo of it (near) or just outside."""
    x_if = (n[0] + 1) // 2
    d = 0 if near else 1
    return [Inj("p", [x_if - radius - d, 3, 5], [x_if - radius - d, 30, 50], seed=1),
            Inj("p", [x_if + radius - 1 + d, 2, 0], [x_if + radius - 1 + d, 20, 63], mode="set", seed=2)]


@pytest.mark.parametrize("radius", [8, 2])
@pytest.mark.parametrize("near", [False, True], ids=["far-keeps-fused", "near-forces-split"])
def test_rank_grid_near_and_far_from_the_x_interface(near, radius):
    n = (75, 40, 64)
    grid_case("iso3dfd", n, (2, 1, 1), near_far(n, radius, near), 4, radius=radius)


def crossing_injs(n, grid, var="p"):
    """A plane across every interface, a decimated box whose phase differs between ranks, and a box around an interface that
    overlaps the plane (two launch groups)."""
    ifs = [(m + g - 1) // g for m, g in zip(n, grid)]
    hi = [m - 1 for m in n]
    return [Inj(var, [0, 0, n[2] // 2], [hi[0], hi[1], n[2] // 2], seed=1),
            Inj(var, [1, 2, 3], hi, stride=[3, 2, 5], t0=2, every=2, nrows=2, mode="set", seed=2),
            Inj(var, [max(0, i - 3) for i in ifs], [min(m - 1, i + 2) for i, m in zip(ifs, n)], seed=3)]


GRIDS = [("1x2x1", (1, 2, 1), (40, 75, 64), ()),
         ("1x1x2", (1, 1, 2), (40, 36, 130), ()),
         ("2x2x1", (2, 2, 1), (75, 61, 64), ()),
         ("3x1x1-uneven", (3, 1, 1), (77, 36, 64), ()),
         ("2x1x1-whole", (2, 1, 1), (75, 40, 64), (("overlap_comms", 0),)),
         ("2x1x1-split", (2, 1, 1), (75, 40, 64), (("fused_halo", 0),))]


@pytest.mark.parametrize("radius", [8, 2])
@pytest.mark.parametrize("name,grid,n,opts", GRIDS, ids=[g[0] for g in GRIDS])
def test_rank_grid_matches_single_rank_loop(name, grid, n, opts, radius):
    grid_case("iso3dfd", n, grid, crossing_injs(n, grid), 4, radius=radius, opts=opts)


def test_awp_elastic_stresses_on_a_rank_grid():
    n, grid = (41, 19, 40), (2, 1, 1)
    injs = crossing_injs(n, grid, "stress_xx") + crossing_injs(n, grid, "stress_yy")[:1]
    grid_case("awp_elastic", n, grid, injs, 4, eb=0)
