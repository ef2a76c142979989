"""Slice correlators and injectors fed from a recorder on the device, bit for bit against the host loop on the same hash-filled
inputs:

    for t in steps:
        run_solution(t, t)
        injectors, sources, recorders (frame[r] = var(u)[box])
        for each correlator with row r due at u:
            b = var(u)[box]                                         (autocorrelation)
                or frames[nrows - 1 - r if reverse else r]          (of a recorder, as it stands now)
            image = image + var(u)[box] * b                         (numpy: each operation rounded to the element type)

(u = t + 1, or t - 1 for a reverse solution; row r = (u - t0) / every when u - t0 is a multiple of `every` and r < nrows).  Every
image, every written var at every valid step and every frame are compared, and on one rank the exact number of correlating
launches."""
import glob
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from tests.test_points_gpu import amp_table, calls, fill, make, outputs, same
from tests.test_slice_injectors_gpu import Inj
from tests.test_slices_gpu import Rec, out_vars
from yask_b200 import capi, multi

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class Cor:
    """A correlator: var, box, window, and its frames: None (autocorrelation), ("self", recorder index) or ("ext", recorder id of
    the forward solution)."""

    def __init__(self, var, first, last, stride=None, t0=1, every=1, nrows=4, src=None, reverse=False):
        self.var, self.first, self.last = var, list(first), list(last)
        self.stride = list(stride) if stride else [1] * len(first)
        self.t0, self.every, self.nrows, self.src, self.reverse = t0, every, nrows, src, reverse

    def row(self, u):
        k = u - self.t0
        return k // self.every if k >= 0 and k % self.every == 0 and k // self.every < self.nrows else None

    def shape(self):
        return tuple((b - a) // k + 1 for a, b, k in zip(self.first, self.last, self.stride))

    def add(self, s, fwd=None):
        src = None if self.src is None else (s if self.src[0] == "self" else fwd)
        return s.add_slice_correlator(self.var, self.first, self.last, self.t0, self.nrows, src=src,
                                      src_id=None if self.src is None else self.src[1], reverse=self.reverse, stride=self.stride,
                                      every=self.every)


def forward_frames(stencil, n, steps, recs, radius, eb, opts=()):
    """A forward solution recording `recs` over `steps` steps: (solution, frames)."""
    f = make(stencil, n, radius, eb, opts)
    fill(f, stencil, [0, 1, 2, 3])
    for r in recs:
        r.add(f)
    f.run_solution(0, steps - 1)
    return f, [f.get_slice_frames(i)[0] for i in range(len(recs))]


def correlate_loop(s, first, last, off, cors, recs=(), ext=(), injs=(), src=None):
    """The host loop: injectors, on-grid sources, recorders of this solution, then the correlators."""
    dt = np.float32 if s.get_element_bytes() == 4 else np.float64
    step = 1 if last >= first else -1
    frames = [np.zeros((r.nrows,) + r.shape(), dt) for r in recs]
    images = [np.zeros(c.shape(), dt) for c in cors]
    for t in range(first, last + step, step):
        s.run_solution(t, t)
        u = t + off
        for j in injs:
            j.apply(s, u)
        if src and 0 <= u - src[2] < len(src[3]):
            var = s.get_var(src[0])
            for i, p in enumerate(src[1]):
                at = [u] + list(p)
                cur = var.get_elements_in_slice(at, at).reshape(-1)[0]
                var.set_elements_in_slice(np.array([dt(cur) + dt(src[3][u - src[2]][i])], dt), at, at)
        for r, f in zip(recs, frames):
            if r.row(u) is not None:
                f[r.row(u)] = r.read(s, u)
        for c, img in zip(cors, images):
            r = c.row(u)
            if r is None:
                continue
            box = s.get_var(c.var).get_elements_in_slice([u] + c.first, [u] + c.last)[tuple(slice(None, None, k) for k in c.stride)]
            if c.src is None:
                b = box
            else:
                fr = frames[c.src[1]] if c.src[0] == "self" else ext[c.src[1]]
                b = fr[c.nrows - 1 - r if c.reverse else r]
            img[...] = img + box * b
    return images, frames


def expected_launches(first, last, off, cors):
    step = 1 if last >= first else -1
    return sum(1 for t in range(first, last + step, step) if any(c.row(t + off) is not None for c in cors))


def single_case(stencil, n, steps, cors, recs=(), fwd_recs=(), radius=0, eb=4, opts=(), reverse=False, splits=None, injs=(), src=None):
    first, last, off = (steps, 1, -1) if reverse else (0, steps - 1, 1)
    fill_steps = list(range(steps, steps + 4)) if reverse else [0, 1, 2, 3]
    fwd, ext = forward_frames(stencil, n, steps, fwd_recs, radius, eb) if fwd_recs else (None, [])
    s = make(stencil, n, radius, eb, opts)
    fill(s, stencil, fill_steps)
    if src:
        s.set_sources(*src)
    for j in injs:
        j.add(s)
    for r in recs:
        r.add(s)
    assert [c.add(s, fwd) for c in cors] == list(range(len(cors)))
    for a, b in calls(first, last, splits):
        s.run_solution(a, b)
    images = [s.get_correlator_image(i) for i in range(len(cors))]
    fields = outputs(s)
    frames = [s.get_slice_frames(i)[0] for i in range(len(recs))]
    launches = int(s.get_option("slice_correlator_launches"))
    tt = s.get_option("tt_launches") if ("block_steps", 2) in opts else "0"
    s.close()
    if fwd:
        fwd.close()
    o = make(stencil, n, radius, eb, opts)
    fill(o, stencil, fill_steps)
    ref_images, ref_frames = correlate_loop(o, first, last, off, cors, recs, ext, injs, src)
    ref_fields = outputs(o)
    o.close()
    for (img, owned), ref in zip(images, ref_images):
        assert owned.all()
        assert same(img, ref), np.argwhere(img != ref)[:5]
    for k in ref_fields:
        assert same(fields[k], ref_fields[k]), k
    for f, rf in zip(frames, ref_frames):
        assert same(f, rf)
    assert tt == "0"
    assert launches == expected_launches(first, last, off, cors), launches


N8 = (40, 36, 64)
FULL, HI = [0, 0, 0], [39, 35, 63]
ISO = {
    "auto-full": dict(cors=[Cor("p", FULL, HI, nrows=6)]),
    "auto-strided": dict(cors=[Cor("p", [1, 2, 3], HI, stride=[2, 3, 5], t0=2, every=2, nrows=3)]),
    "self-forward-every-3": dict(recs=[Rec("p", [1, 0, 2], HI, stride=[3, 1, 2], t0=1, every=3, nrows=3)],
                                 cors=[Cor("p", [1, 0, 2], HI, stride=[3, 1, 2], t0=1, every=3, nrows=2, src=("self", 0))]),
    "self-reversed": dict(recs=[Rec("p", [0, 0, 31], [39, 35, 31], nrows=6)],
                          cors=[Cor("p", [0, 0, 31], [39, 35, 31], t0=1, nrows=6, src=("self", 0), reverse=True)]),
    "fwd-reversed-every-2-short": dict(fwd_recs=[Rec("p", FULL, HI, stride=[1, 2, 1], t0=2, every=2, nrows=3)],
                                       cors=[Cor("p", FULL, HI, stride=[1, 2, 1], t0=1, every=2, nrows=2, src=("ext", 0), reverse=True),
                                             Cor("p", FULL, HI, stride=[1, 2, 1], t0=2, every=3, nrows=2, src=("ext", 0)),
                                             Cor("p", [5, 0, 0], [5, 35, 63], nrows=6)]),
}


@pytest.mark.parametrize("case", list(ISO))
def test_iso3dfd_r8(case):
    single_case("iso3dfd", N8, 6, radius=8, **ISO[case])


@pytest.mark.parametrize("radius", [4, 3], ids=["hand-written-r4", "generated-r3"])
@pytest.mark.parametrize("case", ["auto-strided", "self-forward-every-3", "fwd-reversed-every-2-short"])
def test_iso3dfd_fp64(case, radius):
    """The radius-8 cases on a smaller domain, boxes clipped to it."""
    n = (32, 28, 48)
    clip = lambda c: type(c)(**{**vars(c), "last": [min(a, m - 1) for a, m in zip(c.last, n)]})
    single_case("iso3dfd", n, 6, radius=radius, eb=8, **{k: [clip(c) for c in v] for k, v in ISO[case].items()})


@pytest.mark.parametrize("stencil,n,steps,eb,reverse", [
    ("awp_elastic", (21, 19, 40), 4, 0, False),
    ("3axis", (30, 20, 64), 5, 0, False),
    ("wave2d", (37, 50), 5, 0, False),
    ("test_1d", (70,), 5, 0, False),
    ("test_reverse_2d", (37, 50), 5, 0, True),
])
def test_other_stencils(stencil, n, steps, eb, reverse):
    """An autocorrelation of a decimated box and a correlation with a recorder of the same solution, reversed (awp_elastic: a
    velocity written by stage 1 and a stress by stage 2, both updated in place)."""
    names = ["vel_x", "stress_xx"] if stencil == "awp_elastic" else out_vars(stencil, eb)
    hi = [m - 1 for m in n]
    box = ([1] * len(n), hi, [2] + [3] * (len(n) - 1))
    t0 = -1 if reverse else 1
    recs = [Rec(names[-1], box[0], box[1], box[2], t0=t0 if reverse else 1, nrows=steps)]
    cors = [Cor(names[0], *box, t0=1, nrows=steps), Cor(names[-1], *box, t0=t0 if reverse else 1, nrows=steps, src=("self", 0), reverse=True)]
    single_case(stencil, n, steps, cors, recs=recs, eb=eb, reverse=reverse)


def test_order_within_a_step():
    """An injector, an on-grid source and a recorder on the correlated var: the correlator sees all of them."""
    steps, pts = 5, [[20, 18, 31], [3, 4, 31]]
    injs = [Inj("p", [0, 0, 31], [39, 35, 31], mode="set", nrows=steps)]
    recs = [Rec("p", [0, 0, 30], [39, 35, 32], nrows=steps)]
    cors = [Cor("p", [0, 0, 30], [39, 35, 32], nrows=steps, src=("self", 0)), Cor("p", [0, 0, 31], [39, 35, 31], nrows=steps)]
    single_case("iso3dfd", N8, steps, cors, recs=recs, radius=8, injs=injs, src=("p", pts, 1, amp_table(steps, len(pts), np.float32)))


def test_split_calls_and_tuner():
    cors = [Cor("p", [1, 0, 2], HI, stride=[2, 5, 3], t0=2, every=2, nrows=3), Cor("p", FULL, HI, nrows=7)]
    single_case("iso3dfd", N8, 7, cors, radius=8, splits=[3, 1, 3])
    single_case("iso3dfd", N8, 6, cors[1:], radius=8, opts=(("auto_tune", 1),))


def test_fuse_vars_after_add():
    c = Cor("p", [0, 0, 31], [39, 35, 31], stride=[1, 2, 1], nrows=4)
    a = make("iso3dfd", N8, 8)
    c.add(a)
    b = make("iso3dfd", N8, 8)
    a.get_var("p").fuse_vars(b.get_var("p"))
    fill(a, "iso3dfd", [0, 1])
    a.run_solution(0, 3)
    got = a.get_correlator_image(0)[0]
    a.close()
    b.close()
    o = make("iso3dfd", N8, 8)
    fill(o, "iso3dfd", [0, 1])
    ref = correlate_loop(o, 0, 3, 1, [c])[0][0]
    o.close()
    assert same(got, ref)


@pytest.mark.parametrize("stencil,radius", [("iso3dfd", 2), ("3axis", 1)])
def test_block_steps_fall_back_and_resume(stencil, radius):
    n, opts = (40, 24, 160), (("block_steps", 2),) + ((("tt_variant", 0),) if stencil == "iso3dfd" else ())
    c = Cor("A" if stencil == "3axis" else "p", [0, 5, 0], [39, 5, 159], nrows=4)
    s = make(stencil, n, radius, 4, opts)
    fill(s, stencil, [0, 1])
    c.add(s)
    s.run_solution(0, 3)
    assert s.get_option("tt_launches") == "0" and s.get_option("slice_correlator_launches") == "4"
    img = s.get_correlator_image(0)[0]
    s.clear_slice_correlators()
    s.run_solution(4, 7)
    assert int(s.get_option("tt_launches")) == 2 and s.get_option("slice_correlator_launches") == "4"
    got = outputs(s)
    s.close()
    o = make(stencil, n, radius, 4, opts)
    fill(o, stencil, [0, 1])
    ref_img = correlate_loop(o, 0, 3, 1, [c])[0][0]
    correlate_loop(o, 4, 7, 1, [])
    ref = outputs(o)
    o.close()
    assert same(img, ref_img)
    for k in ref:
        assert same(got[k], ref[k]), k


def shot(fwd_box, steps=6, reverse=True, eb=4):
    """A forward solution recording the box every step, and an adjoint one correlating against it."""
    f = make("iso3dfd", N8, 8, eb)
    fill(f, "iso3dfd", [0, 1])
    f.get_var("p").fill_hash(1, 41, 7, -1, 1)
    f.add_slice("p", *fwd_box, 1, steps)
    a = make("iso3dfd", N8, 8, eb)
    fill(a, "iso3dfd", [0, 1])
    a.add_slice_correlator("p", *fwd_box, 1, steps, src=f, src_id=0, reverse=reverse)
    return f, a


def test_lifetime_of_shared_frames():
    """clear_slices() on the source, and destroying the source, leave the consumer reading the frames as they were."""
    box = ([0, 0, 0], [39, 35, 63])
    results = []
    for how in ("keep", "clear", "destroy"):
        f, a = shot(box)
        f.run_solution(0, 5)
        frames = f.get_slice_frames(0)[0]
        if how == "clear":
            f.clear_slices()
            f.run_solution(6, 8)
        elif how == "destroy":
            f.close()
        a.run_solution(0, 5)
        results.append(a.get_correlator_image(0)[0])
        a.close()
        f.close()
    o = make("iso3dfd", N8, 8)
    fill(o, "iso3dfd", [0, 1])
    ref = correlate_loop(o, 0, 5, 1, [Cor("p", *box, nrows=6, src=("ext", 0), reverse=True)], ext=[frames])[0][0]
    o.close()
    for r in results:
        assert same(r, ref)


def test_cross_solution_order_without_host_sync():
    """The source runs, the consumer runs, the source is refilled and runs again, all enqueued with no sync in between: the
    consumer reads the first run's rows."""
    box = ([0, 0, 0], [39, 35, 63])
    f, a = shot(box)
    f.run_solution(0, 5)
    a.run_solution(0, 5)
    f.get_var("p").fill_hash(0, 99, 5, -1, 1)
    f.run_solution(0, 5)
    a.sync()
    got = a.get_correlator_image(0)[0]
    a.close()
    f.close()
    g, _ = shot(box)
    g.run_solution(0, 5)
    frames = g.get_slice_frames(0)[0]
    g.close()
    o = make("iso3dfd", N8, 8)
    fill(o, "iso3dfd", [0, 1])
    ref = correlate_loop(o, 0, 5, 1, [Cor("p", *box, nrows=6, src=("ext", 0), reverse=True)], ext=[frames])[0][0]
    o.close()
    assert same(got, ref)


def test_past_2_31_elements_per_slot():
    """64-bit offsets: a plane and a decimated box across element 2^31 of a slot, against a recorder of the same solution."""
    from tests.large_domain import crossing_index
    n, steps = (1100, 1024, 1984), 2
    s = make("iso3dfd", n)
    p = s.get_var("p")
    xc = int(crossing_index(p.info))
    assert p.info.slot_elems > 1 << 31 and xc < n[0] - 2
    box = ([xc - 2, 0, 0], [n[0] - 1, n[1] - 1, n[2] - 1], [5, 7, 1])
    rec = Rec("p", *box, nrows=steps)
    cors = [Cor("p", [n[0] - 3, 0, 0], [n[0] - 3, n[1] - 1, n[2] - 1], nrows=steps), Cor("p", *box, nrows=steps, src=("self", 0), reverse=True)]
    fill(s, "iso3dfd", [0, 1])
    rec.add(s)
    for c in cors:
        c.add(s)
    s.run_solution(0, steps - 1)
    got = [s.get_correlator_image(i)[0] for i in range(2)]
    s.close()
    o = make("iso3dfd", n)
    fill(o, "iso3dfd", [0, 1])
    ref = correlate_loop(o, 0, steps - 1, 1, cors, [rec])[0]
    o.close()
    for a, b in zip(got, ref):
        assert same(a, b)


# rank grids in one process: the owned parts of every rank's image merged, against one rank over the global domain
GRIDS = [("2x1x1-fused", (2, 1, 1), (75, 40, 64), ()), ("1x2x1-split", (1, 2, 1), (40, 75, 64), ()),
         ("3x1x1-whole-uneven", (3, 1, 1), (77, 36, 64), (("overlap_comms", 0),))]


@pytest.mark.parametrize("name,grid,n,opts", GRIDS, ids=[g[0] for g in GRIDS])
def test_rank_grid_matches_single_rank(name, grid, n, opts):
    steps, world = 4, int(np.prod(grid))
    hi = [m - 1 for m in n]
    box = ([1, 2, 3], hi, [3, 2, 5])
    recs = [Rec("p", *box, nrows=steps)]
    cors = [Cor("p", [0, 0, 0], hi, nrows=steps), Cor("p", *box, nrows=steps, src=("ext", 0), reverse=True)]
    fwd = [make("iso3dfd", n, 8, 4, opts, grid, r) for r in range(world)]
    multi.connect_local(fwd)
    adj = [make("iso3dfd", n, 8, 4, opts, grid, r) for r in range(world)]
    multi.connect_local(adj)
    for f, a in zip(fwd, adj):
        fill(f, "iso3dfd", [0, 1])
        fill(a, "iso3dfd", [0, 1])
        recs[0].add(f)
    other = make("iso3dfd", n, 8, 4, opts, grid, 1)          # another rank of the grid
    recs[0].add(other)
    with pytest.raises(capi.YaskError, match="rank index"):
        cors[1].add(adj[0], other)
    other.close()
    for f in fwd:
        f.run_solution(0, steps - 1)
    for a, f in zip(adj, fwd):
        cors[0].add(a)
        cors[1].add(a, f)
    for a in adj:
        a.run_solution(0, steps - 1)
    for a in adj:
        a.sync()
    merged = [np.zeros(c.shape(), np.float32) for c in cors]
    frames = np.zeros((steps,) + recs[0].shape(), np.float32)
    for f, a in zip(fwd, adj):
        fr, fo = f.get_slice_frames(0)
        frames[:, fo] = fr[:, fo]
        for i in range(len(cors)):
            img, owned = a.get_correlator_image(i)
            merged[i][owned] = img[owned]
        f.close()
        a.close()
    o = make("iso3dfd", n, 8)
    fill(o, "iso3dfd", [0, 1])
    ref = correlate_loop(o, 0, steps - 1, 1, cors, ext=[frames])[0]
    o.close()
    for m, r in zip(merged, ref):
        assert same(m, r), np.argwhere(m != r)[:5]


@pytest.mark.parametrize("mode", ["add", "set"])
@pytest.mark.parametrize("reverse", [False, True], ids=["forward", "reversed"])
def test_injector_from_recorder_matches_host_frames(mode, reverse):
    """An injector fed from a recorder's device frames gives the bits of add_slice_injector fed with get_slice_frames."""
    steps, box = 5, ([1, 0, 2], [39, 35, 62], [2, 5, 3])
    f = make("iso3dfd", N8, 8)
    fill(f, "iso3dfd", [0, 1])
    f.get_var("p").fill_hash(1, 41, 7, -1, 1)
    f.add_slice("p", *box[:2], 1, steps, stride=box[2])
    f.run_solution(0, steps - 1)
    frames = f.get_slice_frames(0)[0]
    results = []
    for dev in (True, False):
        s = make("iso3dfd", N8, 8)
        fill(s, "iso3dfd", [0, 1])
        if dev:
            s.add_slice_injector_from("p", *box[:2], 2, steps - 1, f, 0, reverse=reverse, stride=box[2], mode=mode)
        else:
            fr = frames[:steps - 1][::-1] if reverse else frames[:steps - 1]
            s.add_slice_injector("p", *box[:2], 2, np.ascontiguousarray(fr), stride=box[2], mode=mode)
        s.run_solution(0, steps - 1)
        results.append((outputs(s), s.get_option("slice_injector_launches")))
        s.close()
    f.close()
    assert results[0][1] == results[1][1] == str(steps - 1)
    for k in results[1][0]:
        assert same(results[0][0][k], results[1][0][k]), k


def test_boundary_replay_r8():
    """A forward run records the six R-deep faces; a second solution writes them back from the device, reversed, with `set`."""
    n, R, steps = N8, 8, 5
    hi = [m - 1 for m in n]
    faces = []
    for d in range(3):
        for lo in (True, False):
            f, l = [0, 0, 0], list(hi)
            if lo:
                l[d] = R - 1
            else:
                f[d] = n[d] - R
            faces.append((f, l))
    fwd = make("iso3dfd", n, 8)
    fill(fwd, "iso3dfd", [0, 1])
    for f, l in faces:
        fwd.add_slice("p", f, l, 1, steps)
    fwd.run_solution(0, steps - 1)
    host = [fwd.get_slice_frames(i)[0] for i in range(len(faces))]
    got = []
    for dev in (True, False):
        s = make("iso3dfd", n, 8)
        fill(s, "iso3dfd", [2, 3])
        for i, (f, l) in enumerate(faces):
            if dev:
                s.add_slice_injector_from("p", f, l, 1, steps, fwd, i, reverse=True, mode="set")
            else:
                s.add_slice_injector("p", f, l, 1, np.ascontiguousarray(host[i][::-1]), mode="set")
        s.run_solution(0, steps - 1)
        got.append(outputs(s))
        s.close()
    fwd.close()
    for k in got[1]:
        assert same(got[0][k], got[1][k]), k


MOD = glob.glob(os.path.join(ROOT, "yask_b200", "lib", "python", "iso3dfd", "yask_kernel*.so"))
SCRIPT = textwrap.dedent("""
    import numpy as np
    import yask_kernel as yk

    steps, n = 4, (40, 36, 64)
    fac, env = yk.yk_factory(), None

    def solution(a):
        global env
        env = env or fac.new_env()
        s = fac.new_solution(env)
        s.set_overall_domain_size_vec(list(n))
        s.prepare_solution()
        s.get_var("v").set_all_elements_same(0.1)
        p = s.get_var("p")
        p.set_all_elements_same(0.375)          # products well above the subnormal range (fp32 runs with FTZ)
        p.set_element(a, [0, 20, 18, 32])
        p.set_element(-0.5, [1, 21, 17, 30])
        return s

    first, last, stride = [0, 0, 1], [39, 35, 63], [1, 2, 3]
    f = solution(0.25)
    assert yk.yk_add_slice(f, "p", first, last, 1, steps, stride) == 0
    f.run_solution(0, steps - 1)
    fr, shape, _ = yk.yk_get_slice_frames(f, 0)
    fr = np.array(fr, np.float32).reshape(shape)
    a = solution(0.75)
    assert yk.yk_add_slice_correlator(a, "p", first, last, 1, steps, f, 0, True, stride) == 0
    assert yk.yk_add_slice_correlator(a, "p", first, last, 1, steps, None, 0, False, stride) == 1
    assert yk.yk_add_slice_injector_from(a, "p", first, last, 3, 1, f, 0, False, stride, 1, False) == 0
    a.run_solution(0, steps - 1)
    assert yk.yk_get_slice_correlator_launches(a) == steps
    img, ishape, owned = yk.yk_get_correlator_image(a, 0)
    auto = np.array(yk.yk_get_correlator_image(a, 1)[0], np.float32).reshape(ishape)
    img = np.array(img, np.float32).reshape(ishape)
    assert list(ishape) == list(shape[1:]) and all(owned)

    b = solution(0.75)
    p = b.get_var("p")
    ref, rauto, fwd = np.zeros_like(img), np.zeros_like(img), np.zeros_like(img)
    for t in range(steps):
        b.run_solution(t)
        u = t + 1
        buf = np.zeros((1, 40, 36, 63), np.float32)
        p.get_elements_in_slice(buf, [u] + first, [u] + last)
        if u == 3:
            buf[0, :, ::2, ::3] = buf[0, :, ::2, ::3] + fr[0]
            p.set_elements_in_slice(buf, [u] + first, [u] + last)
        box = buf[0, :, ::2, ::3]
        ref = ref + box * fr[steps - u]
        rauto = rauto + box * box
        fwd = fwd + box * fr[u - 1]
    assert np.array_equal(img.view(np.uint32), ref.view(np.uint32)), (np.abs(img - ref).max(), np.abs(img - fwd).max(),
                                                                      np.abs(auto - rauto).max(), np.abs(ref).max())
    assert np.array_equal(auto.view(np.uint32), rauto.view(np.uint32))
    yk.yk_clear_slice_correlators(a)
    a.run_solution(steps, steps)
    assert yk.yk_get_slice_correlator_launches(a) == steps
    print("correlators api ok")
""")


@pytest.mark.skipif(not MOD, reason="python module not built")
def test_yask_kernel_module_correlators_match_reference_loop():
    env = dict(os.environ, PYTHONPATH=os.path.dirname(MOD[0]))
    r = subprocess.run([sys.executable, "-c", SCRIPT], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "correlators api ok" in r.stdout
