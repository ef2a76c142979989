"""Frame and image types on the device, bit for bit against the host loop on the same hash-filled inputs.  The loop reads each
box with get_elements_in_slice after a one-step run_solution() and narrows it in numpy: astype(float16 / float32) and the bf16
round-to-nearest-even below; double images accumulate in numpy float64.  Every frame, image and written var is compared, and
the launch counters, which the types must not change."""
import glob
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from tests.test_points_gpu import fill, make, outputs, same
from tests.test_slice_injectors_gpu import Inj
from tests.test_slices_gpu import Rec, due_steps, out_vars, slice_loop
from yask_b200 import multi

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def bf16(a):
    """float32 -> the nearest bfloat16, ties to even, as float32 (NaN stays NaN)."""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    r = (((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16).astype(np.uint32).view(np.float32)
    return np.where(np.isnan(a), np.float32(np.nan), r)


def narrow(a, dtype):
    """A frame of type dtype as the host loop computes it from the element-type box a (bf16 widened to float32)."""
    with np.errstate(over="ignore"):
        if dtype == "bfloat16":
            return bf16(a.astype(np.float32))
        return a if dtype is None else a.astype(dtype)


def same_bits(a, b):
    """Same dtype, shape and bits; NaN where the other is NaN (its payload is not specified)."""
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    it = {2: np.uint16, 4: np.uint32, 8: np.uint64}[a.dtype.itemsize]
    nan = np.isnan(a)
    return np.array_equal(nan, np.isnan(b)) and np.array_equal(a.view(it)[~nan], b.view(it)[~nan])


class TRec(Rec):
    def __init__(self, var, first, last, dtype=None, **kw):
        super().__init__(var, first, last, **kw)
        self.dtype = dtype

    def add(self, s):
        return s.add_slice(self.var, self.first, self.last, self.t0, self.nrows, stride=self.stride, every=self.every, dtype=self.dtype)


class TInj(Inj):
    """A host-fed injector whose frames are held in dtype: the loop applies the frames rounded to T, then to dtype."""

    def __init__(self, var, first, last, dtype=None, frames=None, **kw):
        super().__init__(var, first, last, **kw)
        self.dtype = dtype
        if frames is not None:
            self.frames = frames

    def add(self, s):
        return s.add_slice_injector(self.var, self.first, self.last, self.t0, self.frames, stride=self.stride, every=self.every,
                                    mode=self.mode, dtype=self.dtype)

    def apply(self, s, u):
        r = self.row(u)
        if r is None:
            return
        dt = np.float32 if s.get_element_bytes() == 4 else np.float64
        var = s.get_var(self.var)
        box = var.get_elements_in_slice([u] + self.first, [u] + self.last)
        sl = tuple(slice(None, None, k) for k in self.stride)
        fr = narrow(self.frames[r].astype(dt), self.dtype).astype(dt)
        box[sl] = fr if self.mode == "set" else box[sl] + fr
        var.set_elements_in_slice(np.ascontiguousarray(box), [u] + self.first, [u] + self.last)


def run_case(stencil, n, steps, recs, radius=0, eb=4, reverse=False, injs=()):
    """Typed recorders (and injectors) on the device against the loop; fields must be unchanged by recording."""
    first, last, off = (steps, 1, -1) if reverse else (0, steps - 1, 1)
    fill_steps = list(range(steps, steps + 4)) if reverse else [0, 1, 2, 3]
    s = make(stencil, n, radius, eb)
    fill(s, stencil, fill_steps)
    for j in injs:
        j.add(s)
    assert [r.add(s) for r in recs] == list(range(len(recs)))
    s.run_solution(first, last)
    got = [s.get_slice_frames(i) for i in range(len(recs))]
    fields, launches = outputs(s), int(s.get_option("slice_launches"))
    s.close()
    o = make(stencil, n, radius, eb)
    fill(o, stencil, fill_steps)
    ref = loop(o, first, last, off, recs, injs)
    ref_fields = outputs(o)
    o.close()
    for (f, owned), rf, r in zip(got, ref, recs):
        assert owned.all()
        want = narrow(rf, r.dtype)
        assert same_bits(f, want), (r.dtype, np.argwhere(f.view(np.uint8) != want.view(np.uint8))[:5] if f.dtype == want.dtype else f.dtype)
    for k in ref_fields:
        assert same(fields[k], ref_fields[k]), k
    assert launches == due_steps(first, last, off, recs)


def loop(s, first, last, off, recs, injs=()):
    """slice_loop with the injectors applied first in each step."""
    if not injs:
        return slice_loop(s, first, last, off, recs)
    dt = np.float32 if s.get_element_bytes() == 4 else np.float64
    frames = [np.zeros((r.nrows,) + r.shape(), dt) for r in recs]
    step = 1 if last >= first else -1
    for t in range(first, last + step, step):
        s.run_solution(t, t)
        u = t + off
        for j in injs:
            j.apply(s, u)
        for r, f in zip(recs, frames):
            if r.row(u) is not None:
                f[r.row(u)] = r.read(s, u)
    return frames


N8 = (40, 36, 64)
F32_TYPES = ["float32", "float16", "bfloat16"]


def planes_and_box(n, dtype, nrows):
    hi = [m - 1 for m in n]
    return [TRec("p", [n[0] // 2, 0, 0], [n[0] // 2] + hi[1:], dtype, nrows=nrows),
            TRec("p", [0, n[1] // 2, 0], [hi[0], n[1] // 2, hi[2]], dtype, nrows=nrows),
            TRec("p", [0, 0, n[2] // 2], hi[:2] + [n[2] // 2], dtype, nrows=nrows),
            TRec("p", [1, 2, 3], hi, dtype, stride=[2, 3, 5], t0=2, every=2, nrows=nrows // 2)]


@pytest.mark.parametrize("dtype", F32_TYPES)
def test_iso3dfd_r8_fp32(dtype):
    run_case("iso3dfd", N8, 6, planes_and_box(N8, dtype, 6), radius=8)


@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_iso3dfd_r4_fp64(dtype):
    n = (32, 28, 48)
    run_case("iso3dfd", n, 6, planes_and_box(n, dtype, 6), radius=4, eb=8)


@pytest.mark.parametrize("dtype", F32_TYPES)
@pytest.mark.parametrize("stencil,n,reverse", [("awp_elastic", (21, 19, 40), False), ("wave2d", (37, 50), False),
                                               ("test_reverse_2d", (37, 50), True)])
def test_other_stencils(stencil, n, reverse, dtype):
    """awp_elastic updates its vars in place; wave2d has two domain dims; test_reverse_2d steps backwards."""
    names = ["vel_x", "stress_xx"] if stencil == "awp_elastic" else out_vars(stencil, 0)
    hi = [m - 1 for m in n]
    mid = [n[0] // 2] + [0] * (len(n) - 1)
    recs = [TRec(names[0], [0] * len(n), hi, dtype, stride=[2] + [3] * (len(n) - 1), t0=1, nrows=5),
            TRec(names[-1], mid, [n[0] // 2] + hi[1:], dtype, t0=-1 if reverse else 2, every=2 if reverse else 1, nrows=3)]
    run_case(stencil, n, 5, recs, eb=0, reverse=reverse)


def crafted(eb):
    """Values at the edges of the narrowing: ties at both parities, the ranges' ends, subnormals of each type, signed zeros and
    infinities, a NaN."""
    p = 2.0
    v = [1 + p ** -11, 1 + 3 * p ** -11, 1 + p ** -8, 1 + 3 * p ** -8, 65504, 65519.996, 65520, 1e5, p ** -24, p ** -25,
         3 * p ** -25, p ** -14 - p ** -25, 0.0, -0.0, np.inf, -np.inf, np.nan, 1 / 3]
    if eb == 4:    # float32 subnormals on and between the bf16 grid, and bf16's largest finite value and the tie above it
        extra = np.array([0x00000001, 0x00008000, 0x00018000, 0x00400000, 0x7F7F0000, 0x7F7F8000], np.uint32).view(np.float32)
        return np.concatenate([np.array(v + [-x for x in v], np.float32), extra, -extra])
    # float32's subnormals, their ties and its overflow, from double
    extra = [p ** -149, p ** -150, 3 * p ** -150, 1e-40, 3.4028235677973366e38, 3.4028235677973366e38 * (1 + p ** -25), 1e39]
    return np.array(v + extra + [-x for x in v + extra], np.float64)


@pytest.mark.parametrize("eb", [4, 8])
def test_crafted_elements(eb):
    """A `set` injector in the element type writes the crafted values (the loop writes them with set_elements_in_slice); the
    recorders of every allowed type narrow them in the same step."""
    n, steps = (32, 28, 64), 3
    vals = crafted(eb)
    first, last = [3, 4, 0], [3, 4, len(vals) - 1]
    frames = np.broadcast_to(vals, (steps, 1, 1, len(vals))).copy()
    injs = [TInj("p", first, last, frames=frames, mode="set", nrows=steps)]
    types = F32_TYPES if eb == 4 else ["float64", "float32"]
    recs = [TRec("p", first, last, d, nrows=steps) for d in types]
    run_case("iso3dfd", n, steps, recs, radius=4 if eb == 8 else 8, eb=eb, injs=injs)


@pytest.mark.parametrize("mode", ["set", "add"])
@pytest.mark.parametrize("eb,dtype", [(4, "float32"), (4, "float16"), (4, "bfloat16"), (8, "float64"), (8, "float32")])
def test_injectors_from_host_frames(eb, dtype, mode):
    """Host frames held in dtype and widened on the device; a recorder of the same box sees the injection."""
    n, steps = (32, 28, 48), 5
    injs = [TInj("p", [1, 0, 2], [31, 27, 46], dtype, stride=[2, 5, 3], mode=mode, nrows=steps - 1),
            TInj("p", [0, 0, 20], [31, 27, 20], dtype, mode=mode, t0=2, every=2, nrows=2, seed=1)]
    injs[0].frames[0, 0, 0, :4] = [65519.996, 2.0 ** -25, 3 * 2.0 ** -25, 1 + 2.0 ** -11]     # fp16's largest, subnormal ties, a tie
    recs = [TRec("p", [0, 0, 20], [31, 27, 20], nrows=steps)]
    run_case("iso3dfd", n, steps, recs, radius=4 if eb == 8 else 8, eb=eb, injs=injs)


@pytest.mark.parametrize("dtype", ["float16", "bfloat16", ("float32", 8)])
@pytest.mark.parametrize("reverse", [False, True], ids=["forward", "reversed"])
def test_injector_from_narrowed_recorder(dtype, reverse):
    """An injector fed from a narrowed recorder's device frames gives the bits of a host-fed injector with those frames."""
    dtype, eb = dtype if isinstance(dtype, tuple) else (dtype, 4)
    steps, box = 5, ([1, 0, 2], [31, 27, 46], [2, 5, 3])
    radius = 8 if eb == 4 else 4
    f = make("iso3dfd", (32, 28, 48), radius, eb)
    fill(f, "iso3dfd", [0, 1])
    f.add_slice("p", *box[:2], 1, steps, stride=box[2], dtype=dtype)
    f.run_solution(0, steps - 1)
    frames = f.get_slice_frames(0)[0]
    results = []
    for mode in ("set", "add"):
        for dev in (True, False):
            s = make("iso3dfd", (32, 28, 48), radius, eb)
            fill(s, "iso3dfd", [0, 1])
            if dev:
                s.add_slice_injector_from("p", *box[:2], 2, steps - 1, f, 0, reverse=reverse, stride=box[2], mode=mode)
            else:
                fr = frames[:steps - 1][::-1] if reverse else frames[:steps - 1]
                s.add_slice_injector("p", *box[:2], 2, np.ascontiguousarray(fr), stride=box[2], mode=mode, dtype=dtype)
            s.run_solution(0, steps - 1)
            results.append(outputs(s))
            s.close()
    f.close()
    for a, b in ((0, 1), (2, 3)):
        for k in results[b]:
            assert same(results[a][k], results[b][k]), k


class TCor:
    """A correlator with an image type: b is var(u) (src None) or a row of recorder src of the same solution, read in its type."""

    def __init__(self, var, first, last, image=None, src=None, reverse=False, stride=None, t0=1, every=1, nrows=4):
        self.var, self.first, self.last, self.image, self.src, self.reverse = var, list(first), list(last), image, src, reverse
        self.stride = list(stride) if stride else [1] * len(first)
        self.t0, self.every, self.nrows = t0, every, nrows

    def row(self, u):
        k = u - self.t0
        return k // self.every if k >= 0 and k % self.every == 0 and k // self.every < self.nrows else None

    def shape(self):
        return tuple((b - a) // k + 1 for a, b, k in zip(self.first, self.last, self.stride))

    def add(self, s, fwd=None):
        src = None if self.src is None else (fwd or s)
        return s.add_slice_correlator(self.var, self.first, self.last, self.t0, self.nrows, src=src, src_id=self.src, reverse=self.reverse,
                                      stride=self.stride, every=self.every, image_dtype=self.image)


def correlate(img, box, b, image):
    """One correlated step: in T, product and sum each rounded; in double, the product exact."""
    if image == "float64" and box.dtype == np.float32:
        return img + box.astype(np.float64) * b.astype(np.float64)
    return img + box * b.astype(box.dtype)


def correlate_loop(s, first, last, off, recs, cors, ext=None):
    dt = np.float32 if s.get_element_bytes() == 4 else np.float64
    frames = [np.zeros((r.nrows,) + r.shape(), dt) for r in recs]
    images = [np.zeros(c.shape(), np.float64 if c.image == "float64" else dt) for c in cors]
    step = 1 if last >= first else -1
    for t in range(first, last + step, step):
        s.run_solution(t, t)
        u = t + off
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
                fr = ext[c.src] if ext is not None else narrow(frames[c.src], recs[c.src].dtype)
                b = fr[c.nrows - 1 - r if c.reverse else r]
            img[...] = correlate(img, box, b, c.image)
    return images, [narrow(f, r.dtype) for f, r in zip(frames, recs)]


def correlate_case(n, steps, recs, cors, radius=8, eb=4):
    s = make("iso3dfd", n, radius, eb)
    fill(s, "iso3dfd", [0, 1])
    for r in recs:
        r.add(s)
    assert [c.add(s) for c in cors] == list(range(len(cors)))
    s.run_solution(0, steps - 1)
    images = [s.get_correlator_image(i) for i in range(len(cors))]
    frames = [s.get_slice_frames(i)[0] for i in range(len(recs))]
    fields = outputs(s)
    counts = (int(s.get_option("slice_launches")), int(s.get_option("slice_correlator_launches")))
    s.close()
    o = make("iso3dfd", n, radius, eb)
    fill(o, "iso3dfd", [0, 1])
    ref_images, ref_frames = correlate_loop(o, 0, steps - 1, 1, recs, cors)
    ref_fields = outputs(o)
    o.close()
    for (img, owned), ref in zip(images, ref_images):
        assert owned.all()
        assert same_bits(img, ref), np.argwhere(img != ref)[:5]
    for f, rf in zip(frames, ref_frames):
        assert same_bits(f, rf)
    for k in ref_fields:
        assert same(fields[k], ref_fields[k]), k
    return counts


HI8 = [39, 35, 63]


@pytest.mark.parametrize("image", ["float32", "float64"])
@pytest.mark.parametrize("dtype", F32_TYPES)
def test_correlators_against_narrowed_recorders(dtype, image):
    box = ([1, 0, 2], HI8, [3, 1, 2])
    recs = [TRec("p", box[0], box[1], dtype, stride=box[2], nrows=6)]
    cors = [TCor("p", box[0], box[1], image, src=0, reverse=True, stride=box[2], nrows=6),
            TCor("p", box[0], box[1], image, src=0, stride=box[2], t0=2, every=2, nrows=2),
            TCor("p", [0, 0, 0], HI8, image, nrows=6)]
    assert correlate_case(N8, 6, recs, cors) == (6, 6)


@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_correlators_fp64(dtype):
    n, hi = (32, 28, 48), [31, 27, 47]
    recs = [TRec("p", [0, 0, 0], hi, dtype, stride=[1, 2, 1], nrows=5)]
    cors = [TCor("p", [0, 0, 0], hi, "float64", src=0, reverse=True, stride=[1, 2, 1], nrows=5), TCor("p", [0, 0, 0], hi, nrows=5)]
    assert correlate_case(n, 5, recs, cors, radius=4, eb=8) == (5, 5)


def test_mixed_types_share_one_launch_per_step():
    """f32, f16 and bf16 recorders and correlators of both image types in one solution: one recording and one correlating launch
    per step."""
    recs = [TRec("p", [0, 0, 0], HI8, "float32", nrows=6), TRec("p", [0, 0, 31], [39, 35, 31], "float16", nrows=6),
            TRec("p", [2, 1, 0], HI8, "bfloat16", stride=[4, 3, 2], t0=2, every=2, nrows=3)]
    cors = [TCor("p", [0, 0, 0], HI8, "float64", src=0, reverse=True, nrows=6),
            TCor("p", [0, 0, 31], [39, 35, 31], "float32", src=1, nrows=6),
            TCor("p", [2, 1, 0], HI8, "float64", src=2, stride=[4, 3, 2], t0=2, every=2, nrows=3, reverse=True),
            TCor("p", [0, 0, 0], HI8, "float64", nrows=6), TCor("p", [5, 0, 0], [5, 35, 63], None, nrows=6)]
    assert correlate_case(N8, 6, recs, cors) == (6, 6)


@pytest.mark.parametrize("grid,n", [((2, 1, 1), (75, 40, 64)), ((2, 2, 1), (61, 59, 48))], ids=["2x1x1", "2x2x1"])
def test_rank_grid_matches_single_rank(grid, n):
    """Each rank records its part in bf16 and f16 and correlates a double image against the forward grid's bf16 frames."""
    steps, world = 4, int(np.prod(grid))
    hi = [m - 1 for m in n]
    box = ([1, 2, 3], hi, [3, 2, 5])
    recs = [TRec("p", *box[:2], "bfloat16", stride=box[2], nrows=steps), TRec("p", [0, 0, n[2] // 2], hi[:2] + [n[2] // 2], "float16", nrows=steps)]
    cors = [TCor("p", *box[:2], "float64", src=0, reverse=True, stride=box[2], nrows=steps), TCor("p", [0, 0, 0], hi, "float64", nrows=steps)]
    fwd = [make("iso3dfd", n, 8, 4, (), grid, r) for r in range(world)]
    multi.connect_local(fwd)
    adj = [make("iso3dfd", n, 8, 4, (), grid, r) for r in range(world)]
    multi.connect_local(adj)
    for f, a in zip(fwd, adj):
        fill(f, "iso3dfd", [0, 1])
        fill(a, "iso3dfd", [0, 1])
        for r in recs:
            r.add(f)
    for f in fwd:
        f.run_solution(0, steps - 1)
    for a, f in zip(adj, fwd):
        for c in cors:
            c.add(a, f)
    for a in adj:
        a.run_solution(0, steps - 1)
    for a in adj:
        a.sync()
    frames = [np.zeros((steps,) + r.shape(), np.float32 if r.dtype == "bfloat16" else np.float16) for r in recs]
    images = [np.zeros(c.shape(), np.float64) for c in cors]
    for f, a in zip(fwd, adj):
        for fr, i in zip(frames, range(len(recs))):
            got, owned = f.get_slice_frames(i)
            fr[:, owned] = got[:, owned]
        for img, i in zip(images, range(len(cors))):
            got, owned = a.get_correlator_image(i)
            img[owned] = got[owned]
        assert int(a.get_option("slice_correlator_launches")) == steps
        f.close()
        a.close()
    o = make("iso3dfd", n, 8)
    fill(o, "iso3dfd", [0, 1])
    ref_frames = [narrow(fr, r.dtype) for fr, r in zip(slice_loop(o, 0, steps - 1, 1, recs), recs)]
    o.close()
    for fr, rf in zip(frames, ref_frames):
        assert same_bits(fr, rf)
    o = make("iso3dfd", n, 8)
    fill(o, "iso3dfd", [0, 1])
    ref_images = correlate_loop(o, 0, steps - 1, 1, [], cors, ext=[ref_frames[0]])[0]
    o.close()
    for img, ref in zip(images, ref_images):
        assert same_bits(img, ref), np.argwhere(img != ref)[:5]


def test_past_2_31_elements_per_slot():
    """A bf16 recorder and a double-image correlator against it, on boxes across element 2^31 of a slot."""
    from tests.large_domain import crossing_index
    n, steps = (1100, 1024, 1984), 2
    s = make("iso3dfd", n)
    p = s.get_var("p")
    xc = int(crossing_index(p.info))
    assert p.info.slot_elems > 1 << 31 and xc < n[0] - 2
    box = ([xc - 2, 0, 0], [n[0] - 1, n[1] - 1, n[2] - 1], [5, 7, 1])
    recs = [TRec("p", *box[:2], "bfloat16", stride=box[2], nrows=steps)]
    cors = [TCor("p", *box[:2], "float64", src=0, reverse=True, stride=box[2], nrows=steps)]
    fill(s, "iso3dfd", [0, 1])
    recs[0].add(s)
    cors[0].add(s)
    s.run_solution(0, steps - 1)
    got_f, got_i = s.get_slice_frames(0)[0], s.get_correlator_image(0)[0]
    s.close()
    o = make("iso3dfd", n)
    fill(o, "iso3dfd", [0, 1])
    ref_i, ref_f = correlate_loop(o, 0, steps - 1, 1, recs, cors)
    o.close()
    assert same_bits(got_f, ref_f[0])
    assert same_bits(got_i, ref_i[0])


MOD = glob.glob(os.path.join(ROOT, "yask_b200", "lib", "python", "iso3dfd", "yask_kernel*.so"))
SCRIPT = textwrap.dedent("""
    import numpy as np
    import yask_kernel as yk

    steps, n = 4, (40, 36, 64)
    fac = yk.yk_factory()
    s = fac.new_solution(fac.new_env())
    s.set_overall_domain_size_vec(list(n))
    s.prepare_solution()
    s.get_var("v").set_all_elements_same(0.1)
    p = s.get_var("p")
    p.set_all_elements_same(0.375)
    p.set_element(1 + 2.0 ** -8, [0, 20, 18, 32])
    first, last = [0, 0, 0], [39, 35, 63]
    plane = ([0, 0, 31], [39, 35, 31])
    frames = np.random.default_rng(2).uniform(-4, 4, (1, 40, 36, 1))
    assert yk.yk_add_slice_injector_typed(s, "p", *plane, 2, 1, frames.ravel().tolist(), "float16", set=True) == 0
    assert yk.yk_add_slice(s, "p", first, last, 1, steps) == 0
    assert yk.yk_add_slice_typed(s, "p", first, last, 1, steps, "bfloat16") == 1
    assert yk.yk_add_slice_correlator_typed(s, "p", first, last, 1, steps, "float64") == 0
    s.run_solution(0, steps - 1)
    f32, shape, _ = yk.yk_get_slice_frames(s, 0)
    f32 = np.array(f32, np.float32).reshape(shape)
    b16 = np.array(yk.yk_get_slice_frames(s, 1)[0]).reshape(shape)
    u = f32.view(np.uint32).astype(np.uint64)
    want = (((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16).astype(np.uint32).view(np.float32)
    assert np.array_equal(b16, want.astype(np.float64))
    with np.errstate(over="ignore"):
        assert np.array_equal(f32[1, :, :, 31:32], frames[0].astype(np.float32).astype(np.float16).astype(np.float32))
    img = np.array(yk.yk_get_correlator_image(s, 0)[0]).reshape(shape[1:])
    ref = np.zeros(shape[1:])
    for r in range(steps):
        ref = ref + f32[r].astype(np.float64) * f32[r].astype(np.float64)
    finite = np.isfinite(ref)
    assert np.array_equal(img[finite], ref[finite]) and np.array_equal(np.isfinite(img), finite)
    assert yk.yk_get_slice_launches(s) == steps and yk.yk_get_slice_correlator_launches(s) == steps
    print("typed api ok")
""")


@pytest.mark.skipif(not MOD, reason="python module not built")
def test_yask_kernel_module_typed_calls():
    env = dict(os.environ, PYTHONPATH=os.path.dirname(MOD[0]))
    r = subprocess.run([sys.executable, "-c", SCRIPT], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "typed api ok" in r.stdout
