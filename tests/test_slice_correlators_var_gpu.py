"""Correlators whose b is a var of another solution (add_slice_correlator_var) on the device, bit for bit against the host loop
on the same hash-filled inputs:

    for k in steps:
        g.run_solution(k); a.run_solution(k)
        for each correlator with row r due at u (u = k + 1):
            image = image + a.var(u)[box] * g.src_var(src_t0 + u - t0)[box]      (numpy, in the element or image type)

Every image, every written var of both solutions at every valid step and, on one rank, the exact number of correlating
launches are compared.  The device runs alternate one-step calls of the two solutions with no host sync between them."""
import glob
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from tests.test_points_gpu import fill, make, outputs, same
from tests.test_slice_correlators_gpu import Cor
from tests.test_slices_gpu import Rec
from yask_b200 import capi, multi

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class VCor:
    """A var correlator: consumer var, box, window, and the source var and its first paired step."""

    def __init__(self, var, first, last, stride=None, t0=1, every=1, nrows=4, src_var=None, src_t0=None, image_dtype=None):
        self.var, self.first, self.last = var, list(first), list(last)
        self.stride = list(stride) if stride else [1] * len(first)
        self.t0, self.every, self.nrows = t0, every, nrows
        self.src_var = src_var or var
        self.src_t0 = t0 if src_t0 is None else src_t0
        self.image_dtype = image_dtype

    def row(self, u):
        k = u - self.t0
        return k // self.every if k >= 0 and k % self.every == 0 and k // self.every < self.nrows else None

    def shape(self):
        return tuple((b - a) // k + 1 for a, b, k in zip(self.first, self.last, self.stride))

    def add(self, a, g):
        return a.add_slice_correlator_var(self.var, self.first, self.last, self.t0, self.nrows, g, self.src_var, src_t0=self.src_t0,
                                          stride=self.stride, every=self.every, image_dtype=self.image_dtype)

    def box(self, s, var, step):
        sl = tuple(slice(None, None, k) for k in self.stride)
        return s.get_var(var).get_elements_in_slice([step] + self.first, [step] + self.last)[sl]


def pair(stencil, n, radius, eb, g_stencil=None, g_opts=(), a_opts=(), grid=None, rank=0):
    g = make(g_stencil or stencil, n, radius, eb, g_opts, grid, rank)
    a = make(stencil, n, radius, eb, a_opts, grid, rank)
    return g, a


def filled(g, a, g_stencil, stencil):
    fill(g, g_stencil, [0, 1, 2, 3])
    fill(a, stencil, [0, 1, 2, 3])
    # a differs from g: its step-0 and step-1 fields are shifted by a second hash
    for v in a.get_vars():
        if v.info.is_output and v.info.has_step:
            v.fill_hash(0, 77, 5, -0.5, 0.5)


def host_loop(g, a, steps, cors, off=1):
    """The alternating loop with the correlation in numpy (each get_elements_in_slice syncs its solution)."""
    dt = np.float32 if a.get_element_bytes() == 4 else np.float64
    images = [np.zeros(c.shape(), np.float64 if c.image_dtype == "float64" else dt) for c in cors]
    for k in range(steps):
        g.run_solution(k)
        a.run_solution(k)
        u = k + off
        for c, img in zip(cors, images):
            if c.row(u) is None:
                continue
            x, y = c.box(a, c.var, u), c.box(g, c.src_var, c.src_t0 + u - c.t0)
            if img.dtype == np.float64 and dt == np.float32:
                img[...] = img + x.astype(np.float64) * y.astype(np.float64)
            else:
                img[...] = img + x * y
    return images


def device_loop(g, a, steps):
    for k in range(steps):
        g.run_solution(k)
        a.run_solution(k)


def run_case(stencil, n, steps, cors, radius=0, eb=4, g_stencil=None, g_opts=(), a_opts=(), extra=None):
    g_stencil = g_stencil or stencil
    out = []
    for device in (True, False):
        g, a = pair(stencil, n, radius, eb, g_stencil, g_opts, a_opts)
        filled(g, a, g_stencil, stencil)
        ids = [c.add(a, g) for c in cors]
        assert ids == list(range(len(cors)))
        if extra:
            extra(a)
        if device:
            device_loop(g, a, steps)
            a.sync()
            imgs = [a.get_correlator_image(i)[0] for i in range(len(cors))]
            launches = int(a.get_option("slice_correlator_launches"))
        else:
            a.clear_slice_correlators()
            imgs, launches = host_loop(g, a, steps, cors), None
        out.append((imgs, outputs(g), outputs(a), launches))
        g.close()
        a.close()
    (dev, gd, ad, launches), (ref, gr, ar, _) = out
    for d, r in zip(dev, ref):
        assert d.dtype == r.dtype and same(d, r), np.argwhere(d != r)[:5]
    for x, y in ((gd, gr), (ad, ar)):
        assert x.keys() == y.keys()
        for key in x:
            assert same(x[key], y[key]), key
    return launches


def due_steps(steps, cors, off=1):
    return sum(1 for k in range(steps) if any(c.row(k + off) is not None for c in cors))


N8 = (40, 36, 64)
HI8 = [m - 1 for m in N8]


@pytest.mark.parametrize("case", ["full", "strided", "nrows-short", "double-image"])
def test_iso3dfd_r8_fp32(case):
    steps = 6
    c = {"full": VCor("p", [0, 0, 0], HI8, nrows=steps),
         "strided": VCor("p", [1, 2, 3], HI8, stride=[3, 2, 5], t0=2, every=2, nrows=3, src_t0=1),
         "nrows-short": VCor("p", [0, 0, 0], HI8, nrows=2),
         "double-image": VCor("p", [2, 0, 1], HI8, stride=[1, 3, 1], nrows=steps, image_dtype="float64")}[case]
    launches = run_case("iso3dfd", N8, steps, [c], radius=8)
    assert launches == due_steps(steps, [c])


def test_with_frame_correlator_and_autocorrelation():
    """A var correlator beside a frame correlator and an autocorrelation of one solution: the frame kernel's launch and the var
    kernel's launch right after it, in each step where both kinds are due."""
    steps = 5
    vc = VCor("p", [0, 0, 0], HI8, nrows=steps, every=2)
    rec = Rec("p", [1, 2, 3], HI8, stride=[3, 2, 5], nrows=steps)
    fc = Cor("p", [1, 2, 3], HI8, stride=[3, 2, 5], nrows=steps, src=("self", 0))
    ac = Cor("p", [0, 0, 0], HI8, nrows=steps)
    out = []
    for device in (True, False):
        g, a = pair("iso3dfd", N8, 8, 4)
        filled(g, a, "iso3dfd", "iso3dfd")
        rec.add(a)
        assert ac.add(a) == 0 and vc.add(a, g) == 1
        if device:
            assert a.add_slice_correlator("p", [1, 2, 3], HI8, 1, steps, src=a, src_id=0, stride=[3, 2, 5]) == 2
            device_loop(g, a, steps)
            a.sync()
            out.append([a.get_correlator_image(i)[0] for i in range(3)])
            frame_due = sum(1 for k in range(steps) if ac.row(k + 1) is not None)
            var_due = sum(1 for k in range(steps) if vc.row(k + 1) is not None)
            assert int(a.get_option("slice_correlator_launches")) == frame_due + var_due
        else:
            a.clear_slice_correlators()
            dt = np.float32
            imgs = [np.zeros(ac.shape(), dt), np.zeros(vc.shape(), dt), np.zeros(fc.shape(), dt)]
            for k in range(steps):
                g.run_solution(k)
                a.run_solution(k)
                u = k + 1
                pa = a.get_var("p").get_elements_in_slice([u, 0, 0, 0], [u] + HI8)
                if ac.row(u) is not None:
                    imgs[0] = imgs[0] + pa * pa
                if vc.row(u) is not None:
                    imgs[1] = imgs[1] + pa * g.get_var("p").get_elements_in_slice([u, 0, 0, 0], [u] + HI8)
                if fc.row(u) is not None:
                    b = pa[1::3, 2::2, 3::5]
                    imgs[2] = imgs[2] + b * b
            out.append(imgs)
        g.close()
        a.close()
    for d, r in zip(*out):
        assert same(d, r)


@pytest.mark.parametrize("radius", [4, 3])
def test_iso3dfd_fp64(radius):
    """fp64: the hand-written sweep at radius 4 and the generated kernel at radius 3."""
    n, steps = (30, 28, 48), 5
    cors = [VCor("p", [0, 0, 0], [29, 27, 47], nrows=steps), VCor("p", [1, 1, 2], [29, 27, 47], stride=[2, 3, 2], every=2, nrows=2, src_t0=0)]
    assert run_case("iso3dfd", n, steps, cors, radius=radius, eb=8) == due_steps(steps, cors)


def test_source_with_other_storage():
    """An iso3dfd_sponge source (other vars, other halos) and an iso3dfd source with larger pads."""
    steps = 4
    c = VCor("p", [0, 1, 0], HI8, stride=[1, 2, 1], nrows=steps)
    run_case("iso3dfd", N8, steps, [c], radius=8, g_stencil="iso3dfd_sponge")
    out = []
    for device in (True, False):
        g = capi.Solution("iso3dfd", radius=8)
        g.set_overall_domain_size_vec(N8)
        for d, m in enumerate((20, 24, 40)):
            capi._chk(capi.lib().yb_set_min_pad_size(g._h, d, m))
        g.prepare_solution(0)
        a = make("iso3dfd", N8, 8, 4)
        assert g.get_var("p").info.slot_elems != a.get_var("p").info.slot_elems
        filled(g, a, "iso3dfd", "iso3dfd")
        c.add(a, g)
        if device:
            device_loop(g, a, steps)
            out.append(a.get_correlator_image(0)[0])
        else:
            a.clear_slice_correlators()
            out.append(host_loop(g, a, steps, [c])[0])
        g.close()
        a.close()
    assert same(out[0], out[1])


def test_awp_elastic_in_place():
    """awp_elastic: a multi-stage solution whose vars are updated in place (alloc_t = 1): only the newest step pairs."""
    n, steps = (21, 19, 40), 4
    cors = [VCor("vel_x", [0, 0, 0], [20, 18, 39], nrows=steps), VCor("stress_xx", [1, 0, 2], [20, 18, 39], stride=[2, 1, 3], nrows=steps)]
    assert run_case("awp_elastic", n, steps, cors) == due_steps(steps, cors)


def test_multi_step_run_fits_or_is_refused():
    """A consumer run of several steps is legal when every due step pairs inside the source's valid window; otherwise it is
    refused before anything changes."""
    g, a = pair("iso3dfd", N8, 8, 4)
    filled(g, a, "iso3dfd", "iso3dfd")
    g.run_solution(0, 4)                     # g's p: steps 4, 5
    # a's steps 1..2 would pair with 4..5 (src_t0 = 4): a run of 2 steps fits
    assert VCor("p", [0, 0, 0], HI8, t0=1, nrows=10, src_t0=4).add(a, g) == 0
    a.run_solution(0, 1)
    img1 = a.get_correlator_image(0)[0].copy()
    before = outputs(a)
    with pytest.raises(capi.YaskError) as e:
        a.run_solution(2, 3)                 # u = 3 pairs with step 6 of g: outside [4, 5]
    msg = str(e.value)
    for w in ("slice correlator 0", "step 3 pairs with step 6", "valid steps [4, 5]"):
        assert w in msg, msg
    assert same(a.get_correlator_image(0)[0], img1)
    after = outputs(a)
    assert before.keys() == after.keys() and all(same(before[k], after[k]) for k in before)
    c = VCor("p", [0, 0, 0], HI8)
    ref = np.zeros_like(img1)
    for u in (1, 2):
        ref = ref + c.box(a, "p", u) * c.box(g, "p", u + 3)
    assert same(img1, ref)
    g.close()
    a.close()


def test_unsynced_refill_and_no_recorders():
    """The source has no recorders.  Source runs, consumer runs, the source is refilled and runs, the consumer runs: no host sync,
    and the image is that of the same sequence with a sync after every call."""
    c = VCor("p", [0, 0, 0], HI8, t0=1, nrows=4)
    out = []
    for sync in (False, True):
        g, a = pair("iso3dfd", N8, 8, 4)
        filled(g, a, "iso3dfd", "iso3dfd")
        c.add(a, g)
        seq = [lambda: g.run_solution(0), lambda: a.run_solution(0),
               lambda: g.get_var("p").fill_hash(1, 99, 3, -1, 1), lambda: g.get_var("p").fill_hash(2, 98, 4, -1, 1),
               lambda: g.run_solution(2), lambda: a.run_solution(1), lambda: g.run_solution(3), lambda: a.run_solution(2)]
        for f in seq:
            f()
            if sync:
                g.sync()
                a.sync()
        out.append((a.get_correlator_image(0)[0], outputs(g), outputs(a)))
        g.close()
        a.close()
    (i0, g0, a0), (i1, g1, a1) = out
    assert same(i0, i1)
    for x, y in ((g0, g1), (a0, a1)):
        assert all(same(x[k], y[k]) for k in x)


def test_source_storage_moves():
    """The source's storage changes under an existing correlator: fuse_vars gives it another allocation, and a radius-2 source
    running two-step calls in pairs (block_steps=2) moves its live slots."""
    steps = 4
    c = VCor("p", [0, 0, 0], HI8, t0=2, every=2, nrows=2, src_t0=2)
    out = []
    for device in (True, False):
        g, a = pair("iso3dfd", N8, 8, 4)
        h = make("iso3dfd", N8, 8, 4)
        filled(g, a, "iso3dfd", "iso3dfd")
        fill(h, "iso3dfd", [0, 1])
        c.add(a, g)
        g.run_solution(0)
        a.run_solution(0)
        g.get_var("p").fuse_vars(h.get_var("p"))
        g.run_solution(1)
        if device:
            a.run_solution(1)
            out.append(a.get_correlator_image(0)[0])
        else:
            a.clear_slice_correlators()
            a.run_solution(1)
            out.append(c.box(a, "p", 2) * c.box(g, "p", 2))
        for x in (g, a, h):
            x.close()
    assert same(out[0], out[1])
    # pairs: a radius-2 source with block_steps=2, two steps per call, so each call moves its live slot pair; the consumer
    # correlates every step, the first step of each pair included
    out = []
    c = VCor("p", [0, 0, 0], HI8, t0=1, nrows=6)
    for device in (True, False):
        g, a = pair("iso3dfd", N8, 2, 4, g_opts=(("block_steps", 2),), a_opts=(("block_steps", 2),))
        filled(g, a, "iso3dfd", "iso3dfd")
        c.add(a, g)
        if not device:
            a.clear_slice_correlators()
        img, ptrs = np.zeros(c.shape(), np.float32), []
        for k in range(0, 6, 2):
            g.run_solution(k, k + 1)          # two steps in one fused launch
            ptrs.append(g.get_var("p").device_ptr(k + 2))
            a.run_solution(k, k + 1)
            if not device:
                for u in (k + 1, k + 2):
                    img = img + c.box(a, "p", u) * c.box(g, "p", u)
        assert len(set(ptrs)) == 2, ptrs       # the even steps alternate between the two slot pairs: the bias moved
        if device:
            assert a.get_option("slice_correlator_launches") == "6"
        out.append(a.get_correlator_image(0)[0] if device else img)
        g.close()
        a.close()
    assert same(out[0], out[1])


def test_source_destroyed():
    g, a = pair("iso3dfd", N8, 8, 4)
    filled(g, a, "iso3dfd", "iso3dfd")
    VCor("p", [0, 0, 0], HI8, nrows=4).add(a, g)
    g.run_solution(0)
    a.run_solution(0)
    img = a.get_correlator_image(0)[0].copy()
    assert img.any()
    g.close()
    with pytest.raises(capi.YaskError, match="slice correlator 0: its source solution 'iso3dfd' was destroyed"):
        a.run_solution(1)
    assert same(a.get_correlator_image(0)[0], img)
    a.clear_slice_correlators()
    a.run_solution(1)
    a.close()


GRIDS = [("2x1x1-fused", (2, 1, 1), (75, 40, 64), ()), ("1x2x1-split", (1, 2, 1), (40, 75, 64), ()),
         ("3x1x1-whole-uneven", (3, 1, 1), (77, 36, 64), (("overlap_comms", 0),))]


@pytest.mark.parametrize("name,grid,n,opts", GRIDS, ids=[g[0] for g in GRIDS])
def test_rank_grid_matches_single_rank(name, grid, n, opts):
    steps, world = 4, int(np.prod(grid))
    hi = [m - 1 for m in n]
    cors = [VCor("p", [0, 0, 0], hi, nrows=steps), VCor("p", [1, 2, 3], hi, stride=[3, 2, 5], every=2, nrows=2, src_t0=0)]
    gs = [make("iso3dfd", n, 8, 4, opts, grid, r) for r in range(world)]
    multi.connect_local(gs)
    adj = [make("iso3dfd", n, 8, 4, opts, grid, r) for r in range(world)]
    multi.connect_local(adj)
    for g, a in zip(gs, adj):
        filled(g, a, "iso3dfd", "iso3dfd")
        for c in cors:
            c.add(a, g)
    with pytest.raises(capi.YaskError, match="rank index"):
        cors[0].add(adj[0], gs[1])
    for k in range(steps):
        for g in gs:
            g.run_solution(k)
        for a in adj:
            a.run_solution(k)
    for a in adj:
        a.sync()
    merged = [np.zeros(c.shape(), np.float32) for c in cors]
    for g, a in zip(gs, adj):
        for i in range(len(cors)):
            img, owned = a.get_correlator_image(i)
            merged[i][owned] = img[owned]
        g.close()
        a.close()
    g, a = pair("iso3dfd", n, 8, 4)
    filled(g, a, "iso3dfd", "iso3dfd")
    ref = host_loop(g, a, steps, cors)
    g.close()
    a.close()
    for m, r in zip(merged, ref):
        assert same(m, r), np.argwhere(m != r)[:5]


def test_past_2_31_elements_per_slot():
    """A source whose var slot holds more than 2^31 elements (two such solutions: about 54 GB).  Both steps of the run stay
    valid, so the image is checked against numpy on three x-planes of the decimated box."""
    n, steps = (1290, 1290, 1296), 2
    c = VCor("p", [0, 0, 0], [m - 1 for m in n], stride=[7, 1, 1], nrows=steps)
    g, a = pair("iso3dfd", n, 8, 4)
    assert g.get_var("p").info.slot_elems > 2 ** 31
    for s in (g, a):
        salt = 1 if s is g else 9
        s.get_var("p").fill_hash(0, 5, salt, -1, 1)
        s.get_var("p").fill_hash(1, 6, salt + 1, -1, 1)
        s.get_var("v").fill_hash(0, 7, 3, 0.05, 0.3)
    c.add(a, g)
    device_loop(g, a, steps)
    a.sync()
    img = a.get_correlator_image(0)[0]
    assert img.shape == c.shape()
    for i in (0, c.shape()[0] // 2, c.shape()[0] - 1):
        x = 7 * i
        want = np.zeros(c.shape()[1:], np.float32)
        for u in (1, 2):
            pa = a.get_var("p").get_elements_in_slice([u, x, 0, 0], [u, x, n[1] - 1, n[2] - 1])[0]
            pg = g.get_var("p").get_elements_in_slice([u, x, 0, 0], [u, x, n[1] - 1, n[2] - 1])[0]
            want = want + pa * pg
        assert same(img[i], want), i
    g.close()
    a.close()


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
    g, a = solution(0.25), solution(0.75)
    assert yk.yk_add_slice_correlator(a, "p", first, last, 1, steps) == 0
    assert yk.yk_add_slice_correlator_var(a, "p", first, last, 1, steps, g, "p", 1, stride) == 1
    assert yk.yk_add_slice_correlator_var(a, "p", first, last, 2, 1, g, "p", 2, stride, 1, "float64") == 2
    for t in range(steps):
        g.run_solution(t)
        a.run_solution(t)
    assert yk.yk_get_slice_correlator_launches(a) == 2 * steps
    img, ishape, owned = yk.yk_get_correlator_image(a, 1)
    img = np.array(img, np.float32).reshape(ishape)
    img64 = np.array(yk.yk_get_correlator_image(a, 2)[0]).reshape(ishape)
    assert all(owned)

    g2, b = solution(0.25), solution(0.75)
    ref, ref64 = np.zeros_like(img), np.zeros_like(img64)
    for t in range(steps):
        g2.run_solution(t)
        b.run_solution(t)
        u = t + 1
        x, y = np.zeros((1, 40, 36, 63), np.float32), np.zeros((1, 40, 36, 63), np.float32)
        b.get_var("p").get_elements_in_slice(x, [u] + first, [u] + last)
        g2.get_var("p").get_elements_in_slice(y, [u] + first, [u] + last)
        ref = ref + x[0, :, ::2, ::3] * y[0, :, ::2, ::3]
        if u == 2:
            ref64 = ref64 + x[0, :, ::2, ::3].astype(np.float64) * y[0, :, ::2, ::3].astype(np.float64)
    assert np.array_equal(img.view(np.uint32), ref.view(np.uint32)), np.abs(img - ref).max()
    assert np.array_equal(img64.view(np.uint64), ref64.view(np.uint64))
    print("var correlators api ok")
""")


@pytest.mark.skipif(not MOD, reason="python module not built")
def test_yask_kernel_module():
    env = dict(os.environ, PYTHONPATH=os.path.dirname(MOD[0]))
    r = subprocess.run([sys.executable, "-c", SCRIPT], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "var correlators api ok" in r.stdout
