"""CPU: 3axis, 3axis_with_diags, 3plane and cube at any radius in fp32 and fp64.
  * the oracle (tests/avepts_oracle.py) is bit-exact against the generated restatements of the reference's default-radius builds
    (both contraction modes) and against the unmodified reference built at other radii (tests/golden/<shape>-r<r>*.npz,
    <shape>-fp64-r<r>*.npz) in its default build and with -ffp-contract=off;
  * without a device: routing (default fp32 radius -> generated form, other radii and fp64 -> hand-written form, radius 9 refused),
    the hand-written form declares the generated form's vars, dims and halos, plan_geometry() pads;
  * the radius- and precision-suffixed C++ API libraries and the shapes' Python modules report their radius and precision.
"""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from oracle import oracle as O
from tests import avepts_oracle as A
from tests.helpers import golden_cases, load_golden, regen_inputs
from yask_b200 import capi
from yask_b200.synth import hash_field, var_salt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FP32_RADII, FP64_RADII = (1, 2, 5, 8), (2, 8)
CASES = [p for s in A.SHAPES for r in FP32_RADII for p in golden_cases(f"{s}-r{r}")] + \
        [p for s in A.SHAPES for r in FP64_RADII for p in golden_cases(f"{s}-fp64-r{r}")]


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def test_point_counts_and_order():
    for shape in A.SHAPES:
        for R in range(1, 9):
            pts = A.points(shape, R)
            assert len(pts) == len(set(pts)) == A.npoints(shape, R)
            assert pts[0] == (0, 0, 0) and max(max(abs(c) for c in p) for p in pts) == R
    # the order the reference's compiler emits at radius 4 (oracle/gen/s3axis.gen.h)
    assert A.points("3axis", 2)[:13] == [(0, 0, 0), (-1, 0, 0), (1, 0, 0), (0, -1, 0), (0, 1, 0), (0, 0, -1), (0, 0, 1),
                                         (-2, 0, 0), (2, 0, 0), (0, -2, 0), (0, 2, 0), (0, 0, -2), (0, 0, 2)]


@pytest.mark.parametrize("contract", [0, 1])
@pytest.mark.parametrize("shape", A.SHAPES)
def test_oracle_matches_generated_restatement(shape, contract):
    R, n, steps = A.DEFAULT_RADIUS[shape], (13, 17, 37), 3
    ins = {("A", t): hash_field(30 + t, var_salt("A", t), (-R,) * 3, [i + 2 * R for i in n], -1, 1) for t in (0, 1)}
    gen = O.gen_run(shape, n, steps, ins, contract=contract)
    tl, ref = gen["A"]
    got = A.run(ins[("A", 0)], ins[("A", 1)], shape, R, steps)
    assert tl == steps and np.array_equal(_bits(got), _bits(ref))


def test_fixtures_cover_every_shape_radius_and_build():
    # cube at radius 8 (4913 points) is not among them: the reference's build of it did not complete in the time the others took
    tags = {load_golden(p)[0]["ref_tag"] for p in CASES}
    want = {f"{s}-r{r}{b}.avx512" for s in A.SHAPES for r in FP32_RADII for b in ("", "-strict")} | \
           {f"{s}-fp64-r{r}{b}.avx512" for s in A.SHAPES for r in FP64_RADII for b in ("", "-strict")}
    assert tags == {t for t in want if not t.startswith(("cube-r8", "cube-fp64-r8"))}


@pytest.mark.parametrize("path", CASES, ids=[os.path.basename(p)[:-4] for p in CASES])
def test_oracle_bit_exact_vs_reference(path):
    meta, arrays = load_golden(path)
    shape = meta["ref_tag"].split("-")[0]
    R = int(meta["ref_tag"].split("-r")[1].split("-")[0].split(".")[0])
    ins = regen_inputs(meta)
    ref = arrays[f"A.t{meta['vars']['A']['steps'][1]}"]
    got = A.run(ins[("A", 0)], ins[("A", 1)], shape, R, meta["steps"])[R:-R, R:-R, R:-R]
    assert got.dtype == ref.dtype and np.array_equal(_bits(got), _bits(ref))


def _layout(s):
    out = []
    for v in s.get_vars():
        vi = v.info
        out.append((vi.name, vi.step_alloc, vi.is_output, vi.halo_exchange_l1_norm,
                    [(vi.dims[i].name, vi.dims[i].kind, vi.dims[i].left_halo, vi.dims[i].right_halo) for i in range(vi.num_dims)]))
    return out


def _is_hand_written(s):
    try:
        s.get_option("kernel")      # an option of the hand-written engine only
        return True
    except capi.YaskError:
        return False


@pytest.mark.parametrize("shape", A.SHAPES)
def test_routing(shape):
    d = A.DEFAULT_RADIUS[shape]
    for R, eb, hand in [(0, 4, False), (d, 4, False), (0, 8, True), (d, 8, True)] + \
                       [(r, 4, True) for r in range(1, 9) if r != d] + [(r, 8, True) for r in range(1, 9)]:
        s = capi.Solution(shape, radius=R, elem_bytes=eb)
        try:
            assert s.get_name() == shape and s.get_element_bytes() == eb
            assert _is_hand_written(s) == hand, (R, eb)
            assert s.get_var("A").info.dims[1].left_halo == (R or d)
        finally:
            s.close()
    for eb in (4, 8):
        with pytest.raises(capi.YaskError, match="radius 9 > 8"):
            capi.Solution(shape, radius=9, elem_bytes=eb)


@pytest.mark.parametrize("shape", A.SHAPES)
def test_vars_equal_generated(shape):
    d = A.DEFAULT_RADIUS[shape]
    g = capi.Solution(shape, radius=d, elem_bytes=4)
    h = capi.Solution(shape, radius=d, elem_bytes=8)
    try:
        assert _layout(h) == _layout(g)
        assert [v.get_name() for v in h.get_vars()] == ["A"]
        assert h.get_var("A").info.halo_exchange_l1_norm == A.L1_NORM[shape]
    finally:
        g.close()
        h.close()


@pytest.mark.parametrize("shape,R,eb", [("3axis", 1, 4), ("cube", 8, 8), ("3plane", 5, 4)])
def test_plan_geometry_pads(shape, R, eb):
    s = capi.Solution(shape, radius=R, elem_bytes=eb)
    try:
        s.set_overall_domain_size_vec((40, 33, 70))
        s.plan_geometry()
        vi = s.get_var("A").info
        for i in range(1, vi.num_dims):
            dm = vi.dims[i]
            assert dm.left_pad >= R and dm.right_pad >= R and dm.left_halo == dm.right_halo == R
        z = vi.dims[vi.num_dims - 1]
        assert (z.left_pad * eb) % 128 == 0        # rows start on 128 bytes: the sweep's 16-byte TMA boxes
    finally:
        s.close()


def _lib_report(lib):
    so = os.path.join(ROOT, "yask_b200", "lib", f"libyask_kernel.{lib}.b200.so")
    assert os.path.exists(so), f"csrc/Makefile builds the {lib} API library"
    src = r'''
#include <cstdio>
#include "yask_kernel_api.hpp"
int main() {
    yask::yk_factory f;
    auto env = f.new_env();
    auto s = f.new_solution(env);
    printf("%s %d %d\n", s->get_name().c_str(), s->get_element_bytes(), int(s->get_var("A")->get_left_halo_size("x")));
    return 0;
}
'''
    with tempfile.TemporaryDirectory() as d:
        cpp, exe = os.path.join(d, "eb.cpp"), os.path.join(d, "eb")
        open(cpp, "w").write(src)
        subprocess.run(["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "yask_b200", "include"), cpp,
                        so, "-L" + os.path.join(ROOT, "yask_b200", "lib"), "-lyask_b200",
                        "-Wl,-rpath," + os.path.join(ROOT, "yask_b200", "lib"), "-o", exe], check=True)
        r = subprocess.run([exe], capture_output=True, text=True, timeout=60,
                           env={k: v for k, v in os.environ.items() if not k.startswith("YASK_B200_")})
    assert r.returncode == 0, r.stderr
    return r.stdout.split()


@pytest.mark.parametrize("lib,expect", [("3axis_r1", ["3axis", "4", "1"]), ("3axis_with_diags_r2", ["3axis_with_diags", "4", "2"]),
                                        ("3plane_r1", ["3plane", "4", "1"]), ("cube_r1_fp64", ["cube", "8", "1"]),
                                        ("cube", ["cube", "4", "2"])])
def test_library_suffix_parsing(lib, expect):
    assert _lib_report(lib) == expect


@pytest.mark.parametrize("shape,radius,elem_bytes", [("3axis", None, None), ("3axis", "1", None), ("cube", "3", "8"),
                                                     ("3plane", "8", "4")])
def test_python_module_radius_and_precision(shape, radius, elem_bytes):
    mod = os.path.join(ROOT, "yask_b200", "lib", "python", shape)
    assert os.path.isdir(mod), f"csrc/Makefile builds the {shape} Python module"
    code = r'''
import yask_kernel as yk
fac = yk.yk_factory()
s = fac.new_solution(fac.new_env())
print(s.get_name(), s.get_element_bytes(), s.get_var("A").get_left_halo_size("x"))
'''
    env = {k: v for k, v in os.environ.items() if k not in ("YASK_B200_RADIUS", "YASK_B200_ELEM_BYTES")}
    env.update(PYTHONPATH=mod, CUDA_VISIBLE_DEVICES="")
    if radius:
        env["YASK_B200_RADIUS"] = radius
    if elem_bytes:
        env["YASK_B200_ELEM_BYTES"] = elem_bytes
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120, env=env)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.split() == [shape, elem_bytes or "4", radius or str(A.DEFAULT_RADIUS[shape])]
