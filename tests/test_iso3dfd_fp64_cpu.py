"""CPU: double-precision iso3dfd at the radii of the hand-written fp64 sweep (1, 2, 4, 5, 6, 7).

  * the oracle (oracle/yask_oracle.c, float64) is bit-exact against the unmodified reference built with real_bytes=8 at
    each radius, in its default build and with -ffp-contract=off (tests/golden/iso3dfd-fp64-r<r>*.npz);
  * without a device, the registry creates fp64 iso3dfd at radius 1..8 and refuses radius 9;
  * the iso3dfd_r4_fp64 C++ API library reports 8-byte elements.
"""
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import contract_mode_of, golden_cases, load_golden, regen_inputs
from yask_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FP64_RADII = (1, 2, 4, 5, 6, 7)
CASES = [p for r in FP64_RADII for p in golden_cases(f"iso3dfd-fp64-r{r}")]


def _radius_of(meta):
    return int(meta["ref_tag"].split("-r")[1].split("-")[0].split(".")[0])


def test_fixtures_cover_every_radius_and_both_builds():
    tags = {load_golden(p)[0]["ref_tag"] for p in CASES}
    assert tags == {f"iso3dfd-fp64-r{r}{s}.avx512" for r in FP64_RADII for s in ("", "-strict")}
    assert len(CASES) == 2 * len(tags)     # a small box over 3 steps and a ragged one over 2


@pytest.mark.parametrize("path", CASES, ids=[os.path.basename(p)[:-4] for p in CASES])
def test_oracle_bit_exact_vs_reference_fp64(path):
    meta, arrays = load_golden(path)
    R = _radius_of(meta)
    ins = regen_inputs(meta)
    assert ins[("p", 0)].dtype == np.float64
    mode = contract_mode_of(meta["ref_tag"])
    out = O.iso3dfd_run(ins[("p", 0)], ins[("p", 1)], ins[("v", 0)], R, meta["steps"], mode)
    ref = arrays[f"p.t{meta['vars']['p']['steps'][1]}"]
    got = out[R:-R, R:-R, R:-R]
    assert got.dtype == ref.dtype == np.float64 and got.shape == ref.shape
    assert np.array_equal(got.view(np.uint64), ref.view(np.uint64))
    # the other contraction mode is not what this build does (guards the fixture labels)
    other = O.iso3dfd_run(ins[("p", 0)], ins[("p", 1)], ins[("v", 0)], R, meta["steps"], 2 - mode)
    assert not np.array_equal(other[R:-R, R:-R, R:-R].view(np.uint64), ref.view(np.uint64))


@pytest.mark.parametrize("radius", range(1, 9))
def test_fp64_solution_created_without_device(radius):
    s = capi.Solution("iso3dfd", radius=radius, elem_bytes=8)
    try:
        assert s.get_element_bytes() == 8
    finally:
        s.close()


def test_fp64_radius_above_8_refused():
    with pytest.raises(Exception):
        capi.Solution("iso3dfd", radius=9, elem_bytes=8)


def test_fp64_library_reports_8_byte_elements():
    lib = os.path.join(ROOT, "yask_b200", "lib", "libyask_kernel.iso3dfd_r4_fp64.b200.so")
    assert os.path.exists(lib), "csrc/Makefile builds the iso3dfd_r4_fp64 API library"
    src = r'''
#include <cstdio>
#include "yask_kernel_api.hpp"
int main() {
    yask::yk_factory f;
    auto env = f.new_env();
    auto s = f.new_solution(env);
    printf("%s %d\n", s->get_name().c_str(), s->get_element_bytes());
    return 0;
}
'''
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        cpp, exe = os.path.join(d, "eb.cpp"), os.path.join(d, "eb")
        open(cpp, "w").write(src)
        subprocess.run(["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "yask_b200", "include"), cpp,
                        lib, "-L" + os.path.join(ROOT, "yask_b200", "lib"), "-lyask_b200",
                        "-Wl,-rpath," + os.path.join(ROOT, "yask_b200", "lib"), "-o", exe], check=True)
        r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stderr
    assert r.stdout.split() == ["iso3dfd", "8"]
