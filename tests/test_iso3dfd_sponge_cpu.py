"""CPU: iso3dfd_sponge at any radius in fp32 and fp64.

  * the sponge oracle (tests/sponge_oracle.py) is bit-exact against the generated restatements of the reference's own sponge
    builds (fp32 radius 8, fp64 radius 6) in both contraction modes, and against the unmodified reference built at other radii
    (tests/golden/iso3dfd_sponge-r<r>*.npz, iso3dfd_sponge-fp64-r<r>*.npz) in its default build and with -ffp-contract=off;
  * without a device, the registry creates iso3dfd_sponge at radius 1..8 in both precisions and refuses radius 9, and the
    hand-written form declares the generated form's vars;
  * the iso3dfd_sponge_r4 and iso3dfd_sponge_r4_fp64 C++ API libraries report their solution and element size, and the
    iso3dfd_sponge Python module takes its radius and precision from YASK_B200_RADIUS / YASK_B200_ELEM_BYTES.
"""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import contract_mode_of, golden_cases, load_golden, regen_inputs
from tests.sponge_oracle import iso3dfd_sponge_run
from yask_b200 import capi
from yask_b200.synth import hash_field, var_salt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FP32_RADII, FP64_RADII = (2, 4, 7), (3, 4, 8)
CASES = [p for r in FP32_RADII for p in golden_cases(f"iso3dfd_sponge-r{r}")] + \
        [p for r in FP64_RADII for p in golden_cases(f"iso3dfd_sponge-fp64-r{r}")]


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def sponge_inputs(n, seed, R, dt):
    ins = {("p", t): hash_field(seed, var_salt("p", t), (-R,) * 3, [i + 2 * R for i in n], -1, 1, dt) for t in (0, 1)}
    ins[("v", 0)] = hash_field(seed, var_salt("v", 0), (0, 0, 0), n, 0.05, 0.3, dt)
    for d, name in enumerate(("cr_x", "cr_y", "cr_z")):
        ins[(name, 0)] = hash_field(seed, var_salt(name, 0), (0,), (n[d],), 0.92, 1.0, dt)
    return ins


def run_oracle(ins, R, steps, mode):
    return iso3dfd_sponge_run(ins[("p", 0)], ins[("p", 1)], ins[("v", 0)], ins[("cr_x", 0)], ins[("cr_y", 0)], ins[("cr_z", 0)],
                              R, steps, mode)


@pytest.mark.parametrize("contract", [0, 1])
@pytest.mark.parametrize("stencil,R,dt,n", [("iso3dfd_sponge", 8, np.float32, (13, 9, 35)),
                                            ("iso3dfd_sponge", 8, np.float32, (21, 17, 70)),
                                            ("iso3dfd_sponge_fp64_r6", 6, np.float64, (13, 9, 35)),
                                            ("iso3dfd_sponge_fp64_r6", 6, np.float64, (17, 23, 67))])
def test_oracle_matches_generated_restatement(stencil, R, dt, n, contract):
    steps = 3
    ins = sponge_inputs(n, 40 + R, R, dt)
    gen = O.gen_run(stencil, n, steps, ins, contract=contract)
    tl, ref = gen["p"]
    # generated contraction 1 is the reference's default build: the oracle's mode 2
    got = run_oracle(ins, R, steps, 2 if contract else 0)
    assert tl == steps and got.dtype == ref.dtype == dt
    assert np.array_equal(_bits(got[R:-R, R:-R, R:-R]), _bits(ref[R:-R, R:-R, R:-R]))
    assert np.array_equal(_bits(got), _bits(ref))      # halo cells: p(t-1)'s, untouched


def test_fixtures_cover_every_radius_and_both_builds():
    tags = {load_golden(p)[0]["ref_tag"] for p in CASES}
    assert tags == {f"iso3dfd_sponge-r{r}{s}.avx512" for r in FP32_RADII for s in ("", "-strict")} | \
                   {f"iso3dfd_sponge-fp64-r{r}{s}.avx512" for r in FP64_RADII for s in ("", "-strict")}
    assert len(CASES) == 2 * len(tags)     # a small box over 3 steps and a ragged one over 2


def radius_of(meta):
    return int(meta["ref_tag"].split("-r")[1].split("-")[0].split(".")[0])


@pytest.mark.parametrize("path", CASES, ids=[os.path.basename(p)[:-4] for p in CASES])
def test_oracle_bit_exact_vs_reference(path):
    meta, arrays = load_golden(path)
    R = radius_of(meta)
    ins = regen_inputs(meta)
    mode = contract_mode_of(meta["ref_tag"])
    ref = arrays[f"p.t{meta['vars']['p']['steps'][1]}"]
    got = run_oracle(ins, R, meta["steps"], mode)[R:-R, R:-R, R:-R]
    assert got.dtype == ref.dtype and got.shape == ref.shape
    assert np.array_equal(_bits(got), _bits(ref))
    # the other contraction mode is not what this build does (guards the fixture labels)
    other = run_oracle(ins, R, meta["steps"], 2 - mode)[R:-R, R:-R, R:-R]
    assert not np.array_equal(_bits(other), _bits(ref))


@pytest.mark.parametrize("elem_bytes", [4, 8])
@pytest.mark.parametrize("radius", range(1, 9))
def test_solution_created_without_device(radius, elem_bytes):
    s = capi.Solution("iso3dfd_sponge", radius=radius, elem_bytes=elem_bytes)
    try:
        assert s.get_element_bytes() == elem_bytes
        assert s.get_var("p").info.dims[1].left_halo == radius
    finally:
        s.close()


@pytest.mark.parametrize("elem_bytes", [4, 8])
def test_radius_above_8_refused(elem_bytes):
    with pytest.raises(capi.YaskError, match="radius 9 > 8"):
        capi.Solution("iso3dfd_sponge", radius=9, elem_bytes=elem_bytes)


def _layout(s):
    out = []
    for v in s.get_vars():
        vi = v.info
        out.append((vi.name, vi.step_alloc, vi.is_output, vi.halo_exchange_l1_norm,
                    [(vi.dims[i].name, vi.dims[i].kind, vi.dims[i].left_halo, vi.dims[i].right_halo) for i in range(vi.num_dims)]))
    return out


# the hand-written form at the radius of a generated form (other precision) declares the same vars, in the same order
@pytest.mark.parametrize("hand,generated", [((8, 8), (8, 4)), ((6, 4), (6, 8))])
def test_vars_equal_generated(hand, generated):
    h = capi.Solution("iso3dfd_sponge", radius=hand[0], elem_bytes=hand[1])
    g = capi.Solution("iso3dfd_sponge", radius=generated[0], elem_bytes=generated[1])
    try:
        assert _layout(h) == _layout(g)
        assert [v.get_name() for v in h.get_vars()] == ["p", "v", "cr_x", "cr_y", "cr_z"]
    finally:
        h.close()
        g.close()


@pytest.mark.parametrize("lib,expect", [("iso3dfd_sponge_r4", ["iso3dfd_sponge", "4", "4"]),
                                        ("iso3dfd_sponge_r4_fp64", ["iso3dfd_sponge", "8", "4"])])
def test_library_reports_solution(lib, expect):
    so = os.path.join(ROOT, "yask_b200", "lib", f"libyask_kernel.{lib}.b200.so")
    assert os.path.exists(so), f"csrc/Makefile builds the {lib} API library"
    src = r'''
#include <cstdio>
#include "yask_kernel_api.hpp"
int main() {
    yask::yk_factory f;
    auto env = f.new_env();
    auto s = f.new_solution(env);
    auto p = s->get_var("p");
    printf("%s %d %d\n", s->get_name().c_str(), s->get_element_bytes(), int(p->get_left_halo_size("x")));
    return 0;
}
'''
    with tempfile.TemporaryDirectory() as d:
        cpp, exe = os.path.join(d, "eb.cpp"), os.path.join(d, "eb")
        open(cpp, "w").write(src)
        subprocess.run(["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "yask_b200", "include"), cpp,
                        so, "-L" + os.path.join(ROOT, "yask_b200", "lib"), "-lyask_b200",
                        "-Wl,-rpath," + os.path.join(ROOT, "yask_b200", "lib"), "-o", exe], check=True)
        r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stderr
    assert r.stdout.split() == expect


# the Python module of the iso3dfd_sponge library: YASK_B200_RADIUS / YASK_B200_ELEM_BYTES select the radius and precision, as
# for the C++ library it wraps
@pytest.mark.parametrize("radius,elem_bytes", [(None, None), ("4", None), ("3", "8")])
def test_python_module_radius_and_precision(radius, elem_bytes):
    mod = os.path.join(ROOT, "yask_b200", "lib", "python", "iso3dfd_sponge")
    assert os.path.isdir(mod), "csrc/Makefile builds the iso3dfd_sponge Python module"
    code = r'''
import yask_kernel as yk
fac = yk.yk_factory()
s = fac.new_solution(fac.new_env())
print(s.get_name(), s.get_element_bytes(), s.get_var("p").get_left_halo_size("x"), [v.get_name() for v in s.get_vars()])
'''
    env = {k: v for k, v in os.environ.items() if k not in ("YASK_B200_RADIUS", "YASK_B200_ELEM_BYTES")}
    env.update(PYTHONPATH=mod, CUDA_VISIBLE_DEVICES="")
    if radius:
        env["YASK_B200_RADIUS"] = radius
    if elem_bytes:
        env["YASK_B200_ELEM_BYTES"] = elem_bytes
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120, env=env)
    assert r.returncode == 0, r.stdout + r.stderr
    tok = r.stdout.split()
    assert tok[:3] == ["iso3dfd_sponge", elem_bytes or "4", radius or "8"]
    assert r.stdout.strip().endswith("['p', 'v', 'cr_x', 'cr_y', 'cr_z']")
