"""CPU: x-chunk planning of the iso3dfd sweep launches (yask_b200/csrc/yb_chunk_plan.h), a host-only header compiled with g++."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_sweep_chunk_plan(tmp_path):
    """tests/unit/chunk_plan_test.cpp: x chunks of the iso3dfd sweeps -- balanced, covering the box exactly, lx honoured within the
    bounds, and with the in-kernel signal at least R planes long with the boundary chunks first and the last one swept downwards."""
    exe = str(tmp_path / "chunk_plan_test")
    subprocess.run(["g++", "-std=c++17", "-Wall", os.path.join(ROOT, "tests", "unit", "chunk_plan_test.cpp"), "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.strip() == "OK", r.stdout + r.stderr
