#!/usr/bin/env python
"""Generate the fixtures tests/golden/<shape>-r<r>*.npz and <shape>-fp64-r<r>*.npz of the four average-of-points stencils (3axis,
3axis_with_diags, 3plane, cube) from the UNMODIFIED reference.

The reference fixes radius and element size at build time; tests/golden/build_ref_avepts.sh builds each shape at radius 1, 2, 5
and 8 in fp32 and 2 and 8 in fp64 (real_bytes=8), in the default build and with -ffp-contract=off:

    oracle/build_ref.sh && tests/golden/build_ref_avepts.sh && python tests/golden/make_golden_avepts.py

One ragged box per build (y and z not multiples of the sweep's tile, z not a multiple of 4), 2 steps.  The fixtures are written by
make_golden.gen() in the same format as every other fixture.  Their stencil fields are <shape>_r<r> and <shape>_fp64_r<r>,
names no generated solution has, so the fixture sets of the other tests do not include them.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import oracle as O  # noqa: E402
from tests.golden.make_golden import RANGES, gen  # noqa: E402

SHAPES = ("3axis", "3axis_with_diags", "3plane", "cube")
FP32_RADII = (1, 2, 5, 8)
FP64_RADII = (2, 8)
N, STEPS, SEED = (8, 13, 37), 2, 2024


def main():
    missing = []
    for shape in SHAPES:
        for prec, radii in (("", FP32_RADII), ("fp64-", FP64_RADII)):
            for r in radii:
                stencil = f"{shape}_{prec.replace('-', '_')}r{r}"
                RANGES[stencil] = RANGES[shape]
                for tag in (f"{shape}-{prec}r{r}.avx512", f"{shape}-{prec}r{r}-strict.avx512"):
                    if not O.ref_available(tag):
                        missing.append(tag)
                        continue
                    gen(stencil, tag, N, STEPS, SEED)
    if missing:
        raise SystemExit("make_golden_avepts.py: reference builds missing (tests/golden/build_ref_avepts.sh): " + " ".join(missing))


if __name__ == "__main__":
    main()
