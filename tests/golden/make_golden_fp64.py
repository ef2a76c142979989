#!/usr/bin/env python
"""Generate the double-precision iso3dfd fixtures tests/golden/iso3dfd-fp64-r<r>*.npz from the UNMODIFIED reference.

The reference fixes radius and element size at build time; tests/golden/build_ref_fp64.sh builds its iso3dfd with
real_bytes=8 at the radii of the hand-written fp64 sweep (1, 2, 4, 5, 6, 7), in the default build and with
-ffp-contract=off:

    oracle/build_ref.sh && tests/golden/build_ref_fp64.sh && python tests/golden/make_golden_fp64.py

Per radius and build: a small box over 3 steps, and a ragged one (y not a multiple of the 16-row tile, z over two 64-wide
fp64 tiles, x thinner than 4R from radius 3 up) over 2 steps; about 2 MB for all 24.  The fixtures are written by
make_golden.gen() in the same format as every other fixture.  Their stencil field is iso3dfd_fp64_r<r> (like the generated
fp64 radius-3 fixtures), so the fp32 iso3dfd fixture sets of the other tests do not include them.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import oracle as O  # noqa: E402
from tests.golden.make_golden import RANGES, gen  # noqa: E402

FP64_RADII = (1, 2, 4, 5, 6, 7)


def main():
    missing = []
    for r in FP64_RADII:
        RANGES[f"iso3dfd_fp64_r{r}"] = RANGES["iso3dfd"]
        for tag in (f"iso3dfd-fp64-r{r}.avx512", f"iso3dfd-fp64-r{r}-strict.avx512"):
            if not O.ref_available(tag):
                missing.append(tag)
                continue
            gen(f"iso3dfd_fp64_r{r}", tag, (12, 20, 40), 3, 1234)
            gen(f"iso3dfd_fp64_r{r}", tag, (9, 17, 70), 2, 77)
    if missing:
        raise SystemExit("make_golden_fp64.py: reference builds missing (tests/golden/build_ref_fp64.sh): " + " ".join(missing))


if __name__ == "__main__":
    main()
