#!/usr/bin/env python
"""Generate the iso3dfd_sponge fixtures tests/golden/iso3dfd_sponge-r<r>*.npz and iso3dfd_sponge-fp64-r<r>*.npz from the
UNMODIFIED reference.

The reference fixes radius and element size at build time; tests/golden/build_ref_sponge.sh builds its iso3dfd_sponge at
radius 2, 4 and 7 in fp32 and 3, 4 and 8 in fp64 (real_bytes=8), in the default build and with -ffp-contract=off:

    oracle/build_ref.sh && tests/golden/build_ref_sponge.sh && python tests/golden/make_golden_sponge.py

Per radius and build: a small box over 3 steps, and a ragged one (y not a multiple of the 16-row tile, z over two tiles of the
sweep -- 128 wide in fp32, 64 in fp64 -- x thinner than 4R from radius 3 up) over 2 steps.  The fixtures are written by
make_golden.gen() in the same format as every other fixture.  Their stencil fields are iso3dfd_sponge_r<r> and
iso3dfd_sponge_fp64_r<r>, names no generated solution has, so the fixture sets of the other tests do not include them.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import oracle as O  # noqa: E402
from tests.golden.make_golden import RANGES, gen  # noqa: E402

FP32_RADII = (2, 4, 7)
FP64_RADII = (3, 4, 8)


def main():
    missing = []
    for prec, radii, ragged in (("", FP32_RADII, (9, 17, 150)), ("fp64-", FP64_RADII, (9, 17, 70))):
        for r in radii:
            stencil = f"iso3dfd_sponge_{prec.replace('-', '_')}r{r}"
            RANGES[stencil] = RANGES["iso3dfd_sponge"]
            for tag in (f"iso3dfd_sponge-{prec}r{r}.avx512", f"iso3dfd_sponge-{prec}r{r}-strict.avx512"):
                if not O.ref_available(tag):
                    missing.append(tag)
                    continue
                gen(stencil, tag, (12, 20, 40), 3, 1234)
                gen(stencil, tag, ragged, 2, 77)
    if missing:
        raise SystemExit("make_golden_sponge.py: reference builds missing (tests/golden/build_ref_sponge.sh): " + " ".join(missing))


if __name__ == "__main__":
    main()
