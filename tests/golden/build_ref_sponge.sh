#!/bin/bash
# TEST INFRASTRUCTURE ONLY: fixture generation.
# Builds the UNMODIFIED reference's iso3dfd_sponge at some of the radii the hand-written sponge sweep serves -- fp32 at 2, 4 and 7,
# fp64 (real_bytes=8) at 3, 4 and 8 -- in its default build and with -ffp-contract=off ("-strict"), plus oracle/ref_driver.cpp
# against each kernel library.  Tags: iso3dfd_sponge-r<r>[-strict].<arch> and iso3dfd_sponge-fp64-r<r>[-strict].<arch>.  The
# outputs go where oracle/build_ref.sh puts its own (oracle/_ref/yask, git-ignored); make_golden_sponge.py then writes the
# tests/golden/iso3dfd_sponge-r<r>* and iso3dfd_sponge-fp64-r<r>* fixtures:
#
#     oracle/build_ref.sh && tests/golden/build_ref_sponge.sh && python tests/golden/make_golden_sponge.py
#
# Needs the reference tree (YASK_REFERENCE) and the reference compiler oracle/build_ref.sh builds into tools/_refc.
# 12 kernel builds, about 20 minutes.
set -e
REF=${YASK_REFERENCE:-/root/reference}
ROOT=$(cd "$(dirname "$0")/../.." && pwd)
ORACLE=$ROOT/oracle
OUT=$ORACLE/_ref/yask
ARCH=${1:-avx512}
J=${JOBS:-8}

if [ ! -d "$REF/src/kernel" ]; then
    echo "build_ref_sponge.sh: no reference tree at $REF (set YASK_REFERENCE)" >&2
    exit 1
fi
if [ ! -x "$OUT/bin/yask_compiler.exe" ]; then
    echo "build_ref_sponge.sh: run oracle/build_ref.sh first (it builds the reference compiler)" >&2
    exit 1
fi
LOG=$ORACLE/_ref/build_sponge.log
: > "$LOG"

# suffix  real_bytes  extra-make-args
build_kernel() {
    local suf=$1 rb=$2; shift 2
    local tag="iso3dfd_sponge$suf.$ARCH"
    if [ ! -f "$OUT/lib/libyask_kernel.$tag.so" ] || [ ! -x "$OUT/bin/yask_kernel.$tag.exe" ]; then
        echo "[build_ref_sponge] kernel $tag"
        make -C "$REF/src/kernel" YASK_OUTPUT_DIR="$OUT" stencil=iso3dfd_sponge YK_STENCIL_SUFFIX=$suf arch=$ARCH \
            mpi=0 numa=0 real_bytes=$rb -j$J "$@" default >> "$LOG" 2>&1
    fi
    if [ ! -x "$OUT/bin/ref_driver.$tag" ] || [ "$ORACLE/ref_driver.cpp" -nt "$OUT/bin/ref_driver.$tag" ]; then
        g++ -std=c++17 -O2 -fopenmp -I"$REF/include" "$ORACLE/ref_driver.cpp" \
            -L"$OUT/lib" -Wl,-rpath,'$ORIGIN/../lib' -lyask_kernel.$tag -lrt -o "$OUT/bin/ref_driver.$tag"
    fi
}

for r in 2 4 7; do
    build_kernel "-r$r"        4 radius=$r
    build_kernel "-r$r-strict" 4 radius=$r EXTRA_YK_CXXFLAGS=-ffp-contract=off
done
for r in 3 4 8; do
    build_kernel "-fp64-r$r"        8 radius=$r
    build_kernel "-fp64-r$r-strict" 8 radius=$r EXTRA_YK_CXXFLAGS=-ffp-contract=off
done
strip --strip-debug "$OUT"/lib/libyask_kernel.iso3dfd_sponge-*r*.so "$OUT"/bin/yask_kernel.iso3dfd_sponge-*r*.exe \
    "$OUT"/bin/ref_driver.iso3dfd_sponge-*r* 2>/dev/null || true
if [ "${KEEP_BUILD:-0}" != "1" ]; then rm -rf "$OUT/build"; fi
echo "[build_ref_sponge] done"
