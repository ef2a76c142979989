#!/bin/bash
# TEST INFRASTRUCTURE ONLY: fixture generation.
# Builds the UNMODIFIED reference's iso3dfd in double precision (real_bytes=8) at the radii the hand-written fp64 sweep
# serves (1, 2, 4, 5, 6, 7), in its default build and with -ffp-contract=off ("-strict"), plus oracle/ref_driver.cpp
# against each kernel library.  Tags: iso3dfd-fp64-r<r>[-strict].<arch>, named like the fp64 radius-3 build
# (iso3dfd-fp64-r3).  The outputs go where oracle/build_ref.sh puts its own (oracle/_ref/yask, git-ignored);
# make_golden_fp64.py then writes the tests/golden/iso3dfd-fp64-r<r>* fixtures:
#
#     oracle/build_ref.sh && tests/golden/build_ref_fp64.sh && python tests/golden/make_golden_fp64.py
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
    echo "build_ref_fp64.sh: no reference tree at $REF (set YASK_REFERENCE)" >&2
    exit 1
fi
if [ ! -x "$OUT/bin/yask_compiler.exe" ]; then
    echo "build_ref_fp64.sh: run oracle/build_ref.sh first (it builds the reference compiler)" >&2
    exit 1
fi
LOG=$ORACLE/_ref/build_fp64.log
: > "$LOG"

# suffix  extra-make-args
build_kernel() {
    local suf=$1; shift
    local tag="iso3dfd$suf.$ARCH"
    if [ ! -f "$OUT/lib/libyask_kernel.$tag.so" ] || [ ! -x "$OUT/bin/yask_kernel.$tag.exe" ]; then
        echo "[build_ref_fp64] kernel $tag"
        make -C "$REF/src/kernel" YASK_OUTPUT_DIR="$OUT" stencil=iso3dfd YK_STENCIL_SUFFIX=$suf arch=$ARCH \
            mpi=0 numa=0 real_bytes=8 -j$J "$@" default >> "$LOG" 2>&1
    fi
    if [ ! -x "$OUT/bin/ref_driver.$tag" ] || [ "$ORACLE/ref_driver.cpp" -nt "$OUT/bin/ref_driver.$tag" ]; then
        g++ -std=c++17 -O2 -fopenmp -I"$REF/include" "$ORACLE/ref_driver.cpp" \
            -L"$OUT/lib" -Wl,-rpath,'$ORIGIN/../lib' -lyask_kernel.$tag -lrt -o "$OUT/bin/ref_driver.$tag"
    fi
}

for r in 1 2 4 5 6 7; do
    build_kernel "-fp64-r$r"        radius=$r
    build_kernel "-fp64-r$r-strict" radius=$r EXTRA_YK_CXXFLAGS=-ffp-contract=off
done
strip --strip-debug "$OUT"/lib/libyask_kernel.iso3dfd-fp64-r*.so "$OUT"/bin/yask_kernel.iso3dfd-fp64-r*.exe \
    "$OUT"/bin/ref_driver.iso3dfd-fp64-r* 2>/dev/null || true
if [ "${KEEP_BUILD:-0}" != "1" ]; then rm -rf "$OUT/build"; fi
echo "[build_ref_fp64] done"
