#!/bin/bash
# TEST INFRASTRUCTURE ONLY: fixture generation.
# Builds the UNMODIFIED reference's four "simple" stencils (3axis, 3axis_with_diags, 3plane, cube) at radii the hand-written
# average-of-points sweep serves -- fp32 at 1, 2, 5 and 8, fp64 (real_bytes=8) at 2 and 8 -- in the default build and with
# -ffp-contract=off ("-strict"), plus oracle/ref_driver.cpp against each kernel library.  Tags: <shape>-r<r>[-strict].<arch> and
# <shape>-fp64-r<r>[-strict].<arch>.  The outputs go where oracle/build_ref.sh puts its own (oracle/_ref/yask, git-ignored);
# make_golden_avepts.py then writes the tests/golden/<shape>-r<r>* and <shape>-fp64-r<r>* fixtures:
#
#     oracle/build_ref.sh && tests/golden/build_ref_avepts.sh && python tests/golden/make_golden_avepts.py
#
# Needs the reference tree (YASK_REFERENCE) and the reference compiler oracle/build_ref.sh builds into tools/_refc.
# 48 kernel builds, PAR of them at a time (default 6).
set -e
REF=${YASK_REFERENCE:-/root/reference}
ROOT=$(cd "$(dirname "$0")/../.." && pwd)
ORACLE=$ROOT/oracle
OUT=$ORACLE/_ref/yask
ARCH=${1:-avx512}
J=${JOBS:-2}
PAR=${PAR:-6}

if [ ! -d "$REF/src/kernel" ]; then
    echo "build_ref_avepts.sh: no reference tree at $REF (set YASK_REFERENCE)" >&2
    exit 1
fi
if [ ! -x "$OUT/bin/yask_compiler.exe" ]; then
    echo "build_ref_avepts.sh: run oracle/build_ref.sh first (it builds the reference compiler)" >&2
    exit 1
fi
mkdir -p "$ORACLE/_ref/avepts_logs"

# shape  suffix  real_bytes  extra-make-args
build_kernel() {
    local st=$1 suf=$2 rb=$3; shift 3
    local tag="$st$suf.$ARCH"
    local log="$ORACLE/_ref/avepts_logs/$tag.log"
    if [ ! -f "$OUT/lib/libyask_kernel.$tag.so" ] || [ ! -x "$OUT/bin/yask_kernel.$tag.exe" ]; then
        echo "[build_ref_avepts] kernel $tag"
        make -C "$REF/src/kernel" YASK_OUTPUT_DIR="$OUT" stencil=$st YK_STENCIL_SUFFIX=$suf \
            arch=$ARCH mpi=0 numa=0 real_bytes=$rb -j$J "$@" default > "$log" 2>&1
    fi
    if [ ! -x "$OUT/bin/ref_driver.$tag" ] || [ "$ORACLE/ref_driver.cpp" -nt "$OUT/bin/ref_driver.$tag" ]; then
        g++ -std=c++17 -O2 -fopenmp -I"$REF/include" "$ORACLE/ref_driver.cpp" \
            -L"$OUT/lib" -Wl,-rpath,'$ORIGIN/../lib' -lyask_kernel.$tag -lrt -o "$OUT/bin/ref_driver.$tag"
    fi
}
export -f build_kernel
export REF OUT ORACLE ARCH J

# The first build alone: it also compiles the objects every stencil shares (per arch), which the parallel builds then find
# up to date.  The others have separate per-stencil object trees.
build_kernel 3axis -r1 4 radius=1
{
    for st in 3axis 3axis_with_diags 3plane cube; do
        for r in 1 2 5 8; do
            echo "$st -r$r 4 radius=$r"
            echo "$st -r$r-strict 4 radius=$r EXTRA_YK_CXXFLAGS=-ffp-contract=off"
        done
        for r in 2 8; do
            echo "$st -fp64-r$r 8 radius=$r"
            echo "$st -fp64-r$r-strict 8 radius=$r EXTRA_YK_CXXFLAGS=-ffp-contract=off"
        done
    done
} | xargs -P "$PAR" -L 1 bash -c 'build_kernel "$@"' _
strip --strip-debug "$OUT"/lib/libyask_kernel.{3axis,3axis_with_diags,3plane,cube}-*r*.so \
    "$OUT"/bin/yask_kernel.{3axis,3axis_with_diags,3plane,cube}-*r*.exe "$OUT"/bin/ref_driver.{3axis,3axis_with_diags,3plane,cube}-*r* 2>/dev/null || true
if [ "${KEEP_BUILD:-0}" != "1" ]; then rm -rf "$OUT/build"; fi
echo "[build_ref_avepts] done"
