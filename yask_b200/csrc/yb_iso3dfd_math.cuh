// iso3dfd point arithmetic, shared by every iso3dfd kernel (yb_iso3dfd.cuh, yb_iso3dfd_tt.cuh), in the element type E
// (float or double).
//
// Equation and association order: /root/reference/src/stencils/Iso3dfdStencil.cpp:63-137 (get_next_p):
//   acc = p*c0;  r=1..R: acc += (((((p[x-r]+p[x+r])+p[y-r])+p[y+r])+p[z-r])+p[z+r]) * c_r
//   p(t+1) = ((2*p) - p(t-1)) + acc*v
// FP modes: 0 strict IEEE mul/add, 1 canonical FMA, 2 = the FMA pattern GCC emits for the reference's default build.
// The pattern is the same in both precisions (the reference's fp64 build is the same source with real_bytes=8).
//
// YB_DEVFN is `__device__ __forceinline__` in the product build.  The CTA emulator of the test suite
// (tests/emul/tt_emul.cpp) compiles this header with g++, defines YB_DEVFN as `static inline` and supplies the
// rounded-arithmetic intrinsics of the fp32 path as plain C functions (built with -ffp-contract=off); the fp64 branches
// below are discarded there, so they need no host counterparts.
#pragma once
#ifndef YB_DEVFN
#define YB_DEVFN __device__ __forceinline__
#endif

namespace yb {

template <class E>
YB_DEVFN E iso_add(E a, E b) {
    if constexpr (sizeof(E) == 8) return __dadd_rn(a, b); else return __fadd_rn(a, b);
}
template <class E>
YB_DEVFN E iso_mul(E a, E b) {
    if constexpr (sizeof(E) == 8) return __dmul_rn(a, b); else return __fmul_rn(a, b);
}
template <class E>
YB_DEVFN E iso_fma(E a, E b, E c) {
    if constexpr (sizeof(E) == 8) return __fma_rn(a, b, c); else return __fmaf_rn(a, b, c);
}

template <int MODE, class E>
YB_DEVFN E iso_group(E acc, E pc, E c0, E cr, E xm, E xp, E ym, E yp, E zm, E zp, bool first) {
    E s = iso_add(xm, xp);
    s = iso_add(s, ym);
    s = iso_add(s, yp);
    s = iso_add(s, zm);
    s = iso_add(s, zp);
    if (MODE == 0) {
        if (first) acc = iso_mul(pc, c0);
        return iso_add(acc, iso_mul(s, cr));
    } else if (MODE == 1) {
        if (first) acc = iso_mul(pc, c0);
        return iso_fma(s, cr, acc);
    } else {
        if (first) return iso_fma(pc, c0, iso_mul(s, cr));
        return iso_fma(s, cr, acc);
    }
}

template <int MODE, class E>
YB_DEVFN E iso_final(E acc, E pc, E prev, E v) {
    // 2*p is exact, so fma(2,p,-prev) == round((2*p) - prev): one instruction, same bits.
    E lhs = iso_fma(E(2), pc, -prev);
    if (MODE == 0) return iso_add(lhs, iso_mul(acc, v));
    return iso_fma(acc, v, lhs);
}

}  // namespace yb
