// A box of var storage walked as a dense array: the dense index of a point maps to its element offset in a step slot.  Shared by
// the slice copies, fills and reductions (yb_fill.cu) and the slice recorders (yb_slices.cu), whose decimated boxes are the same
// walk with each storage stride multiplied by the box stride.
#pragma once

namespace yb {

// Dims right-aligned in the 4 entries: n[3] is the innermost (dense fastest) dim, n[i] = 1 and vs[i] = 0 for missing ones.
struct BoxDev {
    int nd;
    long long n[4];        // extents
    long long vs[4];       // storage element stride of one step of the box in each dim
    long long off;         // element offset of the box origin
    long long total;       // n[0] * n[1] * n[2] * n[3]
};

// dense linear index -> storage element offset; also returns per-dim coordinates
__device__ __forceinline__ long long box_offset(const BoxDev& b, long long lin, long long* coord) {
    long long o = b.off;
#pragma unroll
    for (int d = 3; d >= 0; d--) {
        long long c = lin % b.n[d];
        lin /= b.n[d];
        coord[d] = c;
        o += c * b.vs[d];
    }
    return o;
}

}  // namespace yb
