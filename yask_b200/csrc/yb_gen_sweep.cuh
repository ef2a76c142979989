// "Sweep" form of the emitter-generated kernels: TMA-staged shared-memory planes with the same 2.5-D march along x as the
// hand-written iso3dfd kernel, for multi-var stencils (awp_elastic, ssg, ...).  The kernels themselves are written by
// yask_b200/emitter/yask_cuda_emit.py (gen/<name>.gen.cuh); this header holds what they share.
//
// A CTA owns a (TY rows x TZ z) tile, TZ = 32 vectors of VW = 16 B / sizeof(T) elements, and marches over a chunk of x
// planes.  Warp-specialised like the iso3dfd kernel:
//   * a producer warpgroup (one elected lane, registers handed back with setmaxnreg.dec) streams every full-rank var the part
//     reads: each is a TMA *stream* (cp.async.bulk.tensor.3d, box = tile + the stream's y/z reach, first element 16-byte
//     aligned) into its own shared-memory ring of (x reach + PF) plane slots, PF planes ahead of first use.  All loads first
//     needed at sweep iteration j complete on full[j mod (PF+1)]; the slots that iteration j + PF + 1 overwrites are released
//     by done[j mod (PF+1)], on which every consumer warp arrives -- no __syncthreads in the loop.
//   * a var whose x reach is long (ssg: 8 planes) and whose x neighbours are only read at the point's own (y,z) is split
//     into two streams: the current plane with its y/z halo, and a ring of halo-less planes for the x neighbours;
//   * NW consumer warps (setmaxnreg.inc), one warp per tile row: a thread computes VW consecutive z points of its row from
//     128-bit shared-memory loads (z neighbours of the VW points share their vectors), evaluates the part's statement list
//     (same order, same rounding as the direct kernel) and stores 128-bit vectors straight to HBM;
//   * lower-rank vars (1-D sponge arrays, scalars) are read from global memory, hoisted out of the sweep where they do not
//     depend on x.
#pragma once
#include "yb_gen.cuh"
#include "yb_ptx.cuh"

namespace yb { namespace gen {

struct GenSweepParams {
    GenParams g;                               // box, pointers and strides as for the direct kernel
    const CUtensorMap* maps;                   // device array, one per stream: 3-D (z, y, x) view of the var's step slot,
                                               // box (pz, rows, 1); built once per slot combination and cached (yb_gen.cu)
    int px, py, pz;                            // left pads of the shared geometry (tensor coordinate of local index 0)
    int lx, nchunks;                           // planes per sweep chunk, chunks along x
    int nzb, nyb;                              // tiles along z and y
};

// (GenSweepFn, GenSweepStream and GenSweep -- the host-side description filled in by the generated describe() -- are
// declared in yb_gen.cuh next to GenPart.)

#define GEN_SW_FN1(k, M) reinterpret_cast<yb::gen::GenSweepFn>(static_cast<void (*)(const yb::gen::GenSweepParams)>(k<M>))
#define GEN_SW_FN(k, M) yb::gen::GenFnPair<yb::gen::GenSweepFn>{GEN_SW_FN1(k, M), GEN_SW_FN1(k, (M) | yb::gen::GEN_WIDE)}

#ifdef __CUDACC__
// The VW consecutive points of a thread: a 16-byte vector (float x 4, double x 2) or half of one (float x 2, double x 1).
template <typename T, int VW> struct SwVec;
template <> struct SwVec<float, 4> {
    static __device__ __forceinline__ void lds(uint32_t addr, float* o) {
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(o[0]), "=f"(o[1]), "=f"(o[2]), "=f"(o[3]) : "r"(addr));
    }
    static __device__ __forceinline__ void stg(float* p, const float* v) {
        asm volatile("st.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v[0]), "f"(v[1]), "f"(v[2]), "f"(v[3]) : "memory");
    }
};
template <> struct SwVec<float, 2> {
    static __device__ __forceinline__ void lds(uint32_t addr, float* o) {
        asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(o[0]), "=f"(o[1]) : "r"(addr));
    }
    static __device__ __forceinline__ void stg(float* p, const float* v) {
        asm volatile("st.global.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(v[0]), "f"(v[1]) : "memory");
    }
};
template <> struct SwVec<double, 2> {
    static __device__ __forceinline__ void lds(uint32_t addr, double* o) {
        asm volatile("ld.shared.v2.f64 {%0, %1}, [%2];" : "=d"(o[0]), "=d"(o[1]) : "r"(addr));
    }
    static __device__ __forceinline__ void stg(double* p, const double* v) {
        asm volatile("st.global.v2.f64 [%0], {%1, %2};" ::"l"(p), "d"(v[0]), "d"(v[1]) : "memory");
    }
};
template <> struct SwVec<double, 1> {
    static __device__ __forceinline__ void lds(uint32_t addr, double* o) {
        asm volatile("ld.shared.f64 %0, [%1];" : "=d"(o[0]) : "r"(addr));
    }
    static __device__ __forceinline__ void stg(double* p, const double* v) {
        asm volatile("st.global.f64 [%0], %1;" ::"l"(p), "d"(v[0]) : "memory");
    }
};

// position `ahead` further along a ring of `size` (c and ahead < size; all three in the same unit: slots or bytes)
__device__ __forceinline__ uint32_t sw_wrap(uint32_t c, uint32_t ahead, uint32_t size) {
    const uint32_t u = c + ahead;
    return u >= size ? u - size : u;
}

// Producer side: the loads of stream k first needed at sweep iteration j (j == 0: its whole x reach; j > 0: the newest plane).
#define SW_ISSUE(k, OFF, SLOT, NS, XL, XR, YL, ZL)                                                                     \
    if (j == 0) {                                                                                                      \
        for (int dx = (XL); dx <= (XR); dx++)                                                                          \
            tma_load_3d(sw_smem + (OFF) + (dx - (XL)) * (SLOT), &SP.maps[k], bar, SP.pz + z0 + (ZL), SP.py + y0_ + (YL), \
                        SP.px + xs + dx);                                                                              \
    } else {                                                                                                           \
        tma_load_3d(sw_smem + (OFF) + ((j + (XR) - (XL)) % (NS)) * (SLOT), &SP.maps[k], bar, SP.pz + z0 + (ZL),         \
                    SP.py + y0_ + (YL), SP.px + xs + j + (XR));                                                        \
    }
#endif

} }  // namespace yb::gen
