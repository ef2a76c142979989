// Support for emitter-generated stencil kernels (yask_b200/emitter/yask_cuda_emit.py).
// Host side: the tables a generated file fills in (what the reference's generated context ctor encodes,
// /root/reference/src/compiler/lib/YaskKernel.cpp:730-).  Device side: the statement vocabulary
// (RD/WR/C/ADD/SUB/MUL/DIV) the generated kernels are written in.
#pragma once
#include <cuda_runtime.h>

#include <string>
#include <type_traits>
#include <vector>

namespace yb { namespace gen {

constexpr int GEN_MAX_ACC = 96;   // distinct (var, step-offset) pairs one part may touch
// CTA = GEN_BZ x GEN_BY x GEN_BX points (z fastest): neighbouring rows/planes of a point are computed by
// the same CTA, so their reads of shared neighbours hit L1 instead of going back to L2.
#ifndef YB_GEN_BZ
#define YB_GEN_BZ 128
#define YB_GEN_BY 1
#define YB_GEN_BX 1
#endif
constexpr int GEN_BZ = YB_GEN_BZ, GEN_BY = YB_GEN_BY, GEN_BX = YB_GEN_BX;
// Each thread computes several points (rows y, y + GEN_BY, ...): the unrolled bodies are independent, so the
// compiler overlaps their loads -- the kernels are load-latency bound.  4 rows per thread for fp32, 2 for fp64 (4 rows of fp64
// need more registers and lower the occupancy).
__host__ __device__ constexpr int gen_np(int elem_bytes) { return elem_bytes == 4 ? 4 : 2; }
constexpr int GEN_BLOCK = GEN_BZ * GEN_BY * GEN_BX;

struct GenParams {
    int xb, xe, yb, ye, zb, ze;              // box to compute, rank-local domain coordinates
    void* ptr[GEN_MAX_ACC];                  // element (0,0,0) of the var's step slot for each access
    long long sx[GEN_MAX_ACC], sy[GEN_MAX_ACC], sz[GEN_MAX_ACC];   // element strides (0 where the var lacks the dim)
    // All vars that span every domain dim share ONE padded geometry (the engine pads them to the solution's
    // largest halo), so their neighbour offsets dx*SX + dy*SY + dz are computed once and shared by all vars.
    int SX, SY;
    // sub-domain conditions are written over GLOBAL indices: rank offset and overall first/last index per dim
    long long off[3], gfirst[3], glast[3];
    // L2 prefetch (option gen_pf): the CTA asks L2 for the lines of its own (y,z) tile `pfd` planes ahead in x of
    // every full-rank input var, so that the demand loads of the CTA that computes that plane find them in L2.
    int npf, pfd;
    unsigned char pf[GEN_MAX_ACC];
    // CTA order (1-D grid): z blocks fastest, then the y blocks of one y CHUNK, then x, then the next chunk -- the
    // planes x-h..x+h of a chunk (all vars) stay L2-resident while the sweep moves along x, so every element comes
    // from DRAM once even when whole x planes of all vars would not fit in L2 (ssg fp64 512^3: 8 planes x 12 vars
    // x 2 MB).  nzb/nyb/nxb = number of blocks per dim, ychunk = y blocks per chunk.
    int nzb, nyb, nxb, ychunk;
    long long t;   // step index the part is evaluated at (step conditions, IF_STEP)
};

typedef void (*GenKernelFn)(const GenParams);
// Generated kernels come in two addressing forms (template argument MODE | GEN_WIDE): 32-bit element positions, and 64-bit ones
// for slots of 2^31 elements or more.  The 32-bit form is what most sizes run: in the direct kernels the 64-bit one keeps a
// 64-bit base per var live (up to 44 more registers in the kernels of many-var parts), in the sweep kernels it costs the output
// stores an instruction (awp_elastic 0.5 % at 512^3).  yb_gen.cu picks the form from the slots' size.
constexpr int GEN_WIDE = 2;
template <typename F> struct GenFnPair {
    F narrow = nullptr, wide = nullptr;
    F pick(bool w) const { return w ? wide : narrow; }
};
typedef GenFnPair<GenKernelFn> GenKernelPair;

// Sweep variant (yb_gen_sweep.cuh): host-side description of one part's TMA streams; empty when the part has none.
struct GenSweepParams;
typedef void (*GenSweepFn)(const GenSweepParams);
struct GenSweepStream { int acc, xl, xr, yl, yr, zl, zr, rows, pz, slot_bytes, ns, off; };
struct GenSweep {
    GenFnPair<GenSweepFn> fn[2][2];   // [fp64?][mode]; only the solution's element type is emitted
    int ty = 0, tz = 0, threads = 0, occ = 1, smem = 0;               // tile rows x z points, CTA size, CTAs per SM, dynamic smem
    std::vector<GenSweepStream> streams;
};

struct GenVar {
    const char* name;
    std::vector<const char*> dims;   // declared order, step dim first if any
    int alloc_t;
    bool is_output;
    int l1_norm;
    std::vector<int> halo_l, halo_r; // per solution domain dim
    std::vector<int> misc_first, misc_size;   // per declared dim: index range of misc dims (0 size otherwise)
    bool is_scratch = false;         // engine-internal temporary (MAKE_SCRATCH_VAR): not visible through the API
};
struct GenAccess { int var, toff; int misc[2]; };   // misc: constant indices of the var's misc dims, in declared order
struct GenPart {
    const char* name;
    int fp_ops, reads, writes;
    std::vector<GenAccess> acc;
    std::vector<int> outs;           // indices into acc of the written accesses
    GenKernelPair fn[2][2];          // [fp64?][mode: 0 strict, 1 fused]
    // Launch-box bounds derived from the part's sub-domain condition, per domain dim: global index range
    // [lo, hi] with each end = offset relative to 0 / first / last overall index (kind 0/1/2), kind -1 = open.
    struct Bound { int lo_kind, lo_off, hi_kind, hi_off; } bound[3];
    // Scratch part: writes scratch vars over the launch box EXPANDED by the write halo (per kernel slot x,y,z), before
    // the parts that read them (/root/reference/src/kernel/lib/stencil_calc.cpp:128-137, setup.cpp:1182-1228).
    bool is_scratch = false;
    bool conditional = false;        // has a sub-domain or step condition (scratch outputs are zeroed first)
    int wh_l[3] = {0, 0, 0}, wh_r[3] = {0, 0, 0};
    GenSweep sweep;                  // TMA-staged variant of the same statements, when the emitter could build one
};
struct GenStage { const char* name; std::vector<GenPart> parts; };
struct GenStencil {
    std::string name, step_dim;
    int elem_bytes = 4;
    std::vector<std::string> domain_dims;
    std::vector<GenVar> vars;
    std::vector<GenStage> stages;
};

#define GEN_FN1(k, T, M) reinterpret_cast<yb::gen::GenKernelFn>(static_cast<void (*)(const yb::gen::GenParams)>(k<T, M>))
#define GEN_FN(k, T, M) yb::gen::GenKernelPair{GEN_FN1(k, T, M), GEN_FN1(k, T, (M) | yb::gen::GEN_WIDE)}

#ifdef __CUDACC__
// MODE 0: every operation individually rounded, in statement order (== the reference built with
// -ffp-contract=off).  MODE 1: the same, except that the products the reference's DEFAULT build (GCC -O3,
// -ffp-contract=fast) fuses into the addition that consumes them -- worked out by the emitter (contract_like_gcc) and
// written as MAD / MSB / NMAD in the statement lists -- are single fma operations (== the reference's default build).
// Nothing is left to nvcc's own contraction: every operation is an explicitly rounded intrinsic in both modes.
template <typename T> struct GenRn;
template <> struct GenRn<float> {
    static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
    static __device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
    static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
    static __device__ __forceinline__ float div(float a, float b) { return __fdiv_rn(a, b); }
    static __device__ __forceinline__ float fma(float a, float b, float c) { return __fmaf_rn(a, b, c); }
};
template <> struct GenRn<double> {
    static __device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
    static __device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
    static __device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
    static __device__ __forceinline__ double div(double a, double b) { return __ddiv_rn(a, b); }
    static __device__ __forceinline__ double fma(double a, double b, double c) { return __fma_rn(a, b, c); }
};
template <typename T, int MODE> struct GenOp : GenRn<T> {
    using R = GenRn<T>;
    static __device__ __forceinline__ T mad(T a, T b, T c) { return (MODE & 1) == 0 ? R::add(R::mul(a, b), c) : R::fma(a, b, c); }
    static __device__ __forceinline__ T msb(T a, T b, T c) { return (MODE & 1) == 0 ? R::sub(R::mul(a, b), c) : R::fma(a, b, -c); }
    static __device__ __forceinline__ T nmad(T a, T b, T c) { return (MODE & 1) == 0 ? R::sub(c, R::mul(a, b)) : R::fma(-a, b, c); }
    static __device__ __forceinline__ T nmsb(T a, T b, T c) { return (MODE & 1) == 0 ? R::sub(-R::mul(a, b), c) : R::fma(-a, b, -c); }
};

// blockIdx.x -> (x, y, z) block coordinates in chunked sweep order (see GenParams::ychunk)
__device__ __forceinline__ void gen_block_coords(const GenParams& P, int& bx, int& by, int& bz) {
    const unsigned per_chunk = unsigned(P.nzb) * unsigned(P.ychunk) * unsigned(P.nxb);
    const unsigned chunk = blockIdx.x / per_chunk;
    unsigned rem = blockIdx.x - chunk * per_chunk;
    const unsigned y0 = chunk * unsigned(P.ychunk);
    const unsigned yc = min(unsigned(P.ychunk), unsigned(P.nyb) - y0);   // the last chunk may be shorter
    const unsigned per_plane = unsigned(P.nzb) * yc;
    bx = int(rem / per_plane);
    rem -= unsigned(bx) * per_plane;
    by = int(y0 + rem / unsigned(P.nzb));
    bz = int(rem % unsigned(P.nzb));
}

// Element position type of a direct kernel: int in the 32-bit form, long long in the 64-bit one (MODE & GEN_WIDE).
template <int MODE> using GenIdx = typename std::conditional<(MODE & GEN_WIDE) != 0, long long, int>::type;
template <int MODE>
__device__ __forceinline__ GenIdx<MODE> gen_pos(const GenParams& P, int x, int y, int z) {
    return GenIdx<MODE>(x) * P.SX + GenIdx<MODE>(y) * P.SY + z;
}

// One 128-byte line per thread and trip: lines of (GEN_BY * NP) rows x GEN_BZ points x GEN_BX planes per var.
template <typename T, int MODE>
__device__ __forceinline__ void gen_prefetch(const GenParams& P, int x0, int y0, int z0) {
    constexpr int LPR = GEN_BZ * int(sizeof(T)) / 128;              // lines per row
    constexpr int ROWS = GEN_BY * gen_np(int(sizeof(T))) * GEN_BX;
    constexpr int EPL = 128 / int(sizeof(T));                        // elements per line
    const int total = P.npf * (ROWS * LPR);
    for (int i = threadIdx.x; i < total; i += GEN_BLOCK) {
        const int v = i / (ROWS * LPR), r = (i / LPR) % ROWS, l = i % LPR;
        const int xx = x0 + P.pfd + r / (GEN_BY * gen_np(int(sizeof(T)))), yy = y0 + r % (GEN_BY * gen_np(int(sizeof(T)))), zz = z0 + l * EPL;
        if (xx < P.xe && yy < P.ye && zz < P.ze) {
            const T* a = static_cast<const T*>(P.ptr[P.pf[v]]) + gen_pos<MODE>(P, xx, yy, zz);
            asm volatile("prefetch.global.L2 [%0];" ::"l"(a));
        }
    }
}

#define GEN_KERNEL_BEGIN                                                                         \
    int gbx_, gby_, gbz_;                                                                        \
    gen_block_coords(P, gbx_, gby_, gbz_);                                                       \
    const int z = P.zb + gbz_ * GEN_BZ + (threadIdx.x % GEN_BZ);                                 \
    constexpr int GEN_NP = gen_np(int(sizeof(T)));                                               \
    const int y0_ = P.yb + gby_ * (GEN_BY * GEN_NP) + (threadIdx.x / GEN_BZ) % GEN_BY;           \
    const int x = P.xb + gbx_ * GEN_BX + threadIdx.x / (GEN_BZ * GEN_BY);                        \
    if (P.npf) gen_prefetch<T, MODE>(P, P.xb + gbx_ * GEN_BX, P.yb + gby_ * (GEN_BY * GEN_NP), P.zb + gbz_ * GEN_BZ);       \
    if (z >= P.ze || x >= P.xe) return;                                                          \
    _Pragma("unroll") for (int gp_ = 0; gp_ < GEN_NP; gp_++) {                                   \
        const int y = y0_ + gp_ * GEN_BY;                                                        \
        if (y < P.ye) {
#define GEN_KERNEL_END } }
// m = dim mask of the var (x=1, y=2, z=4).  Full-rank vars (m==7) use the shared geometry: one 64-bit position
// per thread, 32-bit neighbour offsets that the compiler shares across vars; lower-rank vars (1-D sponge
// arrays, scalars) take the general strided path.
// The position is 64-bit in the kernels' 64-bit form (slots of 2^31 elements or more; GenIdx); a neighbour offset stays 32-bit
// because it is bounded by the halo times the plane stride, which the engine keeps below 2^31 (GenEngine::check_geometry).
#define GEN_POS gen_pos<MODE>(P, x, y, z)
#define RD(a, m, dx, dy, dz)                                                                                             \
    ((m) == 7 ? static_cast<const T*>(P.ptr[a])[GEN_POS + ((dx) * P.SX + (dy) * P.SY + (dz))]                              \
              : static_cast<const T*>(P.ptr[a])[(x + (dx)) * P.sx[a] + (y + (dy)) * P.sy[a] + (z + (dz)) * P.sz[a]])
#define WR(a, m, v)                                                                                                      \
    do { if ((m) == 7) static_cast<T*>(P.ptr[a])[GEN_POS] = (v);                                                         \
         else static_cast<T*>(P.ptr[a])[x * P.sx[a] + y * P.sy[a] + z * P.sz[a]] = (v); } while (0)
#define C(v) static_cast<T>(v)
#define G(i) ((i) == 0 ? x + P.off[0] : ((i) == 1 ? y + P.off[1] : z + P.off[2]))
#define GT P.t
#define GF(i) P.gfirst[i]
#define GL(i) P.glast[i]
#define ADD(a, b) GenOp<T, MODE>::add(a, b)
#define SUB(a, b) GenOp<T, MODE>::sub(a, b)
#define MUL(a, b) GenOp<T, MODE>::mul(a, b)
#define DIV(a, b) GenOp<T, MODE>::div(a, b)
#define MAD(a, b, c) GenOp<T, MODE>::mad(a, b, c)
#define MSB(a, b, c) GenOp<T, MODE>::msb(a, b, c)
#define NMAD(a, b, c) GenOp<T, MODE>::nmad(a, b, c)
#define NMSB(a, b, c) GenOp<T, MODE>::nmsb(a, b, c)
// DSL math functions (/root/reference/src/kernel/lib/realv.hpp:713-726 call libm per element); CUDA's overloads
// pick the element type.  sqrt/fabs/min/max are exact, the others agree with libm to a few ulps.
#define YF_sqrt(a) sqrt(a)
#define YF_cbrt(a) cbrt(a)
#define YF_fabs(a) fabs(a)
#define YF_erf(a) erf(a)
#define YF_exp(a) exp(a)
#define YF_log(a) log(a)
#define YF_sin(a) sin(a)
#define YF_cos(a) cos(a)
#define YF_atan(a) atan(a)
#define YF_pow(a, b) pow(a, b)
#define YF_min(a, b) ((b) < (a) ? (b) : (a))   /* std::min */
#define YF_max(a, b) ((a) < (b) ? (b) : (a))   /* std::max */
#define YF_sincos(a, s, c) sincos(a, &(s), &(c))
#endif

} }  // namespace yb::gen
