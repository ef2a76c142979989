// iso3dfd point-update kernels for sm_90a.
//
// Equation and association order: /root/reference/src/stencils/Iso3dfdStencil.cpp:63-137
// (get_next_p) as canonicalised by the reference compiler ("-target pseudo", SURVEY.md
// Appendix A) -- this replaces the generated stencil_iso3dfd_part_1::calc_vectors()
// (emitter: /root/reference/src/compiler/lib/Cpp.cpp:377-1175) and the loop hierarchy that
// calls it (/root/reference/src/kernel/lib/context.cpp:631-1174, stencil_calc.hpp:444-860).
//
//   acc = p*c0;  r=1..R: acc += (((((p[x-r]+p[x+r])+p[y-r])+p[y+r])+p[z-r])+p[z+r]) * c_r
//   p(t+1) = ((2*p) - p(t-1)) + acc*v
//
// FP modes (see oracle/yask_oracle.c): 0 strict IEEE mul/add, 1 canonical FMA,
// 2 = FMA pattern GCC 13 emits for the reference's default build (bit-exact vs it).
//
// Every kernel here is written for an element type E, float or double (the reference's real_bytes=4 / 8).  A thread
// moves 16-byte vectors: 4 floats (float4) or 2 doubles (double2).
#pragma once
#include <type_traits>

#include "yb_ptx.cuh"
#include "yb_iso3dfd_math.cuh"

namespace yb {

constexpr int ISO_MAX_R = 8;
constexpr int ISO_MAX_CHUNKS = 40;   // x chunks of one launch (boundary chunks + interior chunks)

// 16-byte vector of the element type: the unit of shared-memory loads, x-queue entries and global stores.
template <class E> struct IsoVec;
template <> struct IsoVec<float> { using V = float4; static constexpr int N = 4; };
template <> struct IsoVec<double> { using V = double2; static constexpr int N = 2; };

template <class E>
struct IsoParamsT {
    E* out;             // &p_next[domain origin]; written in place over p(t-1)
    long long out_sx, out_sy;  // element strides of the p arrays (z stride is 1)
    const E* cur;           // &p_cur[domain origin]  (naive kernel only)
    const E* prev;          // &p_prev[domain origin] (naive kernel only): == out unless the var has extra storage slots
    const E* vel;           // &v[domain origin]      (naive kernel only)
    long long v_sx, v_sy;
    int nx, ny, nz;         // rank-domain sizes
    int x_begin, x_end;     // sub-range of x planes to compute (boundary/interior split)
    int y_begin, y_end;
    int z_begin, z_end;
    int pad_x, pad_y, pad_z;    // p arrays: alloc index of domain origin (TMA coordinates)
    int vpad_x, vpad_y, vpad_z; // v array: same
    int nty, ntz, nchunks;      // tiling of [begin,end): tiles in y,z; chunks along x
    // Every chunk: first plane computed, number of planes, sweep direction (+1 / -1).  Work units are numbered chunk-major,
    // so the chunks listed first are swept first by every CTA.  A multi-rank launch lists the chunk that starts at plane 0
    // (swept upwards) and the chunk that ends at plane nx-1 (swept DOWNWARDS) first: the planes the x neighbours need are
    // then the first R planes of those sweeps.  (A downward sweep gives the same bits: the x neighbours enter the sum as
    // p[x-r] + p[x+r], and IEEE addition commutes.)
    int cx0[ISO_MAX_CHUNKS], clen[ISO_MAX_CHUNKS], cdir[ISO_MAX_CHUNKS];
    int pol_c, pol_h, pol_pv;   // L2 eviction policy of the TMA streams: 0 normal, 1 evict_first, 2 evict_last
    int st_cs;                  // 1: results leave with streaming (evict-first) stores
    int peer_probe;             // DEBUG (option peer_probe): 1 = skip the peer stores (timing probe only: halos are NOT exchanged),
                                // 2 = CTAs start a few microseconds apart so that their boundary phases do not coincide
    // Fused halo exchange: when non-null, the first / last R computed x planes are ALSO stored into the lower /
    // upper x neighbour's halo cells (peer HBM over NVLink), indexed exactly like `out`.
    E* peer_lo;
    E* peer_hi;
    // In-kernel completion signal of the boundary planes (replaces the push + signal kernels that used to follow the
    // sweep): units [0, sig_units) are the units whose sweeps START with boundary planes.  Every consumer warp of the
    // grid arrives once on *sig_counter, right after the R-th plane of its last such unit (system-scope fence first);
    // the arrival that completes the count (sig_total) publishes sig_epoch into the neighbours' flag words with release
    // semantics and resets the counter.  The neighbours' next step, which needs exactly these planes, therefore has them
    // while this rank is still sweeping the rest (the overlap of /root/reference/src/kernel/lib/context.cpp:378-475:
    // exterior first, exchange during the interior) -- and no plane is swept twice or warmed up twice for it.
    int sig_units;
    unsigned int sig_total;
    unsigned int* sig_counter;
    unsigned long long* sig_flag_lo;
    unsigned long long* sig_flag_hi;
    unsigned long long sig_epoch;
    E c[ISO_MAX_R + 1];
    // iso3dfd_sponge (the kernels' SP form): element 0 of the rank domain of the 1-D vars cr_x(x), cr_y(y), cr_z(z).  Their
    // unit-stride dim is padded like every var's, so cr_z's origin sits on a 128-byte boundary and its alloc is a whole number
    // of 16-byte vectors.
    const E* cr_x;
    const E* cr_y;
    const E* cr_z;
};
using IsoParams = IsoParamsT<float>;

// ---------------------------------------------------------------------------------------------
// Reference-order direct kernel: one thread per point, straight global loads (through L1/L2).
// Used for radii/shapes the tiled kernel does not cover and as the on-device cross-check of the
// tiled kernel at sizes the CPU oracle cannot reach.  Any radius 1..8.
// SP: iso3dfd_sponge, p(t+1) *= cr_x(x) * cr_y(y) * cr_z(z) in the reference's statement order
// (/root/reference/src/stencils/Iso3dfdStencil.cpp:212-249): three rounded multiplies, ((p * cr_x) * cr_y) * cr_z, never the
// product of the three factors first (its rounding differs).  No addition follows them, so they are the same in every FP mode.
// ---------------------------------------------------------------------------------------------
template <class E>
__device__ __forceinline__ E iso_sponge(E p, E crx, E cry, E crz) {
    return iso_mul(iso_mul(iso_mul(p, crx), cry), crz);
}

template <class E, int MODE, bool SP = false>
__global__ void __launch_bounds__(256) iso3dfd_direct_kernel(IsoParamsT<E> P, int R) {
    const int z = P.z_begin + blockIdx.x * blockDim.x + threadIdx.x;
    const int y = P.y_begin + blockIdx.y;
    const int x = P.x_begin + blockIdx.z;
    if (z >= P.z_end || y >= P.y_end || x >= P.x_end) return;
    const long long o = (long long)x * P.out_sx + (long long)y * P.out_sy + z;
    const E* pc = P.cur + o;
    const E center = pc[0];
    E acc = 0;
    for (int r = 1; r <= R; r++) {
        acc = iso_group<MODE>(acc, center, P.c[0], P.c[r], pc[-r * P.out_sx], pc[r * P.out_sx], pc[-r * P.out_sy],
                              pc[r * P.out_sy], pc[-r], pc[r], r == 1);
    }
    const E v = P.vel[(long long)x * P.v_sx + (long long)y * P.v_sy + z];
    const E r = iso_final<MODE>(acc, center, P.prev[o], v);
    if constexpr (SP) P.out[o] = iso_sponge(r, P.cr_x[x], P.cr_y[y], P.cr_z[z]);
    else P.out[o] = r;
}

// ---------------------------------------------------------------------------------------------
// Tiled TMA kernel ("2.5-D sweep").
//
// A CTA owns a (TY x TZ) column of the (y,z) plane and sweeps it along x (the outermost,
// largest-stride axis) over a chunk of planes.  A thread owns two vertically adjacent rows x four
// z-consecutive points for every plane of the sweep.
//
//   * x neighbours: a 2R+1 deep register queue of the thread's own quads, rotated by register moves.
//   * y,z neighbours: the current plane with halo, (TY+2R) x (TZ+2HZ) elements, staged in shared
//     memory by ONE TMA box load (cp.async.bulk.tensor.3d, box depth 1).
//   * the queue is fed by a second, halo-less TMA box R planes ahead of the current one;
//     p(t-1) and v tiles arrive the same way (evict-first: they are streamed exactly once).
//   * a ring of STAGES such stage buffers is filled by a producer warpgroup (one elected lane) running
//     STAGES-1 sweep steps ahead; full/empty mbarriers, no __syncthreads in the sweep loop.
//   * results leave as 128-bit coalesced stores straight over p(t-1) (the reference's
//     2-slot write-back, /root/reference/src/compiler/lib/Var.cpp:435-464).
//
// Persistent grid: one CTA per SM; work units (y-tile, z-tile, x-chunk) are dealt round-robin so
// that the units in flight at any time are neighbours in (y,z) and share their halos through L2.
// ---------------------------------------------------------------------------------------------
struct IsoMaps {
    CUtensorMap h;  // p_cur, box (TZ+2HZ, TY+2R, 1)
    CUtensorMap c;  // p_cur, box (TZ, TY, 1)
    CUtensorMap p;  // p_prev, box (TZ, TY, 1)
    CUtensorMap v;  // v,      box (TZ, TY, 1)
};

// Sweep position of a CTA in its flattened (unit, iteration) sequence.
struct IsoCursor {
    int unit;      // current work unit
    int it;        // iteration within unit: 0 .. n_it-1
    int n_it;      // lx_unit + 2R
    int x0, y0, z0;  // unit origin (domain coordinates); x0 = first plane computed
    int dir;         // sweep direction along x
    int stage;
    uint32_t phase;
};

template <class T, class PT>
__device__ __forceinline__ void iso_unit_setup(IsoCursor& cu, const PT& P) {
    int u = cu.unit;
    const int tz = u % P.ntz; u /= P.ntz;
    const int ty = u % P.nty; u /= P.nty;
    cu.z0 = P.z_begin + tz * T::TZ;
    cu.y0 = P.y_begin + ty * T::TY;
    cu.x0 = P.cx0[u];
    cu.dir = P.cdir[u];
    cu.n_it = P.clen[u] + 2 * T::R;
    cu.it = 0;
}

// ---------------------------------------------------------------------------------------------
// Thread layout ("row pairs").
//
// The first version of this kernel (one row x 4 z per thread, sweep loop unrolled 2R+1 times) was limited by shared-memory wavefronts (23 LDS.128 per 4 points,
// every y neighbour loaded once per point) and by instruction-cache misses of the unrolled body.  Hence:
//   * a thread owns TWO vertically adjacent rows x 4 z (8 points; 2 z and 4 points in fp64).  The y window of the pair is
//     18 rows, each loaded ONCE and used by both rows: 16+8 neighbour loads per 8 points
//     instead of 2 x 20 -- 40 % fewer shared-memory wavefronts per point;
//   * the x queue is rotated by register moves (loop NOT unrolled 2R+1 times), so the whole
//     sweep body fits the instruction cache.
// ---------------------------------------------------------------------------------------------
// E = double: a thread's rows are one double2 wide, so the same thread layout covers half the z extent (TZ = 2 * TZQ)
// with the same registers per x-queue entry, and the z halo rounds up to whole double2 vectors.
template <int R_, int TYP_, int TZQ_, int STAGES_, class E_ = float>
struct IsoTile2 {
    using E = E_;
    using V = typename IsoVec<E>::V;
    static constexpr int VW = IsoVec<E>::N;     // elements per 16-byte vector
    static constexpr int ES = int(sizeof(E));
    static constexpr int R = R_, TYP = TYP_, TZQ = TZQ_, STAGES = STAGES_;
    static constexpr int TY = 2 * TYP;
    static constexpr int TZ = VW * TZQ;
    static constexpr int HZ = (R + VW - 1) / VW * VW;
    static constexpr int ZQ = HZ / VW;
    static constexpr int HP = TZ + 2 * HZ;
    static constexpr int HROWS = TY + 2 * R;
    static constexpr int THREADS = TYP * TZQ;
    static constexpr int NWARPS = THREADS / 32;
    static constexpr int QN = 2 * R + 1;
    // setmaxnreg split of a CTA with a producer warpgroup (128 x PROD_REGS + THREADS x CONS_REGS <= 64K registers).  The fp64
    // producer keeps twice the fp32 budget: its unit bookkeeping then stays in registers (24 spill a few bytes to the stack).
    static constexpr int PROD_REGS = sizeof(E) == 8 ? 48 : 24;
    static constexpr int CONS_REGS = sizeof(E) == 8 ? 224 : 240;
    static constexpr uint32_t H_BYTES = HROWS * HP * ES;
    static constexpr uint32_t C_BYTES = TY * TZ * ES;
    static constexpr uint32_t H_OFF = 0;
    static constexpr uint32_t C_OFF = (H_BYTES + 127) / 128 * 128;
    static constexpr uint32_t P_OFF = C_OFF + C_BYTES;
    static constexpr uint32_t V_OFF = P_OFF + C_BYTES;
    static constexpr uint32_t STAGE_BYTES = V_OFF + C_BYTES;
    static constexpr uint32_t BAR_OFF = STAGES * STAGE_BYTES;
    static constexpr uint32_t SMEM_BYTES = BAR_OFF + 2 * STAGES * 8 + 128;
    static_assert(THREADS % 32 == 0, "whole warps");
    static_assert(C_BYTES % 128 == 0, "TMA destination alignment");
};

// Boundary-phase completion (see IsoParams::sig_*): called once per consumer warp, by all of its lanes.  Out of line in the
// plain sweep; the sponge form (SP) inlines it, since the registers live across the call spilled there.
template <class PT>
__device__ __forceinline__ void iso_boundary_arrive_inl(const PT& P, int lane) {
    __threadfence_system();          // this lane's peer stores are ordered before what follows, at system scope
    __syncwarp();
    if (lane == 0) {
        const unsigned int prev = atomicAdd(P.sig_counter, 1u);
        if (prev + 1u == P.sig_total) {            // every warp of the grid has finished its boundary units
            __threadfence_system();
            atomicExch(P.sig_counter, 0u);         // ready for the next launch (stream-ordered after this one)
            if (P.sig_flag_lo) asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(P.sig_flag_lo), "l"(P.sig_epoch) : "memory");
            if (P.sig_flag_hi) asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(P.sig_flag_hi), "l"(P.sig_epoch) : "memory");
        }
    }
}
template <class PT>
__device__ __noinline__ void iso_boundary_arrive(const PT& P, int lane) { iso_boundary_arrive_inl(P, lane); }

__device__ __forceinline__ void f4_to_arr(const float4& v, float* a) { a[0] = v.x; a[1] = v.y; a[2] = v.z; a[3] = v.w; }
__device__ __forceinline__ void f4_to_arr(const double2& v, double* a) { a[0] = v.x; a[1] = v.y; }
__device__ __forceinline__ void arr_to_v(const float* a, float4& v) { v = make_float4(a[0], a[1], a[2], a[3]); }
__device__ __forceinline__ void arr_to_v(const double* a, double2& v) { v = make_double2(a[0], a[1]); }

// One sweep step of a consumer thread: p(t+1) of its two rows (a, b) at plane xo, and the stores.  Shared by the sweep kernels
// (iso3dfd_tma2_kernel, iso3dfd_tma3_kernel), which differ only in how p(t) reaches shared memory.
//   qa, qb  the rows' x queues; window q[B .. B+2R], centre q[B+R]
//   h       row a's centre in the haloed p(t) plane (T::HP elements per row; row b is the next row)
//   pv, v   row a in the p(t-1) and v tiles (T::TZ elements per row)
//   oa      row a's output vector; row b is P.out_sy further on
// Results leave as 128-bit stores where the row's vector is whole and aligned (scalars on ragged edges).  The fused halo
// exchange (peer stores into the x neighbours' halo cells) is compiled for fp32 only: the engine never fuses an fp64
// sweep, and leaving the out-of-line signal call out keeps its registers free of call spills.
// SP (iso3dfd_sponge): both rows' results are scaled by the sponge factors in `sg` (iso_sponge) before every store, the peer
// stores included.
template <class E>
struct IsoSpongeRegs {
    E x;                    // cr_x of the plane computed now
    E ya, yb;               // cr_y of rows a and b
    E z[IsoVec<E>::N];      // cr_z of the thread's vector
};

// Default `pv_load` of iso_rows_update: the caller waited for the p(t-1) and v tiles before the call.
struct IsoPvLoaded {
    template <class F>
    __device__ __forceinline__ void operator()(F&& load) const { load(); }
};

// pv_load(load) runs load(), the reads of the p(t-1) and v vectors.  They come after the stencil sums, so a caller that has
// not yet waited for those tiles can wait inside pv_load, with the sums' arithmetic as cover for the load.
template <class T, int MODE, int B, int QL, bool SP = false, class PvLoad = IsoPvLoaded>
__device__ __forceinline__ void iso_rows_update(const IsoParamsT<typename T::E>& P, const typename T::V (&qa)[QL],
                                                const typename T::V (&qb)[QL], const uint8_t* h, const uint8_t* pv,
                                                const uint8_t* v, typename T::E* oa, int xo, int nva, int nvb, bool vec_ok,
                                                const IsoSpongeRegs<typename T::E>* sg = nullptr, PvLoad pv_load = {}) {
    using E = typename T::E;
    using V = typename T::V;
    constexpr int R = T::R, ZQ = T::ZQ, VW = T::VW, ES = T::ES;
    constexpr bool FUSED = sizeof(E) == 4;
    if constexpr (MODE == 3) {
        // DEBUG (mem_probe=1): memory-system ceiling probe -- same TMA traffic and stores, no stencil math.
        static_assert(sizeof(E) == 4, "the memory probe is compiled for fp32 only");
        const float4 pva = *reinterpret_cast<const float4*>(pv);
        const float4 vva = *reinterpret_cast<const float4*>(v);
        const float4 pvb = *reinterpret_cast<const float4*>(pv + T::TZ * 4);
        const float4 vvb = *reinterpret_cast<const float4*>(v + T::TZ * 4);
        const float4 ha = *reinterpret_cast<const float4*>(h);
        float4 ra = make_float4(pva.x + vva.x * qa[B + R].x, pva.y + vva.y * ha.y, pva.z + vva.z, pva.w + vva.w);
        float4 rb = make_float4(pvb.x + vvb.x * qb[B + R].x, pvb.y + vvb.y, pvb.z + vvb.z, pvb.w + vvb.w);
        if (vec_ok && nva == 4) stg128(oa, ra);
        if (vec_ok && nvb == 4) stg128(oa + P.out_sy, rb);
    } else {
        const E* hp = reinterpret_cast<const E*>(h);
        E pa[VW], pb[VW];
        f4_to_arr(qa[B + R], pa);
        f4_to_arr(qb[B + R], pb);
        // z windows of both rows (centre quads come from the queue)
        E za[VW * (2 * ZQ + 1)], zb[VW * (2 * ZQ + 1)];
#pragma unroll
        for (int k = -ZQ; k <= ZQ; k++) {
            if (k == 0) { f4_to_arr(qa[B + R], &za[VW * ZQ]); f4_to_arr(qb[B + R], &zb[VW * ZQ]); continue; }
            f4_to_arr(*reinterpret_cast<const V*>(hp + VW * k), &za[VW * (k + ZQ)]);
            f4_to_arr(*reinterpret_cast<const V*>(hp + T::HP + VW * k), &zb[VW * (k + ZQ)]);
        }
        E acca[VW] = {}, accb[VW] = {};
        // y window: w(k) = hp + (k - R) * HP ; row a centre = w(R), row b centre = w(R+1)
        E wlo_prev[VW], whi_prev[VW];   // w(R - (r-1)) and w(R+1 + (r-1)) from the previous radius
        f4_to_arr(qa[B + R], wlo_prev);   // r=1: row b's y-1 neighbour is row a's centre
        f4_to_arr(qb[B + R], whi_prev);   //      row a's y+1 neighbour is row b's centre
#pragma unroll
        for (int r = 1; r <= R; r++) {
            E wlo[VW], whi[VW], xm[VW], xp[VW];
            f4_to_arr(*reinterpret_cast<const V*>(hp - r * T::HP), wlo);        // row a - r
            f4_to_arr(*reinterpret_cast<const V*>(hp + (r + 1) * T::HP), whi);  // row b + r
            f4_to_arr(qa[B + R - r], xm); f4_to_arr(qa[B + R + r], xp);
#pragma unroll
            for (int i = 0; i < VW; i++)   // row a: y-r = wlo, y+r = w(R+r) = previous whi
                acca[i] = iso_group<MODE>(acca[i], pa[i], P.c[0], P.c[r], xm[i], xp[i], wlo[i], whi_prev[i],
                                          za[VW * ZQ + i - r], za[VW * ZQ + i + r], r == 1);
            f4_to_arr(qb[B + R - r], xm); f4_to_arr(qb[B + R + r], xp);
#pragma unroll
            for (int i = 0; i < VW; i++)   // row b: y-r = w(R+1-r) = previous wlo, y+r = whi
                accb[i] = iso_group<MODE>(accb[i], pb[i], P.c[0], P.c[r], xm[i], xp[i], wlo_prev[i], whi[i],
                                          zb[VW * ZQ + i - r], zb[VW * ZQ + i + r], r == 1);
#pragma unroll
            for (int i = 0; i < VW; i++) { wlo_prev[i] = wlo[i]; whi_prev[i] = whi[i]; }
        }
        E pva[VW], vva[VW], pvb[VW], vvb[VW], ea[VW], eb[VW];
        pv_load([&] {
            f4_to_arr(*reinterpret_cast<const V*>(pv), pva);
            f4_to_arr(*reinterpret_cast<const V*>(v), vva);
            f4_to_arr(*reinterpret_cast<const V*>(pv + T::TZ * ES), pvb);
            f4_to_arr(*reinterpret_cast<const V*>(v + T::TZ * ES), vvb);
        });
#pragma unroll
        for (int i = 0; i < VW; i++) ea[i] = iso_final<MODE>(acca[i], pa[i], pva[i], vva[i]);
#pragma unroll
        for (int i = 0; i < VW; i++) eb[i] = iso_final<MODE>(accb[i], pb[i], pvb[i], vvb[i]);
        if constexpr (SP) {
#pragma unroll
            for (int i = 0; i < VW; i++) {
                ea[i] = iso_sponge(ea[i], sg->x, sg->ya, sg->z[i]);
                eb[i] = iso_sponge(eb[i], sg->x, sg->yb, sg->z[i]);
            }
        }
        V ra, rb;
        arr_to_v(ea, ra); arr_to_v(eb, rb);
        E* ob = oa + P.out_sy;
        if (vec_ok && nva == VW) { if (P.st_cs) stg128_cs(oa, ra); else stg128(oa, ra); }
        else {
#pragma unroll
            for (int i = 0; i < VW && i < nva; i++) oa[i] = ea[i];
        }
        if (vec_ok && nvb == VW) { if (P.st_cs) stg128_cs(ob, rb); else stg128(ob, rb); }
        else {
#pragma unroll
            for (int i = 0; i < VW && i < nvb; i++) ob[i] = eb[i];
        }
        // fused halo exchange: boundary planes also go straight into the x neighbours' halo cells
        E* peer = !FUSED ? nullptr : (P.peer_lo != nullptr && xo < R) ? P.peer_lo : ((P.peer_hi != nullptr && xo >= P.nx - R) ? P.peer_hi : nullptr);
        if (peer != nullptr && P.peer_probe != 1) {
            E* qa_ = peer + (oa - P.out);
            E* qb_ = qa_ + P.out_sy;
            if (vec_ok && nva == VW) stg128(qa_, ra);
            else {
#pragma unroll
                for (int i = 0; i < VW && i < nva; i++) qa_[i] = ea[i];
            }
            if (vec_ok && nvb == VW) stg128(qb_, rb);
            else {
#pragma unroll
                for (int i = 0; i < VW && i < nvb; i++) qb_[i] = eb[i];
            }
        }
    }
}

// PW = 1: a dedicated producer warp (warp NWARPS) issues the TMA loads, so no compute warp carries the
//         issue code (with 2 warps per scheduler a straggling warp 0 delays every stage hand-over).
// U  = 2: the sweep loop handles two planes per trip and rotates the x queues by two entries every second
//         plane (half the register moves of U = 1) at the price of one extra queue entry per row.
// SP = true: iso3dfd_sponge.  The sponge factors live in registers: cr_z (one 16-byte vector) and cr_y (two rows) are loaded
//         once per work unit, cr_x one plane ahead of the plane it scales, in the chunk's sweep direction.
template <class T, int MODE, int PW = 0, int U = 1, bool SP = false>
__global__ void __launch_bounds__(T::THREADS + 128 * PW, 1)
iso3dfd_tma2_kernel(const __grid_constant__ IsoMaps M, const __grid_constant__ IsoParamsT<typename T::E> P) {
    using E = typename T::E;
    using V = typename T::V;
    constexpr int R = T::R, QN = T::QN, ZQ = T::ZQ, VW = T::VW, ES = T::ES;
    constexpr int QL = QN + (U - 1);          // queue entries kept per row
    constexpr bool FUSED = sizeof(E) == 4;    // see iso_rows_update
    // setmaxnreg split: the fp32 sponge form gives its producer warpgroup 32 registers (at 24 it spilled at radius 1-4), which
    // leaves its consumers 232 of the 168 x 384 the CTA is launched with
    constexpr int PROD_REGS = (SP && FUSED) ? 32 : T::PROD_REGS;
    constexpr int CONS_REGS = (SP && FUSED) ? 232 : T::CONS_REGS;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 127u) & ~127u;
    uint8_t* sbase = smem_raw + (base - smem_u32(smem_raw));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(sbase + T::BAR_OFF);
    uint64_t* empty_bar = full_bar + T::STAGES;

    const int tid = threadIdx.x;
    const int lane = tid & 31;
    const int nunits = P.nty * P.ntz * P.nchunks;
    const int prod_tid = PW ? T::THREADS : 0;

    if (tid == 0) {
        tma_prefetch_desc(&M.h); tma_prefetch_desc(&M.c); tma_prefetch_desc(&M.p); tma_prefetch_desc(&M.v);
        for (int s = 0; s < T::STAGES; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], T::NWARPS); }
        fence_barrier_init();
    }
    __syncthreads();

    // ---- producer -----------------------------------------------------------------------------------
    IsoCursor pr;
    pr.unit = blockIdx.x; pr.stage = 0; pr.phase = 0; pr.it = 0; pr.n_it = 0; pr.x0 = pr.y0 = pr.z0 = 0; pr.dir = 1;
    const uint64_t pol_pv = l2_policy(P.pol_pv), pol_c = l2_policy(P.pol_c), pol_h = l2_policy(P.pol_h);
    bool pr_live = (tid == prod_tid) && (pr.unit < nunits);
    if (pr_live) iso_unit_setup<T>(pr, P);

    auto produce_one = [&]() {
        mbar_wait(&empty_bar[pr.stage], pr.phase ^ 1u);
        uint8_t* st = sbase + pr.stage * T::STAGE_BYTES;
        uint64_t* fb = &full_bar[pr.stage];
        const bool compute = pr.it >= 2 * R;
        mbar_arrive_expect_tx(fb, compute ? (T::H_BYTES + 3 * T::C_BYTES) : T::C_BYTES);
        const int cz = P.pad_z + pr.z0, cy = P.pad_y + pr.y0;
        tma_load_3d_hint(st + T::C_OFF, &M.c, fb, cz, cy, P.pad_x + pr.x0 + pr.dir * (pr.it - R), pol_c);
        if (compute) {
            const int xo = pr.x0 + pr.dir * (pr.it - 2 * R);
            tma_load_3d_hint(st + T::H_OFF, &M.h, fb, cz - T::HZ, cy - R, P.pad_x + xo, pol_h);
            tma_load_3d_hint(st + T::P_OFF, &M.p, fb, cz, cy, P.pad_x + xo, pol_pv);
            tma_load_3d_hint(st + T::V_OFF, &M.v, fb, P.vpad_z + pr.z0, P.vpad_y + pr.y0, P.vpad_x + xo, pol_pv);
        }
        if (++pr.stage == T::STAGES) { pr.stage = 0; pr.phase ^= 1u; }
        if (++pr.it == pr.n_it) {
            pr.unit += gridDim.x;
            if (pr.unit < nunits) iso_unit_setup<T>(pr, P); else pr_live = false;
        }
    };
    if (PW) {
        // Warp-specialised register budget (setmaxnreg works on whole warpgroups): the producer warpgroup
        // hands its registers back, the two consumer warpgroups take them.
        if (tid >= T::THREADS) {          // producer warpgroup: one lane streams every load of this CTA, then exits
            asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PROD_REGS));
            while (pr_live) produce_one();
            return;
        }
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONS_REGS));
    } else if (tid == 0) {
        for (int k = 0; k < T::STAGES - 1 && pr_live; k++) produce_one();
    }

    if (P.peer_probe == 2) __nanosleep((blockIdx.x & 7u) * 2000u);
    // ---- consumer ------------------------------------------------------------------------------------
    const int rp = tid / T::TZQ;           // row pair 0..TYP-1  (rows 2rp, 2rp+1)
    const int quad = tid % T::TZQ;
    const uint32_t h_own = ((2 * rp + R) * T::HP + T::HZ + VW * quad) * ES;  // row a centre in H
    const uint32_t c_own = (2 * rp * T::TZ + VW * quad) * ES;               // row a in C/P/V tiles

    IsoCursor cu;
    cu.stage = 0; cu.phase = 0;
    V qa[QL], qb[QL];
#pragma unroll
    for (int k = 0; k < QL; k++) { const E zero[VW] = {}; arr_to_v(zero, qa[k]); qb[k] = qa[k]; }

    bool sig_pending = FUSED && P.sig_counter != nullptr;
    auto arrive = [&]() { if constexpr (SP) iso_boundary_arrive_inl(P, lane); else iso_boundary_arrive(P, lane); };
    for (cu.unit = blockIdx.x; cu.unit < nunits; cu.unit += gridDim.x) {
        if (sig_pending && cu.unit >= P.sig_units) { arrive(); sig_pending = false; }   // (a CTA without boundary-first units)
        iso_unit_setup<T>(cu, P);
        const int ya = cu.y0 + 2 * rp;
        const int zq = cu.z0 + VW * quad;
        const int nz_ok = max(0, min(VW, P.z_end - zq));
        const int nva = (ya < P.y_end) ? nz_ok : 0;
        const int nvb = (ya + 1 < P.y_end) ? nz_ok : 0;
        E* out_a = P.out + (long long)ya * P.out_sy + zq + (long long)cu.x0 * P.out_sx;       // plane x0; step s -> + dir*s planes
        const long long out_step = (long long)cu.dir * P.out_sx;
        const bool vec_ok = ((reinterpret_cast<uintptr_t>(out_a) & 15) == 0);
        // this warp's boundary planes are complete after plane R-1 of its last boundary-first unit
        const bool sig_here = sig_pending && cu.unit < P.sig_units && cu.unit + int(gridDim.x) >= P.sig_units;
        IsoSpongeRegs<E> sg;
        [[maybe_unused]] E crx_next;       // cr_x of the next plane to compute
        if constexpr (SP) {
            // zq < z_end keeps the vector inside cr_z's allocation (whole 16-byte vectors from a 128-byte aligned origin); a
            // thread without points in z takes ones
            if (nz_ok > 0) f4_to_arr(*reinterpret_cast<const V*>(P.cr_z + zq), sg.z);
            else {
#pragma unroll
                for (int i = 0; i < VW; i++) sg.z[i] = E(1);
            }
            sg.ya = nva > 0 ? P.cr_y[ya] : E(1);
            sg.yb = nvb > 0 ? P.cr_y[ya + 1] : E(1);
            crx_next = P.cr_x[cu.x0];
        }

        // One sweep step.  B = index of the oldest live queue entry after the push (window = q[B .. B+2R]).
        auto step = [&](auto Bc, const int it) {
            constexpr int B = decltype(Bc)::value;
            if (!PW && tid == 0 && pr_live) produce_one();

            const uint8_t* st = sbase + cu.stage * T::STAGE_BYTES;
            mbar_wait(&full_bar[cu.stage], cu.phase);

            // push plane x0 - R + it into the x queues
            if (B == 0) {
#pragma unroll
                for (int k = 0; k + U < QL; k++) { qa[k] = qa[k + U]; qb[k] = qb[k + U]; }
            }
            qa[B + QN - 1] = *reinterpret_cast<const V*>(st + T::C_OFF + c_own);
            qb[B + QN - 1] = *reinterpret_cast<const V*>(st + T::C_OFF + c_own + T::TZ * ES);

            if (it >= 2 * R) {
                if constexpr (SP) {
                    sg.x = crx_next;
                    if (it + 1 < cu.n_it) crx_next = P.cr_x[cu.x0 + cu.dir * (it + 1 - 2 * R)];   // used at the next step
                }
                iso_rows_update<T, MODE, B, QL, SP>(P, qa, qb, st + T::H_OFF + h_own, st + T::P_OFF + c_own, st + T::V_OFF + c_own,
                                                    out_a + (long long)(it - 2 * R) * out_step, cu.x0 + cu.dir * (it - 2 * R), nva, nvb,
                                                    vec_ok, &sg);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[cu.stage]);
            if (++cu.stage == T::STAGES) { cu.stage = 0; cu.phase ^= 1u; }
            if (sig_here && it == 3 * R - 1) { arrive(); sig_pending = false; }
        };

        if (U == 1) {
#pragma unroll 1
            for (int it = 0; it < cu.n_it; it++) step(std::integral_constant<int, 0>{}, it);
        } else {
            // trip = [rotate by 2, push] then [push]: the second plane lands one entry further along
#pragma unroll 1
            for (int it = 0; it < cu.n_it; it += 2) {
                step(std::integral_constant<int, 0>{}, it);
                if (it + 1 < cu.n_it) step(std::integral_constant<int, U - 1>{}, it + 1);
            }
        }
    }
    if (sig_pending) arrive();
}

// ---------------------------------------------------------------------------------------------
// Resident-plane sweep (fp32): every p(t) plane is loaded ONCE, with its halo, into a ring of NS shared-memory slots.
//
// The sweep kernel above loads each plane twice: halo-less R steps ahead to feed the x queues, and again with its halo when it
// becomes the current plane.  Between the two fetches a CTA streams ~R planes of traffic, and the whole grid together about as
// much as the H100's L2 holds, so the second fetch goes back to HBM.  Here the slot that receives plane x+R feeds the queues
// from its centre rows and stays resident until plane x is computed, R steps later, from its halo rows; only then do the
// consumer warps release it.  Queue-only planes (the R planes before a chunk and the R after it) take the halo-less box and are
// released at once.  p(t-1) and v arrive in a ring of their own, NPV stages.  NS = R + 1 + (planes of prefetch).
// Thread layout, x queues (two planes per trip), producer warpgroup and arithmetic are those of iso3dfd_tma2_kernel<T,MODE,1,2>.
// ---------------------------------------------------------------------------------------------
template <int R_, int TYP_, int TZQ_, int NS_, int NPV_>
struct IsoTile3 : IsoTile2<R_, TYP_, TZQ_, 1, float> {
    using Base = IsoTile2<R_, TYP_, TZQ_, 1, float>;
    static constexpr int NS = NS_, NPV = NPV_;
    static_assert(NS > R_ + 1, "a slot lives R + 1 sweep steps; at least one more is prefetch");
    static constexpr uint32_t SLOT_BYTES = (Base::H_BYTES + 127) / 128 * 128;
    static constexpr uint32_t PV_OFF = NS * SLOT_BYTES;
    static constexpr uint32_t PV_BYTES = 2 * Base::C_BYTES;     // p(t-1) tile, then v tile
    static constexpr uint32_t BAR_OFF = PV_OFF + NPV * PV_BYTES;
    static constexpr uint32_t SMEM_BYTES = BAR_OFF + 2 * (NS + NPV) * 8 + 128;
    static_assert(SMEM_BYTES <= 232448, "over the sm_90 opt-in shared memory per block");
};

template <class T, int MODE>
__global__ void __launch_bounds__(T::THREADS + 128, 1)
iso3dfd_tma3_kernel(const __grid_constant__ IsoMaps M, const __grid_constant__ IsoParams P) {
    using V = float4;
    constexpr int R = T::R, QN = T::QN, NS = T::NS, NPV = T::NPV, ES = 4;
    constexpr int QL = QN + 1;                // two planes per trip: one extra queue entry per row
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 127u) & ~127u;
    uint8_t* sbase = smem_raw + (base - smem_u32(smem_raw));
    uint64_t* h_full = reinterpret_cast<uint64_t*>(sbase + T::BAR_OFF);
    uint64_t* h_empty = h_full + NS;
    uint64_t* pv_full = h_empty + NS;
    uint64_t* pv_empty = pv_full + NPV;

    const int tid = threadIdx.x;
    const int lane = tid & 31;
    const int nunits = P.nty * P.ntz * P.nchunks;

    if (tid == 0) {
        tma_prefetch_desc(&M.h); tma_prefetch_desc(&M.c); tma_prefetch_desc(&M.p); tma_prefetch_desc(&M.v);
        for (int s = 0; s < NS; s++) { mbar_init(&h_full[s], 1); mbar_init(&h_empty[s], T::NWARPS); }
        for (int s = 0; s < NPV; s++) { mbar_init(&pv_full[s], 1); mbar_init(&pv_empty[s], T::NWARPS); }
        fence_barrier_init();
    }
    __syncthreads();

    // ---- producer warpgroup: one lane streams every load of this CTA, then exits -------------------------------------
    if (tid >= T::THREADS) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(T::PROD_REGS));
        if (tid != T::THREADS) return;
        const uint64_t pol_pv = l2_policy(P.pol_pv), pol_c = l2_policy(P.pol_c), pol_h = l2_policy(P.pol_h);
        int hs = 0, ps = 0;
        uint32_t hph = 0, pph = 0;
        IsoCursor pr;
        for (pr.unit = blockIdx.x; pr.unit < nunits; pr.unit += gridDim.x) {
            iso_unit_setup<T>(pr, P);
            const int lx = pr.n_it - 2 * R;
            const int cz = P.pad_z + pr.z0, cy = P.pad_y + pr.y0;
            for (int it = 0; it < pr.n_it; it++) {
                // plane x0 + dir*(it - R): haloed if it is computed (at step it + R), else queue-only
                const bool halo = it >= R && it < lx + R;
                mbar_wait(&h_empty[hs], hph ^ 1u);
                mbar_arrive_expect_tx(&h_full[hs], halo ? T::H_BYTES : T::C_BYTES);
                const int xp = P.pad_x + pr.x0 + pr.dir * (it - R);
                if (halo) tma_load_3d_hint(sbase + hs * T::SLOT_BYTES, &M.h, &h_full[hs], cz - T::HZ, cy - R, xp, pol_h);
                else tma_load_3d_hint(sbase + hs * T::SLOT_BYTES, &M.c, &h_full[hs], cz, cy, xp, pol_c);
                if (++hs == NS) { hs = 0; hph ^= 1u; }
                if (it >= 2 * R) {      // p(t-1) and v of the plane computed at step it
                    const int xo = pr.x0 + pr.dir * (it - 2 * R);
                    uint8_t* pv = sbase + T::PV_OFF + ps * T::PV_BYTES;
                    mbar_wait(&pv_empty[ps], pph ^ 1u);
                    mbar_arrive_expect_tx(&pv_full[ps], T::PV_BYTES);
                    tma_load_3d_hint(pv, &M.p, &pv_full[ps], cz, cy, P.pad_x + xo, pol_pv);
                    tma_load_3d_hint(pv + T::C_BYTES, &M.v, &pv_full[ps], P.vpad_z + pr.z0, P.vpad_y + pr.y0, P.vpad_x + xo, pol_pv);
                    if (++ps == NPV) { ps = 0; pph ^= 1u; }
                }
            }
        }
        return;
    }
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(T::CONS_REGS));

    if (P.peer_probe == 2) __nanosleep((blockIdx.x & 7u) * 2000u);
    // ---- consumers ---------------------------------------------------------------------------------------------------
    const int rp = tid / T::TZQ;           // row pair 0..TYP-1  (rows 2rp, 2rp+1)
    const int quad = tid % T::TZQ;
    const uint32_t h_own = ((2 * rp + R) * T::HP + T::HZ + 4 * quad) * ES;   // row a centre in a haloed slot
    const uint32_t c_own = (2 * rp * T::TZ + 4 * quad) * ES;                 // row a in a halo-less slot / the p(t-1), v tiles

    int hs = 0, ps = 0;
    uint32_t hph = 0, pph = 0;
    V qa[QL], qb[QL];
#pragma unroll
    for (int k = 0; k < QL; k++) { qa[k] = make_float4(0.f, 0.f, 0.f, 0.f); qb[k] = qa[k]; }

    bool sig_pending = P.sig_counter != nullptr;
    IsoCursor cu;
    for (cu.unit = blockIdx.x; cu.unit < nunits; cu.unit += gridDim.x) {
        if (sig_pending && cu.unit >= P.sig_units) { iso_boundary_arrive(P, lane); sig_pending = false; }   // (a CTA without boundary-first units)
        iso_unit_setup<T>(cu, P);
        const int lx = cu.n_it - 2 * R;
        const int ya = cu.y0 + 2 * rp;
        const int zq = cu.z0 + 4 * quad;
        const int nz_ok = max(0, min(4, P.z_end - zq));
        const int nva = (ya < P.y_end) ? nz_ok : 0;
        const int nvb = (ya + 1 < P.y_end) ? nz_ok : 0;
        float* out_a = P.out + (long long)ya * P.out_sy + zq + (long long)cu.x0 * P.out_sx;
        const long long out_step = (long long)cu.dir * P.out_sx;
        const bool vec_ok = ((reinterpret_cast<uintptr_t>(out_a) & 15) == 0);
        const bool sig_here = sig_pending && cu.unit < P.sig_units && cu.unit + int(gridDim.x) >= P.sig_units;

        // One sweep step: push plane x0 - R + it into the queues (slot hs); from step 2R on compute plane x0 + (it - 2R), whose
        // haloed slot arrived R steps ago.  B = index of the oldest live queue entry after the push.
        auto step = [&](auto Bc, const int it) {
            constexpr int B = decltype(Bc)::value;
            const bool halo = it >= R && it < lx + R;
            const uint8_t* sl = sbase + hs * T::SLOT_BYTES;
            mbar_wait(&h_full[hs], hph);
            if (B == 0) {
#pragma unroll
                for (int k = 0; k + 2 < QL; k++) { qa[k] = qa[k + 2]; qb[k] = qb[k + 2]; }
            }
            const uint32_t own = halo ? h_own : c_own;
            qa[B + QN - 1] = *reinterpret_cast<const V*>(sl + own);
            qb[B + QN - 1] = *reinterpret_cast<const V*>(sl + own + (halo ? T::HP : T::TZ) * ES);

            const bool compute = it >= 2 * R;
            const int hc = hs >= R ? hs - R : hs - R + NS;     // slot of the plane computed now
            if (compute) {
                const uint8_t* pv = sbase + T::PV_OFF + ps * T::PV_BYTES;
                // p(t-1) and v are first read by iso_final, after the stencil sums: wait for them there, so the sums cover
                // their load.  The memory probe (MODE 3) reads them first and keeps the wait it is measured with.
                if constexpr (MODE == 3) mbar_wait(&pv_full[ps], pph);
                iso_rows_update<T, MODE, B>(P, qa, qb, sbase + hc * T::SLOT_BYTES + h_own, pv + c_own, pv + T::C_BYTES + c_own,
                                            out_a + (long long)(it - 2 * R) * out_step, cu.x0 + cu.dir * (it - 2 * R), nva, nvb, vec_ok,
                                            nullptr, [&](auto&& load) { mbar_wait(&pv_full[ps], pph); load(); });
            }
            __syncwarp();
            if (lane == 0) {
                if (compute) { mbar_arrive(&pv_empty[ps]); mbar_arrive(&h_empty[hc]); }
                if (!halo) mbar_arrive(&h_empty[hs]);
            }
            if (compute && ++ps == NPV) { ps = 0; pph ^= 1u; }
            if (++hs == NS) { hs = 0; hph ^= 1u; }
            if (sig_here && it == 3 * R - 1) { iso_boundary_arrive(P, lane); sig_pending = false; }
        };
        // trip = [rotate by 2, push] then [push]: the second plane lands one entry further along
#pragma unroll 1
        for (int it = 0; it < cu.n_it; it += 2) {
            step(std::integral_constant<int, 0>{}, it);
            if (it + 1 < cu.n_it) step(std::integral_constant<int, 1>{}, it + 1);
        }
    }
    if (sig_pending) iso_boundary_arrive(P, lane);
}

}  // namespace yb
