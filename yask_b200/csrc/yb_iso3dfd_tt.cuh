// Temporal tile for iso3dfd: TWO time steps per sweep, the intermediate step held in shared memory.
//
// What it replaces: the reference's temporal blocking of a block of points over several steps
// (/root/reference/src/kernel/lib/context.cpp:657-681 calc_block: block steps "-bt"; :838-1003 the shifted
// micro-block shapes per step; option parsing /root/reference/src/kernel/lib/settings.cpp "-bt").  There the block that
// stays in cache is a trapezoid whose base shrinks by the radius per step; here the tile that stays in shared memory
// is extended by the radius per step instead ("overlapped tiling": the step-1 ring is computed redundantly by the
// neighbouring CTAs, so no CTA ever waits for another one) -- same arithmetic per point, same bits.
//
// One CTA owns a (TY x TZ) tile of the (y,z) plane and marches along x.  Per sweep iteration j (g = running count):
//   loads   : p(t) plane xl = x0 + j - 2R over the tile + 2R rows / 2*HZ1 columns     -> ring of 2R+1+PF planes
//             p(t-1), v  plane x1 = xl - R  over the tile + R rows / HZ1 columns        -> rings of PF+1 planes
//             (three TMA 3-D boxes, cp.async.bulk.tensor; completion on full[g mod (PF+1)])
//   step 1  : p(t+1) at plane x1 over the tile + R ring, from the p(t) ring -> p1 ring (shared memory, 2R+2 planes);
//             the tile's own part also goes to HBM (slot of t+1).  Points outside the global domain take p(t-1): the value
//             the reference's two-slot storage holds in the halo cells of p(t+1) (/root/reference/src/compiler/lib/Var.cpp:435-464).
//             Points in the R ring beyond a rank interface are computed like any other (TTParams::ext_lo / ext_hi): the
//             reference's wave-front extension of a rank, whose halos are exchanged once per pair of steps.
//   barrier : __syncthreads (the only one per iteration); then thread 0 issues the loads of iteration g+PF
//   step 2  : p(t+2) at plane x2 = x1 - R over the tile, from the p1 ring (x2-R..x2+R), p(t) plane x2 (the oldest plane of
//             the p ring, "prev") and v(x2) (read from global/L2 into a register before step 1) -> HBM (slot of t+2).
//
// (Form XQ = 1, below: the x neighbours of both steps come from per-thread register queues instead of the rings, which then
// only span R+1 / R+2 planes.)
//
// HBM traffic per point and PAIR of steps: read p(t-1), p(t), v, write p(t+1), p(t+2) = 20 B (+ halo overlap) against
// 2 x 16 B for two one-step sweeps.  Overlapping tiles read halo cells of BOTH input steps, so the two results cannot
// overwrite them in place: the var gets a spare pair of storage slots and fused launches ping-pong between the pairs
// (yb_core.h Var::extra_slots / slot_bias, yb_iso3dfd.cu).
// Shared memory bounds the radius: R = 2 needs 227 KB at tile 16 x 128 in the first form (R = 3 would leave an 8-row tile
// that recomputes 86 % of step 1) -- hence "where the radius allows" = R <= 2.
// The first form reads every neighbour from shared memory; the XQ form keeps x neighbours in register queues.
//
// Every function that touches tile data is written once (YB_DEVFN) and is ALSO compiled by g++ into the test suite's CTA
// emulator (tests/emul/tt_emul.cpp: threads run in a loop, TMA boxes are copied by the host), which checks the ring /
// index logic bit for bit against the oracle on a machine without a GPU.
#pragma once
#include <stdint.h>

#include "yb_iso3dfd_math.cuh"

#ifndef YB_DEVMEM      // member functions: the emulator's YB_DEVFN is `static inline`, which a member must not be
#ifdef YB_TT_HOST_EMUL
#define YB_DEVMEM inline
#else
#define YB_DEVMEM __device__ __forceinline__
#endif
#endif

namespace yb {

constexpr int TT_MAX_CHUNKS = 40;
constexpr int TT_MAX_R = 2;

struct TTParams {
    float* out1;               // &p(t+1)[domain origin]
    float* out2;               // &p(t+2)[domain origin]
    const float* vel;          // &v[domain origin]
    long long p_sx, p_sy;      // element strides of the p slots (z stride 1)
    long long v_sx, v_sy;
    int nx, ny, nz;            // rank-domain sizes (the temporal tile runs on whole rank domains)
    // Step-1 points with -ext_lo[d] <= index < n[d] + ext_hi[d] in every dim (x, y, z) are computed; the others lie outside the
    // GLOBAL domain and take p(t-1).  0 on a side at the global boundary (so a zero-initialised TTParams describes one rank); R on a
    // side with a neighbour rank, whose halos hold p(t) 2R deep and p(t-1), v R deep, so that the step-1 ring there is what the
    // neighbour computes for its own points.
    int ext_lo[3], ext_hi[3];
    int pad_x, pad_y, pad_z;   // p: alloc index of the domain origin (TMA coordinates)
    int vpad_x, vpad_y, vpad_z;
    int nty, ntz, nchunks;     // tiles in y and z, chunks along x
    int cx0[TT_MAX_CHUNKS], clen[TT_MAX_CHUNKS];   // first plane and number of planes of every chunk
    float c[TT_MAX_R + 1];
    // L2 policy, as in the one-step kernel: the p(t) box is the stream whose halo rows the neighbouring
    // tiles re-read (0 normal, 1 evict_first, 2 evict_last); results are not read again during the launch (st_cs: streaming stores)
    int pol_p, st_cs;
};

struct alignas(16) TTVec4 { float x, y, z, w; };

// XQ = 1: the x neighbours of BOTH steps live in per-thread register queues (2R+1 vectors per owned vector, shifted by one plane
// per iteration), as in the one-step kernel: the p(t) ring then only spans the planes between arrival and use as the y/z
// centre plane (R+1), the p1 ring R+2, and a thread issues 9 + 6 instead of 13 + 12 shared-memory loads per pair of vectors.
template <int R_, int TY_, int TZ_, int PF_, int THREADS_, int XQ_ = 0>
struct TTile {
    static constexpr int R = R_, TY = TY_, TZ = TZ_, PF = PF_, THREADS = THREADS_, XQ = XQ_;
    static constexpr int QN = 2 * R + 1;
    static constexpr int HZ1 = (R + 3) / 4 * 4;       // z reach of one step, in whole 16-byte vectors
    static constexpr int ZQ = HZ1 / 4;
    static constexpr int IY = TY + 4 * R, IZ = TZ + 4 * HZ1;     // p(t) box: every vector of the step-1 region finds its reach
    static constexpr int S1Y = TY + 2 * R, S1Z = TZ + 2 * HZ1;   // step-1 region = box of the p(t-1) and v loads
    static constexpr int S1Q = S1Z / 4, S1_ITEMS = S1Y * S1Q;
    static constexpr int S2Q = TZ / 4, S2_ITEMS = TY * S2Q, S2_ROUNDS = (S2_ITEMS + THREADS - 1) / THREADS;
    // XQ: a thread's first S2_ROUNDS step-1 vectors ARE its step-2 vectors (so that a step-1 result enters the step-2 queue
    // without leaving the thread); the vectors of the ring around the tile are dealt out after them
    static constexpr int S1_EXTRA = S1_ITEMS - S2_ITEMS;
    static constexpr int S1_ROUNDS = XQ ? S2_ROUNDS + (S1_EXTRA + THREADS - 1) / THREADS : (S1_ITEMS + THREADS - 1) / THREADS;
    static constexpr int NP = (XQ ? R + 1 : 2 * R + 1) + PF;   // p(t) ring
    static constexpr int N1 = (XQ ? R : 2 * R) + 2;   // p(t+1) ring: one more than the planes step 2 reads, so that step 1 of iteration g
                                                      // never writes a plane step 2 of iteration g-1 may still be reading
    static constexpr int NS = PF + 1;           // p(t-1) / v rings and full barriers
    static constexpr uint32_t P_BYTES = IY * IZ * 4, S_BYTES = S1Y * S1Z * 4;
    static constexpr uint32_t P_SLOT = (P_BYTES + 127) / 128 * 128, S_SLOT = (S_BYTES + 127) / 128 * 128;
    static constexpr uint32_t P_OFF = 0;
    static constexpr uint32_t P1_OFF = P_OFF + NP * P_SLOT;
    static constexpr uint32_t PV_OFF = P1_OFF + N1 * S_SLOT;
    static constexpr uint32_t V_OFF = PV_OFF + NS * S_SLOT;
    static constexpr uint32_t BAR_OFF = V_OFF + NS * S_SLOT;
    static constexpr uint32_t SMEM_BYTES = BAR_OFF + NS * 8 + 128;
    static_assert(R >= 1 && R <= TT_MAX_R, "radius");
    static_assert(TZ % 4 == 0 && IZ <= 256 && IY <= 256, "TMA box limits");
    static_assert(SMEM_BYTES <= 232448, "shared memory of one CTA");
};

// Position of a CTA in its sequence of work units (tile, x chunk).
struct TTCursor {
    int unit, j, n_it;     // j: iteration within the unit, 0 .. n_it-1 (n_it = chunk length + 4R)
    int cx0, len, y0, z0;  // chunk and tile origin, domain coordinates
};

template <class T>
YB_DEVFN void tt_unit_setup(TTCursor& cu, const TTParams& P) {
    int u = cu.unit;
    const int tz = u % P.ntz; u /= P.ntz;
    const int ty = u % P.nty; u /= P.nty;
    cu.z0 = tz * T::TZ;
    cu.y0 = ty * T::TY;
    cu.cx0 = P.cx0[u];
    cu.len = P.clen[u];
    cu.n_it = cu.len + 4 * T::R;
    cu.j = 0;
}

// The three boxes of one iteration: shared-memory offset and first element coordinates (z, y, x) in the padded arrays.
struct TTLoads {
    uint32_t p_off, pv_off, v_off, bytes;
    bool step1;                 // p(t-1) and v boxes are loaded (iteration >= 2R)
    int pz, py, px;             // p(t) box
    int sz, sy, sx;             // p(t-1) box
    int vz, vy, vx;             // v box
};

template <class T>
YB_DEVFN TTLoads tt_loads(const TTParams& P, const TTCursor& cu, unsigned g) {
    TTLoads L;
    L.step1 = cu.j >= 2 * T::R;
    L.p_off = T::P_OFF + (g % T::NP) * T::P_SLOT;
    L.pv_off = T::PV_OFF + (g % T::NS) * T::S_SLOT;
    L.v_off = T::V_OFF + (g % T::NS) * T::S_SLOT;
    L.bytes = T::P_BYTES + (L.step1 ? 2 * T::S_BYTES : 0);
    L.pz = P.pad_z + cu.z0 - 2 * T::HZ1; L.py = P.pad_y + cu.y0 - 2 * T::R; L.px = P.pad_x + cu.cx0 + cu.j - 2 * T::R;
    L.sz = P.pad_z + cu.z0 - T::HZ1;     L.sy = P.pad_y + cu.y0 - T::R;     L.sx = P.pad_x + cu.cx0 + cu.j - 3 * T::R;
    L.vz = P.vpad_z + cu.z0 - T::HZ1;    L.vy = P.vpad_y + cu.y0 - T::R;    L.vx = P.vpad_x + cu.cx0 + cu.j - 3 * T::R;
    return L;
}

// Shared-memory vector load / store.  The emulator hooks both (YB_TT_SMEM_HOOKS) to detect data races between threads inside
// one barrier interval -- the one class of error a sequential emulation of the threads cannot produce by itself.
#ifdef YB_TT_SMEM_HOOKS
void tt_hook_smem_read(const float* p);
void tt_hook_smem_write(const float* p);
YB_DEVFN TTVec4 tt_ld4(const float* p) { tt_hook_smem_read(p); return *reinterpret_cast<const TTVec4*>(p); }
YB_DEVFN void tt_sts4(float* p, const TTVec4& v) { tt_hook_smem_write(p); *reinterpret_cast<TTVec4*>(p) = v; }
#else
YB_DEVFN TTVec4 tt_ld4(const float* p) { return *reinterpret_cast<const TTVec4*>(p); }
YB_DEVFN void tt_sts4(float* p, const TTVec4& v) { *reinterpret_cast<TTVec4*>(p) = v; }
#endif
YB_DEVFN void tt_v2a(const TTVec4& v, float* a) { a[0] = v.x; a[1] = v.y; a[2] = v.z; a[3] = v.w; }

#ifndef YB_TT_HOST_EMUL
YB_DEVFN void tt_stg4(float* p, const TTVec4& v, int cs) {
    if (cs) asm volatile("st.global.cs.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
    else asm volatile("st.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
YB_DEVFN TTVec4 tt_ldg4(const float* p) {
    TTVec4 v;
    asm volatile("ld.global.nc.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}
#else
YB_DEVFN void tt_stg4(float* p, const TTVec4& v, int) { p[0] = v.x; p[1] = v.y; p[2] = v.z; p[3] = v.w; }
YB_DEVFN TTVec4 tt_ldg4(const float* p) { return *reinterpret_cast<const TTVec4*>(p); }
#endif

// Result vector -> global memory; `nv` leading lanes are inside the domain.
YB_DEVFN void tt_store(float* o, const float* r, int nv, int cs) {
    if (nv >= 4 && (reinterpret_cast<uintptr_t>(o) & 15) == 0) {
        TTVec4 v{r[0], r[1], r[2], r[3]};
        tt_stg4(o, v, cs);
    } else {
        if (nv > 0) o[0] = r[0];
        if (nv > 1) o[1] = r[1];
        if (nv > 2) o[2] = r[2];
        if (nv > 3) o[3] = r[3];
    }
}

// What a thread needs to know about its vectors ("items"), fixed for a whole work unit: worked out once per unit so that the
// sweep loop carries no divisions, bounds tests or 64-bit address arithmetic beyond one add per store.
//   step 1: item k = vector (row, q) of the step-1 region, k < S1_ROUNDS;  step 2: vector (row, q) of the tile, k < S2_ROUNDS.
template <class T>
struct TTThread {
    int io1[T::S1_ROUNDS];          // element offset of the vector in a p(t) plane; -1: no such item
    int so1[T::S1_ROUNDS];          // ... in a step-1-region plane (p1, p(t-1), v)
    int in1[T::S1_ROUNDS];          // bit i: lane i lies inside the domain in y and z
    int nv1[T::S1_ROUNDS];          // lanes to store to p(t+1) (0: the vector is not part of the tile / outside the domain)
    long long g1[T::S1_ROUNDS];     // gy * p_sy + gz
    int so2[T::S2_ROUNDS];          // element offset in a step-1-region plane; -1: no such item
    int io2[T::S2_ROUNDS];          // ... in a p(t) plane
    int nv2[T::S2_ROUNDS];          // lanes to store to p(t+2) = lanes of v to read
    long long g2[T::S2_ROUNDS];     // gy * p_sy + gz
    long long gv[T::S2_ROUNDS];     // gy * v_sy + gz
    // XQ only: the thread's own vectors of p(t) planes xl-2R .. xl (q1) and of p(t+1) planes x1-2R .. x1 (q2), newest last
    TTVec4 q1[T::S1_ROUNDS][T::QN];
    TTVec4 q2[T::S2_ROUNDS][T::QN];
};

template <class T>
YB_DEVFN void tt_thread_setup(TTThread<T>& th, const TTParams& P, const TTCursor& cu, int tid) {
    constexpr int R = T::R;
#pragma unroll
    for (int k = 0; k < T::S1_ROUNDS; k++) {
        const int item = tid + k * T::THREADS;
        th.io1[k] = -1; th.so1[k] = 0; th.in1[k] = 0; th.nv1[k] = 0; th.g1[k] = 0;
        int row = 0, q = 0;
        bool have = false;
        if (!T::XQ) {
            have = item < T::S1_ITEMS;
            row = item / T::S1Q; q = item - row * T::S1Q;
        } else if (k < T::S2_ROUNDS) {          // the thread's step-2 vectors
            have = item < T::S2_ITEMS;
            row = item / T::S2Q + R; q = item % T::S2Q + T::ZQ;
        } else {                                // ring around the tile: R rows above, R rows below, ZQ vectors left and right
            int e = tid + (k - T::S2_ROUNDS) * T::THREADS;
            have = e < T::S1_EXTRA;
            constexpr int TOP = R * T::S1Q;
            if (e < TOP) { row = e / T::S1Q; q = e % T::S1Q; }
            else if (e < 2 * TOP) { e -= TOP; row = R + T::TY + e / T::S1Q; q = e % T::S1Q; }
            else { e -= 2 * TOP; row = R + e / (2 * T::ZQ); const int c = e % (2 * T::ZQ); q = c < T::ZQ ? c : T::S2Q + c; }
        }
        if (have) {
            const int gy = cu.y0 - R + row, gz = cu.z0 - T::HZ1 + 4 * q;
            th.io1[k] = (row + R) * T::IZ + T::HZ1 + 4 * q;   // p(t) planes start at row y0-2R, column z0-2*HZ1
            th.so1[k] = row * T::S1Z + 4 * q;                 // step-1 planes start at row y0-R, column z0-HZ1
            int m = 0;
            if (gy >= -P.ext_lo[1] && gy < P.ny + P.ext_hi[1])
                for (int i = 0; i < 4; i++) if (gz + i >= -P.ext_lo[2] && gz + i < P.nz + P.ext_hi[2]) m |= 1 << i;
            th.in1[k] = m;
            const bool centre = row >= R && row < R + T::TY && q >= T::ZQ && q < T::ZQ + T::S2Q;
            if (centre && gy < P.ny && gz < P.nz) {
                th.nv1[k] = P.nz - gz < 4 ? P.nz - gz : 4;
                th.g1[k] = (long long)gy * P.p_sy + gz;
            }
        }
    }
#pragma unroll
    for (int k = 0; k < T::S2_ROUNDS; k++) {
        const int item = tid + k * T::THREADS;
        th.so2[k] = -1; th.io2[k] = 0; th.nv2[k] = 0; th.g2[k] = 0; th.gv[k] = 0;
        if (item < T::S2_ITEMS) {
            const int row = item / T::S2Q, q = item - row * T::S2Q;
            const int gy = cu.y0 + row, gz = cu.z0 + 4 * q;
            th.so2[k] = (row + R) * T::S1Z + T::HZ1 + 4 * q;
            th.io2[k] = (row + 2 * R) * T::IZ + 2 * T::HZ1 + 4 * q;
            if (gy < P.ny && gz < P.nz) {
                th.nv2[k] = P.nz - gz < 4 ? P.nz - gz : 4;
                th.g2[k] = (long long)gy * P.p_sy + gz;
                th.gv[k] = (long long)gy * P.v_sy + gz;
            }
        }
    }
}

// Ring positions of the current iteration g (uniform over the CTA), advanced without divisions.
YB_DEVFN int tt_wrap(int i, int n) { return i < 0 ? i + n : (i >= n ? i - n : i); }
template <class T>
struct TTRing {
    int gp, g1, gs;        // g mod NP, g mod N1, g mod NS
    uint32_t parity;       // (g / NS) & 1: phase parity of full[gs]
    YB_DEVMEM void start() { gp = g1 = gs = 0; parity = 0; }
    YB_DEVMEM void advance() {
        if (++gp == T::NP) gp = 0;
        if (++g1 == T::N1) g1 = 0;
        if (++gs == T::NS) { gs = 0; parity ^= 1u; }
    }
    // plane loaded (p) / produced (p1) `back` iterations ago
    YB_DEVMEM const float* p(const uint8_t* sm, int back) const { return reinterpret_cast<const float*>(sm + T::P_OFF + tt_wrap(gp - back, T::NP) * T::P_SLOT); }
    YB_DEVMEM const float* p1(const uint8_t* sm, int back) const { return reinterpret_cast<const float*>(sm + T::P1_OFF + tt_wrap(g1 - back, T::N1) * T::S_SLOT); }
};

// v(x2) of the thread's step-2 vectors, fetched before step 1 so that the latency hides behind it.
template <class T>
YB_DEVFN void tt_load_v(const TTParams& P, const TTCursor& cu, const TTThread<T>& th, int j, TTVec4* vreg) {
    if (j < 4 * T::R) return;
    const float* vx = P.vel + (long long)(cu.cx0 + j - 4 * T::R) * P.v_sx;
#pragma unroll
    for (int k = 0; k < T::S2_ROUNDS; k++) {
        vreg[k] = TTVec4{0.f, 0.f, 0.f, 0.f};
        const int nv = th.nv2[k];
        if (nv == 0) continue;
        const float* vp = vx + th.gv[k];
        if (nv == 4 && (reinterpret_cast<uintptr_t>(vp) & 15) == 0) vreg[k] = tt_ldg4(vp);
        else {
            vreg[k].x = vp[0];
            if (nv > 1) vreg[k].y = vp[1];
            if (nv > 2) vreg[k].z = vp[2];
            if (nv > 3) vreg[k].w = vp[3];
        }
    }
}

// One vector (4 z-consecutive points) of the star: centre plane `pc`, the x neighbours' planes, row pitch `pitch`.
// `o` = element offset of the vector in each plane.  Returns acc[4] and the centre values.
template <class T, int MODE>
YB_DEVFN void tt_star(const TTParams& P, const float* pc, const float* const* pxm, const float* const* pxp, int pitch, int o,
                      float* acc, float* centre) {
    constexpr int R = T::R, HZ1 = T::HZ1, ZQ = T::ZQ;
    float zw[4 + 2 * HZ1];
#pragma unroll
    for (int kq = -ZQ; kq <= ZQ; kq++) tt_v2a(tt_ld4(pc + o + 4 * kq), &zw[4 * (kq + ZQ)]);
#pragma unroll
    for (int i = 0; i < 4; i++) { centre[i] = zw[HZ1 + i]; acc[i] = 0.f; }
#pragma unroll
    for (int r = 1; r <= R; r++) {
        float xm[4], xp[4], ym[4], yp[4];
        tt_v2a(tt_ld4(pxm[r - 1] + o), xm);
        tt_v2a(tt_ld4(pxp[r - 1] + o), xp);
        tt_v2a(tt_ld4(pc + o - r * pitch), ym);
        tt_v2a(tt_ld4(pc + o + r * pitch), yp);
#pragma unroll
        for (int i = 0; i < 4; i++)
            acc[i] = iso_group<MODE>(acc[i], centre[i], P.c[0], P.c[r], xm[i], xp[i], ym[i], yp[i], zw[HZ1 + i - r], zw[HZ1 + i + r], r == 1);
    }
}

// Step 1 of iteration j: p(t+1) at plane x1 = cx0 + j - 3R over the step-1 region.
//   p(t) plane x1 was loaded R iterations ago, planes x1 -/+ r were loaded R +/- r iterations ago.
template <class T, int MODE>
YB_DEVFN void tt_step1(uint8_t* sm, const TTParams& P, const TTCursor& cu, const TTThread<T>& th, const TTRing<T>& rg, int j) {
    constexpr int R = T::R;
    if (j < 2 * R) return;
    const int x1 = cu.cx0 + j - 3 * R;
    const float* pc = rg.p(sm, R);
    const float *pxm[R], *pxp[R];
#pragma unroll
    for (int r = 1; r <= R; r++) { pxm[r - 1] = rg.p(sm, R + r); pxp[r - 1] = rg.p(sm, R - r); }
    const float* prevp = reinterpret_cast<const float*>(sm + T::PV_OFF + rg.gs * T::S_SLOT);
    const float* vp = reinterpret_cast<const float*>(sm + T::V_OFF + rg.gs * T::S_SLOT);
    float* p1 = reinterpret_cast<float*>(sm + T::P1_OFF + rg.g1 * T::S_SLOT);
    const bool x_in = x1 >= -P.ext_lo[0] && x1 < P.nx + P.ext_hi[0];
    const bool x_store = x1 >= cu.cx0 && x1 < cu.cx0 + cu.len;
    float* o1 = P.out1 + (long long)x1 * P.p_sx;
#pragma unroll
    for (int k = 0; k < T::S1_ROUNDS; k++) {
        const int io = th.io1[k];
        if (io >= 0) {
            const int so = th.so1[k];
            float acc[4], centre[4], pv[4], vv[4], res[4];
            tt_star<T, MODE>(P, pc, pxm, pxp, T::IZ, io, acc, centre);
            tt_v2a(tt_ld4(prevp + so), pv);
            tt_v2a(tt_ld4(vp + so), vv);
            // points outside the domain keep p(t-1): what the halo cells of p(t+1) hold in the reference's two-slot storage
            const int m = x_in ? th.in1[k] : 0;
#pragma unroll
            for (int i = 0; i < 4; i++) res[i] = iso_final<MODE>(acc[i], centre[i], pv[i], vv[i]);
            if (m != 15) {
#pragma unroll
                for (int i = 0; i < 4; i++) if (!((m >> i) & 1)) res[i] = pv[i];
            }
            tt_sts4(p1 + so, TTVec4{res[0], res[1], res[2], res[3]});
            if (x_store && th.nv1[k] > 0) tt_store(o1 + th.g1[k], res, th.nv1[k], P.st_cs);
        }
    }
}

// Step 2 of iteration j: p(t+2) at plane x2 = cx0 + j - 4R over the tile.
//   p1 plane x2 was produced R iterations ago (x2 +/- r: R -/+ r ago); p(t) plane x2 ("prev") was loaded 2R iterations ago.
template <class T, int MODE>
YB_DEVFN void tt_step2(uint8_t* sm, const TTParams& P, const TTCursor& cu, const TTThread<T>& th, const TTRing<T>& rg, int j, const TTVec4* vreg) {
    constexpr int R = T::R;
    if (j < 4 * R) return;
    const int x2 = cu.cx0 + j - 4 * R;
    const float* pc = rg.p1(sm, R);
    const float *pxm[R], *pxp[R];
#pragma unroll
    for (int r = 1; r <= R; r++) { pxm[r - 1] = rg.p1(sm, R + r); pxp[r - 1] = rg.p1(sm, R - r); }
    const float* prevp = rg.p(sm, 2 * R);
    float* o2 = P.out2 + (long long)x2 * P.p_sx;
#pragma unroll
    for (int k = 0; k < T::S2_ROUNDS; k++) {
        const int so = th.so2[k];
        if (so >= 0 && th.nv2[k] > 0) {
            float acc[4], centre[4], pv[4], vv[4], res[4];
            tt_star<T, MODE>(P, pc, pxm, pxp, T::S1Z, so, acc, centre);
            tt_v2a(tt_ld4(prevp + th.io2[k]), pv);
            tt_v2a(vreg[k], vv);
#pragma unroll
            for (int i = 0; i < 4; i++) res[i] = iso_final<MODE>(acc[i], centre[i], pv[i], vv[i]);
            tt_store(o2 + th.g2[k], res, th.nv2[k], P.st_cs);
        }
    }
}

// ---- XQ = 1 -------------------------------------------------------------------------------------------------------------
// One vector of the star with the centre and the x neighbours taken from a register queue `qv` (qv[R] = centre plane, qv[R -/+ r]
// = planes -/+ r); y and z neighbours from the shared-memory plane `pc`.
template <class T, int MODE>
YB_DEVFN void tt_star_q(const TTParams& P, const float* pc, int pitch, int o, const TTVec4* qv, float* acc, float* centre) {
    constexpr int R = T::R, HZ1 = T::HZ1, ZQ = T::ZQ;
    float zw[4 + 2 * HZ1];
#pragma unroll
    for (int kq = -ZQ; kq <= ZQ; kq++) {
        if (kq == 0) tt_v2a(qv[R], &zw[4 * ZQ]);
        else tt_v2a(tt_ld4(pc + o + 4 * kq), &zw[4 * (kq + ZQ)]);
    }
#pragma unroll
    for (int i = 0; i < 4; i++) { centre[i] = zw[HZ1 + i]; acc[i] = 0.f; }
#pragma unroll
    for (int r = 1; r <= R; r++) {
        float xm[4], xp[4], ym[4], yp[4];
        tt_v2a(qv[R - r], xm);
        tt_v2a(qv[R + r], xp);
        tt_v2a(tt_ld4(pc + o - r * pitch), ym);
        tt_v2a(tt_ld4(pc + o + r * pitch), yp);
#pragma unroll
        for (int i = 0; i < 4; i++)
            acc[i] = iso_group<MODE>(acc[i], centre[i], P.c[0], P.c[r], xm[i], xp[i], ym[i], yp[i], zw[HZ1 + i - r], zw[HZ1 + i + r], r == 1);
    }
}

// Step 1, XQ: EVERY iteration pushes the thread's vectors of the newest p(t) plane (xl = cx0 + j - 2R) into q1; from
// iteration 2R on p(t+1) at plane x1 = xl - R is computed (q1[R] = plane x1) and the results of the thread's step-2 vectors
// are pushed into q2.
template <class T, int MODE>
YB_DEVFN void tt_step1_xq(uint8_t* sm, const TTParams& P, const TTCursor& cu, TTThread<T>& th, const TTRing<T>& rg, int j) {
    constexpr int R = T::R, QN = T::QN;
    const int x1 = cu.cx0 + j - 3 * R;
    const float* pnew = rg.p(sm, 0);
    const float* pc = rg.p(sm, R);
    const float* prevp = reinterpret_cast<const float*>(sm + T::PV_OFF + rg.gs * T::S_SLOT);
    const float* vp = reinterpret_cast<const float*>(sm + T::V_OFF + rg.gs * T::S_SLOT);
    float* p1 = reinterpret_cast<float*>(sm + T::P1_OFF + rg.g1 * T::S_SLOT);
    const bool x_in = x1 >= -P.ext_lo[0] && x1 < P.nx + P.ext_hi[0];
    const bool x_store = x1 >= cu.cx0 && x1 < cu.cx0 + cu.len;
    float* o1 = P.out1 + (long long)x1 * P.p_sx;
#pragma unroll
    for (int k = 0; k < T::S1_ROUNDS; k++) {
        // The queues shift on EVERY iteration and for every k, outside all conditions (a queue that is modified under a
        // branch costs a register move per entry at the join); a thread without this item shifts garbage it never uses.
        const int io = th.io1[k];
        const bool have = io >= 0;
#pragma unroll
        for (int i = 0; i + 1 < QN; i++) th.q1[k][i] = th.q1[k][i + 1];
        th.q1[k][QN - 1] = tt_ld4(pnew + (have ? io : 0));
        TTVec4 rv{0.f, 0.f, 0.f, 0.f};
        if (have && j >= 2 * R) {
            const int so = th.so1[k];
            float acc[4], centre[4], pv[4], vv[4], res[4];
            tt_star_q<T, MODE>(P, pc, T::IZ, io, th.q1[k], acc, centre);
            tt_v2a(tt_ld4(prevp + so), pv);
            tt_v2a(tt_ld4(vp + so), vv);
            const int m = x_in ? th.in1[k] : 0;
#pragma unroll
            for (int i = 0; i < 4; i++) res[i] = iso_final<MODE>(acc[i], centre[i], pv[i], vv[i]);
            if (m != 15) {
#pragma unroll
                for (int i = 0; i < 4; i++) if (!((m >> i) & 1)) res[i] = pv[i];
            }
            rv = TTVec4{res[0], res[1], res[2], res[3]};
            tt_sts4(p1 + so, rv);
            if (x_store && th.nv1[k] > 0) tt_store(o1 + th.g1[k], res, th.nv1[k], P.st_cs);
        }
        if (k < T::S2_ROUNDS) {
#pragma unroll
            for (int i = 0; i + 1 < QN; i++) th.q2[k][i] = th.q2[k][i + 1];
            th.q2[k][QN - 1] = rv;
        }
    }
}

// Step 2, XQ: p(t+2) at plane x2 = x1 - R: centre and x neighbours from q2 (q2[R] = plane x2), y / z neighbours from the p1
// plane produced R iterations ago, "prev" = p(t) at plane x2 = the oldest entry of q1.
template <class T, int MODE>
YB_DEVFN void tt_step2_xq(uint8_t* sm, const TTParams& P, const TTCursor& cu, const TTThread<T>& th, const TTRing<T>& rg, int j, const TTVec4* vreg) {
    constexpr int R = T::R;
    if (j < 4 * R) return;
    const int x2 = cu.cx0 + j - 4 * R;
    const float* pc = rg.p1(sm, R);
    float* o2 = P.out2 + (long long)x2 * P.p_sx;
#pragma unroll
    for (int k = 0; k < T::S2_ROUNDS; k++) {
        const int so = th.so2[k];
        if (so >= 0 && th.nv2[k] > 0) {
            float acc[4], centre[4], pv[4], vv[4], res[4];
            tt_star_q<T, MODE>(P, pc, T::S1Z, so, th.q2[k], acc, centre);
            tt_v2a(th.q1[k][0], pv);
            tt_v2a(vreg[k], vv);
#pragma unroll
            for (int i = 0; i < 4; i++) res[i] = iso_final<MODE>(acc[i], centre[i], pv[i], vv[i]);
            tt_store(o2 + th.g2[k], res, th.nv2[k], P.st_cs);
        }
    }
}

// The sweep of one CTA, written once for both back ends.  BE supplies the execution model:
//   threads(f)   run f(tid) for every thread of the CTA        (device: f(threadIdx.x); emulator: a loop)
//   once(f)      run f() on the producer thread                  (device: thread 0)
//   barrier()    CTA-wide barrier                                (device: __syncthreads)
//   issue(L, b)  start the TMA box loads L, completing on full barrier b
//   wait_full(b, parity)  block until that phase of barrier b has completed
//   thread(tid)  the thread's TTThread; vreg(tid): its S2_ROUNDS vectors of v that live across step 1
// Ring-slot reuse (all indexed by the CTA's running iteration count g, across unit boundaries):
//   p(t) slot of iteration g+PF held iteration g-2R-1: last read by step 1 / step 2 ("prev") of iteration g-1;
//   p(t-1) / v slot and full barrier of g+PF held iteration g-1: read / waited on in iteration g-1;
//   -> the loads of iteration g+PF are issued right after the barrier of iteration g.
//   p1 slot of iteration g held iteration g-2R-2: last read by step 2 of iteration g-2, which the barrier of g-1 closes.
template <class T, int MODE, class BE>
YB_DEVFN void tt_sweep(BE& be, uint8_t* sm, const TTParams& P, int first_unit, int unit_stride) {
    const int nunits = P.nty * P.ntz * P.nchunks;
    // producer cursor: PF iterations ahead of the sweep (only the producer thread's copy advances)
    TTCursor pr;
    pr.unit = first_unit; pr.j = 0; pr.n_it = 0; pr.cx0 = pr.len = pr.y0 = pr.z0 = 0;
    unsigned pg = 0;
    bool pr_live = pr.unit < nunits;
    if (pr_live) tt_unit_setup<T>(pr, P);
    auto produce_one = [&]() {
        const TTLoads L = tt_loads<T>(P, pr, pg);
        be.issue(L, int(pg % T::NS));
        pg++;
        if (++pr.j == pr.n_it) {
            pr.unit += unit_stride;
            if (pr.unit < nunits) tt_unit_setup<T>(pr, P); else pr_live = false;
        }
    };
    be.once([&]() { for (int k = 0; k < T::PF && pr_live; k++) produce_one(); });

    TTCursor cu;
    TTRing<T> rg;
    rg.start();
    for (cu.unit = first_unit; cu.unit < nunits; cu.unit += unit_stride) {
        tt_unit_setup<T>(cu, P);
        be.threads([&](int tid) { tt_thread_setup<T>(be.thread(tid), P, cu, tid); });
#pragma unroll 1
        for (int j = 0; j < cu.n_it; j++) {
            be.threads([&](int tid) { tt_load_v<T>(P, cu, be.thread(tid), j, be.vreg(tid)); });
            be.wait_full(rg.gs, rg.parity);
            be.threads([&](int tid) {
                if (T::XQ) tt_step1_xq<T, MODE>(sm, P, cu, be.thread(tid), rg, j);
                else tt_step1<T, MODE>(sm, P, cu, be.thread(tid), rg, j);
            });
            be.barrier();     // p1 plane of this iteration visible; every thread is done with iteration g-1
            be.once([&]() { if (pr_live) produce_one(); });     // loads of iteration g+PF
            be.threads([&](int tid) {
                if (T::XQ) tt_step2_xq<T, MODE>(sm, P, cu, be.thread(tid), rg, j, be.vreg(tid));
                else tt_step2<T, MODE>(sm, P, cu, be.thread(tid), rg, j, be.vreg(tid));
            });
            rg.advance();
        }
    }
}

}  // namespace yb

#ifndef YB_TT_HOST_EMUL
#include "yb_ptx.cuh"

namespace yb {

struct TTMaps {
    CUtensorMap pin;   // p(t),   box (IZ, IY, 1)
    CUtensorMap prev;  // p(t-1), box (S1Z, S1Y, 1)
    CUtensorMap v;     // v,      box (S1Z, S1Y, 1)
};

template <class T>
struct TTDevice {
    uint8_t* sbase;
    uint64_t* full_bar;
    const TTMaps* M;
    uint64_t pol_p;        // L2 policy of the p(t) box
    TTVec4 v[T::S2_ROUNDS];
    TTThread<T> th;
    __device__ __forceinline__ TTThread<T>& thread(int) { return th; }
    template <class F> __device__ __forceinline__ void threads(F f) { f(int(threadIdx.x)); }
    template <class F> __device__ __forceinline__ void once(F f) { if (threadIdx.x == 0) f(); }
    __device__ __forceinline__ void barrier() { __syncthreads(); }
    __device__ __forceinline__ void wait_full(int b, uint32_t parity) { mbar_wait_or_trap(&full_bar[b], parity); }
    __device__ __forceinline__ TTVec4* vreg(int) { return v; }
    __device__ __forceinline__ void issue(const TTLoads& L, int b) {
        uint64_t* fb = &full_bar[b];
        mbar_arrive_expect_tx(fb, L.bytes);
        tma_load_3d_hint(sbase + L.p_off, &M->pin, fb, L.pz, L.py, L.px, pol_p);
        if (L.step1) {
            tma_load_3d(sbase + L.pv_off, &M->prev, fb, L.sz, L.sy, L.sx);
            tma_load_3d(sbase + L.v_off, &M->v, fb, L.vz, L.vy, L.vx);
        }
    }
};

template <class T, int MODE>
__global__ void __launch_bounds__(T::THREADS, 1)
iso3dfd_tt2_kernel(const __grid_constant__ TTMaps M, const __grid_constant__ TTParams P) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 127u) & ~127u;
    TTDevice<T> be;
    be.sbase = smem_raw + (base - smem_u32(smem_raw));
    be.full_bar = reinterpret_cast<uint64_t*>(be.sbase + T::BAR_OFF);
    be.M = &M;
    be.pol_p = l2_policy(P.pol_p);
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&M.pin); tma_prefetch_desc(&M.prev); tma_prefetch_desc(&M.v);
        for (int s = 0; s < T::NS; s++) mbar_init(&be.full_bar[s], 1);
        fence_barrier_init();
    }
    __syncthreads();
    tt_sweep<T, MODE>(be, be.sbase, P, int(blockIdx.x), int(gridDim.x));
}

}  // namespace yb
#endif
