// Average-of-points stencils for sm_90a: 3axis, 3axis_with_diags, 3plane and cube at any radius 1..8, fp32 or fp64.
//
// Equation: the reference's src/stencils/SimpleStencils.cpp.  AvePtsStencil::define starts from the centre point, the shape's
// add_points adds its points (AxisStencil, DiagStencil, PlaneStencil and CubeStencil, each after its base class's) and the sum is
// multiplied by 1.0 / pts.  The reference's compiler front-end flattens the chain of `v += a + b + ...` into ONE left-to-right
// sum in the order the points are written, then one multiply (oracle/gen/s3axis.gen.h at radius 4):
//
//   A(t+1) = (((A(0,0,0) + A(-1,0,0)) + A(+1,0,0)) + ... ) * (1/pts)
//
// Both kernels here add in exactly that order, one rounded addition per point, so they give the reference's bits.  No product
// feeds an addition, so every FP mode computes the same bits and the kernels have no FP-mode variants.
#pragma once
#include "yb_iso3dfd.cuh"
#include "yb_ptx.cuh"

namespace yb {

enum AvpShape { AVP_3AXIS = 0, AVP_DIAGS = 1, AVP_PLANE = 2, AVP_CUBE = 3 };
constexpr int AVP_MAX_R = 8;
constexpr int AVP_MAX_CHUNKS = 40;

template <class E>
struct AvpParamsT {
    E* out;                 // element (0,0,0) of the rank domain in the slot of t+1
    const E* cur;           // the same in the slot of t (direct kernel only)
    long long sx, sy;       // element strides of A (z stride is 1)
    int x_begin, x_end, y_begin, y_end, z_begin, z_end;     // box to compute, rank-domain coordinates
    int pad_x, pad_y, pad_z;                                 // alloc index of the domain origin (TMA coordinates)
    int nty, ntz, nchunks;                                   // (y, z) tiles of the box and x chunks
    int cx0[AVP_MAX_CHUNKS], clen[AVP_MAX_CHUNKS];           // every chunk's first plane and number of planes
    E scale;                                                  // 1/pts, as the reference's generated code holds it
};

// The points after the centre of shapes up to 3plane, in the reference's order: f(dx, dy, dz) once per axis and diagonal point, fp
// once per in-plane point.  With a compile-time radius (the sweep kernel) the axis and diagonal loops unroll and those points'
// offsets are constants; the in-plane loops, 12 R (R - 1) points, stay loops (unrolled, their loads spill at radius 3 and up).
template <int SHAPE, class F, class FP>
__device__ __forceinline__ void avp_star_points(int R, F&& f, FP&& fp) {
#pragma unroll
    for (int r = 1; r <= R; r++) { f(-r, 0, 0); f(r, 0, 0); f(0, -r, 0); f(0, r, 0); f(0, 0, -r); f(0, 0, r); }
    if constexpr (SHAPE >= AVP_DIAGS) {
#pragma unroll
        for (int r = 1; r <= R; r++) {
            f(-r, -r, 0); f(r, -r, 0); f(-r, r, 0); f(r, r, 0);
            f(-r, 0, -r); f(r, 0, r); f(-r, 0, r); f(r, 0, -r);
            f(0, -r, -r); f(0, r, r); f(0, -r, r); f(0, r, -r);
        }
    }
    if constexpr (SHAPE >= AVP_PLANE) {
#pragma unroll 1
        for (int r = 1; r <= R; r++) {
#pragma unroll 1
            for (int m = r + 1; m <= R; m++) {
                fp(-r, -m, 0); fp(-m, -r, 0); fp(r, m, 0); fp(m, r, 0); fp(-r, m, 0); fp(-m, r, 0); fp(r, -m, 0); fp(m, -r, 0);
                fp(-r, 0, -m); fp(-m, 0, -r); fp(r, 0, m); fp(m, 0, r); fp(-r, 0, m); fp(-m, 0, r); fp(r, 0, -m); fp(m, 0, -r);
                fp(0, -r, -m); fp(0, -m, -r); fp(0, r, m); fp(0, m, r); fp(0, -r, m); fp(0, -m, r); fp(0, r, -m); fp(0, m, -r);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------------------
// Reference-order direct kernel: one thread per point, straight global loads.  Thin slabs, boxes whose z start is off a 16-byte
// boundary, kernel=direct and the on-device cross-check of the sweep.
// ---------------------------------------------------------------------------------------------------------------------------------
template <class E, int SHAPE>
__global__ void __launch_bounds__(128) avepts_direct_kernel(AvpParamsT<E> P, int R) {
    const int z = P.z_begin + blockIdx.x * blockDim.x + threadIdx.x;
    const int y = P.y_begin + blockIdx.y;
    const int x = P.x_begin + blockIdx.z;
    if (z >= P.z_end || y >= P.y_end || x >= P.x_end) return;
    const long long o = (long long)x * P.sx + (long long)y * P.sy + z;
    const E* c = P.cur + o;
    E acc = c[0];
    auto add = [&](int dx, int dy, int dz) { acc = acc + c[dx * P.sx + dy * P.sy + dz]; };
    avp_star_points<SHAPE>(R, add, add);
    if constexpr (SHAPE == AVP_CUBE) {
        for (int rx = 1; rx <= R; rx++)
            for (int ry = 1; ry <= R; ry++)
                for (int rz = 1; rz <= R; rz++) {
                    const long long px = rx * P.sx, py = ry * P.sy;
                    acc = acc + c[px + py + rz];
                    acc = acc + c[px - py - rz];
                    acc = acc + c[px + py - rz];
                    acc = acc + c[px - py + rz];
                    acc = acc + c[-px + py + rz];
                    acc = acc + c[-px - py - rz];
                    acc = acc + c[-px + py - rz];
                    acc = acc + c[-px - py + rz];
                }
    }
    P.out[o] = acc * P.scale;
}

// ---------------------------------------------------------------------------------------------------------------------------------
// TMA-staged sweep along x.
//
// A CTA owns a (TY x TZ) column of the (y, z) plane and sweeps it along x over a chunk of planes.  A producer warp (one lane) loads
// every plane of A(t) the chunk reads -- the tile plus R rows and HZ columns of halo -- ONCE, with one TMA box load, into a ring of
// NS = 2R+1+PF shared-memory slots: the 2R+1 planes one output plane reads, plus PF planes of prefetch.  A slot is released when the
// output plane R above it is done, so the diagonal, in-plane and octant points, which read other x planes at (y, z) offsets, come
// from shared memory like the centre plane's.  full/empty mbarriers, no __syncthreads in the sweep.
//
// A consumer thread owns one 16-byte vector of one row (4 fp32 or 2 fp64 points) and adds its points in the reference's order.  A
// point at a z offset that is not a whole vector is assembled from the two aligned vectors it straddles.  The cube's octant points,
// 8 R^3 of them, take their values from register windows instead: for each (rx, ry) the four rows (+-rx, +-ry) are loaded once as
// whole vectors over the z window [-HZ, VW + HZ), and the 8 R points of that (rx, ry) read them by constant register index.  Results
// leave as 128-bit streaming stores into the slot of t+1 (scalars on ragged edges).
//
// Persistent grid: units (z tile, y tile, x chunk) are dealt round-robin, so the units in flight are neighbours in (y, z) and share
// their halos through L2.
// ---------------------------------------------------------------------------------------------------------------------------------
template <int SHAPE_, int R_, class E_, int TY_, int TZ_, int PF_>
struct AvpTile {
    using E = E_;
    using V = typename IsoVec<E>::V;
    static constexpr int SHAPE = SHAPE_, R = R_, TY = TY_, TZ = TZ_, PF = PF_;
    static constexpr int VW = IsoVec<E>::N;
    static constexpr int ES = int(sizeof(E));
    static constexpr int HZ = (R + VW - 1) / VW * VW;           // z halo of a plane, whole vectors
    static constexpr int HP = TZ + 2 * HZ;                      // elements per row of a staged plane
    static constexpr int HROWS = TY + 2 * R;
    static constexpr int TZV = TZ / VW;                         // threads per row
    static constexpr int THREADS = TY * TZV;                    // consumer threads; one producer warp follows them
    static constexpr int NWARPS = THREADS / 32;
    static constexpr int NS = 2 * R + 1 + PF;
    static constexpr uint32_t PLANE_BYTES = uint32_t(HROWS) * HP * ES;
    static constexpr uint32_t SLOT_BYTES = (PLANE_BYTES + 127) / 128 * 128;
    static constexpr uint32_t BAR_OFF = NS * SLOT_BYTES;
    static constexpr uint32_t SMEM_BYTES = BAR_OFF + 2 * NS * 8 + 128;
    static_assert(THREADS % 32 == 0, "whole warps");
    static_assert(TZ % VW == 0 && HP <= 256 && HROWS <= 256, "TMA box limits");
    static_assert(SMEM_BYTES <= 232448, "over the sm_90 opt-in shared memory per block");
};

// The VW values of the point dz elements past the thread's vector at `p` (shared memory).
template <class T>
__device__ __forceinline__ void avp_load_point(const uint8_t* p, int dz, typename T::E (&v)[T::VW]) {
    using E = typename T::E;
    using V = typename T::V;
    constexpr int VW = T::VW;
    const int lo = (dz + 64) / VW - 64 / VW;                    // floor(dz / VW)
    const int sh = dz - lo * VW;
    E a[VW];
    f4_to_arr(*reinterpret_cast<const V*>(p + lo * 16), a);
    if (sh == 0) {
#pragma unroll
        for (int i = 0; i < VW; i++) v[i] = a[i];
    } else {
        E b[VW];
        f4_to_arr(*reinterpret_cast<const V*>(p + (lo + 1) * 16), b);
#pragma unroll
        for (int i = 0; i < VW; i++) v[i] = i + sh < VW ? a[i + sh] : b[i + sh - VW];
    }
}

// The sum, in the reference's order, of the points of one 16-byte vector staged in shared memory: pl[R + dx] is the vector in the
// plane dx away (dx = -R..R), plane(dx) the same for a run-time dx, and rows are ROWB bytes apart.  acc comes back unscaled.
template <class T, int ROWB, class PF>
__device__ __forceinline__ void avp_sum(const uint8_t* const* pl, PF&& plane, typename T::E (&acc)[T::VW]) {
    using E = typename T::E;
    using V = typename T::V;
    constexpr int R = T::R, VW = T::VW, ES = T::ES, HZ = T::HZ;
    avp_load_point<T>(pl[R], 0, acc);
    avp_star_points<T::SHAPE>(
        R,
        [&](int dx, int dy, int dz) {
            E v[VW];
            avp_load_point<T>(pl[R + dx] + dy * ROWB, dz, v);
#pragma unroll
            for (int i = 0; i < VW; i++) acc[i] = acc[i] + v[i];
        },
        [&](int dx, int dy, int dz) {       // run-time offsets: one scalar load per element
            const E* v = reinterpret_cast<const E*>(plane(dx) + dy * ROWB) + dz;
#pragma unroll
            for (int i = 0; i < VW; i++) acc[i] = acc[i] + v[i];
        });
    if constexpr (T::SHAPE == AVP_CUBE) {
        constexpr int WN = VW + 2 * HZ;
#pragma unroll 1
        for (int rx = 1; rx <= R; rx++) {
#pragma unroll 1
            for (int ry = 1; ry <= R; ry++) {
                // rows (rx, ry), (rx, -ry), (-rx, ry), (-rx, -ry) over the z window [-HZ, VW + HZ)
                E w[4][WN];
                const uint8_t *px = plane(rx), *mx = plane(-rx);
                const uint8_t* ro[4] = {px + ry * ROWB, px - ry * ROWB, mx + ry * ROWB, mx - ry * ROWB};
#pragma unroll
                for (int k = 0; k < 4; k++)
#pragma unroll
                    for (int c = 0; c < WN / VW; c++)
                        f4_to_arr(*reinterpret_cast<const V*>(ro[k] + (c * VW - HZ) * ES), &w[k][c * VW]);
#pragma unroll
                for (int rz = 1; rz <= R; rz++)
#pragma unroll
                    for (int i = 0; i < VW; i++) {
                        E a = acc[i];
                        a = a + w[0][HZ + i + rz];      // ( rx,  ry,  rz)
                        a = a + w[1][HZ + i - rz];      // ( rx, -ry, -rz)
                        a = a + w[0][HZ + i - rz];      // ( rx,  ry, -rz)
                        a = a + w[1][HZ + i + rz];      // ( rx, -ry,  rz)
                        a = a + w[2][HZ + i + rz];      // (-rx,  ry,  rz)
                        a = a + w[3][HZ + i - rz];      // (-rx, -ry, -rz)
                        a = a + w[2][HZ + i - rz];      // (-rx,  ry, -rz)
                        a = a + w[3][HZ + i + rz];      // (-rx, -ry,  rz)
                        acc[i] = a;
                    }
            }
        }
    }
}

template <class T>
__global__ void __launch_bounds__(T::THREADS + 32, 1)
avepts_sweep_kernel(const __grid_constant__ CUtensorMap M, const __grid_constant__ AvpParamsT<typename T::E> P) {
    using E = typename T::E;
    using V = typename T::V;
    constexpr int R = T::R, NS = T::NS, VW = T::VW, ES = T::ES, HZ = T::HZ, HP = T::HP;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 127u) & ~127u;
    uint8_t* sbase = smem_raw + (base - smem_u32(smem_raw));
    uint64_t* full = reinterpret_cast<uint64_t*>(sbase + T::BAR_OFF);
    uint64_t* empty = full + NS;

    const int tid = threadIdx.x;
    const int lane = tid & 31;
    const int nunits = P.nty * P.ntz * P.nchunks;
    if (tid == 0) {
        tma_prefetch_desc(&M);
        for (int s = 0; s < NS; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], T::NWARPS); }
        fence_barrier_init();
    }
    __syncthreads();

    // unit -> (z tile, y tile, chunk): first plane, planes, tile origin
    auto unit_of = [&](int u, int& x0, int& len, int& y0, int& z0) {
        const int tz = u % P.ntz; u /= P.ntz;
        const int ty = u % P.nty; u /= P.nty;
        z0 = P.z_begin + tz * T::TZ;
        y0 = P.y_begin + ty * T::TY;
        x0 = P.cx0[u];
        len = P.clen[u];
    };

    // ---- producer warp: one lane loads planes x0-R .. x0+len-1+R of every unit of this CTA, in order ----
    if (tid >= T::THREADS) {
        if (tid != T::THREADS) return;
        uint32_t g = 0;
        for (int u = blockIdx.x; u < nunits; u += gridDim.x) {
            int x0, len, y0, z0;
            unit_of(u, x0, len, y0, z0);
            for (int k = 0; k < len + 2 * R; k++, g++) {
                const int s = int(g % NS);
                mbar_wait(&empty[s], ((g / NS) & 1u) ^ 1u);
                mbar_arrive_expect_tx(&full[s], T::PLANE_BYTES);
                tma_load_3d(sbase + s * T::SLOT_BYTES, &M, &full[s], P.pad_z + z0 - HZ, P.pad_y + y0 - R, P.pad_x + x0 - R + k);
            }
        }
        return;
    }

    // ---- consumers ----
    const int ty = tid / T::TZV;
    const int q = tid % T::TZV;
    const uint32_t own = uint32_t(((ty + R) * HP + HZ + VW * q) * ES);      // the thread's vector in a slot
    uint32_t g0 = 0;                                                        // sequence number of the unit's first plane
    auto wait_plane = [&](uint32_t g) { mbar_wait(&full[g % NS], (g / NS) & 1u); };
    for (int u = blockIdx.x; u < nunits; u += gridDim.x) {
        int x0, len, y0, z0;
        unit_of(u, x0, len, y0, z0);
        const int y = y0 + ty, zq = z0 + VW * q;
        const int nv = y < P.y_end ? max(0, min(VW, P.z_end - zq)) : 0;
        E* out = P.out + (long long)y * P.sy + zq + (long long)x0 * P.sx;
        const bool vec_ok = (reinterpret_cast<uintptr_t>(out) & 15) == 0;
        for (int k = 0; k < 2 * R; k++) wait_plane(g0 + k);
#pragma unroll 1
        for (int j = 0; j < len; j++) {
            wait_plane(g0 + j + 2 * R);
            const uint32_t gc = g0 + j + R;                                 // the plane computed now
            // the thread's vector in plane gc + dx, dx = -R..R: every point is one of these plus a constant offset
            const uint8_t* pl[2 * R + 1];
#pragma unroll
            for (int d = 0; d < 2 * R + 1; d++) pl[d] = sbase + ((gc + d - R) % NS) * T::SLOT_BYTES + own;
            // the same for a run-time dx (an index into pl[] would put it in local memory)
            auto plane = [&](int dx) { return sbase + ((gc + dx) % NS) * T::SLOT_BYTES + own; };
            E acc[VW];
            avp_sum<T, HP * ES>(pl, plane, acc);
            E res[VW];
#pragma unroll
            for (int i = 0; i < VW; i++) res[i] = acc[i] * P.scale;
            E* o = out + (long long)j * P.sx;
            if (vec_ok && nv == VW) {
                V rv;
                arr_to_v(res, rv);
                stg128_cs(o, rv);
            } else {
#pragma unroll
                for (int i = 0; i < VW; i++)
                    if (i < nv) o[i] = res[i];
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[(g0 + j) % NS]);
        }
        __syncwarp();
        if (lane == 0)
            for (int k = len; k < len + 2 * R; k++) mbar_arrive(&empty[(g0 + k) % NS]);
        g0 += len + 2 * R;
    }
}

}  // namespace yb
