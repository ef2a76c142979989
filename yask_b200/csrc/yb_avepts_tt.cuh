// Temporal tile of the average-of-points stencils (option block_steps / -bt 2): steps t+1 and t+2 in one sweep along x.
//
// A step reads only A(t), so a pair reads A(t) once and writes A(t+2) once; A(t+1) stays in shared memory and is stored only by the
// pair that ends a run_solution() call, whose two steps form the API's window of valid steps.  Storage is the iso3dfd tile's
// (yb_core.h Var::extra_slots / slot_bias): the live pair of slots holds A(t) and the slot of A(t+1); the launch writes A(t+2)
// (and A(t+1)) into their partners in the spare pair, which then becomes the live one.
//
// A CTA owns a (TY x TZ) column of the (y, z) plane, as in avepts_sweep_kernel.  One producer lane loads every plane of A(t) the
// chunk reads -- the tile plus 2R rows and 2 HZ columns -- once, with one TMA box, into a ring of 2R+1+PF slots.  The consumers
//   1. compute step 1 over the tile plus R rows and HZ columns, whole vectors, into a ring of 2R+2 step-1 planes;
//   2. wait at a barrier of the consumer warps only;
//   3. compute step 2 over the tile from the 2R+1 step-1 planes around it, and store it.
// The step-1 ring has one plane more than step 2 reads, so one barrier per plane orders both hazards: the plane step 1 writes in an
// iteration was last read by step 2 two iterations earlier.
//
// Both steps add their points through avp_sum (yb_avepts.cuh), so the point order and the bits are those of the one-step sweep.
// Step-1 points outside the domain are not computed: they are the halo cells of the slot of t+1 (kernels never write halo cells, so
// they hold what the user or the previous run left there), read from global memory on the tiles that touch the boundary.
#pragma once
#include "yb_avepts.cuh"

namespace yb {

template <class E>
struct AvpTTParamsT : AvpParamsT<E> {       // box = the whole rank domain; out = slot of A(t+2)
    E* out1;                                // slot of A(t+1) in the spare pair, or null: A(t+1) is not stored
    const E* halo1;                         // slot of A(t+1) in the live pair: the step-1 values outside the domain
};

template <int SHAPE_, int R_, class E_, int TY_, int TZ_, int PF_>
struct AvpTTile {
    using E = E_;
    using V = typename IsoVec<E>::V;
    static constexpr int SHAPE = SHAPE_, R = R_, TY = TY_, TZ = TZ_, PF = PF_;
    static constexpr int VW = IsoVec<E>::N;
    static constexpr int ES = int(sizeof(E));
    static constexpr int HZ = (R + VW - 1) / VW * VW;           // z halo of a step, whole vectors
    static constexpr int IP = TZ + 4 * HZ;                      // elements per row of a staged A(t) plane
    static constexpr int IROWS = TY + 4 * R;
    static constexpr int SP = TZ + 2 * HZ;                      // elements per row of a step-1 plane
    static constexpr int SROWS = TY + 2 * R;
    static constexpr int SV = SP / VW;                          // vectors per step-1 row
    static constexpr int TZV = TZ / VW;
    static constexpr int THREADS = TY * TZV;                    // consumer threads; one producer warp follows them
    static constexpr int NWARPS = THREADS / 32;
    static constexpr int NS = 2 * R + 1 + PF;                   // A(t) ring
    static constexpr int NS1 = 2 * R + 2;                       // step-1 ring
    static constexpr uint32_t IN_BYTES = uint32_t(IROWS) * IP * ES;
    static constexpr uint32_t IN_SLOT = (IN_BYTES + 127) / 128 * 128;
    static constexpr uint32_t S1_SLOT = (uint32_t(SROWS) * SP * ES + 127) / 128 * 128;
    static constexpr uint32_t S1_OFF = NS * IN_SLOT;
    static constexpr uint32_t BAR_OFF = S1_OFF + NS1 * S1_SLOT;
    static constexpr uint32_t SMEM_BYTES = BAR_OFF + 2 * NS * 8 + 128;
    static_assert(THREADS % 32 == 0, "whole warps");
    static_assert(TZ % VW == 0 && IP <= 256 && IROWS <= 256, "TMA box limits");
    static_assert(SMEM_BYTES <= 232448, "over the sm_90 opt-in shared memory per block");
};

__device__ __forceinline__ void avp_consumer_bar(int threads) {
    asm volatile("bar.sync 1, %0;" ::"r"(threads) : "memory");
}

template <class T>
__global__ void __launch_bounds__(T::THREADS + 32, 1)
avepts_tt2_kernel(const __grid_constant__ CUtensorMap M, const __grid_constant__ AvpTTParamsT<typename T::E> P) {
    using E = typename T::E;
    using V = typename T::V;
    constexpr int R = T::R, NS = T::NS, NS1 = T::NS1, VW = T::VW, ES = T::ES, HZ = T::HZ;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 127u) & ~127u;
    uint8_t* sbase = smem_raw + (base - smem_u32(smem_raw));
    uint8_t* s1base = sbase + T::S1_OFF;
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

    auto unit_of = [&](int u, int& x0, int& len, int& y0, int& z0) {
        const int tz = u % P.ntz; u /= P.ntz;
        const int ty = u % P.nty; u /= P.nty;
        z0 = P.z_begin + tz * T::TZ;
        y0 = P.y_begin + ty * T::TY;
        x0 = P.cx0[u];
        len = P.clen[u];
    };

    // ---- producer warp: one lane loads planes x0-2R .. x0+len-1+2R of every unit of this CTA, in order ----
    if (tid >= T::THREADS) {
        if (tid != T::THREADS) return;
        uint32_t g = 0;
        for (int u = blockIdx.x; u < nunits; u += gridDim.x) {
            int x0, len, y0, z0;
            unit_of(u, x0, len, y0, z0);
            for (int k = 0; k < len + 4 * R; k++, g++) {
                const int s = int(g % NS);
                mbar_wait(&empty[s], ((g / NS) & 1u) ^ 1u);
                mbar_arrive_expect_tx(&full[s], T::IN_BYTES);
                tma_load_3d(sbase + s * T::IN_SLOT, &M, &full[s], P.pad_z + z0 - 2 * HZ, P.pad_y + y0 - 2 * R, P.pad_x + x0 - 2 * R + k);
            }
        }
        return;
    }

    // ---- consumers ----
    const int ty = tid / T::TZV;
    const int q = tid % T::TZV;
    const uint32_t own2 = uint32_t(((ty + R) * T::SP + HZ + VW * q) * ES);      // the thread's step-2 vector in a step-1 plane
    uint32_t g0 = 0;            // sequence number of the unit's first A(t) plane
    uint32_t g1 = 0;            // sequence number of the unit's first step-1 plane
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
        for (int j = 0; j < len + 2 * R; j++) {
            // ---- step 1 at plane xs = x0 - R + j from A(t) planes j .. j + 2R of the unit ----
            wait_plane(g0 + j + 2 * R);
            const int xs = x0 - R + j;
            uint8_t* s1 = s1base + ((g1 + j) % NS1) * T::S1_SLOT;
            const bool x_in = xs >= 0 && xs < P.x_end, x_halo = xs >= -R && xs < P.x_end + R;
            const bool store1 = P.out1 != nullptr && j >= R && j < len + R;
#pragma unroll 1
            for (int w = tid; w < T::SROWS * T::SV; w += T::THREADS) {
                const int r = w / T::SV, c = w % T::SV;
                const int ys = y0 - R + r, zs = z0 - HZ + VW * c;
                const uint32_t off = uint32_t(((r + R) * T::IP + HZ + VW * c) * ES);
                const uint8_t* pl[2 * R + 1];
#pragma unroll
                for (int d = 0; d < 2 * R + 1; d++) pl[d] = sbase + ((g0 + j + d) % NS) * T::IN_SLOT + off;
                auto plane = [&](int dx) { return sbase + ((g0 + j + R + dx) % NS) * T::IN_SLOT + off; };
                E acc[VW];
                avp_sum<T, T::IP * ES>(pl, plane, acc);
                E res[VW];
#pragma unroll
                for (int i = 0; i < VW; i++) res[i] = acc[i] * P.scale;
                const bool y_in = ys >= 0 && ys < P.y_end;
                if (!(x_in && y_in && zs >= 0 && zs + VW <= P.z_end)) {
                    // outside the domain: the halo cells of A(t+1); farther out no step-2 point of the domain reads it
                    const bool yz_halo = x_halo && ys >= -R && ys < P.y_end + R;
                    const E* h = P.halo1 + (long long)xs * P.sx + (long long)ys * P.sy + zs;
#pragma unroll
                    for (int i = 0; i < VW; i++) {
                        const int z = zs + i;
                        if (!(x_in && y_in && z >= 0 && z < P.z_end)) res[i] = (yz_halo && z >= -R && z < P.z_end + R) ? h[i] : E(0);
                    }
                }
                V rv;
                arr_to_v(res, rv);
                *reinterpret_cast<V*>(s1 + (r * T::SP + VW * c) * ES) = rv;
                if (store1 && r >= R && r < R + T::TY && c >= HZ / VW && c < HZ / VW + T::TZV && y_in) {
                    const int n1 = max(0, min(VW, P.z_end - zs));
                    E* o = P.out1 + (long long)xs * P.sx + (long long)ys * P.sy + zs;
                    if (n1 == VW && (reinterpret_cast<uintptr_t>(o) & 15) == 0) {
                        stg128_cs(o, rv);
                    } else {
#pragma unroll
                        for (int i = 0; i < VW; i++)
                            if (i < n1) o[i] = res[i];
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[(g0 + j) % NS]);     // A(t) plane j has no later reader
            avp_consumer_bar(T::THREADS);
            // ---- step 2 at plane x0 + i, i = j - 2R, from step-1 planes i .. i + 2R ----
            if (j >= 2 * R) {
                const int i2 = j - 2 * R;
                const uint8_t* pl[2 * R + 1];
#pragma unroll
                for (int d = 0; d < 2 * R + 1; d++) pl[d] = s1base + ((g1 + i2 + d) % NS1) * T::S1_SLOT + own2;
                auto plane = [&](int dx) { return s1base + ((g1 + i2 + R + dx) % NS1) * T::S1_SLOT + own2; };
                E acc[VW];
                avp_sum<T, T::SP * ES>(pl, plane, acc);
                E res[VW];
#pragma unroll
                for (int i = 0; i < VW; i++) res[i] = acc[i] * P.scale;
                E* o = out + (long long)i2 * P.sx;
                if (vec_ok && nv == VW) {
                    V rv;
                    arr_to_v(res, rv);
                    stg128_cs(o, rv);
                } else {
#pragma unroll
                    for (int i = 0; i < VW; i++)
                        if (i < nv) o[i] = res[i];
                }
            }
        }
        __syncwarp();
        if (lane == 0)
            for (int k = len + 2 * R; k < len + 4 * R; k++) mbar_arrive(&empty[(g0 + k) % NS]);
        g0 += len + 4 * R;
        g1 += len + 2 * R;
    }
}

}  // namespace yb
