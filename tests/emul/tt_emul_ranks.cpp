// TEST INFRASTRUCTURE ONLY -- the CTA emulator of tt_emul.cpp on ONE RANK of a rank grid (tests/test_temporal_ranks_cpu.py).
//
// Same back end (threads in a loop, TMA boxes copied by the host, eager / lazy completion, race detector, NaN-poisoned shared
// memory), same kernel code; the one difference is TTParams::ext_lo / ext_hi: on a side with a neighbour rank the step-1 ring
// is computed from the halos (p(t) 2R deep, p(t-1) and v R deep) instead of taking p(t-1).  Built by the test into a library
// of its own, so tt_emul.cpp and its library stay what tests/test_temporal_cpu.py checks.
#include "tt_emul.cpp"

namespace {

template <class T, int MODE>
int run_ext(const float* pprev, const float* pcur, const float* vel, float* out1, float* out2, const int* n, const int* ppad, const int* vpad,
            const float* coef, int grid, int nchunks, int lazy, const int* ext_lo, const int* ext_hi) {
    const long long pz = n[2] + 2 * ppad[2], py = n[1] + 2 * ppad[1], px = n[0] + 2 * ppad[0];
    const long long vz = n[2] + 2 * vpad[2], vy = n[1] + 2 * vpad[1], vx = n[0] + 2 * vpad[0];
    TTParams P{};
    P.p_sy = pz; P.p_sx = pz * py; P.v_sy = vz; P.v_sx = vz * vy;
    const long long porg = ppad[0] * P.p_sx + ppad[1] * P.p_sy + ppad[2];
    P.out1 = out1 + porg; P.out2 = out2 + porg;
    P.vel = vel + vpad[0] * P.v_sx + vpad[1] * P.v_sy + vpad[2];
    P.nx = n[0]; P.ny = n[1]; P.nz = n[2];
    for (int d = 0; d < 3; d++) { P.ext_lo[d] = ext_lo[d]; P.ext_hi[d] = ext_hi[d]; }
    P.pad_x = ppad[0]; P.pad_y = ppad[1]; P.pad_z = ppad[2];
    P.vpad_x = vpad[0]; P.vpad_y = vpad[1]; P.vpad_z = vpad[2];
    for (int r = 0; r <= T::R; r++) P.c[r] = coef[r];
    P.nty = (P.ny + T::TY - 1) / T::TY;
    P.ntz = (P.nz + T::TZ - 1) / T::TZ;
    if (nchunks < 1 || nchunks > TT_MAX_CHUNKS || nchunks > P.nx) return -1;
    P.nchunks = nchunks;
    for (int k = 0; k < nchunks; k++) {
        const long long x0 = (long long)P.nx * k / nchunks, x1 = (long long)P.nx * (k + 1) / nchunks;
        P.cx0[k] = int(x0); P.clen[k] = int(x1 - x0);
    }
    for (int blk = 0; blk < grid; blk++) {
        Emul<T> be;
        be.lazy = lazy != 0;
        be.pin = Tensor{pcur, pz, py, px, P.p_sy, P.p_sx};
        be.prev = Tensor{pprev, pz, py, px, P.p_sy, P.p_sx};
        be.v = Tensor{vel, vz, vy, vx, P.v_sy, P.v_sx};
        g_race.reset(be.smem.data(), be.smem.size());
        tt_sweep<T, MODE>(be, be.smem.data(), P, blk, grid);
        if (be.error) return be.error;
        if (g_race.races) return 6;
        for (auto& b : be.bars) if (b.armed) return 5;
    }
    return 0;
}

template <class T>
int run_ext_mode(int mode, const float* a, const float* b, const float* c, float* d, float* e, const int* n, const int* pp, const int* vp,
                 const float* coef, int grid, int nchunks, int lazy, const int* lo, const int* hi) {
    switch (mode) {
        case 0: return run_ext<T, 0>(a, b, c, d, e, n, pp, vp, coef, grid, nchunks, lazy, lo, hi);
        case 1: return run_ext<T, 1>(a, b, c, d, e, n, pp, vp, coef, grid, nchunks, lazy, lo, hi);
        default: return run_ext<T, 2>(a, b, c, d, e, n, pp, vp, coef, grid, nchunks, lazy, lo, hi);
    }
}

}  // namespace

// As tt_emul_run, plus `ext_lo` / `ext_hi` (TTParams): R on a side with a neighbour rank, 0 at the global boundary.
extern "C" int tt_emul_run_ext(int radius, int variant, int mode, const float* pprev, const float* pcur, const float* vel, float* out1, float* out2,
                               const int* n, const int* ppad, const int* vpad, const float* coef, int grid, int nchunks, int lazy,
                               const int* ext_lo, const int* ext_hi) {
#define YB_EXT_CASE(r, v, ...) \
    if (radius == r && variant == v) return run_ext_mode<__VA_ARGS__>(mode, pprev, pcur, vel, out1, out2, n, ppad, vpad, coef, grid, nchunks, lazy, ext_lo, ext_hi);
    YB_EXT_CASE(1, 0, TTile<1, 16, 128, 3, 256>)
    YB_EXT_CASE(2, 0, TTile<2, 16, 128, 2, 256>)
    YB_EXT_CASE(1, 1, TTile<1, 4, 16, 2, 32>)
    YB_EXT_CASE(2, 1, TTile<2, 4, 16, 1, 32>)
    YB_EXT_CASE(1, 2, TTile<1, 16, 128, 3, 256, 1>)
    YB_EXT_CASE(2, 2, TTile<2, 16, 128, 3, 256, 1>)
    YB_EXT_CASE(1, 3, TTile<1, 4, 16, 2, 32, 1>)
    YB_EXT_CASE(2, 3, TTile<2, 4, 16, 1, 32, 1>)
    YB_EXT_CASE(1, 4, TTile<1, 16, 128, 3, 512, 0>)
    YB_EXT_CASE(2, 4, TTile<2, 16, 128, 2, 512, 0>)
    YB_EXT_CASE(1, 5, TTile<1, 16, 128, 3, 512, 1>)
    YB_EXT_CASE(2, 5, TTile<2, 16, 128, 3, 512, 1>)
#undef YB_EXT_CASE
    return -2;
}
