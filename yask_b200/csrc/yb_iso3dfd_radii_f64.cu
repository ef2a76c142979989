// iso3dfd tiled kernel in double precision: the default variant of yb_iso3dfd_radii.cu (producer warpgroup, 2 planes per
// trip) with E = double.  A thread owns two rows x one double2, so the 256 consumer threads cover a 16 (y) x 64 (z) tile
// and an x-queue entry takes the same 4 registers as in fp32; a stage is then at most 43 KB (radius 7), and the 5-stage
// ring fits in shared memory.
//
// The boundary planes are not stored into the x neighbours (fused_ok = false): multi-rank runs take the exterior /
// interior split with a separate halo exchange.
#include "yb_iso3dfd_tiles.h"

namespace yb {

namespace {
template <int R>
TileCfgT<double> make_cfg_f64(const char* name) {
    using T = IsoTile2<R, 8, 32, 5, double>;
    return TileCfgT<double>{false, name, T::TY, T::TZ, T::HP, T::HROWS, T::THREADS + 128, T::SMEM_BYTES,
                            {iso3dfd_tma2_kernel<T, 0, 1, 2>, iso3dfd_tma2_kernel<T, 1, 1, 2>, iso3dfd_tma2_kernel<T, 2, 1, 2>, nullptr}};
}
}  // namespace

const TileCfgT<double>* iso_radius_cfg_f64(int radius) {
    static const TileCfgT<double> cfgs[6] = {make_cfg_f64<1>("fp64 r1 16x64 PW U2"), make_cfg_f64<2>("fp64 r2 16x64 PW U2"),
                                             make_cfg_f64<4>("fp64 r4 16x64 PW U2"), make_cfg_f64<5>("fp64 r5 16x64 PW U2"),
                                             make_cfg_f64<6>("fp64 r6 16x64 PW U2"), make_cfg_f64<7>("fp64 r7 16x64 PW U2")};
    switch (radius) {
        case 1: return &cfgs[0];
        case 2: return &cfgs[1];
        case 4: return &cfgs[2];
        case 5: return &cfgs[3];
        case 6: return &cfgs[4];
        case 7: return &cfgs[5];
        default: return nullptr;
    }
}

}  // namespace yb
