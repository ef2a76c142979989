// iso3dfd_sponge in double precision: the sweep of yb_iso3dfd_radii_f64.cu (tile 16x64, producer warpgroup, 2 planes per trip)
// in its SP form (see yb_iso3dfd_sponge.cu), for radius 1, 2, 3, 4, 5, 7 and 8.  As in plain fp64 the boundary planes are not
// stored into the x neighbours (fused_ok = false): multi-rank runs take the exterior / interior split.
#include "yb_iso3dfd_tiles.h"

namespace yb {

namespace {
template <int R>
TileCfgT<double> make_sponge_cfg_f64(const char* name) {
    using T = IsoTile2<R, 8, 32, 5, double>;
    // radius 8: a stage is 45,056 B, so the 5-stage ring and its barriers take 225,488 B of the 227 KB opt-in
    static_assert(T::SMEM_BYTES <= 232448, "over the sm_90 opt-in shared memory per block");
    return TileCfgT<double>{false, name, T::TY, T::TZ, T::HP, T::HROWS, T::THREADS + 128, T::SMEM_BYTES,
                            {iso3dfd_tma2_kernel<T, 0, 1, 2, true>, iso3dfd_tma2_kernel<T, 1, 1, 2, true>,
                             iso3dfd_tma2_kernel<T, 2, 1, 2, true>, nullptr}};
}
}  // namespace

const TileCfgT<double>* iso_sponge_cfg_f64(int radius) {
    static const TileCfgT<double> cfgs[7] = {
        make_sponge_cfg_f64<1>("fp64 sponge r1 16x64 PW U2"), make_sponge_cfg_f64<2>("fp64 sponge r2 16x64 PW U2"),
        make_sponge_cfg_f64<3>("fp64 sponge r3 16x64 PW U2"), make_sponge_cfg_f64<4>("fp64 sponge r4 16x64 PW U2"),
        make_sponge_cfg_f64<5>("fp64 sponge r5 16x64 PW U2"), make_sponge_cfg_f64<7>("fp64 sponge r7 16x64 PW U2"),
        make_sponge_cfg_f64<8>("fp64 sponge r8 16x64 PW U2")};
    switch (radius) {
        case 1: case 2: case 3: case 4: case 5: return &cfgs[radius - 1];
        case 7: return &cfgs[5];
        case 8: return &cfgs[6];
        default: return nullptr;
    }
}

}  // namespace yb
