// iso3dfd_sponge on the iso3dfd sweep: the default variant of yb_iso3dfd_radii.cu (tile 16x128, producer warpgroup, 2 planes
// per trip) compiled in its SP form, which scales every result by cr_x(x) * cr_y(y) * cr_z(z) before it is stored, for radius
// 1..7.  The fused peer stores and the in-kernel signal of the plain kernel stay: they store the scaled value.  The fp64 form is
// in yb_iso3dfd_sponge_f64.cu (own translation unit: the instantiations compile in parallel).
#include "yb_iso3dfd_tiles.h"

namespace yb {

namespace {
template <int R>
TileCfg make_sponge_cfg(const char* name) {
    using T = IsoTile2<R, 8, 32, 5>;
    return TileCfg{true, name, T::TY, T::TZ, T::HP, T::HROWS, T::THREADS + 128, T::SMEM_BYTES,
                   {iso3dfd_tma2_kernel<T, 0, 1, 2, true>, iso3dfd_tma2_kernel<T, 1, 1, 2, true>, iso3dfd_tma2_kernel<T, 2, 1, 2, true>,
                    nullptr}};
}
}  // namespace

const TileCfg* iso_sponge_cfg(int radius) {
    static const TileCfg cfgs[7] = {make_sponge_cfg<1>("sponge r1 16x128 PW U2"), make_sponge_cfg<2>("sponge r2 16x128 PW U2"),
                                    make_sponge_cfg<3>("sponge r3 16x128 PW U2"), make_sponge_cfg<4>("sponge r4 16x128 PW U2"),
                                    make_sponge_cfg<5>("sponge r5 16x128 PW U2"), make_sponge_cfg<6>("sponge r6 16x128 PW U2"),
                                    make_sponge_cfg<7>("sponge r7 16x128 PW U2")};
    return (radius >= 1 && radius <= 7) ? &cfgs[radius - 1] : nullptr;
}

}  // namespace yb
