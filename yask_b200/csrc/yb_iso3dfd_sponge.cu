// iso3dfd_sponge on the iso3dfd sweep: the default variant of yb_iso3dfd_radii.cu (tile 16x128, producer warpgroup, 2 planes
// per trip) compiled in its SP form, which scales every result by cr_x(x) * cr_y(y) * cr_z(z) before it is stored, for radius
// 1..7.  The fused peer stores and the in-kernel signal of the plain kernel stay: they store the scaled value.  The fp64 form is
// in yb_iso3dfd_sponge_f64.cu (own translation unit: the instantiations compile in parallel).
#include "yb_iso3dfd_tiles.h"

namespace yb {

const TileCfg* iso_sponge_cfg(int radius) {
    static const TileCfg cfgs[7] = {
        iso_default_cfg<1, float, true>("sponge r1 16x128 PW U2"), iso_default_cfg<2, float, true>("sponge r2 16x128 PW U2"),
        iso_default_cfg<3, float, true>("sponge r3 16x128 PW U2"), iso_default_cfg<4, float, true>("sponge r4 16x128 PW U2"),
        iso_default_cfg<5, float, true>("sponge r5 16x128 PW U2"), iso_default_cfg<6, float, true>("sponge r6 16x128 PW U2"),
        iso_default_cfg<7, float, true>("sponge r7 16x128 PW U2")};
    return iso_cfg_of_radius(cfgs, radius);
}

}  // namespace yb
