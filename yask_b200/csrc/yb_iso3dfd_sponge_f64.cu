// iso3dfd_sponge in double precision: the sweep of yb_iso3dfd_radii_f64.cu (tile 16x64, producer warpgroup, 2 planes per trip)
// in its SP form (see yb_iso3dfd_sponge.cu), for radius 1, 2, 3, 4, 5, 7 and 8.  As in plain fp64 the boundary planes are not
// stored into the x neighbours: multi-rank runs take the exterior / interior split.  At radius 8 a stage is 45,056 B, so the
// 5-stage ring and its barriers take 225,488 B of the 227 KB opt-in.
#include "yb_iso3dfd_tiles.h"

namespace yb {

const TileCfgT<double>* iso_sponge_cfg_f64(int radius) {
    static const TileCfgT<double> cfgs[8] = {
        iso_default_cfg<1, double, true>("fp64 sponge r1 16x64 PW U2"), iso_default_cfg<2, double, true>("fp64 sponge r2 16x64 PW U2"),
        iso_default_cfg<3, double, true>("fp64 sponge r3 16x64 PW U2"), iso_default_cfg<4, double, true>("fp64 sponge r4 16x64 PW U2"),
        iso_default_cfg<5, double, true>("fp64 sponge r5 16x64 PW U2"), {},
        iso_default_cfg<7, double, true>("fp64 sponge r7 16x64 PW U2"), iso_default_cfg<8, double, true>("fp64 sponge r8 16x64 PW U2")};
    return iso_cfg_of_radius(cfgs, radius);
}

}  // namespace yb
