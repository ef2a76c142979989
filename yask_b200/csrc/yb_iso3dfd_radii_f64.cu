// iso3dfd tiled kernel in double precision: the default variant of yb_iso3dfd_radii.cu (producer warpgroup, 2 planes per
// trip) with E = double.  A thread owns two rows x one double2, so the 256 consumer threads cover a 16 (y) x 64 (z) tile
// and an x-queue entry takes the same 4 registers as in fp32; a stage is then at most 43 KB (radius 7), and the 5-stage
// ring fits in shared memory.
//
// The boundary planes are not stored into the x neighbours (the kernel's FUSED is fp32 only): multi-rank runs take the
// exterior / interior split with a separate halo exchange.
#include "yb_iso3dfd_tiles.h"

namespace yb {

const TileCfgT<double>* iso_radius_cfg_f64(int radius) {
    static const TileCfgT<double> cfgs[7] = {
        iso_default_cfg<1, double>("fp64 r1 16x64 PW U2"), iso_default_cfg<2, double>("fp64 r2 16x64 PW U2"), {},
        iso_default_cfg<4, double>("fp64 r4 16x64 PW U2"), iso_default_cfg<5, double>("fp64 r5 16x64 PW U2"),
        iso_default_cfg<6, double>("fp64 r6 16x64 PW U2"), iso_default_cfg<7, double>("fp64 r7 16x64 PW U2")};
    return iso_cfg_of_radius(cfgs, radius);
}

}  // namespace yb
