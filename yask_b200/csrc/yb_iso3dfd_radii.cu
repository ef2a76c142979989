// iso3dfd tiled kernel (default variant: tile 16x128, producer warpgroup, 2 planes per trip) for radius 1..7.
// Same template as the radius-8 product kernel (yb_iso3dfd.cuh); kept in its own translation unit so the
// instantiations compile in parallel with yb_iso3dfd.cu.
#include "yb_iso3dfd_tiles.h"

namespace yb {

const TileCfg* iso_radius_cfg(int radius) {
    static const TileCfg cfgs[7] = {iso_default_cfg<1, float>("r1 16x128 PW U2"), iso_default_cfg<2, float>("r2 16x128 PW U2"),
                                    iso_default_cfg<3, float>("r3 16x128 PW U2"), iso_default_cfg<4, float>("r4 16x128 PW U2"),
                                    iso_default_cfg<5, float>("r5 16x128 PW U2"), iso_default_cfg<6, float>("r6 16x128 PW U2"),
                                    iso_default_cfg<7, float>("r7 16x128 PW U2")};
    return iso_cfg_of_radius(cfgs, radius);
}

}  // namespace yb
