// Table entry describing one compiled variant of the iso3dfd tiled kernels (yb_iso3dfd.cu / yb_iso3dfd_radii*.cu).
#pragma once
#include "yb_iso3dfd.cuh"

namespace yb {

template <class E>
struct TileCfgT {
    typedef void (*Fn)(const IsoMaps, const IsoParamsT<E>);
    bool fused_ok;      // kernel can store boundary planes into the x neighbours (gen2 PW/U variants)
    const char* name;
    int ty, tz, hp, hrows, threads;
    uint32_t smem;
    Fn fn[4];           // per FP mode (3 = debug memory-only probe, fp32 gen2 only)
};
using TileCfg = TileCfgT<float>;


// The default variant (tile 16x128, producer warpgroup, 2 planes per trip) instantiated for radius 1..7;
// radius 8 has the full variant table in yb_iso3dfd.cu.  Returns nullptr for other radii.
const TileCfg* iso_radius_cfg(int radius);

// Double precision (yb_iso3dfd_radii_f64.cu): the same sweep with a 16x64 tile, for radius 1, 2, 4, 5, 6 and 7.  Radius 3
// and 8 are served by the emitter-generated kernels (yb_stencils.cpp), so they have no entry here: returns nullptr.
const TileCfgT<double>* iso_radius_cfg_f64(int radius);

// iso3dfd_sponge (yb_iso3dfd_sponge.cu): the same default variant in its SP form, fp32 at radius 1..7 and fp64 at radius 1, 2, 3,
// 4, 5, 7 and 8.  fp32 radius 8 and fp64 radius 6 are served by the emitter-generated kernels (yb_stencils.cpp): nullptr.
const TileCfg* iso_sponge_cfg(int radius);
const TileCfgT<double>* iso_sponge_cfg_f64(int radius);

}  // namespace yb
