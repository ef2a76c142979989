// Table entry describing one compiled variant of the iso3dfd tiled kernels (yb_iso3dfd.cu / yb_iso3dfd_radii*.cu).
#pragma once
#include "yb_iso3dfd.cuh"

namespace yb {

template <class E>
struct TileCfgT {
    typedef void (*Fn)(const IsoMaps, const IsoParamsT<E>);
    const char* name;
    int ty, tz, hp, hrows, threads;
    uint32_t smem;
    Fn fn[4];           // per FP mode (3 = debug memory-only probe, fp32 radius 8 only)
};
using TileCfg = TileCfgT<float>;

// The entry of iso3dfd_tma2_kernel<T, MODE, PW, U, SP>; PROBE: mode 3 (the memory-only probe, option mem_probe) is compiled too.
template <class T, int PW, int U, bool PROBE = false, bool SP = false>
TileCfgT<typename T::E> iso_tile_cfg(const char* name) {
    static_assert(T::SMEM_BYTES <= 232448, "over the sm_90 opt-in shared memory per block");
    TileCfgT<typename T::E> c{name, T::TY, T::TZ, T::HP, T::HROWS, T::THREADS + 128 * PW, T::SMEM_BYTES,
                              {iso3dfd_tma2_kernel<T, 0, PW, U, SP>, iso3dfd_tma2_kernel<T, 1, PW, U, SP>,
                               iso3dfd_tma2_kernel<T, 2, PW, U, SP>, nullptr}};
    if constexpr (PROBE) c.fn[3] = iso3dfd_tma2_kernel<T, 3, PW, U, SP>;
    return c;
}

// The default variant at radius R: producer warpgroup, 2 planes per trip, tile 16x128 in fp32 and 16x64 in fp64 (a thread owns
// two rows x one 16-byte vector in both).
template <int R, class E, bool SP = false>
TileCfgT<E> iso_default_cfg(const char* name) { return iso_tile_cfg<IsoTile2<R, 8, 32, 5, E>, 1, 2, false, SP>(name); }

// Entry of a table indexed by radius - 1 (a value-initialised entry is a radius with no compiled variant), nullptr outside it.
template <class E, int N>
const TileCfgT<E>* iso_cfg_of_radius(const TileCfgT<E> (&cfgs)[N], int radius) {
    return (radius >= 1 && radius <= N && cfgs[radius - 1].fn[0]) ? &cfgs[radius - 1] : nullptr;
}

// The default variant instantiated for radius 1..7; radius 8 has the full variant table in yb_iso3dfd.cu.  Returns nullptr for
// other radii.
const TileCfg* iso_radius_cfg(int radius);

// Double precision (yb_iso3dfd_radii_f64.cu): the same sweep with a 16x64 tile, for radius 1, 2, 4, 5, 6 and 7.  Radius 3
// and 8 are served by the emitter-generated kernels (yb_stencils.cpp), so they have no entry here: returns nullptr.
const TileCfgT<double>* iso_radius_cfg_f64(int radius);

// iso3dfd_sponge (yb_iso3dfd_sponge.cu): the same default variant in its SP form, fp32 at radius 1..7 and fp64 at radius 1, 2, 3,
// 4, 5, 7 and 8.  fp32 radius 8 and fp64 radius 6 are served by the emitter-generated kernels (yb_stencils.cpp): nullptr.
const TileCfg* iso_sponge_cfg(int radius);
const TileCfgT<double>* iso_sponge_cfg_f64(int radius);

}  // namespace yb
