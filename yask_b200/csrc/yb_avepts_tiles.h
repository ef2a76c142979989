// Table entries of the average-of-points sweep kernels (yb_avepts.cuh), one per (shape, radius, element type).  The tables are
// instantiated one shape per translation unit (yb_avepts_<shape>.cu) and read by the engine (yb_avepts.cu).
#pragma once
#include <utility>

#include "yb_avepts.cuh"

namespace yb {

template <class E>
struct AvpCfgT {
    typedef void (*Fn)(const CUtensorMap, const AvpParamsT<E>);
    int ty, tz, hp, hrows, threads;
    uint32_t smem;
    Fn fn;
};

// Tile per radius and element type: 16 rows x 64 fp32 / 32 fp64 columns, 256 consumer threads (one 16-byte vector each), 2 planes
// of prefetch -- 1 for fp64 radius 8, whose 18 slots of 12 KB then fit the 227 KB opt-in (fp32 radius 8: 19 slots of 10 KB).
template <int SHAPE, int R, class E>
using AvpTileOf = AvpTile<SHAPE, R, E, 16, sizeof(E) == 4 ? 64 : 32, (sizeof(E) == 8 && R == 8) ? 1 : 2>;

template <class T>
AvpCfgT<typename T::E> avp_cfg() {
    return AvpCfgT<typename T::E>{T::TY, T::TZ, T::HP, T::HROWS, T::THREADS + 32, T::SMEM_BYTES, avepts_sweep_kernel<T>};
}

template <int SHAPE, class E, int... Rm1>
const AvpCfgT<E>* avp_table_of(std::integer_sequence<int, Rm1...>) {
    static const AvpCfgT<E> t[] = {avp_cfg<AvpTileOf<SHAPE, Rm1 + 1, E>>()...};
    return t;
}

// The entries of radius 1..AVP_MAX_R of one shape (index radius - 1); defined in yb_avepts_<shape>.cu.
template <int SHAPE, class E>
const AvpCfgT<E>* avp_table();
#define YB_AVP_TABLE_DECL(SHAPE)                         \
    template <>                                          \
    const AvpCfgT<float>* avp_table<SHAPE, float>();     \
    template <>                                          \
    const AvpCfgT<double>* avp_table<SHAPE, double>();
YB_AVP_TABLE_DECL(AVP_3AXIS)
YB_AVP_TABLE_DECL(AVP_DIAGS)
YB_AVP_TABLE_DECL(AVP_PLANE)
YB_AVP_TABLE_DECL(AVP_CUBE)

#define YB_AVP_TABLES(SHAPE)                                                                                                 \
    template <>                                                                                                              \
    const AvpCfgT<float>* avp_table<SHAPE, float>() { return avp_table_of<SHAPE, float>(std::make_integer_sequence<int, AVP_MAX_R>{}); } \
    template <>                                                                                                              \
    const AvpCfgT<double>* avp_table<SHAPE, double>() { return avp_table_of<SHAPE, double>(std::make_integer_sequence<int, AVP_MAX_R>{}); }

}  // namespace yb
