// Table entries of the average-of-points sweep kernels (yb_avepts.cuh), one per (shape, radius, element type).  The tables are
// instantiated one shape per translation unit (yb_avepts_<shape>.cu) and read by the engine (yb_avepts.cu).
#pragma once
#include <utility>

#include "yb_avepts.cuh"
#include "yb_avepts_tt.cuh"

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

// ---- temporal tile (yb_avepts_tt.cuh) ----
template <class E>
struct AvpTTCfgT {
    typedef void (*Fn)(const CUtensorMap, const AvpTTParamsT<E>);
    int ty, tz, ip, irows, threads;
    uint32_t smem;
    Fn fn;              // null: no tile for this radius, block_steps has no effect
};
constexpr int AVP_TT_MAX_R = 2;

// The one-step sweep's tile: 16 rows x 64 fp32 / 32 fp64 columns, 256 consumer threads, 2 planes of prefetch.
template <int SHAPE, int R, class E>
using AvpTTileOf = AvpTTile<SHAPE, R, E, 16, sizeof(E) == 4 ? 64 : 32, 2>;

template <int SHAPE, int R, class E, bool ON>
AvpTTCfgT<E> avp_tt_cfg() {
    if constexpr (ON) {
        using T = AvpTTileOf<SHAPE, R, E>;
        return AvpTTCfgT<E>{T::TY, T::TZ, T::IP, T::IROWS, T::THREADS + 32, T::SMEM_BYTES, avepts_tt2_kernel<T>};
    } else {
        return AvpTTCfgT<E>{};
    }
}

// Entries of radius 1..AVP_TT_MAX_R of one shape (index radius - 1); defined in yb_avepts_<shape>.cu with the largest radius that
// has a tile in fp32 and in fp64 (0: none).
template <int SHAPE, class E>
const AvpTTCfgT<E>* avp_tt_table();
#define YB_AVP_TT_TABLE_DECL(SHAPE)                       \
    template <>                                           \
    const AvpTTCfgT<float>* avp_tt_table<SHAPE, float>(); \
    template <>                                           \
    const AvpTTCfgT<double>* avp_tt_table<SHAPE, double>();
YB_AVP_TT_TABLE_DECL(AVP_3AXIS)
YB_AVP_TT_TABLE_DECL(AVP_DIAGS)
YB_AVP_TT_TABLE_DECL(AVP_PLANE)
YB_AVP_TT_TABLE_DECL(AVP_CUBE)

#define YB_AVP_TT_TABLES(SHAPE, RMAX_F32, RMAX_F64)                                                                  \
    template <>                                                                                                      \
    const AvpTTCfgT<float>* avp_tt_table<SHAPE, float>() {                                                           \
        static const AvpTTCfgT<float> t[AVP_TT_MAX_R] = {avp_tt_cfg<SHAPE, 1, float, (RMAX_F32 >= 1)>(),             \
                                                         avp_tt_cfg<SHAPE, 2, float, (RMAX_F32 >= 2)>()};            \
        return t;                                                                                                    \
    }                                                                                                                \
    template <>                                                                                                      \
    const AvpTTCfgT<double>* avp_tt_table<SHAPE, double>() {                                                         \
        static const AvpTTCfgT<double> t[AVP_TT_MAX_R] = {avp_tt_cfg<SHAPE, 1, double, (RMAX_F64 >= 1)>(),           \
                                                          avp_tt_cfg<SHAPE, 2, double, (RMAX_F64 >= 2)>()};          \
        return t;                                                                                                    \
    }

}  // namespace yb
