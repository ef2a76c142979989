// 3axis_with_diags sweep kernels, radius 1..8, fp32 and fp64 (yb_avepts_tiles.h).
#include "yb_avepts_tiles.h"

namespace yb {
YB_AVP_TABLES(AVP_DIAGS)
YB_AVP_TT_TABLES(AVP_DIAGS, 0, 0)     // no temporal tile: slower with pairs on an H100 (README)
}  // namespace yb
