// 3axis sweep kernels, radius 1..8, fp32 and fp64, and its temporal tile at radius 1 and 2 (yb_avepts_tiles.h).
#include "yb_avepts_tiles.h"

namespace yb {
YB_AVP_TABLES(AVP_3AXIS)
YB_AVP_TT_TABLES(AVP_3AXIS, 2, 2)
}  // namespace yb
