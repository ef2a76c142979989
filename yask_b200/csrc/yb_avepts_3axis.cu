// 3axis sweep kernels, radius 1..8, fp32 and fp64 (yb_avepts_tiles.h).
#include "yb_avepts_tiles.h"

namespace yb {
YB_AVP_TABLES(AVP_3AXIS)
}  // namespace yb
