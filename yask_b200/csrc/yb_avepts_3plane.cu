// 3plane sweep kernels, radius 1..8, fp32 and fp64 (yb_avepts_tiles.h).
#include "yb_avepts_tiles.h"

namespace yb {
YB_AVP_TABLES(AVP_PLANE)
}  // namespace yb
