// x chunks of the iso3dfd sweep launches (yb_iso3dfd.cu): how many, and which planes each covers.  Host code only.
#pragma once
#include <stdint.h>

#include <algorithm>

namespace yb {

// Number of x chunks of a sweep over nx planes with ntile (y, z) tiles on at most gmax CTAs, in [min_nc, max_nc].  lx > 0 asks for
// chunks of lx planes.  Otherwise the count that minimises (rounds of units per CTA) x (chunk length + 0.4 x warm-up planes): long
// chunks amortise the planes a chunk loads before its first result, short ones balance the last round.
inline int chunk_count(int64_t nx, int64_t ntile, int gmax, int lx, int warm, int min_nc, int64_t max_nc) {
    if (lx > 0) return int(std::max<int64_t>(min_nc, std::min<int64_t>((nx + lx - 1) / lx, max_nc)));
    double best = 1e30;
    int nc_best = min_nc;
    for (int64_t nc = min_nc; nc <= max_nc; nc++) {
        const int64_t l = (nx + nc - 1) / nc;
        const int64_t rounds = (ntile * nc + gmax - 1) / gmax;
        const double cost = double(rounds) * (double(l) + warm * 0.4);
        if (cost < best * 0.999) { best = cost; nc_best = int(nc); }
    }
    return nc_best;
}

// Balanced partition of [b, b + n) into nc chunks (lengths differ by at most one plane), in launch order: first plane swept (x0),
// planes (len) and, when dir is non-null, direction (+1 / -1).  lo_first lists the chunk that starts at plane b first; hi_first
// lists the chunk that ends at plane b + n - 1 next and sweeps it downwards, unless that is the same chunk.  Returns the number of
// chunks listed for lo_first / hi_first.
inline int chunk_partition(int64_t b, int64_t n, int nc, bool lo_first, bool hi_first, int* x0, int* len, int* dir) {
    const bool hi_down = hi_first && !(nc == 1 && lo_first);
    int k = 0;
    auto put = [&](int c) {
        const int64_t c0 = b + n * c / nc, c1 = b + n * (c + 1) / nc;
        const bool down = hi_down && c == nc - 1;
        x0[k] = int(down ? c1 - 1 : c0);
        len[k] = int(c1 - c0);
        if (dir) dir[k] = down ? -1 : 1;
        k++;
    };
    if (lo_first) put(0);
    if (hi_down) put(nc - 1);
    const int nfirst = k;
    for (int c = lo_first ? 1 : 0; c < (hi_down ? nc - 1 : nc); c++) put(c);
    return nfirst;
}

}  // namespace yb
