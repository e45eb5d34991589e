// ls_fused_c.cu -- profiling instantiations (per-phase cycle counters) and the 4-column instantiations
#include "ls_pcg_fused.cuh"
#include "ls_fused_inst.h"

namespace {
using lsf::fused_fn;
constexpr int W = lsf::PWARPS, WS = lsf::PT_SMALL / 32;
}  // namespace

const void *ls_fused_fn_misc(int K, int res, int nw, int pat, int sync, int prof) {
    if (K == 3 && prof && nw == W) {
        if (sync == 0 && res == 1) return pat ? fused_fn<3, 1, W, true, 0, true>() : fused_fn<3, 1, W, false, 0, true>();
        if (sync == 0 && res == 2) return pat ? fused_fn<3, 2, W, true, 0, true>() : fused_fn<3, 2, W, false, 0, true>();
        if (sync == 1 && res == 2) return pat ? fused_fn<3, 2, W, true, 1, true>() : fused_fn<3, 2, W, false, 1, true>();
        if (sync == 1 && res == 3) return pat ? fused_fn<3, 3, W, true, 1, true>() : fused_fn<3, 3, W, false, 1, true>();
        if (sync == 1 && res == 4) return pat ? fused_fn<3, 4, W, true, 1, true>() : fused_fn<3, 4, W, false, 1, true>();
    }
    if (K == 3 && prof && nw == WS && sync == 1 && res == 4)
        return pat ? fused_fn<3, 4, WS, true, 1, true>() : fused_fn<3, 4, WS, false, 1, true>();
    if (K == 4 && !prof && !pat && nw == W) {
        if (sync == 0 && res == 0) return fused_fn<4, 0, W, false, 0, false>();
        if (sync == 0 && res == 1) return fused_fn<4, 1, W, false, 0, false>();
        if (sync == 0 && res == 2) return fused_fn<4, 2, W, false, 0, false>();
        if (sync == 1 && res == 2) return fused_fn<4, 2, W, false, 1, false>();
        if (sync == 1 && res == 4) return fused_fn<4, 4, W, false, 1, false>();
    }
    return nullptr;
}
