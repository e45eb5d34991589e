// ls_fused_b.cu -- fused solver with the Chebyshev polynomial preconditioner (K = 3)
#include "ls_pcg_fused.cuh"
#include "ls_fused_inst.h"

namespace {
using lsf::fused_fn;
constexpr int W = lsf::PWARPS, WS = lsf::PT_SMALL / 32;
}  // namespace

const void *ls_fused_fn_cheb(int res, int nw, int pat, int sync) {
    if (sync == 0 && nw == W) {
        if (res == 0) return pat ? fused_fn<3, 0, W, true, 0, false, true>() : fused_fn<3, 0, W, false, 0, false, true>();
        if (res == 1) return pat ? fused_fn<3, 1, W, true, 0, false, true>() : fused_fn<3, 1, W, false, 0, false, true>();
        if (res == 2) return pat ? fused_fn<3, 2, W, true, 0, false, true>() : fused_fn<3, 2, W, false, 0, false, true>();
    }
    if (sync == 0 && nw == WS && res == 2)
        return pat ? fused_fn<3, 2, WS, true, 0, false, true>() : fused_fn<3, 2, WS, false, 0, false, true>();
    if (sync == 1 && nw == W && res == 2)
        return pat ? fused_fn<3, 2, W, true, 1, false, true>() : fused_fn<3, 2, W, false, 1, false, true>();
    return nullptr;
}
