// ls_fused_a.cu -- production instantiations of the fused solver (K = 3, Jacobi)
#include "ls_pcg_fused.cuh"
#include "ls_fused_inst.h"

namespace {
using lsf::fused_fn;
constexpr int W = lsf::PWARPS, WS = lsf::PT_SMALL / 32;
}  // namespace

const void *ls_fused_fn_jacobi(int res, int nw, int pat, int sync) {
    if (sync == 0 && nw == W) {
        if (res == 0) return pat ? fused_fn<3, 0, W, true, 0, false>() : fused_fn<3, 0, W, false, 0, false>();
        if (res == 1) return pat ? fused_fn<3, 1, W, true, 0, false>() : fused_fn<3, 1, W, false, 0, false>();
        if (res == 2) return pat ? fused_fn<3, 2, W, true, 0, false>() : fused_fn<3, 2, W, false, 0, false>();
    }
    if (sync == 0 && nw == WS && res == 2) return pat ? fused_fn<3, 2, WS, true, 0, false>() : fused_fn<3, 2, WS, false, 0, false>();
    if (sync == 1 && nw == W && res == 2) return pat ? fused_fn<3, 2, W, true, 1, false>() : fused_fn<3, 2, W, false, 1, false>();
    if (sync == 1 && nw == W && res == 3) return pat ? fused_fn<3, 3, W, true, 1, false>() : fused_fn<3, 3, W, false, 1, false>();
    // one cluster, published rows in distributed shared memory (meshes of a few thousand vertices)
    if (sync == 1 && nw == W && res == 4) return pat ? fused_fn<3, 4, W, true, 1, false>() : fused_fn<3, 4, W, false, 1, false>();
    if (sync == 1 && nw == WS && res == 4) return pat ? fused_fn<3, 4, WS, true, 1, false>() : fused_fn<3, 4, WS, false, 1, false>();
    return nullptr;
}
