// ls_fused_batch.cu -- batch instantiations of the fused solver: one thread-block cluster per mesh, many meshes per launch
// (K = 3; Jacobi: RES 3 for a mesh on one CTA, RES 2 for a cluster of 1..16 CTAs; Chebyshev: RES 2 on a cluster of 1..16 CTAs)
#include "ls_pcg_fused.cuh"
#include "ls_fused_inst.h"

namespace {
using lsf::fused_fn;
constexpr int W = lsf::PWARPS;
}  // namespace

const void *ls_fused_fn_batch(int res, int pat) {
    if (res == 3) return pat ? fused_fn<3, 3, W, true, 1, false, false, true>() : fused_fn<3, 3, W, false, 1, false, false, true>();
    if (res == 2) return pat ? fused_fn<3, 2, W, true, 1, false, false, true>() : fused_fn<3, 2, W, false, 1, false, false, true>();
    return nullptr;
}

const void *ls_fused_fn_batch_cheb(int pat) {
    return pat ? fused_fn<3, 2, W, true, 1, false, true, true>() : fused_fn<3, 2, W, false, 1, false, true, true>();
}
