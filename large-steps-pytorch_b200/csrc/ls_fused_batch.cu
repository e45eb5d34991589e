// ls_fused_batch.cu -- batch instantiations of the fused solver: one thread-block cluster per mesh, many meshes per launch
// (K = 3; Jacobi: RES 3 for a mesh on one CTA, RES 2 for a cluster of 1..16 CTAs; Chebyshev: RES 2 on a cluster of 1..16 CTAs)
#include "ls_pcg_fused.cuh"
#include "ls_fused_inst.h"

namespace {
#ifndef LS_ZH
#define LS_ZH 1   // publish the preconditioned residual as bf16 rows (ls_pcg_fused.cuh "ZH"), as the single-mesh instantiations do
#endif
template <int RES, bool PAT>
const void *bfn() {
    constexpr bool ZH = (LS_ZH != 0) && RES != 3;
    return (const void *)lsf::pcg_fused_kernel<3, RES, lsf::PWARPS, PAT, 1, false, false, ZH, true>;
}
// Chebyshev: fp32 rows (the iterates need full precision), as the single-mesh Chebyshev instantiations
template <bool PAT>
const void *bfn_cheb() {
    return (const void *)lsf::pcg_fused_kernel<3, 2, lsf::PWARPS, PAT, 1, false, true, false, true>;
}
}  // namespace

const void *ls_fused_fn_batch(int res, int pat) {
    if (res == 3) return pat ? bfn<3, true>() : bfn<3, false>();
    if (res == 2) return pat ? bfn<2, true>() : bfn<2, false>();
    return nullptr;
}

const void *ls_fused_fn_batch_cheb(int pat) { return pat ? bfn_cheb<true>() : bfn_cheb<false>(); }
