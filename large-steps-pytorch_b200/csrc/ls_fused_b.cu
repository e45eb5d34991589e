// ls_fused_b.cu -- fused solver with the Chebyshev polynomial preconditioner (K = 3)
#include "ls_pcg_fused.cuh"
#include "ls_fused_inst.h"

namespace {
#ifndef LS_ZH
#define LS_ZH 1   // publish the preconditioned residual as bf16 rows (ls_pcg_fused.cuh "ZH"); -DLS_ZH=0 builds the fp32-row variant for A/B
#endif
// ZH applies to the 3-column Jacobi instantiations that publish through global memory
template <int K, int RES, int NW, bool PAT, int SYNC, bool PROF, bool CHEB = false>
const void *ffn() {
    constexpr bool ZH = (LS_ZH != 0) && K == 3 && !CHEB && RES != 3;
    return (const void *)lsf::pcg_fused_kernel<K, RES, NW, PAT, SYNC, PROF, CHEB, ZH>;
}
constexpr int W = lsf::PWARPS, WS = lsf::PT_SMALL / 32;
}  // namespace

const void *ls_fused_fn_cheb(int res, int nw, int pat, int sync) {
    if (sync == 0 && nw == W) {
        if (res == 0) return pat ? ffn<3, 0, W, true, 0, false, true>() : ffn<3, 0, W, false, 0, false, true>();
        if (res == 1) return pat ? ffn<3, 1, W, true, 0, false, true>() : ffn<3, 1, W, false, 0, false, true>();
        if (res == 2) return pat ? ffn<3, 2, W, true, 0, false, true>() : ffn<3, 2, W, false, 0, false, true>();
    }
    if (sync == 0 && nw == WS && res == 2) return pat ? ffn<3, 2, WS, true, 0, false, true>() : ffn<3, 2, WS, false, 0, false, true>();
    if (sync == 1 && nw == W && res == 2) return pat ? ffn<3, 2, W, true, 1, false, true>() : ffn<3, 2, W, false, 1, false, true>();
    return nullptr;
}
