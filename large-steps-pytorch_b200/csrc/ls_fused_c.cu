// ls_fused_c.cu -- profiling instantiations (per-phase cycle counters) and the 4-column instantiations
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

const void *ls_fused_fn_misc(int K, int res, int nw, int pat, int sync, int prof) {
    if (K == 3 && prof && nw == W) {
        if (sync == 0 && res == 1) return pat ? ffn<3, 1, W, true, 0, true>() : ffn<3, 1, W, false, 0, true>();
        if (sync == 0 && res == 2) return pat ? ffn<3, 2, W, true, 0, true>() : ffn<3, 2, W, false, 0, true>();
        if (sync == 1 && res == 2) return pat ? ffn<3, 2, W, true, 1, true>() : ffn<3, 2, W, false, 1, true>();
        if (sync == 1 && res == 3) return pat ? ffn<3, 3, W, true, 1, true>() : ffn<3, 3, W, false, 1, true>();
        if (sync == 1 && res == 4) return pat ? ffn<3, 4, W, true, 1, true>() : ffn<3, 4, W, false, 1, true>();
    }
    if (K == 3 && prof && nw == WS && sync == 1 && res == 4) return pat ? ffn<3, 4, WS, true, 1, true>() : ffn<3, 4, WS, false, 1, true>();
    if (K == 4 && !prof && !pat && nw == W) {
        if (sync == 0 && res == 0) return ffn<4, 0, W, false, 0, false>();
        if (sync == 0 && res == 1) return ffn<4, 1, W, false, 0, false>();
        if (sync == 0 && res == 2) return ffn<4, 2, W, false, 0, false>();
        if (sync == 1 && res == 2) return ffn<4, 2, W, false, 1, false>();
        if (sync == 1 && res == 4) return ffn<4, 4, W, false, 1, false>();
    }
    return nullptr;
}
