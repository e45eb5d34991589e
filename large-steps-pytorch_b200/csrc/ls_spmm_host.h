// ls_spmm_host.h -- host-side interface of the SpMM launcher shared by ls_spmm.cu and ls_pcg_graph.cu
#pragma once
#include "ls_spmm_kernel.cuh"

namespace lsk {
struct SpmmCfg {
    int stages, cap, unroll, hint, debug;
};
void spmm_config(SpmmCfg *cfg);
// solver_layout = true: SoA planes + dot epilogue (in-solver); false: AoS, no epilogue (public to_differential)
int spmm_prepare(int K, bool solver_layout, const SpmmCfg &cfg, int *ctas_per_sm);
int spmm_launch(int K, bool solver_layout, const SpmmCfg &cfg, const SpmmArgs &a, int grid, cudaStream_t stream);
int spmm_grid_for(int64_t V, int sm_count, int occ);
int spmm_plan(const int *rowptr, const int *part, int G, int cap, int4 *desc, int *desc_cnt, int *overflow,
              cudaStream_t stream);
}  // namespace lsk
