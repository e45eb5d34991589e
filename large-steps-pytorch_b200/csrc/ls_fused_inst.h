// ls_fused_inst.h -- where the instantiations of lsf::pcg_fused_kernel live (four translation units, compiled in parallel; each
// instantiates through lsf::fused_fn in ls_pcg_fused.cuh, which sets the ZH flag)
#pragma once
// K = 3, Jacobi, production:  RES 0..2 x {768, 256 threads (RES 2)} x pattern/general on the grid; one CTA / cluster at RES 2, 3
const void *ls_fused_fn_jacobi(int res, int nw, int pat, int sync);
// K = 3 with the Chebyshev polynomial preconditioner
const void *ls_fused_fn_cheb(int res, int nw, int pat, int sync);
// profiling instantiations (per-phase cycle counters) and K = 4
const void *ls_fused_fn_misc(int K, int res, int nw, int pat, int sync, int prof);
// batches (one cluster per mesh, K = 3, Jacobi, 768 threads): RES 3 (one CTA) or 2, pattern/general; kernel parameter lsf::BatchParams
const void *ls_fused_fn_batch(int res, int pat);
// batches with the Chebyshev polynomial preconditioner: RES 2 on a cluster of 1..16 CTAs, pattern/general
const void *ls_fused_fn_batch_cheb(int pat);
