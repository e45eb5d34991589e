/*
 * largesteps_b200_diag.h -- diagnostics and timing harnesses of libls_b200.so.  NOT part of the drop-in boundary
 * (include/largesteps_b200.h): nothing on the product path calls these; bench.py and the tests do.
 */
#ifndef LARGESTEPS_B200_DIAG_H
#define LARGESTEPS_B200_DIAG_H

#include "largesteps_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* in-solver SpMM of the handle's own matrix copy on SoA planes, for profiling the dominant kernel:
 *   runs `launches` back-to-back launches of the solver's SpMM+dot kernel on its internal p/Ap planes.  */
int ls_pcg_bench_spmm(void *handle, int k, int launches, void *stream);
/* timing harness for the in-solver SpMM, launched back-to-back from C (a Python-level loop is launch-bound):
 *   `launches` launches rotating over `n_handles` handles (use enough handles that matrix+vectors exceed L2 for an
 *   HBM-cold number, one handle for the L2-resident number).  which: 0 SpMM+dot, 4 SpMM without the dot-product
 *   epilogue (the plain SpMV of BASELINE's metric); any other value is LS_ERR_BAD_ARG. */
int ls_pcg_bench(void **handles, int n_handles, int k, int which, int launches, void *stream);
/* input and output of the handle's stand-alone SpMM (what ls_pcg_bench with which = 0 or 4 and ls_pcg_bench_spmm launch),
 * so that a test reads exactly what the timed launches compute.  Both are stream-ordered; x, y and dot are device memory.
 *   put: x (V, k) row-major in the caller's vertex numbering -> the SpMM's input p (rows of 1, 2, 4 floats for k = 1, 2, 3|4,
 *        in the handle's own numbering when it re-ordered its copy; unused lanes and the padding rows up to V rounded up to
 *        32 are 0).  It also sets rows 0 .. V-1 of the k output planes and the k dot products to NaN, so that a row or a dot
 *        product the next launch does not write reads back as NaN.
 *   get: y (V, k) row-major in the caller's numbering <- the k output planes; dot (k doubles, may be NULL) <- the p.Ap
 *        epilogue's result.  The handle's next solve re-initialises everything put and the launches touched.            */
int ls_pcg_spmv_put(void *handle, int k, const float *x, void *stream);
int ls_pcg_spmv_get(void *handle, int k, float *y, double *dot, void *stream);
/* the plan ls_pcg_batch_create makes, as a pure host function (no device needed): for mesh i with nslices[i] slices of 32
 * rows, pat[i] != 0 for the pattern-only matrix copy and cheb[i] = 1 for a handle whose preconditioner is Chebyshev (precond 2),
 * 0 for Jacobi (cheb = NULL: all Jacobi), given max_smem bytes of shared memory per CTA, writes its cluster size (1, 2, 4, 8,
 * 16), residency level (3: one CTA with the gathered vector in shared memory, else 2) and plan group (0 .. n_groups - 1,
 * numbered in order of first appearance; one launch each).  A Chebyshev mesh keeps two more vectors in shared memory (the
 * iterate and the direction, 24 B per row) and always runs at RES 2, also on one CTA; its cluster is the smallest that holds
 * it at that size.  Groups are keyed by (preconditioner, pattern copy, RES, cluster size).  LS_ERR_BAD_ARG, naming the mesh,
 * when a mesh does not fit one cluster of 16, and for any other value in cheb[].                                           */
int ls_pcg_batch_plan_ex(int n, const int32_t *nslices, const int32_t *pat, const int32_t *cheb, int max_smem,
                         int32_t *cluster, int32_t *res, int32_t *group, int32_t *n_groups);
/* the fused solver's launch plan ls_pcg_create makes, as a pure host function (no device needed), with the plan's environment
 * switches (LS_PCG_MODE, _CLUSTER, _RES, _ONECTA, _CLRES, _SMALLCTA) read from the process environment: for a mesh of nslices
 * slices of 32 rows with its SELL-32 copy, k = 3 (the instantiations for k = 1..3) or 4, pat != 0 for the pattern-only matrix copy,
 * precond as ls_pcg_create, on a device with sm_count SMs, max_smem bytes of shared memory per CTA and cooperative launch if
 * coop != 0, writes out8 = [fused solver on (0: graph mode), grid, cluster size (0: cooperative grid), residency level, threads per
 * CTA, preconditioner (auto resolved), shared-memory bytes per CTA, slices per CTA].  These are the values ls_pcg_describe reports
 * for a handle whose device accepts the plan.                                                                                     */
int ls_pcg_plan(int nslices, int k, int pat, int precond, int sm_count, int max_smem, int coop, int64_t *out8);
/* the handle's pattern-only matrix copy (on when every off-diagonal value is the same): info4 = [on, slices, slices stored,
 * words in use].  Identical compact slices share one stored copy unless LS_PCG_PATSHARE=0 was set at ls_pcg_create.  With
 * poff (slices + 1 ints) and words (words in use) both non-NULL and the copy on, also copies the slice offsets (bit 0: wide,
 * bits 1-4: pairs per row, 15 = up to the next slice's offset) and the words to the host.                                */
int ls_pcg_pattern_copy(void *handle, int64_t *info4, int32_t *poff, uint32_t *words, void *stream);
/* with LS_PCG_PROFILE set in the environment the fused kernel's CTA 0 accumulates SM-clock cycles per phase of
 * the last solve: out8 = [phase A (SpMV + x/p/s update), all-reduce of p.s, phase B (r, z), all-reduce of
 * r.z / r.r (publishes z), true-residual restarts, 0, restarts, iterations]                                            */
int ls_pcg_phase_cycles(void *handle, int64_t *out, int n /* 8, or 8 + 8*grid for the per-CTA table (.., smid, it) */, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* LARGESTEPS_B200_DIAG_H */
