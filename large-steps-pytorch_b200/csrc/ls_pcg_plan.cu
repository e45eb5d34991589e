// ls_pcg_plan.cu -- the launch plans of the fused solver (single mesh: plan_fused, auto_precond) and of the batched solve, with
// the environment switches they read.  Host code only, no CUDA call: ls_pcg_plan and ls_pcg_batch_plan_ex run them without a
// device, and ls_pcg_create / ls_pcg_batch_create then ask the device whether it accepts the plan.
#include <stdlib.h>
#include <string.h>
#include "ls_pcg_handle.h"
#include "ls_fused_inst.h"

#ifndef LS_CLRES_DEFAULT
#define LS_CLRES_DEFAULT 0     // slices (x 32 vertices); 0 = off: measured slower than the cooperative grid, see CLRES_CS
#endif

using namespace lspcg;

namespace {

static int env_int(const char *name, int dflt) {
    const char *e = getenv(name);
    return (e && e[0]) ? atoi(e) : dflt;
}

// LS_PCG_CLRES=N (opt-in): meshes of (one CTA's worth) < slices <= N run as ONE cluster of 16 CTAs with every vector -- the
// published rows included -- in (distributed) shared memory: RES = 4 of ls_pcg_fused.cuh; inside the iteration nothing but matrix
// entries comes from global memory.  It is off by default because the cooperative grid with the Chebyshev steps is faster on
// these sizes: the gathers go through distributed shared memory (14 remote 8-byte loads per row), a cluster synchronisation that
// carries a deterministic reduction (fp64 shuffle trees, 16 remote stores, barrier.cluster with release/acquire, fixed-order
// re-sum) costs far more than a bare barrier.cluster, and 16 SMs are 16 SMs.
constexpr int CLRES_CS = 16;

// slices per CTA that fit in max_smem bytes of shared memory at residency level res (sync = 1: the one-CTA / cluster layout)
int slices_per_cta(int K, int res, int pat, int cheb, int sync, int max_smem) {
    if (res == 0) return 1 << 30;
    int n = 0;
    while (lsf::fused_smem_bytes(K, res, n + 1, pat, cheb, sync) <= (size_t)max_smem) ++n;
    return n;
}

constexpr int BATCH_CS_MAX = 16;

}  // namespace

namespace lspcg {

// instantiation table of the fused solver (ls_pcg_fused.cuh): (K, RES, NW, PAT, SYNC, PROF, CHEB) -> kernel, or NULL when that
// combination is not built.  The instantiations live in three translation units (ls_fused_a/b/c.cu) so that they compile in parallel.
const void *fused_fn(int K, int res, int nw, int pat, int sync, int prof, int cheb) {
    if (cheb) return (K == 3 && !prof) ? ls_fused_fn_cheb(res, nw, pat, sync) : nullptr;
    if (K == 3 && !prof) return ls_fused_fn_jacobi(res, nw, pat, sync);
    return ls_fused_fn_misc(K, res, nw, pat, sync, prof);
}

PlanEnv plan_env() {
    const char *mode = getenv("LS_PCG_MODE"), *small = getenv("LS_PCG_SMALLCTA");
    PlanEnv e;
    e.graph = mode && (mode[0] == 'g' || mode[0] == 'G');
    e.cluster = env_int("LS_PCG_CLUSTER", -1);
    e.res = env_int("LS_PCG_RES", -1);
    e.onecta = env_int("LS_PCG_ONECTA", lsf::PWARPS);
    e.clres = env_int("LS_PCG_CLRES", LS_CLRES_DEFAULT);
    e.small_cta = !(small && small[0] == '0');
    return e;
}

CreateEnv create_env() {
    const char *pat = getenv("LS_PCG_PATTERN"), *engine = getenv("LS_SPMM_ENGINE");
    CreateEnv e;
    e.force_reorder = getenv("LS_FORCE_REORDER") != nullptr;
    e.pattern = !(pat && pat[0] == '0');
    e.patshare = env_int("LS_PCG_PATSHARE", 1) != 0;
    e.csr = engine && (engine[0] == 'c' || engine[0] == 'C');
    const int m = env_int("LS_PCG_CHEB_M", 4);
    e.cheb_m = m < 2 ? 2 : (m > 8 ? 8 : m);
    e.refine = env_int("LS_PCG_REFINE", 1);
    e.sell_tma = env_int("LS_SELL_TMA", 3);
    e.sell_pf = env_int("LS_SELL_PF", 1024);
    return e;
}

// precond = 3 (auto) -> 1 or 2.  The polynomial pays where the iteration is synchronisation-bound and its vectors fit in shared
// memory -- the cooperative grid at residency level 2 (V = 1e6, whose vectors do not fit, and the single CTA, which is issue-bound,
// run Jacobi) -- and not where one cluster holds everything in shared memory: a synchronisation costs a tenth there, plain CG's
// fewer SpMVs win.
int auto_precond(int nslices, int sm_count, int max_smem, const PlanEnv &env) {
    if (nslices <= env.onecta) return 1;
    if (env.cluster != 0 && nslices <= env.clres) return 1;
    const int g = sm_count < nslices ? sm_count : nslices;
    const int nsl_max = (nslices + g - 1) / g;
    // (sized with 4 bytes more per row than the general copy needs, as when the pattern copy kept its diagonal there)
    const bool fits = lsf::fused_smem_bytes(3, 2, nsl_max, 0, 1, 0) + (size_t)nsl_max * 32 * 4 <= (size_t)max_smem;
    return fits ? 2 : 1;
}

// Small meshes (the CTA-resident rows of <= 16 SMs hold them) run on ONE CTA or, on request, as ONE thread-block cluster;
// everything else as a cooperative grid with one CTA per SM.  Host code only: ls_pcg_plan runs it without a device.
FusedPlan plan_fused(int nslices, int K, int pat, int cheb, int sm_count, int max_smem, int coop, const PlanEnv &env) {
    FusedPlan p{};
    if (env.graph) return p;
    const int W = lsf::PWARPS;
    // ---- one CTA (everything, including the gathered vector, in shared memory) or, on request, one cluster
    // A cluster of 16 is slower than the cooperative grid for mid-size meshes: 16 SMs give 16 SMs' worth of L2 bandwidth and
    // cluster.sync flushes L1 each time, so it is opt-in (LS_PCG_CLUSTER=N).
    int cs = 0;
    if (env.cluster != 0) {
        // one CTA only while every warp has at most one slice: beyond that the single SM is instruction-issue bound and the
        // cooperative grid wins despite its two grid synchronisations per iteration
        if (nslices <= env.onecta) cs = 1;
        else if (!cheb && nslices <= env.clres) cs = CLRES_CS;
        if (env.cluster > 0) cs = env.cluster;
        if (cs > 0 && (nslices + cs - 1) / cs > slices_per_cta(K, 2, pat, cheb, 1, max_smem)) cs = 0;
    }
    if (cs > 0) {
        const int nsl_max = (nslices + cs - 1) / cs;
        const bool res3 = cs == 1 && K == 3 && !cheb && nsl_max <= slices_per_cta(K, 3, pat, cheb, 1, max_smem);
        int res = (res3 && !(env.res >= 0 && env.res < 3)) ? 3 : 2;
        int nw = W;
        int cap4 = slices_per_cta(K, 4, pat, cheb, 1, max_smem);
        if (cap4 > 63) cap4 = 63;   // (63: the owner of a row is found by a 16-bit multiply)
        if (cs > 1 && !cheb && nsl_max <= cap4 && !(env.res >= 0 && env.res < 4)) {
            res = 4;
            if (K == 3 && nsl_max <= lsf::PT_SMALL / 32 && env.small_cta) nw = lsf::PT_SMALL / 32;
        }
        if (res == 4 && !fused_fn(K, res, nw, pat, 1, 0, cheb)) { res = 2; nw = W; }
        if (fused_fn(K, res, nw, pat, 1, 0, cheb)) return {1, cs, cs, res, nw, 1, nsl_max, lsf::fused_smem_bytes(K, res, nsl_max, pat, cheb, 1)};
    }
    // ---- cooperative grid, one CTA per SM
    if (!coop) return p;
    int g = sm_count < nslices ? sm_count : nslices;
    if (g > 255) g = 255;
    if (g < 1) g = 1;
    const int nsl_max = (nslices + g - 1) / g;
    int res = nsl_max <= slices_per_cta(K, 2, pat, cheb, 0, max_smem) ? 2 : (nsl_max <= slices_per_cta(K, 1, pat, cheb, 0, max_smem) ? 1 : 0);
    if (env.res >= 0 && env.res < res) res = env.res;
    int nw = W;
    if (K == 3 && res == 2 && nsl_max <= 16 && env.small_cta) nw = lsf::PT_SMALL / 32;
    if (!fused_fn(K, res, nw, pat, 0, 0, cheb)) return p;
    return {1, g, 0, res, nw, 0, nsl_max, lsf::fused_smem_bytes(K, res, nsl_max, pat, cheb, 0)};
}

}  // namespace lspcg

extern "C" int ls_pcg_plan(int nslices, int k, int pat, int precond, int sm_count, int max_smem, int coop, int64_t *out8) {
    LS_REQUIRE(out8 != nullptr, "out8 is NULL");
    LS_REQUIRE(nslices >= 1, "nslices must be positive");
    LS_REQUIRE(k == 3 || k == 4, "k must be 3 or 4 (the column counts of the fused kernel's instantiations)");
    LS_REQUIRE(precond >= 0 && precond <= 3, "precond must be 0 (none), 1 (Jacobi), 2 (Chebyshev polynomial over Jacobi) or 3 (auto)");
    LS_REQUIRE(sm_count >= 1 && max_smem > 0, "sm_count and max_smem must be positive");
    const PlanEnv env = plan_env();
    if (precond == 3) precond = auto_precond(nslices, sm_count, max_smem, env);
    const int cheb = (k == 3 && precond == 2) ? 1 : 0;
    const FusedPlan p = plan_fused(nslices, k, (k == 3 && pat) ? 1 : 0, cheb, sm_count, max_smem, coop ? 1 : 0, env);
    const int64_t o[8] = {p.on, p.grid, p.cluster, p.res, p.nw * 32, precond, (int64_t)p.smem, p.nsl_max};
    memcpy(out8, o, sizeof(o));
    return LS_OK;
}

extern "C" int ls_pcg_batch_plan_ex(int n, const int32_t *nslices, const int32_t *pat, const int32_t *cheb, int max_smem,
                                    int32_t *cluster, int32_t *res, int32_t *group, int32_t *n_groups) {
    LS_REQUIRE(n >= 1, "the batch is empty");
    LS_REQUIRE(nslices && pat && cluster && res && group && n_groups, "NULL pointer");
    LS_REQUIRE(max_smem > 0, "max_smem must be positive");
    int keys[2 * 2 * 2 * 5] = {0};   // (preconditioner, pattern copy, RES 2 / 3, cluster size 1 2 4 8 16) -> group id + 1
    int ng = 0;
    for (int i = 0; i < n; ++i) {
        LS_REQUIRE(nslices[i] >= 1, "every mesh needs at least one slice of 32 rows");
        const int c = cheb ? cheb[i] : 0;
        if (c != 0 && c != 1) {
            ls_set_error("bad argument: cheb[%d] = %d: 0 (Jacobi) or 1 (Chebyshev)", i, c);
            return LS_ERR_BAD_ARG;
        }
        const int p = pat[i] ? 1 : 0;
        const int cap2 = slices_per_cta(3, 2, p, c, 1, max_smem), cap3 = c ? 0 : slices_per_cta(3, 3, p, 0, 1, max_smem);
        int cs = 1, lg = 0;
        while (cs <= BATCH_CS_MAX && (nslices[i] + cs - 1) / cs > cap2) {
            cs *= 2;
            ++lg;
        }
        if (cs > BATCH_CS_MAX) {
            ls_set_error("bad argument: mesh %d has %d rows; one cluster of %d CTAs holds at most %d rows with its matrix copy%s "
                         "(%d per CTA): solve it on its own (ls_pcg_solve, from_differential)",
                         i, 32 * nslices[i], BATCH_CS_MAX, 32 * cap2 * BATCH_CS_MAX, c ? " and the Chebyshev vectors" : "", 32 * cap2);
            return LS_ERR_BAD_ARG;
        }
        // one CTA: everything, the gathered vector included, in shared memory where it fits (as the single-mesh solve);
        // a Chebyshev mesh runs at RES 2 on any cluster, as the single-mesh solve runs it on one CTA
        const int r = (cs == 1 && nslices[i] <= cap3) ? 3 : 2;
        int &key = keys[((c * 2 + p) * 2 + (r - 2)) * 5 + lg];
        if (key == 0) key = ++ng;
        cluster[i] = cs;
        res[i] = r;
        group[i] = key - 1;
    }
    *n_groups = ng;
    return LS_OK;
}
