// ls_pcg.cu -- preconditioned conjugate gradients for M X = B, all K columns in one pass (sm_90a): the handle and its
// workspace carve, the C entry points create / solve / destroy, and the fused solver's device checks and launch.  The other
// concerns live beside it (ls_pcg_handle.h lists them): the matrix copies, the graph-mode solver, the launch plans, the batch.
//
// Replaces the reference's solve plug-ins (largesteps/solvers.py:26-39 CholeskySolver -> cholespy/CHOLMOD,
// solvers.py:41-126 ConjugateGradientSolver -> ~12 eager torch kernels + 1 host sync per iteration per axis).
//
// Two execution modes share the handle, the data layout and the per-column arithmetic:
//   * fused (ls_pcg_fused.cuh): the whole solve is ONE kernel with two grid synchronisations per iteration, in-kernel warm
//     start and true-residual guard, optional Chebyshev polynomial preconditioner -- the default for every k in 1..4;
//     cooperative grid (one CTA per SM), one CTA for tiny meshes, or (opt-in) one thread-block cluster;
//   * graph (ls_pcg_graph.cu): three kernels per iteration replayed as a CUDA graph -- the fallback when the fused kernel
//     cannot run (no cooperative launch, no SELL-32 copy, or its launch refused).
//
// Data layout in HBM (all inside the caller-provided workspace):
//   CSR copy  rowptr (V+1) int32, col (nnz) int32, val (nnz) fp32, padded so 16-byte TMA granules never leave it;
//             optionally re-ordered P A P^T (Morton order of the vertices, kept only if it gathers more coherently)
//   SELL-32   soff (V/32+1), ent (padded nnz) int2 {col, val}: the fast SpMM engine's copy
//   dinv      Vp fp32                      Jacobi 1/diag (0 in the padding)
//   x r Ap    K planes of Vp fp32 each     SoA: plane k holds column k; Vp = V rounded up to 32 (zero padded)
//   p         Vp rows of PW floats         PW = 1, 2, 4 for K = 1, 2, 3|4: a gather of p[col] is one load
//   ctrl      PcgCtrl                      device-resident scalars: the iteration never returns to the host for them
// Columns carry their own alpha/beta and freeze independently when ||r_k|| <= rtol ||b_k||, which is exactly the
// reference's "one CG per axis" (solvers.py:115-118) run in lock-step.  Dot products accumulate in fp64.
#include <new>
#include <string.h>
#include <stdlib.h>
#include "ls_pcg_handle.h"

using namespace lspcg;

namespace {

// Takes 256-byte aligned regions of the workspace one after the other; with no base it only counts (NULL pointers).
struct Carve {
    char *base;
    size_t off = 0;
    template <class T>
    T *take(size_t count) {
        T *p = base ? reinterpret_cast<T *>(base + off) : nullptr;
        off = ls_align_up(off + count * sizeof(T), 256);
        return p;
    }
    PcgHandle::Span since(size_t from) const { return {base ? base + from : nullptr, off - from}; }
};

// Lays the handle's regions out in the workspace (h may be a scratch handle when only the size is wanted) and returns the total.
// The two runs marked `zeroed` are what has to start at zero: the vector planes with their padding rows, the scalars and the
// counters.  The matrix copies between them are written in full by ls_pcg_create: at V = 1e6 that is ~100 MB of memset
// instead of ~500 MB.
size_t carve_handle(PcgHandle &h, char *base, int64_t V, int64_t nnz, int k_max, int grid_cap) {
    Carve c{base};
    const int64_t Vp = (V + 31) / 32 * 32;
    const long long sell_cap = (long long)nnz + nnz / 2 + 32768;
    constexpr int RING_SLOTS = 32768;              // fast all-reduce slots (64 B each): 2 per iteration
    h.Vp = Vp;
    h.nslices = (int)(Vp / 32);
    h.sell_cap = h.pat_cap = sell_cap;
    h.ring_slots = RING_SLOTS;
    h.rowptr = c.take<int>(V + 1 + 8);
    h.col = c.take<int>(nnz + 8);
    h.val = c.take<float>(nnz + 8);
    size_t from = c.off;
    h.dinv = c.take<float>(Vp);
    h.x = c.take<float>(Vp * k_max);
    h.r = c.take<float>(Vp * k_max);
    h.p = c.take<float>(Vp * 4);                   // p: rows of PW <= 4 floats
    h.Ap = c.take<float>(Vp * k_max);
    h.pv = c.take<float>(Vp * k_max);
    h.z2 = c.take<float>(Vp * 4);
    h.cy = c.take<float>(Vp * k_max);
    h.cd = c.take<float>(Vp * k_max);
    h.graph.part = c.take<int>(grid_cap + 1);
    h.graph.desc = c.take<int4>((size_t)grid_cap * lsk::SPMM_BMAX);
    h.graph.desc_cnt = c.take<int>(grid_cap);
    h.zeroed[0] = c.since(from);
    h.soff = c.take<int>(Vp / 32 + 2);
    h.ent = c.take<int2>(sell_cap);
    from = c.off;
    h.perm = c.take<int>(V + 8);
    h.inv = c.take<int>(V + 8);
    h.scan = c.take<int>(ls_scan_scratch_elems(V + 1));
    h.ctrl = c.take<PcgCtrl>(1);
    h.part_spmm = c.take<double>((size_t)grid_cap * KMAX);
    h.part_vec = c.take<double>((size_t)grid_cap * 3 * KMAX);
    h.gbar = c.take<lsf::GridBar>(8);
    h.partials = c.take<double>(2 * lsf::NVMAX * 256);
    h.dbg = c.take<long long>(8 + 8 * 256);
    h.ring = c.take<unsigned long long>((size_t)RING_SLOTS * 8);
    h.tickets = c.take<unsigned int>(16);
    h.info = c.take<float>(16);
    h.flags = c.take<int>(16);
    h.zeroed[1] = c.since(from);
    // pattern-only copy (always carved: the workspace size must not depend on the environment)
    h.poff = c.take<int>(Vp / 32 + 2);
    h.pcol = c.take<unsigned int>(sell_cap);        // words: a wide pair (8 bytes) holds two of the general copy's 8-byte entries
    h.pcls = c.take<unsigned char>(Vp);
    h.pcls_tab = c.take<unsigned long long>(lsk::PAT_CLASSES + 8);
    h.patmm = c.take<unsigned int>(16);
    h.gersh = c.take<float>(16);
    return c.off;
}

// Prepares the plan's kernel and asks the device whether it runs: one cluster resident, or every CTA of the grid co-resident.
bool device_accepts(const void *fn, const FusedPlan &p, const LsDevInfo &di) {
    if (p.cluster > 1) return cluster_fits(fn, p.cluster, p.nw * 32, p.smem, di);   // (a cluster plan's grid is one cluster)
    bool ok = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, di.max_smem_optin) == cudaSuccess;
    if (ok && p.sync == 0) {
        int occ = 0;
        ok = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, p.nw * 32, p.smem) == cudaSuccess && occ >= 1 &&
             occ * di.sm_count >= p.grid;
    }
    cudaGetLastError();
    return ok;
}

// The fused solver's configuration for one K: the plan, checked on the device.  A one-CTA or cluster plan the device refuses
// falls back to the cooperative grid; without cooperative launch, or with the grid refused, the fused solver stays off.
void configure_fused(PcgHandle *h, const LsDevInfo &di, const PlanEnv &env, int K, PcgHandle::FusedCfg *c) {
    memset(c, 0, sizeof(*c));
    if (!h->sell_on) return;
    const int cheb = (K == 3 && h->cheb_m > 1) ? 1 : 0;
    const int pat = (K == 3 && h->pat_on) ? 1 : 0;
    int coop = 0;
    if (cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, di.device) != cudaSuccess) {
        coop = 0;
        cudaGetLastError();
    }
    auto kernel = [&](const FusedPlan &q, int prof) { return fused_fn(K, q.res, q.nw, pat, q.sync, prof, cheb); };
    FusedPlan p = plan_fused(h->nslices, K, pat, cheb, di.sm_count, di.max_smem_optin, coop, env);
    if (p.on && p.sync == 1 && !device_accepts(kernel(p, 0), p, di)) {
        PlanEnv grid_only = env;
        grid_only.cluster = 0;
        p = plan_fused(h->nslices, K, pat, cheb, di.sm_count, di.max_smem_optin, coop, grid_only);
    }
    if (!p.on || (p.sync == 0 && !device_accepts(kernel(p, 0), p, di))) return;
    static_cast<FusedPlan &>(*c) = p;
    c->pat = pat;
    c->fn = kernel(p, 0);
    c->fn_prof = kernel(p, 1);   // (NULL with the Chebyshev steps: no profiling instantiation)
    if (c->fn_prof) {
        cudaFuncSetAttribute(c->fn_prof, cudaFuncAttributeMaxDynamicSharedMemorySize, di.max_smem_optin);
        if (p.cluster > 8) cudaFuncSetAttribute(c->fn_prof, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    }
    cudaGetLastError();
}

// Launches the fused solver; -1 when the launch is refused (the graph-mode solver then runs), else an LS_* status.
int solve_fused(PcgHandle *h, const float *b, float *x, const float *x0, int k, float rtol, int maxit, float *info,
                cudaStream_t stream) {
    PcgHandle::FusedCfg &c = h->fused[k == 4 ? 1 : 0];
    lsf::FusedArgs a{};
    fused_handle_args(h, c.nsl_max, a);
    a.kb = k;
    if (k == 4) a.cheb_m = 0;     // (the K = 4 instantiations carry the Jacobi preconditioner only)
    a.b = b;
    a.out = x;
    a.x0 = x0;
    a.rtol = rtol;
    a.maxit = maxit;
    a.bar = h->gbar;
    a.partials = h->partials;
    a.info = info;
    const bool prof = getenv("LS_PCG_PROFILE") != nullptr && c.fn_prof != nullptr;
    a.dbg = prof ? h->dbg : nullptr;
    const void *fn = prof ? c.fn_prof : c.fn;
    void *params[] = {(void *)&a};
    cudaError_t ce;
    if (c.sync == 1) {
        if (c.cluster > 1) {
            cudaLaunchAttribute at;
            const cudaLaunchConfig_t lc = cluster_launch(c.grid, c.cluster, c.nw * 32, c.smem, stream, &at);
            ce = cudaLaunchKernelExC(&lc, fn, params);
        } else {
            ce = cudaLaunchKernel(fn, dim3(1), dim3(c.nw * 32), params, c.smem, stream);
        }
    } else {
        LS_CUDA_TRY(cudaMemsetAsync(h->gbar, 0, sizeof(lsf::GridBar), stream));
        long long need = 2LL * maxit + 64;
        if (need > h->ring_slots) need = h->ring_slots;
        const char *e = getenv("LS_PCG_FASTRED");
        a.ring = h->ring;
        a.ring_slots = (e && e[0] == '0') ? 0 : (int)need;
        if (e && atoi(e) > 0 && atoi(e) < a.ring_slots) a.ring_slots = atoi(e);
        if (a.ring_slots > 0) LS_CUDA_TRY(cudaMemsetAsync(h->ring, 0, (size_t)a.ring_slots * 64, stream));
        ce = cudaLaunchCooperativeKernel(fn, dim3(c.grid), dim3(c.nw * 32), params, c.smem, stream);
    }
    if (ce != cudaSuccess) {
        // e.g. a partitioned device (MPS / MIG limits) that cannot co-schedule the grid: not fatal, the graph-mode solver
        // computes the same thing; remember the failure so later solves go there directly
        cudaGetLastError();
        c.on = 0;
        ls_set_error("launch of the fused solver failed (%s); using the graph-mode solver", cudaGetErrorString(ce));
        return -1;
    }
    g_ls_launches.fetch_add(1, std::memory_order_relaxed);
    return LS_OK;
}

// The fused solver where it is configured and its launch is accepted, else the graph-mode solver
int solve_k(PcgHandle *h, int k, const float *b, float *x, const float *x0, float rtol, int maxit, float *info_dev,
            float *info_host, cudaStream_t stream) {
    float *info = info_dev ? info_dev : h->info;
    int rc = -1;
    if (h->fused[k == 4 ? 1 : 0].on) rc = solve_fused(h, b, x, x0, k, rtol, maxit, info, stream);
    if (rc == -1) rc = solve_graph(h, k, b, x, x0, rtol, maxit, info, stream);
    if (rc) return rc;
    return finish_info(info, info_host, 1, false, rtol, maxit, stream);
}

// Everything ls_pcg_create does once the handle is carved.  Host round trips: at most two in copy_matrix, one in read_back and one
// in build_pattern_copy.  Flag errors are reported last, after the fused solver is configured.
int build_solver(PcgHandle *h, const int *rowptr, const int *col, const float *val, const int *perm, const LsDevInfo &di,
                 cudaStream_t stream) {
    const PlanEnv env = plan_env();
    const CreateEnv ce = create_env();
    h->refine = ce.refine;
    h->graph.sell_tma = ce.sell_tma;
    h->graph.sell_pf = ce.sell_pf;
    for (const PcgHandle::Span &z : h->zeroed) LS_CUDA_TRY(cudaMemsetAsync(z.at, 0, z.bytes, stream));
    int rc = copy_matrix(h, rowptr, col, val, perm, ce.force_reorder, stream);
    if (rc) return rc;
    rc = graph_geometry(h, stream);
    if (rc) return rc;
    rc = sell_copy(h, stream);
    if (rc) return rc;
    if (h->precond == 3) h->precond = auto_precond(h->nslices, di.sm_count, di.max_smem_optin, env);
    Readback rb;
    rc = read_back(h, ce, rb, stream);
    if (rc) return rc;
    h->graph.planned = (rb.flags[1] == 0) ? 1 : 0;
    if (ce.pattern && h->sell_on && rb.mm[0] == rb.mm[1]) {
        rc = build_pattern_copy(h, rb.mm[0], ce.patshare, stream);
        if (rc) return rc;
    }
    if (h->precond == 2 && rb.gersh > 0.f) {
        h->cheb_m = ce.cheb_m;
        chebyshev_coefficients(rb.gersh, h->cheb_m, h->cheb_c0, h->cheb_c1, h->cheb_c2);
    }
    configure_fused(h, di, env, 3, &h->fused[0]);
    if (h->k_max >= 4) configure_fused(h, di, env, 4, &h->fused[1]);
    return flag_error(rb.flags[0]);
}

}  // namespace

namespace lspcg {

// launch configuration of `grid` CTAs in clusters of `cluster` CTAs; `at` receives the cluster attribute the configuration points to
cudaLaunchConfig_t cluster_launch(int grid, int cluster, int threads, size_t smem, cudaStream_t stream, cudaLaunchAttribute *at) {
    cudaLaunchConfig_t lc = {};
    lc.gridDim = dim3(grid);
    lc.blockDim = dim3(threads);
    lc.dynamicSmemBytes = smem;
    lc.stream = stream;
    at->id = cudaLaunchAttributeClusterDimension;
    at->val.clusterDim.x = cluster;
    at->val.clusterDim.y = 1;
    at->val.clusterDim.z = 1;
    lc.attrs = at;
    lc.numAttrs = 1;
    return lc;
}

// Prepares `fn` and asks the device whether it can run one cluster of `cluster` CTAs with `smem` bytes of shared memory each.
// The shared-memory attribute is per function and device, shared by every handle: always the device maximum, never a per-handle size.
bool cluster_fits(const void *fn, int cluster, int threads, size_t smem, const LsDevInfo &di) {
    bool ok = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, di.max_smem_optin) == cudaSuccess;
    if (ok && cluster > 8) ok = cudaFuncSetAttribute(fn, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) == cudaSuccess;
    if (ok) {
        cudaLaunchAttribute at;
        const cudaLaunchConfig_t lc = cluster_launch(cluster, cluster, threads, smem, 0, &at);
        int ncl = 0;
        ok = cudaOccupancyMaxActiveClusters(&ncl, fn, &lc) == cudaSuccess && ncl >= 1;
    }
    cudaGetLastError();
    return ok;
}

// the fused kernel's arguments that depend on the handle only (the single-mesh solve and the batch table share them)
void fused_handle_args(const PcgHandle *h, int nsl_max, lsf::FusedArgs &a) {
    a.V = (int)h->V;
    a.Vp = h->Vp;
    a.nslices = h->nslices;
    a.nsl_max = nsl_max;
    a.soff = h->soff;
    a.ent = h->ent;
    a.poff = h->poff;
    a.pcol = h->pcol;
    a.pcls = h->pcls;
    a.pcls_tab = h->pcls_tab;
    a.offc = h->offc;
    a.pat_l1 = h->pat_shared;
    a.dinv = h->dinv;
    a.x = h->x;
    a.pv = h->pv;
    a.r = h->r;
    a.s = h->Ap;
    a.z = h->p;
    a.z2 = h->z2;
    a.cy = h->cy;
    a.cd = h->cd;
    a.perm = h->has_perm ? h->perm : nullptr;
    a.refine = h->refine;
    a.theta = h->theta;
    a.cheb_m = h->cheb_m;
    a.cheb_c0 = h->cheb_c0;
    for (int j = 0; j < 8; ++j) {
        a.cheb_c1[j] = h->cheb_c1[j];
        a.cheb_c2[j] = h->cheb_c2[j];
    }
}

// Brings n 8-float status records [iterations, status, relres of columns 0..3, 0, 0] (one per mesh) back to info_host and
// reports the first breakdown (status 3), else the first mesh that reached maxit (status 2).  A batch's messages name the mesh
// and give its 3 columns, the single solve's give 4.
int finish_info(const float *info, float *info_host, int n, bool batch, float rtol, int maxit, cudaStream_t stream) {
    if (!info_host) return LS_OK;
    LS_CUDA_TRY(cudaMemcpyAsync(info_host, info, 8 * sizeof(float) * (size_t)n, cudaMemcpyDefault, stream));
    LS_CUDA_TRY(cudaStreamSynchronize(stream));
    for (const int st : {3, 2})
        for (int i = 0; i < n; ++i) {
            const float *r = info_host + 8 * i;
            if ((int)r[1] != st) continue;
            char mesh[32] = "", relres[64] = "";
            if (batch) snprintf(mesh, sizeof(mesh), "mesh %d: ", i);
            if (st == 3) {
                ls_set_error("%sCG breakdown after %d iterations (matrix not SPD or NaN in the right-hand side)", mesh, (int)r[0]);
                return LS_ERR_BREAKDOWN;
            }
            for (int j = 0, len = 0; j < (batch ? 3 : 4); ++j)
                len += snprintf(relres + len, sizeof(relres) - len, " %g", (double)r[2 + j]);
            ls_set_error("%sPCG did not reach rtol=%g within maxit=%d (relres%s)", mesh, (double)rtol, maxit, relres);
            return LS_ERR_NOT_CONVERGED;
        }
    return LS_OK;
}

}  // namespace lspcg

extern "C" int ls_pcg_workspace_bytes(int64_t V, int64_t nnz, int k_max, size_t *bytes_out) {
    LS_REQUIRE(bytes_out != nullptr, "bytes_out is NULL");
    LS_REQUIRE(V > 0 && nnz > 0 && V < (int64_t)0x7ffffff0 && nnz < (int64_t)0x7ffffff0, "size out of range");
    LS_REQUIRE(k_max >= 1 && k_max <= KMAX, "k_max must be in [1,4]");
    PcgHandle scratch{};
    *bytes_out = carve_handle(scratch, nullptr, V, nnz, k_max, GRID_CAP);
    return LS_OK;
}

extern "C" int ls_pcg_create(void **handle_out, int64_t V, int64_t nnz, const int32_t *rowptr, const int32_t *col,
                             const float *val, const int32_t *perm_new2old, int precond, int k_max, void *workspace,
                             size_t workspace_bytes, void *stream_) {
    LS_REQUIRE(handle_out != nullptr, "handle_out is NULL");
    *handle_out = nullptr;
    LS_REQUIRE(V > 0 && nnz > 0 && V < (int64_t)0x7ffffff0 && nnz < (int64_t)0x7ffffff0, "size out of range");
    LS_REQUIRE(k_max >= 1 && k_max <= KMAX, "k_max must be in [1,4]");
    LS_REQUIRE(precond >= 0 && precond <= 3, "precond must be 0 (none), 1 (Jacobi), 2 (Chebyshev polynomial over Jacobi) or 3 (auto)");
    LS_REQUIRE(rowptr && col && val, "NULL CSR pointer");
    LS_REQUIRE(workspace != nullptr && ((uintptr_t)workspace & 255) == 0, "workspace NULL or not 256-byte aligned");
    LsDevInfo di;
    int rc = ls_dev_info(&di);
    if (rc) return rc;
    size_t need = 0;
    ls_pcg_workspace_bytes(V, nnz, k_max, &need);
    if (workspace_bytes < need) {
        ls_set_error("PCG workspace too small: %zu < %zu", workspace_bytes, need);
        return LS_ERR_WORKSPACE;
    }
    PcgHandle *h = new (std::nothrow) PcgHandle();
    LS_REQUIRE(h != nullptr, "out of host memory");
    memset(h, 0, sizeof(*h));
    h->ws_bytes = carve_handle(*h, (char *)workspace, V, nnz, k_max, GRID_CAP);
    h->V = V;
    h->nnz = nnz;
    h->k_max = k_max;
    h->precond = precond;
    h->device = di.device;
    h->sm_count = di.sm_count;
    h->max_smem_optin = di.max_smem_optin;
    h->theta = 3.0f;
    rc = build_solver(h, rowptr, col, val, perm_new2old, di, (cudaStream_t)stream_);
    if (rc) {
        ls_pcg_destroy(h);
        return rc;
    }
    *handle_out = h;
    return LS_OK;
}

extern "C" int ls_pcg_solve(void *handle, const float *b, float *x, const float *x0, int k, float rtol, int maxit,
                            float *info_dev, float *info_host, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    PcgHandle *h = (PcgHandle *)handle;
    LS_REQUIRE(h != nullptr, "handle is NULL");
    LS_REQUIRE(b != nullptr && x != nullptr, "b or x is NULL");
    LS_REQUIRE(k >= 1 && k <= h->k_max, "k out of range for this handle");
    LS_REQUIRE(rtol > 0.f && maxit > 0, "rtol and maxit must be positive");
    int dev = -1;
    LS_CUDA_TRY(cudaGetDevice(&dev));
    LS_REQUIRE(dev == h->device, "handle was created on a different device");
    return solve_k(h, k, b, x, x0, rtol, maxit, info_dev, info_host, stream);
}

extern "C" int ls_pcg_set_refinement(void *handle, int max_restarts, float theta) {
    PcgHandle *h = (PcgHandle *)handle;
    LS_REQUIRE(h != nullptr, "handle is NULL");
    LS_REQUIRE(max_restarts >= 0 && max_restarts <= 8, "max_restarts must be in [0, 8]");
    LS_REQUIRE(theta >= 1.0f && theta < 1e6f, "theta must be >= 1");
    h->refine = max_restarts;
    h->theta = theta;
    return LS_OK;
}

extern "C" int ls_pcg_destroy(void *handle) {
    PcgHandle *h = (PcgHandle *)handle;
    if (!h) return LS_OK;
    graph_destroy(h->graph);
    delete h;
    return LS_OK;
}

extern "C" int ls_pcg_phase_cycles(void *handle, int64_t *out, int n, void *stream_) {
    PcgHandle *h = (PcgHandle *)handle;
    LS_REQUIRE(h != nullptr && out != nullptr, "NULL pointer");
    LS_REQUIRE(n >= 8 && n <= 8 + 8 * 256, "n out of range");
    LS_CUDA_TRY(cudaMemcpyAsync(out, h->dbg, (size_t)n * sizeof(long long), cudaMemcpyDeviceToHost, (cudaStream_t)stream_));
    LS_CUDA_TRY(cudaStreamSynchronize((cudaStream_t)stream_));
    return LS_OK;
}

extern "C" int ls_pcg_describe(void *handle, int64_t *out8) {
    PcgHandle *h = (PcgHandle *)handle;
    LS_REQUIRE(h != nullptr && out8 != nullptr, "NULL pointer");
    const PcgHandle::FusedCfg &fc = h->fused[0];
    if (fc.on) {   // fused two-synchronisation solver: [engine, padded entries, grid, cluster size, mode 10 + RES, preconditioner, threads, re-ordered]
        out8[0] = fc.pat ? 2 : 1;
        out8[1] = h->sell_entries;
        out8[2] = fc.grid;
        out8[3] = fc.cluster;
        out8[4] = 10 + fc.res;
        out8[5] = (h->cheb_m > 1) ? 2 : h->precond;    // preconditioner actually in use (auto resolved)
        out8[6] = fc.nw * 32;
        out8[7] = h->has_perm;
        return LS_OK;
    }
    // graph-mode solver: [engine, padded entries, SpMM grid, vector grid, 0, 0, planned, re-ordered]
    out8[0] = h->sell_on;                 // 1 = SELL-32 engine, 0 = TMA-staged CSR engine
    out8[1] = h->sell_entries;            // padded entries of the SELL copy
    out8[2] = h->sell_on ? h->graph.sell_grid : h->graph.spmm_grid;
    out8[3] = h->graph.vec_grid;
    out8[4] = 0;                          // mode: graph of 3 kernels (1 and 2 are retired, 10 + RES is the fused solver)
    out8[5] = 0;
    out8[6] = h->graph.planned;
    out8[7] = h->has_perm;
    return LS_OK;
}
