// ls_pcg_batch.cu -- batches: many independent meshes per launch, one thread-block cluster per mesh (ls_pcg_fused.cuh, BATCH).
// Each mesh keeps its own handle (ls_pcg_create); the batch holds a device table of their fused-kernel arguments, grouped by the
// batch plan (ls_pcg_batch_plan_ex, ls_pcg_plan.cu), one launch per group.
#include <vector>
#include "ls_pcg_handle.h"
#include "ls_fused_inst.h"

using namespace lspcg;

namespace {

struct BatchGroup {
    int first, count;     // entries [first, first + count) of the table
    int cluster, res, pat, cheb;
    size_t smem;
    const void *fn;
};

struct PcgBatch {
    int n, device, k_max;
    lsf::BatchEntry *tab;   // device: n entries, grouped
    float *info;            // device: 8 n floats (used when the caller passes no info_dev)
    std::vector<BatchGroup> groups;
};

void batch_free(PcgBatch *b) {
    if (!b) return;
    if (b->tab) cudaFree(b->tab);
    if (b->info) cudaFree(b->info);
    delete b;
}

// the batch's device table (from the host table `host`) and info records
int batch_upload(PcgBatch *b, const std::vector<lsf::BatchEntry> &host, cudaStream_t stream) {
    const size_t n = host.size();
    LS_CUDA_TRY(cudaMalloc((void **)&b->tab, sizeof(lsf::BatchEntry) * n));
    LS_CUDA_TRY(cudaMalloc((void **)&b->info, 8 * sizeof(float) * n));
    LS_CUDA_TRY(cudaMemcpyAsync(b->tab, host.data(), sizeof(lsf::BatchEntry) * n, cudaMemcpyHostToDevice, stream));
    LS_CUDA_TRY(cudaMemsetAsync(b->info, 0, 8 * sizeof(float) * n, stream));
    LS_CUDA_TRY(cudaStreamSynchronize(stream));   // (the host table goes when the create returns)
    return LS_OK;
}
}  // namespace

extern "C" int ls_pcg_batch_create(void **batch_out, void *const *handles, int n, void *stream_) try {
    cudaStream_t stream = (cudaStream_t)stream_;
    LS_REQUIRE(batch_out != nullptr, "batch_out is NULL");
    *batch_out = nullptr;
    LS_REQUIRE(handles != nullptr && n >= 1, "no handles");
    for (int i = 0; i < n; ++i) {
        LS_REQUIRE(handles[i] != nullptr, "NULL handle");
        for (int j = 0; j < i; ++j) LS_REQUIRE(handles[j] != handles[i], "a handle appears twice (its workspace can serve one mesh at a time)");
    }
    LsDevInfo di;
    int rc = ls_dev_info(&di);
    if (rc) return rc;
    std::vector<int32_t> ns(n), pt(n), ch(n), cs(n), rs(n), gr(n);
    int kmin = KMAX;
    for (int i = 0; i < n; ++i) {
        const PcgHandle *h = (const PcgHandle *)handles[i];
        if (h->device != di.device) {
            ls_set_error("bad argument: mesh %d: its handle was created on another device", i);
            return LS_ERR_BAD_ARG;
        }
        if (!h->sell_on) {
            ls_set_error("mesh %d: rows too long for the SELL-32 copy the batch solver streams; solve it on its own (ls_pcg_solve)", i);
            return LS_ERR_UNSUPPORTED;
        }
        ns[i] = h->nslices;
        pt[i] = h->pat_on;
        ch[i] = h->cheb_m > 1 ? 1 : 0;   // the handle's own preconditioner (precond 2, or 3 resolved to Chebyshev)
        if (h->k_max < kmin) kmin = h->k_max;
    }
    int ng = 0;
    rc = ls_pcg_batch_plan_ex(n, ns.data(), pt.data(), ch.data(), di.max_smem_optin, cs.data(), rs.data(), gr.data(), &ng);
    if (rc) return rc;
    // table: the meshes of group 0, then group 1, ... (batch order inside a group); packed rows in batch order
    std::vector<long long> row0(n, 0);
    for (int i = 1; i < n; ++i) row0[i] = row0[i - 1] + ((const PcgHandle *)handles[i - 1])->V;
    std::vector<lsf::BatchEntry> host(n);
    std::vector<BatchGroup> groups(ng);
    int e = 0;
    for (int g = 0; g < ng; ++g) {
        BatchGroup &G = groups[g];
        G.first = e;
        for (int i = 0; i < n; ++i) {
            if (gr[i] != g) continue;
            const PcgHandle *h = (const PcgHandle *)handles[i];
            G.cluster = cs[i];
            G.res = rs[i];
            G.pat = pt[i] ? 1 : 0;
            G.cheb = ch[i];
            const int nsl_max = (h->nslices + cs[i] - 1) / cs[i];
            const size_t sm = lsf::fused_smem_bytes(3, rs[i], nsl_max, G.pat, G.cheb, 1);
            if (sm > G.smem) G.smem = sm;
            fused_handle_args(h, nsl_max, host[e].a);   // (Chebyshev: the handle's polynomial travels in the entry)
            host[e].row0 = row0[i];
            host[e].mesh = i;
            ++e;
            ++G.count;
        }
        G.fn = G.cheb ? (G.res == 2 ? ls_fused_fn_batch_cheb(G.pat) : nullptr) : ls_fused_fn_batch(G.res, G.pat);
        if (!G.fn) {
            ls_set_error("batch instantiation (RES %d, pattern %d, Chebyshev %d) is not built", G.res, G.pat, G.cheb);
            return LS_ERR_UNSUPPORTED;
        }
        if (!cluster_fits(G.fn, G.cluster, lsf::PWARPS * 32, G.smem, di)) {
            ls_set_error("this device cannot run a cluster of %d CTAs with %zu bytes of shared memory each", G.cluster, G.smem);
            return LS_ERR_UNSUPPORTED;
        }
    }
    PcgBatch *b = new PcgBatch();
    b->n = n;
    b->device = di.device;
    b->k_max = kmin;
    b->groups = std::move(groups);
    rc = batch_upload(b, host, stream);
    if (rc) {
        batch_free(b);
        return rc;
    }
    *batch_out = b;
    return LS_OK;
} catch (const std::bad_alloc &) {
    ls_set_error("out of host memory");
    return LS_ERR_BAD_ARG;
}

extern "C" int ls_pcg_batch_solve(void *batch, const float *b, float *x, const float *x0, int k, float rtol, int maxit,
                                  float *info_dev, float *info_host, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    PcgBatch *B = (PcgBatch *)batch;
    LS_REQUIRE(B != nullptr, "batch is NULL");
    LS_REQUIRE(b != nullptr && x != nullptr, "b or x is NULL");
    LS_REQUIRE(k >= 1 && k <= 3 && k <= B->k_max, "k must be in [1, 3] (and within every handle's k_max)");
    LS_REQUIRE(rtol > 0.f && maxit > 0, "rtol and maxit must be positive");
    int dev = -1;
    LS_CUDA_TRY(cudaGetDevice(&dev));
    LS_REQUIRE(dev == B->device, "batch was created on a different device");
    float *info = info_dev ? info_dev : B->info;
    for (const BatchGroup &G : B->groups) {
        lsf::BatchParams p{};
        p.tab = B->tab + G.first;
        p.b = b;
        p.out = x;
        p.x0 = x0;
        p.info = info;
        p.kb = k;
        p.rtol = rtol;
        p.maxit = maxit;
        void *params[] = {(void *)&p};
        cudaLaunchAttribute at;
        const cudaLaunchConfig_t lc = cluster_launch(G.count * G.cluster, G.cluster, lsf::PWARPS * 32, G.smem, stream, &at);
        LS_CUDA_TRY(cudaLaunchKernelExC(&lc, G.fn, params));
        g_ls_launches.fetch_add(1, std::memory_order_relaxed);
    }
    return finish_info(info, info_host, B->n, true, rtol, maxit, stream);
}

extern "C" int ls_pcg_batch_destroy(void *batch) {
    batch_free((PcgBatch *)batch);
    return LS_OK;
}
