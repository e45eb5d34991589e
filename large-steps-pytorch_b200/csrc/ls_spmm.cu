// ls_spmm.cu -- SpMM launch plumbing + the public y = A x entry point (AoS (V,k) torch layout).
// Replaces the torch sparse `M @ v` of parameterize.py:30 (to_differential) and scripts/main.py:192-195.
#include <stdlib.h>
#include "ls_spmm_kernel.cuh"
#include "ls_spmm_host.h"

namespace lsk {

// runtime tuning knobs (LS_SPMM_* environment variables exist for sweeps only)
void spmm_config(SpmmCfg *cfg) {
    static SpmmCfg s = {0, 0, 0, 0, 0};
    if (s.stages == 0) {
        auto geti = [](const char *name, int dflt, int lo, int hi) {
            const char *e = getenv(name);
            int v = e ? atoi(e) : dflt;
            return v < lo ? lo : (v > hi ? hi : v);
        };
        s.stages = geti("LS_SPMM_STAGES", 2, 2, SPMM_MAX_STAGES);
        s.cap = SPMM_NT * geti("LS_SPMM_CAPMUL", 8, 2, 24);
        s.unroll = 8;
        s.hint = geti("LS_SPMM_HINT", 1, 0, 2);   // in-solver matrix stream: L2 evict_first
        s.debug = geti("LS_SPMM_DEBUG", 0, 0, 3);  // diagnostics only
    }
    *cfg = s;
}

namespace {
template <int K, bool X4, bool YSOA, bool DOT, int U>
int prepare_t(const SpmmCfg &cfg, int *ctas_per_sm) {
    static thread_local int cached_dev = -1, cached_occ = 0, cached_st = 0, cached_cap = 0;
    LsDevInfo di;
    int rc = ls_dev_info(&di);
    if (rc) return rc;
    if (cached_dev != di.device || cached_st != cfg.stages || cached_cap != cfg.cap) {
        size_t smem = spmm_smem_bytes(cfg.stages, cfg.cap);
        if ((int)smem > di.max_smem_optin) {
            ls_set_error("SpMM stage configuration needs %zu bytes of shared memory, device allows %d", smem, di.max_smem_optin);
            return LS_ERR_UNSUPPORTED;
        }
        LS_CUDA_TRY(cudaFuncSetAttribute(spmm_tma_kernel<K, X4, YSOA, DOT, U>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        int occ = 0;
        LS_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, spmm_tma_kernel<K, X4, YSOA, DOT, U>, SPMM_THREADS, smem));
        if (occ < 1) occ = 1;
        cached_dev = di.device;
        cached_occ = occ;
        cached_st = cfg.stages;
        cached_cap = cfg.cap;
    }
    *ctas_per_sm = cached_occ;
    return LS_OK;
}

template <int K, bool X4, bool YSOA, bool DOT, int U>
int launch_t(const SpmmArgs &a, int grid, cudaStream_t stream) {
    size_t smem = spmm_smem_bytes(a.stages, a.cap);
    spmm_tma_kernel<K, X4, YSOA, DOT, U><<<grid, SPMM_THREADS, smem, stream>>>(a);
    LS_LAUNCH_CHECK();
    return LS_OK;
}
}  // namespace

#define LS_SPMM_DISPATCH(FN, ...)                                                                         \
    do {                                                                                                  \
        if (solver_layout) { /* x = solver p rows (1/2/4 floats), y = SoA planes, dot epilogue */          \
            switch (K) {                                                                                  \
                case 1: return FN<1, false, true, true, 8>(__VA_ARGS__);                                  \
                case 2: return FN<2, false, true, true, 8>(__VA_ARGS__);                                  \
                case 3: return FN<3, true, true, true, 8>(__VA_ARGS__);                                   \
                case 4: return FN<4, true, true, true, 8>(__VA_ARGS__);                                   \
            }                                                                                             \
        } else {             /* public: x, y = (V,k) row-major */                                          \
            switch (K) {                                                                                  \
                case 1: return FN<1, false, false, false, 8>(__VA_ARGS__);                                \
                case 2: return FN<2, false, false, false, 8>(__VA_ARGS__);                                \
                case 3: return FN<3, false, false, false, 8>(__VA_ARGS__);                                \
                case 4: return FN<4, false, false, false, 8>(__VA_ARGS__);                                \
            }                                                                                             \
        }                                                                                                 \
        ls_set_error("SpMM: k=%d out of range [1,4]", K);                                                 \
        return LS_ERR_BAD_ARG;                                                                            \
    } while (0)

int spmm_prepare(int K, bool solver_layout, const SpmmCfg &cfg, int *ctas_per_sm) {
    LS_SPMM_DISPATCH(prepare_t, cfg, ctas_per_sm);
}

int spmm_launch(int K, bool solver_layout, const SpmmCfg &cfg, const SpmmArgs &a, int grid, cudaStream_t stream) {
    LS_SPMM_DISPATCH(launch_t, a, grid, stream);
}

int spmm_grid_for(int64_t V, int sm_count, int occ) {
    int64_t g = (V + 63) / 64;
    int64_t cap = (int64_t)sm_count * occ;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (int)g;
}

// plan kernel: one thread per CTA of the SpMM grid writes that CTA's block descriptors
static __global__ void spmm_plan_kernel(const int *__restrict__ rowptr, const int *__restrict__ part, int G, int cap,
                                 int4 *__restrict__ desc, int *__restrict__ desc_cnt, int *__restrict__ overflow) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= G) return;
    int r = part[c];
    const int r_end = part[c + 1];
    int n = 0;
    int s_nz = (r < r_end) ? rowptr[r] : 0;
    while (r < r_end) {
        int e_nz, direct;
        const int nr = spmm_block_extent(rowptr, r, r_end, s_nz, cap, &e_nz, &direct);
        if (n < SPMM_BMAX) desc[(size_t)c * SPMM_BMAX + n] = make_int4(r, nr | (direct << 16), s_nz, e_nz);
        ++n;
        r += nr;
        s_nz = e_nz;
    }
    desc_cnt[c] = n;
    if (n > SPMM_BMAX) atomicOr(overflow, 1);
}

int spmm_plan(const int *rowptr, const int *part, int G, int cap, int4 *desc, int *desc_cnt, int *overflow,
              cudaStream_t stream) {
    spmm_plan_kernel<<<(G + 127) / 128, 128, 0, stream>>>(rowptr, part, G, cap, desc, desc_cnt, overflow);
    LS_LAUNCH_CHECK();
    return LS_OK;
}

}  // namespace lsk

extern "C" int ls_spmm_csr_f32(int64_t V, const int32_t *rowptr, const int32_t *col, const float *val, const float *x,
                               int64_t ldx, float *y, int64_t ldy, int k, void *stream_) {
    using namespace lsk;
    cudaStream_t stream = (cudaStream_t)stream_;
    LS_REQUIRE(V >= 0 && V < (int64_t)0x7ffffff0, "V out of range");
    LS_REQUIRE(k >= 1, "k must be >= 1");
    LS_REQUIRE(ldx >= k && ldy >= k, "leading dimension smaller than k");
    if (V == 0) return LS_OK;
    LS_REQUIRE(rowptr && col && val && x && y, "NULL pointer");
    LS_REQUIRE((((uintptr_t)rowptr | (uintptr_t)col | (uintptr_t)val) & 15) == 0,
               "rowptr/col/val must be 16-byte aligned (TMA bulk copies)");
    LsDevInfo di;
    int rc = ls_dev_info(&di);
    if (rc) return rc;
    SpmmCfg cfg;
    spmm_config(&cfg);
    for (int k0 = 0; k0 < k; k0 += 4) {
        const int kk = (k - k0) < 4 ? (k - k0) : 4;
        SpmmArgs a{};
        a.V = (int)V;
        a.stages = cfg.stages;
        a.cap = cfg.cap;
        a.hint = 0;
        a.rowptr = rowptr;
        a.col = col;
        a.val = val;
        a.x = x + k0;
        a.y = y + k0;
        a.ldx = ldx;
        a.ldy = ldy;
        int occ = 1;
        rc = spmm_prepare(kk, false, cfg, &occ);
        if (rc) return rc;
        rc = spmm_launch(kk, false, cfg, a, spmm_grid_for(V, di.sm_count, occ), stream);
        if (rc) return rc;
    }
    return LS_OK;
}

// ---- gradient of y = A x with respect to A's values: gval[e] = sum_{q < k} gy[row_e, q] x[col_e, q], q in order ----------
// A sampled dense-dense product over A's CSR pattern, a streaming gather like the SpMM.  Eight lanes per row (a mesh row
// holds ~7 entries): the lanes of a row read consecutive col entries and write consecutive gval entries, and the four rows
// of a warp are consecutive, so both streams are coalesced; the row of gy is one broadcast load per lane group.  Gathers of
// x go through L1 and L2: neighbouring rows share columns, and x (12 MB at V = 10^6, k = 3) fits the H100's 50 MB L2, so
// each row of x comes from HBM about once.
// Byte model per call: 4 (V+1) rowptr + 4 nnz col + 4 k V gy + 4 k V x + 4 nnz gval = 8 nnz + 4 (V+1) + 8 k V, the SpMM's.
// Every entry is one thread's fixed-order sum: no atomics, bit-reproducible.
namespace {
constexpr int GV_LANES = 8;
constexpr int GV_THREADS = 256;

template <int K>   // K = 0: k read at run time
__global__ void __launch_bounds__(GV_THREADS) k_spmm_grad_val(int V, const int *__restrict__ rowptr, const int *__restrict__ col,
                                                              const float *__restrict__ x, long long ldx,
                                                              const float *__restrict__ gy, long long ldgy, int k,
                                                              float *__restrict__ gval) {
    const long long t = (long long)blockIdx.x * GV_THREADS + threadIdx.x;
    const long long r = t / GV_LANES;
    if (r >= V) return;
    const int kk = K > 0 ? K : k;
    const int s = rowptr[r], e = rowptr[r + 1];
    const float *g = gy + r * ldgy;
    for (int j = s + (int)(t % GV_LANES); j < e; j += GV_LANES) {
        const float *xr = x + (long long)__ldg(col + j) * ldx;
        float acc = 0.f;
#pragma unroll
        for (int q = 0; q < (K > 0 ? K : 1); ++q) acc = fmaf(__ldg(g + q), __ldg(xr + q), acc);
        if (K == 0)
            for (int q = 1; q < kk; ++q) acc = fmaf(__ldg(g + q), __ldg(xr + q), acc);
        gval[j] = acc;
    }
}
}  // namespace

extern "C" int ls_spmm_csr_grad_val_f32(int64_t V, const int32_t *rowptr, const int32_t *col, const float *x, int64_t ldx,
                                        const float *gy, int64_t ldgy, int k, float *gval, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    LS_REQUIRE(V >= 0 && V < (int64_t)0x7ffffff0, "V out of range");
    LS_REQUIRE(k >= 1, "k must be >= 1");
    LS_REQUIRE(ldx >= k && ldgy >= k, "leading dimension smaller than k");
    if (V == 0) return LS_OK;
    LS_REQUIRE(rowptr && col && x && gy && gval, "NULL pointer");
    const unsigned grid = (unsigned)((V * GV_LANES + GV_THREADS - 1) / GV_THREADS);
    switch (k) {
        case 1: k_spmm_grad_val<1><<<grid, GV_THREADS, 0, stream>>>((int)V, rowptr, col, x, ldx, gy, ldgy, k, gval); break;
        case 2: k_spmm_grad_val<2><<<grid, GV_THREADS, 0, stream>>>((int)V, rowptr, col, x, ldx, gy, ldgy, k, gval); break;
        case 3: k_spmm_grad_val<3><<<grid, GV_THREADS, 0, stream>>>((int)V, rowptr, col, x, ldx, gy, ldgy, k, gval); break;
        case 4: k_spmm_grad_val<4><<<grid, GV_THREADS, 0, stream>>>((int)V, rowptr, col, x, ldx, gy, ldgy, k, gval); break;
        default: k_spmm_grad_val<0><<<grid, GV_THREADS, 0, stream>>>((int)V, rowptr, col, x, ldx, gy, ldgy, k, gval); break;
    }
    LS_LAUNCH_CHECK();
    return LS_OK;
}
