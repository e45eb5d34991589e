// ls_spmm_kernel.cuh -- the CSR SpMM kernel of the library (sm_90a): y = A x for K right-hand-side columns.
//
// Roofline: HBM.  Algorithmic bytes per launch = 8 nnz + 4 (V+1) + 8 K V  (SURVEY.md section 8 d).
//
// Design (rows have ~7 non-zeros on a triangle mesh, so neither warp-per-row nor naive thread-per-row coalesces):
//   * persistent CTAs, each owning a contiguous, nnz-balanced range of rows (`part`);
//   * a producer warp streams, per block of <= NT rows, the *contiguous* col/val/rowptr slices of that block into a
//     shared-memory ring with 1-D TMA bulk copies (cp.async.bulk + mbarrier complete_tx) -- 2/3 of all bytes of the
//     kernel never touch the LSU or the register file on their way in.  With a plan (`desc`, built once per matrix)
//     the producer knows every block boundary up front and issues the first copies one L2 round trip after launch;
//   * NT consumer threads take one row each out of shared memory (odd stride -> conflict-free), gather x through
//     L1 (neighbouring rows share neighbours, so the gather is mostly L1/L2 hits), and write y coalesced;
//   * optional epilogue: the K dot products x_k . y_k (p.Ap of CG) reduced deterministically across the grid.
//
// Layouts: x is always row-major (V, ldx) -- the public torch layout, and the solver's p (rows of 1/2/4 floats; X4 = rows
//          are 16-byte aligned float4, gathered with one LDG.128); y is row-major (V, ldy) or, YSOA, K planes of ldy floats.
// In the solver this kernel is the general fallback (very long rows, heavy SELL padding); the fast path is
// ls_sell_kernel.cuh.
#pragma once
#include "ls_common.cuh"

namespace lsk {

constexpr int SPMM_NT = 256;            // consumer threads = max rows per block
constexpr int SPMM_THREADS = SPMM_NT + 32;
constexpr int SPMM_MAX_STAGES = 4;
constexpr int SPMM_RP = SPMM_NT + 8;    // rowptr ints per stage
constexpr int SPMM_HDR_BYTES = 64 + 1088;   // barriers + reduction scratch
constexpr int SPMM_BMAX = 64;           // plan: max blocks per CTA (else the on-the-fly producer is used)

struct SpmmArgs {
    int V;
    int stages;             // 2..4
    int cap;                // col/val elements per stage, multiple of 4
    int hint;               // L2 policy of the matrix stream: 0 none, 1 evict_first, 2 evict_last
    int debug;              // diagnostics only (LS_SPMM_DEBUG): 1 = skip the x gathers, 2 = skip the y stores
    const int *rowptr;
    const int *col;
    const float *val;
    const float *x;
    float *y;
    long long ldx, ldy;
    const int *part;        // [gridDim.x + 1] row boundaries, or NULL for an even split
    const int4 *desc;       // plan: [gridDim.x][SPMM_BMAX] (r0, nr | direct<<16, s_nz, e_nz), or NULL
    const int *desc_cnt;    // plan: blocks per CTA
    const int *done;        // optional early-exit flag (device), NULL if unused
    double *partials;       // [K][gridDim.x]    (DOT only)
    unsigned int *ticket;   //                   (DOT only)
    double *dot_out;        // [K]               (DOT only)
};

inline size_t spmm_stage_bytes(int cap) { return 16 + (size_t)SPMM_RP * 4 + (size_t)cap * 8; }
inline size_t spmm_smem_bytes(int stages, int cap) { return SPMM_HDR_BYTES + (size_t)stages * spmm_stage_bytes(cap); }

template <int K, bool X4>
__device__ __forceinline__ void load_x(const float *__restrict__ x, long long ld, int c, float (&v)[K]) {
    if (X4) {
        const float4 t = __ldg(reinterpret_cast<const float4 *>(x) + c);
        const float tt[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
        for (int k = 0; k < K; ++k) v[k] = tt[k];
    } else {
#pragma unroll
        for (int k = 0; k < K; ++k) v[k] = __ldg(x + (size_t)c * ld + k);
    }
}

// Decide the extent of the block that starts at row r (nnz offset s_nz): at most NT rows, at most cap-4 elements
// counted from the 16-byte aligned start.  Returns nr; *e_out = rowptr[r+nr]; *direct = 1 for a row longer than a stage.
__device__ __forceinline__ int spmm_block_extent(const int *__restrict__ rowptr, int r, int r_end, int s_nz, int cap,
                                                 int *e_out, int *direct) {
    int nr = min(SPMM_NT, r_end - r);
    int e_nz = rowptr[r + nr];
    const int s_a = s_nz & ~3;
    *direct = 0;
    if (e_nz - s_a > cap - 4) {
        int lo = 0, hi = nr;   // invariant: `lo` rows fit
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (rowptr[r + mid] - s_a <= cap - 4) lo = mid;
            else hi = mid - 1;
        }
        if (lo == 0) {   // a single row longer than a stage: its consumer reads it straight from global
            nr = 1;
            *direct = 1;
        } else {
            nr = lo;
        }
        e_nz = rowptr[r + nr];
    }
    *e_out = e_nz;
    return nr;
}

template <int K, bool X4, bool YSOA, bool DOT, int U>
__global__ void __launch_bounds__(SPMM_THREADS) spmm_tma_kernel(const SpmmArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    if (a.done != nullptr && *reinterpret_cast<const volatile int *>(a.done) != 0) return;

    uint64_t *full = reinterpret_cast<uint64_t *>(smem_raw);
    uint64_t *empty = full + SPMM_MAX_STAGES;
    double *red = reinterpret_cast<double *>(smem_raw + 64);
    unsigned char *stage_base = smem_raw + SPMM_HDR_BYTES;
    const int stages = a.stages, cap = a.cap;
    const size_t stage_bytes = 16 + (size_t)SPMM_RP * 4 + (size_t)cap * 8;

    const int tid = threadIdx.x;
    const int G = gridDim.x, cta = blockIdx.x;
    int r_begin, r_end;
    if (a.part) {
        r_begin = a.part[cta];
        r_end = a.part[cta + 1];
    } else {
        r_begin = (int)((long long)a.V * cta / G);
        r_end = (int)((long long)a.V * (cta + 1) / G);
    }

    if (tid == 0) {
        for (int s = 0; s < stages; ++s) {
            ls_mbar_init(&full[s], 1);
            ls_mbar_init(&empty[s], SPMM_NT / 32);
        }
        ls_fence_mbar_init();
    }
    __syncthreads();

    if (tid >= SPMM_NT) {
        // ===================== producer warp =====================
        const int lane = tid - SPMM_NT;
        uint64_t policy = 0;
        if (a.hint == 1) policy = ls_policy_evict_first();
        else if (a.hint == 2) policy = ls_policy_evict_last();
        auto issue = [&](int st, int use, int r, int nr, int direct, int s_nz, int e_nz) {
            unsigned char *S = stage_base + (size_t)st * stage_bytes;
            int *hdr = reinterpret_cast<int *>(S);
            int *s_rp = reinterpret_cast<int *>(S + 16);
            int *s_col = s_rp + SPMM_RP;
            float *s_val = reinterpret_cast<float *>(s_col + cap);
            if (use > 0) ls_mbar_wait(&empty[st], (use - 1) & 1);
            const int s_a = s_nz & ~3;
            const int e_a = (e_nz + 3) & ~3;
            const int r_a = r & ~3;
            const int rp_n = ((r + nr + 1 + 3) & ~3) - r_a;
            hdr[0] = r;
            hdr[1] = nr;
            hdr[2] = s_a;
            hdr[3] = direct;
            const uint32_t nbytes_cv = direct ? 0u : (uint32_t)(e_a - s_a) * 4u;
            const uint32_t nbytes_rp = (uint32_t)rp_n * 4u;
            ls_mbar_expect_tx(&full[st], nbytes_rp + 2u * nbytes_cv);
            ls_bulk_g2s(s_rp, a.rowptr + r_a, nbytes_rp, &full[st]);
            if (nbytes_cv) {
                if (a.hint) {
                    ls_bulk_g2s_hint(s_col, a.col + s_a, nbytes_cv, &full[st], policy);
                    ls_bulk_g2s_hint(s_val, a.val + s_a, nbytes_cv, &full[st], policy);
                } else {
                    ls_bulk_g2s(s_col, a.col + s_a, nbytes_cv, &full[st]);
                    ls_bulk_g2s(s_val, a.val + s_a, nbytes_cv, &full[st]);
                }
            }
        };
        if (a.desc != nullptr) {
            // planned: all descriptors of this CTA arrive with one coalesced load; lane 0 issues
            const int nb = a.desc_cnt[cta];
            const int4 *D = a.desc + (size_t)cta * SPMM_BMAX;
            int4 d0 = (lane < nb) ? D[lane] : make_int4(0, 0, 0, 0);
            int4 d1 = (lane + 32 < nb) ? D[lane + 32] : make_int4(0, 0, 0, 0);
            int st = 0, use = 0;
            for (int b = 0; b < nb; ++b) {
                const int4 src = (b < 32) ? d0 : d1;
                int4 d;
                d.x = __shfl_sync(0xffffffffu, src.x, b & 31);
                d.y = __shfl_sync(0xffffffffu, src.y, b & 31);
                d.z = __shfl_sync(0xffffffffu, src.z, b & 31);
                d.w = __shfl_sync(0xffffffffu, src.w, b & 31);
                if (lane == 0) issue(st, use, d.x, d.y & 0xffff, d.y >> 16, d.z, d.w);
                if (++st == stages) {
                    st = 0;
                    ++use;
                }
            }
        } else if (lane == 0 && r_begin < r_end) {
            // unplanned (public SpMM on foreign matrices): block boundaries found on the fly
            int r = r_begin;
            int s_nz = a.rowptr[r];
            int st = 0, use = 0;
            while (r < r_end) {
                int e_nz, direct;
                const int nr = spmm_block_extent(a.rowptr, r, r_end, s_nz, cap, &e_nz, &direct);
                issue(st, use, r, nr, direct, s_nz, e_nz);
                r += nr;
                s_nz = e_nz;
                if (++st == stages) {
                    st = 0;
                    ++use;
                }
            }
        }
    } else {
        // ===================== consumers: one row per thread =====================
        double dacc[K];
#pragma unroll
        for (int k = 0; k < K; ++k) dacc[k] = 0.0;
        int r = r_begin;
        int st = 0, use = 0;
        while (r < r_end) {
            const unsigned char *S = stage_base + (size_t)st * stage_bytes;
            const int *hdr = reinterpret_cast<const int *>(S);
            const int *s_rp = reinterpret_cast<const int *>(S + 16);
            const int *s_col = s_rp + SPMM_RP;
            const float *s_val = reinterpret_cast<const float *>(s_col + cap);
            ls_mbar_wait(&full[st], use & 1);
            const int r0 = hdr[0], nr = hdr[1], s_a = hdr[2], direct = hdr[3];
            if (tid < nr) {
                const int row = r0 + tid;
                const int off = (r0 & 3) + tid;
                const int j0 = s_rp[off], j1 = s_rp[off + 1];
                float acc[K];
#pragma unroll
                for (int k = 0; k < K; ++k) acc[k] = 0.f;
                if (!direct) {
                    const int *sc = s_col + (j0 - s_a);
                    const float *sv = s_val + (j0 - s_a);
                    const int len = j1 - j0;
                    // U entries per pass, all gathers of a pass in flight together; slots past the row end are
                    // predicated to (own row, weight 0) -- an L1 hit that keeps the pass branch-free
                    for (int j = 0; j < len; j += U) {
                        int c[U];
                        float w[U];
                        float xv[U][K];
#pragma unroll
                        for (int u = 0; u < U; ++u) {
                            const bool ok = (j + u) < len;
                            c[u] = ok ? sc[j + u] : row;
                            w[u] = ok ? sv[j + u] : 0.f;
                        }
                        if (a.debug & 1) {
#pragma unroll
                            for (int u = 0; u < U; ++u)
#pragma unroll
                                for (int k = 0; k < K; ++k) xv[u][k] = (float)(c[u] & 7);
                        } else {
#pragma unroll
                            for (int u = 0; u < U; ++u) load_x<K, X4>(a.x, a.ldx, c[u], xv[u]);
                        }
#pragma unroll
                        for (int u = 0; u < U; ++u)
#pragma unroll
                            for (int k = 0; k < K; ++k) acc[k] = fmaf(w[u], xv[u][k], acc[k]);
                    }
                } else {
                    for (int j = j0; j < j1; ++j) {
                        const int c = __ldg(a.col + j);
                        const float w = __ldg(a.val + j);
                        float xv[K];
                        load_x<K, X4>(a.x, a.ldx, c, xv);
#pragma unroll
                        for (int k = 0; k < K; ++k) acc[k] = fmaf(w, xv[k], acc[k]);
                    }
                }
                if (a.debug & 2) {
                    if (acc[0] == 1.2345e-30f) a.y[row] = acc[0];
                } else if (YSOA) {
#pragma unroll
                    for (int k = 0; k < K; ++k) a.y[(size_t)k * a.ldy + row] = acc[k];
                } else {
#pragma unroll
                    for (int k = 0; k < K; ++k) a.y[(size_t)row * a.ldy + k] = acc[k];
                }
                if (DOT) {
                    float xr[K];
                    load_x<K, X4>(a.x, a.ldx, row, xr);
#pragma unroll
                    for (int k = 0; k < K; ++k) dacc[k] += (double)xr[k] * (double)acc[k];
                }
            }
            __syncwarp();
            if ((tid & 31) == 0) ls_mbar_arrive(&empty[st]);
            r = r0 + nr;
            if (++st == stages) {
                st = 0;
                ++use;
            }
        }
        if (DOT) {
            double tot[K];
            const bool last = ls_grid_reduce<K>(dacc, tot, a.partials, a.ticket, red, tid, SPMM_NT, 1, cta, G);
            if (last && tid == 0) {
#pragma unroll
                for (int k = 0; k < K; ++k) a.dot_out[k] = tot[k];
            }
        }
    }
}

}  // namespace lsk
