// ls_pcg_graph.cu -- the graph-mode solver, the fallback when the fused kernel cannot run (no cooperative launch, no SELL-32
// copy, LS_PCG_MODE=graph, or its launch refused): one iteration = three kernels, a CUDA graph of CHUNK iterations replayed until
// a device-side `done` flag is seen --
//   K1  Ap = A p, pAp_k = p_k.Ap_k                     (SELL-32 or TMA-staged CSR SpMM + deterministic grid reduction)
//   K2  x += a p; r -= a Ap; rz' = r.(dinv r); rr = r.r (fused update + 2K dot products; last CTA does the
//       scalar state transition: beta, convergence per column, iteration count, done flag)
//   K3  p = dinv r + beta p
// This file also holds every launch of the stand-alone SpMV kernels (spmm_sell_kernel, spmm_sell_tma_kernel, the CSR engine in
// solver layout) and the diagnostics that drive them.
#include "ls_pcg_handle.h"

using namespace lspcg;

namespace {

constexpr int VEC_THREADS = 256;
constexpr int CHUNK = 8;   // CG iterations per graph launch

// nnz-balanced contiguous row partition: part[c] = first row r with weight(r) >= c * total / G,
// weight(r) = 2 * rowptr[r] + 5 * r   (~ bytes/4 streamed per non-zero and per row)
__global__ void k_partition(int64_t V, const int *__restrict__ rowptr, int G, int *__restrict__ part) {
    int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c > G) return;
    if (c == G) {
        part[c] = (int)V;
        return;
    }
    long long total = 2LL * rowptr[V] + 5LL * V;
    long long target = total * c / G;
    int64_t lo = 0, hi = V;
    while (lo < hi) {
        int64_t mid = (lo + hi) >> 1;
        long long w = 2LL * rowptr[mid] + 5LL * mid;
        if (w < target) lo = mid + 1;
        else hi = mid;
    }
    part[c] = (int)lo;
}

// ---- solve kernels --------------------------------------------------------------------------------
struct VecArgs {
    int64_t V, Vp;
    float *x, *r, *p, *Ap;
    const float *dinv;
    PcgCtrl *ctrl;
    double *partials;
    unsigned int *ticket;
    const int *perm;   // new -> old row of the caller's (V,K) arrays, or NULL
};

// cold start: x = 0, r = b, p = z = dinv r;  warm (stage 2): r = b - Ap (Ap = A x0 from K1), p = z
template <int K, bool WARM>
__global__ void __launch_bounds__(VEC_THREADS) k_init(VecArgs a, const float *__restrict__ b, float rtol, int maxit,
                                                      int only_if_restart) {
    __shared__ double red[3 * K * 32 + 3 * K + 1];
    if (only_if_restart && *reinterpret_cast<volatile int *>(&a.ctrl->restart) == 0) return;
    double acc[3 * K];   // [rz | bb | rr]
#pragma unroll
    for (int i = 0; i < 3 * K; ++i) acc[i] = 0.0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.V; i += (int64_t)gridDim.x * blockDim.x) {
        const float di = a.dinv[i];
        const int64_t io = a.perm ? a.perm[i] : i;
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const float bv = b[io * K + k];
            float rv = bv;
            if (WARM) rv = bv - a.Ap[(size_t)k * a.Vp + i];
            else a.x[(size_t)k * a.Vp + i] = 0.f;
            const float z = di * rv;
            a.r[(size_t)k * a.Vp + i] = rv;
            a.p[(size_t)i * lsk::PRow<K>::PW + k] = z;
            acc[k] += (double)rv * (double)z;
            acc[K + k] += (double)bv * (double)bv;
            acc[2 * K + k] += (double)rv * (double)rv;
        }
        if (K == 3) a.p[(size_t)i * 4 + 3] = 0.f;
    }
    double tot[3 * K];
    const bool last = ls_grid_reduce<3 * K>(acc, tot, a.partials, a.ticket, red, threadIdx.x, VEC_THREADS, 1,
                                            blockIdx.x, gridDim.x);
    if (last && threadIdx.x == 0) {
        PcgCtrl *c = a.ctrl;
        int all = 1, worse = 0;
        const double rtol2 = (double)rtol * (double)rtol;
        for (int k = 0; k < K; ++k) {
            // a warm start whose residual exceeds ||b|| is worse than x = 0 and, in fp32, caps the attainable
            // accuracy at eps * kappa * ||x0|| / ||x||: fall back to the cold start (the reference CG has no such
            // guard, solvers.py:107-110, and loses accuracy when the gradient scale changes between steps)
            if (WARM && tot[2 * K + k] > tot[K + k]) worse = 1;
            c->rz[k] = tot[k];
            c->bb[k] = tot[K + k];
            c->rr[k] = tot[2 * K + k];
            c->pAp[k] = 1.0;
            c->beta[k] = 0.f;
            const int cv = tot[2 * K + k] <= rtol2 * tot[K + k];   // b_k == 0, or the warm start is already good enough
            c->conv[k] = cv;
            all &= cv;
        }
        for (int k = K; k < KMAX; ++k) {
            c->conv[k] = 1;
            c->rr[k] = 0.0;
            c->bb[k] = 0.0;
        }
        c->rtol2 = rtol * rtol;
        c->maxit = maxit;
        c->it = 0;
        c->k = K;
        c->restart = worse;
        c->done = (all && !worse) ? 1 : 0;
    }
}

// warm start stage 1: x = x0 (AoS -> SoA), p = x0 (SpMM input), done = 0 so that K1 runs
template <int K>
__global__ void __launch_bounds__(VEC_THREADS) k_warm_load(VecArgs a, const float *__restrict__ x0) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.V; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t io = a.perm ? a.perm[i] : i;
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const float v = x0[io * K + k];
            a.x[(size_t)k * a.Vp + i] = v;
            a.p[(size_t)i * lsk::PRow<K>::PW + k] = v;
        }
        if (K == 3) a.p[(size_t)i * 4 + 3] = 0.f;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) a.ctrl->done = 0;
}

__device__ __forceinline__ float4 ld4(const float *p) { return *reinterpret_cast<const float4 *>(p); }
__device__ __forceinline__ void st4(float *p, float4 v) { *reinterpret_cast<float4 *>(p) = v; }

// p is stored as rows of PW floats (PW = 1, 2, 4 for K = 1, 2, 3|4) so that the SpMM gathers one row with one load.
// These helpers move the 4 rows 4*i4 .. 4*i4+3 between that layout and per-column float4 registers.
template <int K>
__device__ __forceinline__ void load_p_rows(const float *p, int64_t i4, float4 (&pv)[K]) {
    constexpr int PW = lsk::PRow<K>::PW;
    if (PW == 1) {
        pv[0] = ld4(p + 4 * i4);
    } else if (PW == 2) {
        const float4 a = ld4(p + 8 * i4), b = ld4(p + 8 * i4 + 4);     // rows (0,1) and (2,3)
        pv[0] = make_float4(a.x, a.z, b.x, b.z);
        if (K > 1) pv[K > 1 ? 1 : 0] = make_float4(a.y, a.w, b.y, b.w);
    } else {
        const float4 r0 = ld4(p + 16 * i4), r1 = ld4(p + 16 * i4 + 4), r2 = ld4(p + 16 * i4 + 8), r3 = ld4(p + 16 * i4 + 12);
        pv[0] = make_float4(r0.x, r1.x, r2.x, r3.x);
        if (K > 1) pv[K > 1 ? 1 : 0] = make_float4(r0.y, r1.y, r2.y, r3.y);
        if (K > 2) pv[K > 2 ? 2 : 0] = make_float4(r0.z, r1.z, r2.z, r3.z);
        if (K > 3) pv[K > 3 ? 3 : 0] = make_float4(r0.w, r1.w, r2.w, r3.w);
    }
}
template <int K>
__device__ __forceinline__ void store_p_rows(float *p, int64_t i4, const float4 (&pv)[K]) {
    constexpr int PW = lsk::PRow<K>::PW;
    if (PW == 1) {
        st4(p + 4 * i4, pv[0]);
    } else if (PW == 2) {
        const float4 &c0 = pv[0], &c1 = pv[K > 1 ? 1 : 0];
        st4(p + 8 * i4, make_float4(c0.x, c1.x, c0.y, c1.y));
        st4(p + 8 * i4 + 4, make_float4(c0.z, c1.z, c0.w, c1.w));
    } else {
        const float4 &c0 = pv[0], &c1 = pv[K > 1 ? 1 : 0], &c2 = pv[K > 2 ? 2 : 0];
        const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
        const float4 &c3 = (K > 3) ? pv[K > 3 ? 3 : 0] : z;
        st4(p + 16 * i4, make_float4(c0.x, c1.x, c2.x, c3.x));
        st4(p + 16 * i4 + 4, make_float4(c0.y, c1.y, c2.y, c3.y));
        st4(p + 16 * i4 + 8, make_float4(c0.z, c1.z, c2.z, c3.z));
        st4(p + 16 * i4 + 12, make_float4(c0.w, c1.w, c2.w, c3.w));
    }
}

// scalar state transition run by the last CTA of K2: beta, per-column convergence, iteration count, done flag
template <int K>
__device__ __forceinline__ void pcg_transition(PcgCtrl *c, const double (&tot)[2 * K]) {
    int all = 1, bad = 0;
    for (int k = 0; k < K; ++k) {
        if (c->conv[k]) continue;
        const double pAp = c->pAp[k];
        if (!(pAp > 0.0) || !(tot[k] == tot[k])) bad = 1;   // not SPD, or NaN crept in
        const double rz_old = c->rz[k];
        c->beta[k] = (rz_old > 0.0) ? (float)(tot[k] / rz_old) : 0.f;
        c->rz[k] = tot[k];
        c->rr[k] = tot[K + k];
        const int cv = tot[K + k] <= (double)c->rtol2 * c->bb[k];
        c->conv[k] = cv;
        if (cv) c->beta[k] = 0.f;
        all &= cv;
    }
    const int it = c->it + 1;
    c->it = it;
    if (bad) c->done = 3;
    else if (all) c->done = 1;
    else if (it >= c->maxit) c->done = 2;
}

// K3: p = dinv r + beta p   (same loads-first structure as K2)
template <int K>
__global__ void __launch_bounds__(VEC_THREADS, 4) k_pupdate(VecArgs a) {
    PcgCtrl *c = a.ctrl;
    const int64_t n4 = a.Vp >> 2;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    float4 d, pv[K], rv[K];
    auto load = [&](int64_t j) {
        d = ld4(a.dinv + 4 * j);
        load_p_rows<K>(a.p, j, pv);
#pragma unroll
        for (int k = 0; k < K; ++k) rv[k] = ld4(a.r + (size_t)k * a.Vp + 4 * j);
    };
    if (i < n4) load(i);
    if (*reinterpret_cast<volatile int *>(&c->done) != 0) return;
    float beta[K];
#pragma unroll
    for (int k = 0; k < K; ++k) beta[k] = c->beta[k];
    for (bool first = true; i < n4; i += stride, first = false) {
        if (!first) load(i);
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const float be = beta[k];
            pv[k].x = fmaf(be, pv[k].x, d.x * rv[k].x);
            pv[k].y = fmaf(be, pv[k].y, d.y * rv[k].y);
            pv[k].z = fmaf(be, pv[k].z, d.z * rv[k].z);
            pv[k].w = fmaf(be, pv[k].w, d.w * rv[k].w);
        }
        store_p_rows<K>(a.p, i, pv);
    }
}

// K2: x += alpha p, r -= alpha Ap, rz' = r.(dinv r), rr = r.r ; last CTA: scalar state transition.
// One float4 of rows per thread, one column at a time (4-5 float4 loads in flight, ~80 registers); the vector loads of
// the first column are issued BEFORE the dependent scalar chain (done flag -> pAp/rz -> fp64 divide) so it hides under them.
template <int K>
__global__ void __launch_bounds__(VEC_THREADS, 3) k_update_cs(VecArgs a) {
    __shared__ double red[2 * K * 32 + 2 * K + 1];
    PcgCtrl *c = a.ctrl;
    const int64_t n4 = a.Vp >> 2;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    float4 d = make_float4(0.f, 0.f, 0.f, 0.f), x0, r0, q0, pv[K];
    if (i0 < n4) {   // issued before the dependent scalar chain below
        d = ld4(a.dinv + 4 * i0);
        load_p_rows<K>(a.p, i0, pv);
        x0 = ld4(a.x + 4 * i0);
        r0 = ld4(a.r + 4 * i0);
        q0 = ld4(a.Ap + 4 * i0);
    }
    if (*reinterpret_cast<volatile int *>(&c->done) != 0) return;
    float alpha[K];
#pragma unroll
    for (int k = 0; k < K; ++k) {
        const double pAp = c->pAp[k];
        alpha[k] = (c->conv[k] || !(pAp > 0.0)) ? 0.f : (float)(c->rz[k] / pAp);
    }
    double acc[2 * K];
#pragma unroll
    for (int q = 0; q < 2 * K; ++q) acc[q] = 0.0;
    for (int64_t i = i0; i < n4; i += stride) {
        if (i != i0) {
            d = ld4(a.dinv + 4 * i);
            load_p_rows<K>(a.p, i, pv);
        }
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const size_t o = (size_t)k * a.Vp + 4 * i;
            float4 xv, rv, qv;
            if (k == 0 && i == i0) {
                xv = x0; rv = r0; qv = q0;
            } else {
                xv = ld4(a.x + o); rv = ld4(a.r + o); qv = ld4(a.Ap + o);
            }
            const float al = alpha[k];
            const float4 pk = pv[k];
            xv.x = fmaf(al, pk.x, xv.x); xv.y = fmaf(al, pk.y, xv.y); xv.z = fmaf(al, pk.z, xv.z); xv.w = fmaf(al, pk.w, xv.w);
            rv.x = fmaf(-al, qv.x, rv.x); rv.y = fmaf(-al, qv.y, rv.y); rv.z = fmaf(-al, qv.z, rv.z); rv.w = fmaf(-al, qv.w, rv.w);
            st4(a.x + o, xv);
            st4(a.r + o, rv);
            const float r2x = rv.x * rv.x, r2y = rv.y * rv.y, r2z = rv.z * rv.z, r2w = rv.w * rv.w;
            acc[k] += (double)(d.x * r2x) + (double)(d.y * r2y) + (double)(d.z * r2z) + (double)(d.w * r2w);
            acc[K + k] += (double)r2x + (double)r2y + (double)r2z + (double)r2w;
        }
    }
    double tot[2 * K];
    const bool last = ls_grid_reduce<2 * K>(acc, tot, a.partials, a.ticket, red, threadIdx.x, VEC_THREADS, 1,
                                            blockIdx.x, gridDim.x);
    if (last && threadIdx.x == 0) pcg_transition<K>(c, tot);
}

// x (SoA) -> out (AoS), info
template <int K>
__global__ void __launch_bounds__(VEC_THREADS) k_final(VecArgs a, float *__restrict__ out, float *__restrict__ info) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.V; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t io = a.perm ? a.perm[i] : i;
#pragma unroll
        for (int k = 0; k < K; ++k) out[io * K + k] = a.x[(size_t)k * a.Vp + i];
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        const PcgCtrl *c = a.ctrl;
        float tmp[8];
        tmp[0] = (float)c->it;
        tmp[1] = (float)c->done;
        for (int k = 0; k < KMAX; ++k) tmp[2 + k] = (k < K && c->bb[k] > 0.0) ? (float)sqrt(c->rr[k] / c->bb[k]) : 0.f;
        tmp[6] = tmp[7] = 0.f;
        for (int j = 0; j < 8; ++j)
            if (info) info[j] = tmp[j];
    }
}

VecArgs vec_args(PcgHandle *h, int which_ticket) {
    VecArgs a;
    a.V = h->V;
    a.Vp = h->Vp;
    a.x = h->x;
    a.r = h->r;
    a.p = h->p;
    a.Ap = h->Ap;
    a.dinv = h->dinv;
    a.ctrl = h->ctrl;
    a.partials = h->part_vec;
    a.ticket = h->tickets + which_ticket;
    a.perm = h->has_perm ? h->perm : nullptr;
    return a;
}

lsk::SpmmArgs spmm_args(PcgHandle *h, int K, bool with_done) {
    lsk::SpmmArgs s{};
    s.V = (int)h->V;
    s.stages = h->graph.cfg.stages;
    s.cap = h->graph.cfg.cap;
    s.hint = h->graph.cfg.hint;
    s.debug = h->graph.cfg.debug;
    s.desc = h->graph.planned ? h->graph.desc : nullptr;
    s.desc_cnt = h->graph.desc_cnt;
    s.rowptr = h->rowptr;
    s.col = h->col;
    s.val = h->val;
    s.x = h->p;
    s.y = h->Ap;
    s.ldx = (K == 1) ? 1 : (K == 2 ? 2 : 4);   // p rows
    s.ldy = h->Vp;
    s.part = h->graph.part;
    s.done = with_done ? &h->ctrl->done : nullptr;
    s.partials = h->part_spmm;
    s.ticket = h->tickets + 0;
    s.dot_out = h->ctrl->pAp;
    return s;
}

// TMA-staged SELL SpMM (ls_sell_kernel.cuh): per-warp shared-memory rings fed by cp.async.bulk, launched with programmatic
// stream serialisation so that its matrix prefetch overlaps the tail of the previous kernel in the stream.
template <int K, bool DOT, int NW, int DEPTH, int MINB>
int launch_sell_tma_t(PcgHandle *h, const lsk::SellArgs &a, cudaStream_t s) {
    static bool prepared = false;
    const size_t smem = lsk::sell_tma_smem_bytes(NW, DEPTH);
    if (!prepared) {
        LS_CUDA_TRY(cudaFuncSetAttribute(lsk::spmm_sell_tma_kernel<K, DOT, NW, DEPTH, MINB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        prepared = true;
    }
    cudaLaunchConfig_t lc = {};
    int g = h->nslices < h->sm_count * MINB ? h->nslices : h->sm_count * MINB;
    lc.gridDim = dim3(g < 1 ? 1 : g);
    lc.blockDim = dim3(NW * 32);
    lc.dynamicSmemBytes = smem;
    lc.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    lc.attrs = at;
    lc.numAttrs = (h->graph.sell_tma >= 10) ? 0 : 1;   // LS_SELL_TMA >= 10: same kernels without PDL (A/B)
    LS_CUDA_TRY(cudaLaunchKernelEx(&lc, lsk::spmm_sell_tma_kernel<K, DOT, NW, DEPTH, MINB>, a));
    g_ls_launches.fetch_add(1, std::memory_order_relaxed);
    return LS_OK;
}
template <int K, bool DOT = true>
int launch_sell_tma(PcgHandle *h, const lsk::SellArgs &a, cudaStream_t s) {
    if constexpr (K == 3) {
        switch (h->graph.sell_tma % 10) {
            case 2: return launch_sell_tma_t<K, DOT, 24, 4, 1>(h, a, s);
            case 4: return launch_sell_tma_t<K, DOT, 16, 6, 1>(h, a, s);
            case 5: return launch_sell_tma_t<K, DOT, 16, 3, 2>(h, a, s);   // two CTAs per SM: the next launch's prefetch overlaps this one's tail
            case 6: return launch_sell_tma_t<K, DOT, 24, 2, 2>(h, a, s);
            case 7: return launch_sell_tma_t<K, DOT, 16, 2, 2>(h, a, s);   // 2 x 66 KB of rings: ~95 KB of L1 left for the gathers
            default: break;
        }
    }
    if (h->graph.sell_tma % 10 == 1) return launch_sell_tma_t<K, DOT, 32, 3, 1>(h, a, s);
    return launch_sell_tma_t<K, DOT, 32, 2, 1>(h, a, s);
}

// Ap = A p on the SELL-32 copy, with pAp = p.Ap (the DOT = false kernels ignore the dot-product pointers)
lsk::SellArgs sell_args(const PcgHandle *h, bool with_done) {
    lsk::SellArgs a{};
    a.V = (int)h->V;
    a.nslices = h->nslices;
    a.soff = h->soff;
    a.ent = h->ent;
    a.p = h->p;
    a.y = h->Ap;
    a.ldy = h->Vp;
    a.done = with_done ? &h->ctrl->done : nullptr;
    a.partials = h->part_spmm;
    a.ticket = h->tickets + 0;
    a.dot_out = h->ctrl->pAp;
    a.pf_halo = h->graph.sell_pf;
    return a;
}

template <int K>
int launch_spmm(PcgHandle *h, bool with_done, cudaStream_t s) {
    if (h->sell_on) {
        const lsk::SellArgs a = sell_args(h, with_done);
        if (h->graph.sell_tma) return launch_sell_tma<K>(h, a, s);
        lsk::spmm_sell_kernel<K, true><<<h->graph.sell_grid, lsk::SELL_THREADS, 0, s>>>(a);
        LS_LAUNCH_CHECK();
        return LS_OK;
    }
    return lsk::spmm_launch(K, true, h->graph.cfg, spmm_args(h, K, with_done), h->graph.spmm_grid, s);
}

template <int K>
int launch_iteration(PcgHandle *h, cudaStream_t s) {
    int rc = launch_spmm<K>(h, true, s);
    if (rc) return rc;
    k_update_cs<K><<<h->graph.vec_grid, VEC_THREADS, 0, s>>>(vec_args(h, 1));
    LS_LAUNCH_CHECK();
    k_pupdate<K><<<h->graph.vec_grid, VEC_THREADS, 0, s>>>(vec_args(h, 1));
    LS_LAUNCH_CHECK();
    return LS_OK;
}

// host-side resources only the graph-mode solver needs: created on its first use (they cost ~0.3 ms at handle creation)
int graph_host_resources(PcgHandle *h) {
    if (h->graph.cap_stream) return LS_OK;
    LS_CUDA_TRY(cudaStreamCreateWithFlags(&h->graph.cap_stream, cudaStreamNonBlocking));
    LS_CUDA_TRY(cudaEventCreateWithFlags(&h->graph.ev[0], cudaEventDisableTiming));
    LS_CUDA_TRY(cudaEventCreateWithFlags(&h->graph.ev[1], cudaEventDisableTiming));
    LS_CUDA_TRY(cudaMallocHost((void **)&h->graph.pinned_done, 64));
    return LS_OK;
}

template <int K>
int build_graph(PcgHandle *h) {
    if (h->graph.exec[K]) return LS_OK;
    {
        const int rc0 = graph_host_resources(h);
        if (rc0) return rc0;
    }
    cudaGraph_t g = nullptr;
    LS_CUDA_TRY(cudaStreamBeginCapture(h->graph.cap_stream, cudaStreamCaptureModeThreadLocal));
    int rc = LS_OK;
    for (int i = 0; i < CHUNK && rc == LS_OK; ++i) rc = launch_iteration<K>(h, h->graph.cap_stream);
    cudaError_t e = cudaStreamEndCapture(h->graph.cap_stream, &g);
    if (rc) {
        if (g) cudaGraphDestroy(g);
        return rc;
    }
    LS_CUDA_TRY(e);
    // launches recorded during capture were counted once; replays are counted in solve
    e = cudaGraphInstantiate(&h->graph.exec[K], g, 0);
    cudaGraphDestroy(g);
    LS_CUDA_TRY(e);
    return LS_OK;
}

template <int K>
int solve_graph_k(PcgHandle *h, const float *b, float *x, const float *x0, float rtol, int maxit, float *info,
                  cudaStream_t stream) {
    PcgHandle::Graph &g = h->graph;
    int occ;
    int rc = lsk::spmm_prepare(K, true, g.cfg, &occ);
    if (rc) return rc;
    rc = build_graph<K>(h);
    if (rc) return rc;
    VecArgs va = vec_args(h, 1);
    if (x0) {
        k_warm_load<K><<<g.vec_grid, VEC_THREADS, 0, stream>>>(va, x0);
        LS_LAUNCH_CHECK();
        rc = launch_spmm<K>(h, false, stream);
        if (rc) return rc;
        k_init<K, true><<<g.vec_grid, VEC_THREADS, 0, stream>>>(va, b, rtol, maxit, 0);
        LS_LAUNCH_CHECK();
        k_init<K, false><<<g.vec_grid, VEC_THREADS, 0, stream>>>(va, b, rtol, maxit, 1);   // runs only if `restart`
        LS_LAUNCH_CHECK();
    } else {
        k_init<K, false><<<g.vec_grid, VEC_THREADS, 0, stream>>>(va, b, rtol, maxit, 0);
        LS_LAUNCH_CHECK();
    }
    // iterate: replay the CHUNK-iteration graph; the device `done` flag of chunk c-1 is checked while chunk c runs
    // (kernels of a chunk enqueued after convergence see `done` and return immediately).
    int launched = 0, nq = 0;
    bool finished = false;
    while (!finished) {
        LS_CUDA_TRY(cudaGraphLaunch(g.exec[K], stream));
        g_ls_launches.fetch_add(3 * CHUNK, std::memory_order_relaxed);
        LS_CUDA_TRY(cudaMemcpyAsync(&g.pinned_done[nq & 1], &h->ctrl->done, sizeof(int), cudaMemcpyDeviceToHost, stream));
        LS_CUDA_TRY(cudaEventRecord(g.ev[nq & 1], stream));
        ++nq;
        launched += CHUNK;
        if (nq >= 2) {
            LS_CUDA_TRY(cudaEventSynchronize(g.ev[(nq - 2) & 1]));
            if (g.pinned_done[(nq - 2) & 1] != 0) finished = true;
        }
        if (!finished && launched >= maxit) {   // every iteration maxit allows is enqueued: drain
            LS_CUDA_TRY(cudaEventSynchronize(g.ev[(nq - 1) & 1]));
            finished = true;
        }
    }
    k_final<K><<<g.vec_grid, VEC_THREADS, 0, stream>>>(va, x, info);
    LS_LAUNCH_CHECK();
    return LS_OK;
}

template <int K>
int bench_one(PcgHandle *h, int which, cudaStream_t stream) {
    if (which == 4 && K == 3 && h->sell_on && h->graph.sell_tma)   // pure y = A p, no dot-product epilogue (the SpMV of BASELINE's metric)
        return launch_sell_tma<3, false>(h, sell_args(h, false), stream);
    return launch_spmm<K>(h, false, stream);
}

// p (rows of pw floats, new numbering) <- x (V, k) row-major in the caller's numbering; unused lanes and padding rows 0.
// The k planes of Ap: rows < V NaN (a row no launch writes reads back as NaN), padding rows 0 (as the solver keeps them).
__global__ void k_spmv_put(int64_t V, int64_t Vp, int k, int pw, const int *__restrict__ perm, const float *__restrict__ x,
                           float *__restrict__ p, float *__restrict__ Ap, double *__restrict__ dot) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < Vp * pw; i += stride) {
        const int64_t row = i / pw;
        const int c = (int)(i - row * pw);
        float v = 0.f;
        if (row < V && c < k) v = x[(perm ? (int64_t)perm[row] : row) * k + c];
        p[i] = v;
    }
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < Vp * k; i += stride)
        Ap[i] = (i % Vp < V) ? __int_as_float(0x7fc00000) : 0.f;
    if (blockIdx.x == 0 && threadIdx.x < KMAX) dot[threadIdx.x] = __longlong_as_double(0x7ff8000000000000ll);
}
// y (V, k) row-major in the caller's numbering <- the k planes of Ap
__global__ void k_spmv_get(int64_t V, int64_t Vp, int k, const int *__restrict__ perm, const float *__restrict__ Ap,
                           float *__restrict__ y) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < V * k; i += stride) {
        const int64_t row = i / k;
        const int c = (int)(i - row * k);
        y[(perm ? (int64_t)perm[row] : row) * k + c] = Ap[(size_t)c * Vp + row];
    }
}

}  // namespace

namespace lspcg {

// The graph-mode solver's launch geometry: the CSR engine's grid, its nnz-balanced row partition and block plan (every CTA's
// block boundaries, so the producer warp never chases rowptr at run time), the SELL-32 kernel's grid and the vector kernels' grid.
int graph_geometry(PcgHandle *h, cudaStream_t stream) {
    PcgHandle::Graph &g = h->graph;
    lsk::spmm_config(&g.cfg);
    int occ = 1;
    const int rc = lsk::spmm_prepare(3, true, g.cfg, &occ);
    if (rc) return rc;
    g.spmm_grid = lsk::spmm_grid_for(h->V, h->sm_count, occ);
    if (g.spmm_grid > GRID_CAP) g.spmm_grid = GRID_CAP;
    int socc = 0;
    LS_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&socc, lsk::spmm_sell_kernel<3, true>, lsk::SELL_THREADS, 0));
    if (socc < 1) socc = 1;
    int64_t sg = ((int64_t)h->nslices + lsk::SELL_WARPS - 1) / lsk::SELL_WARPS;   // >= one slice per warp
    if (sg > (int64_t)h->sm_count * socc) sg = (int64_t)h->sm_count * socc;
    if (sg > GRID_CAP) sg = GRID_CAP;
    if (sg < 1) sg = 1;
    g.sell_grid = (int)sg;
    int64_t vg = (h->Vp / 4 + VEC_THREADS - 1) / VEC_THREADS;   // one float4 per thread per column
    if (vg > GRID_CAP) vg = GRID_CAP;                           // beyond that the kernels grid-stride
    if (vg < 1) vg = 1;
    g.vec_grid = (int)vg;
    k_partition<<<(g.spmm_grid + 1 + 127) / 128, 128, 0, stream>>>(h->V, h->rowptr, g.spmm_grid, g.part);
    LS_LAUNCH_CHECK();
    return lsk::spmm_plan(h->rowptr, g.part, g.spmm_grid, g.cfg.cap, g.desc, g.desc_cnt, h->flags + 1, stream);
}

int solve_graph(PcgHandle *h, int k, const float *b, float *x, const float *x0, float rtol, int maxit, float *info,
                cudaStream_t stream) {
    switch (k) {
        case 1: return solve_graph_k<1>(h, b, x, x0, rtol, maxit, info, stream);
        case 2: return solve_graph_k<2>(h, b, x, x0, rtol, maxit, info, stream);
        case 3: return solve_graph_k<3>(h, b, x, x0, rtol, maxit, info, stream);
        default: return solve_graph_k<4>(h, b, x, x0, rtol, maxit, info, stream);
    }
}

void graph_destroy(PcgHandle::Graph &g) {
    for (int k = 0; k <= KMAX; ++k)
        if (g.exec[k]) cudaGraphExecDestroy(g.exec[k]);
    if (g.ev[0]) cudaEventDestroy(g.ev[0]);
    if (g.ev[1]) cudaEventDestroy(g.ev[1]);
    if (g.cap_stream) cudaStreamDestroy(g.cap_stream);
    if (g.pinned_done) cudaFreeHost(g.pinned_done);
}

}  // namespace lspcg

extern "C" int ls_pcg_bench_spmm(void *handle, int k, int launches, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    PcgHandle *h = (PcgHandle *)handle;
    LS_REQUIRE(h != nullptr, "handle is NULL");
    LS_REQUIRE(k >= 1 && k <= h->k_max, "k out of range for this handle");
    int occ;
    int rc = lsk::spmm_prepare(k, true, h->graph.cfg, &occ);
    if (rc) return rc;
    for (int i = 0; i < launches; ++i) {
        switch (k) {
            case 1: rc = launch_spmm<1>(h, false, stream); break;
            case 2: rc = launch_spmm<2>(h, false, stream); break;
            case 3: rc = launch_spmm<3>(h, false, stream); break;
            default: rc = launch_spmm<4>(h, false, stream); break;
        }
        if (rc) return rc;
    }
    return LS_OK;
}

extern "C" int ls_pcg_bench(void **handles, int n_handles, int k, int which, int launches, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    LS_REQUIRE(handles != nullptr && n_handles >= 1, "no handles");
    LS_REQUIRE(which == 0 || which == 4, "which: 0 SpMM+dot, 4 SpMM without the dot epilogue");
    for (int i = 0; i < n_handles; ++i) {
        PcgHandle *h = (PcgHandle *)handles[i];
        LS_REQUIRE(h != nullptr, "NULL handle");
        LS_REQUIRE(k >= 1 && k <= h->k_max, "k out of range for this handle");
        int occ;
        int rc = lsk::spmm_prepare(k, true, h->graph.cfg, &occ);
        if (rc) return rc;
    }
    for (int i = 0; i < launches; ++i) {
        PcgHandle *h = (PcgHandle *)handles[i % n_handles];
        int rc;
        switch (k) {
            case 1: rc = bench_one<1>(h, which, stream); break;
            case 2: rc = bench_one<2>(h, which, stream); break;
            case 3: rc = bench_one<3>(h, which, stream); break;
            default: rc = bench_one<4>(h, which, stream); break;
        }
        if (rc) return rc;
    }
    return LS_OK;
}

extern "C" int ls_pcg_spmv_put(void *handle, int k, const float *x, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    PcgHandle *h = (PcgHandle *)handle;
    LS_REQUIRE(h != nullptr && x != nullptr, "NULL pointer");
    LS_REQUIRE(k >= 1 && k <= h->k_max, "k out of range for this handle");
    const int pw = k == 1 ? 1 : (k == 2 ? 2 : 4);
    int64_t g = (h->Vp * pw + 255) / 256;
    if (g > GRID_CAP) g = GRID_CAP;
    k_spmv_put<<<(unsigned)g, 256, 0, stream>>>(h->V, h->Vp, k, pw, h->has_perm ? h->perm : nullptr, x, h->p, h->Ap, h->ctrl->pAp);
    LS_LAUNCH_CHECK();
    return LS_OK;
}

extern "C" int ls_pcg_spmv_get(void *handle, int k, float *y, double *dot, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    PcgHandle *h = (PcgHandle *)handle;
    LS_REQUIRE(h != nullptr && y != nullptr, "NULL pointer");
    LS_REQUIRE(k >= 1 && k <= h->k_max, "k out of range for this handle");
    int64_t g = (h->V * k + 255) / 256;
    if (g > GRID_CAP) g = GRID_CAP;
    k_spmv_get<<<(unsigned)g, 256, 0, stream>>>(h->V, h->Vp, k, h->has_perm ? h->perm : nullptr, h->Ap, y);
    LS_LAUNCH_CHECK();
    if (dot) LS_CUDA_TRY(cudaMemcpyAsync(dot, h->ctrl->pAp, (size_t)k * sizeof(double), cudaMemcpyDeviceToDevice, stream));
    return LS_OK;
}

extern "C" int64_t ls_pcg_spmm_bytes(void *handle, int k) {
    PcgHandle *h = (PcgHandle *)handle;
    if (!h) return 0;
    return 8 * h->nnz + 4 * (h->V + 1) + 8 * (int64_t)k * h->V;
}
