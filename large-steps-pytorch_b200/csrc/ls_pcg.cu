// ls_pcg.cu -- preconditioned conjugate gradients for M X = B, all K columns in one pass (sm_90a):
// handle / workspace management, solver configuration, the graph-mode solver and the C entry points.
//
// Replaces the reference's solve plug-ins (largesteps/solvers.py:26-39 CholeskySolver -> cholespy/CHOLMOD,
// solvers.py:41-126 ConjugateGradientSolver -> ~12 eager torch kernels + 1 host sync per iteration per axis).
//
// Two execution modes share the handle, the data layout and the per-column arithmetic:
//   * fused (ls_pcg_fused.cuh): the whole solve is ONE kernel with two grid synchronisations per iteration, in-kernel warm
//     start and true-residual guard, optional Chebyshev polynomial preconditioner -- the default for every k in 1..4;
//     cooperative grid (one CTA per SM), one CTA for tiny meshes, or (opt-in) one thread-block cluster;
//   * graph (this file): one iteration = three kernels, a CUDA graph of CHUNK iterations replayed until a device-side
//     `done` flag is seen -- the fallback when the fused kernel cannot run (no cooperative launch, no SELL-32 copy, or its
//     launch refused):
//       K1  Ap = A p, pAp_k = p_k.Ap_k                     (SELL-32 or TMA-staged CSR SpMM + deterministic grid reduction)
//       K2  x += a p; r -= a Ap; rz' = r.(dinv r); rr = r.r (fused update + 2K dot products; last CTA does the
//           scalar state transition: beta, convergence per column, iteration count, done flag)
//       K3  p = dinv r + beta p
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
#include <vector>
#include <string.h>
#include <stdlib.h>
#include "ls_spmm_host.h"
#include "ls_sell_kernel.cuh"
#include "ls_pcg_fused.cuh"
#include "ls_fused_inst.h"

#ifndef LS_CLRES_DEFAULT
#define LS_CLRES_DEFAULT 0     // slices (x 32 vertices); 0 = off: measured slower than the cooperative grid, see CLRES_CS
#endif

namespace {

constexpr int KMAX = 4;
constexpr int VEC_THREADS = 256;
constexpr int CHUNK = 8;   // CG iterations per graph launch

struct PcgCtrl {
    double rz[KMAX], pAp[KMAX], rr[KMAX], bb[KMAX];
    float beta[KMAX];
    float rtol2;
    int maxit;
    int it;
    int done;        // 0 running, 1 converged, 2 maxit reached, 3 breakdown
    int conv[KMAX];  // column frozen
    int k;
    int restart;     // warm start was worse than a cold start for some column: redo the initialisation from x = 0
};

// How the fused solver runs a mesh for one K (plan_fused).  on = 0: it does not, the graph-mode solver runs.
struct FusedPlan {
    int on, grid, cluster, res, nw, sync, nsl_max;   // nw warps per CTA; sync 1: one CTA or one cluster (cluster = grid), 0: grid
    size_t smem;
};

struct PcgHandle {
    int64_t V, nnz, Vp;
    int k_max, precond;
    int device;
    int sm_count;
    // workspace carve-out (device)
    int *rowptr, *col;
    float *val, *dinv;
    float *x, *r, *p, *Ap;
    int *part;
    PcgCtrl *ctrl;
    double *part_spmm, *part_vec;
    unsigned int *tickets;   // [0] spmm, [1] vec
    float *info;
    int *flags;
    // launch geometry
    lsk::SpmmCfg cfg;
    int spmm_grid;
    int vec_grid;
    int4 *desc;
    int *desc_cnt;
    int *perm;       // new -> old row (NULL-equivalent when has_perm == 0)
    int *inv;        // old -> new
    int *scan;
    int has_perm;
    int planned;
    // SELL-32 engine (fast path)
    int *soff;
    int2 *ent;
    long long sell_cap;      // capacity of `ent` in entries
    long long sell_entries;  // padded entry count
    int nslices;
    int sell_on;
    int sell_grid;
    // pattern-only copy for matrices with one common off-diagonal value (ls_sell_kernel.cuh "PAT"; LS_PCG_PATTERN=0 switches it off)
    int *poff;
    unsigned int *pcol;
    unsigned char *pcls;     // diagonal class per row
    unsigned long long *pcls_tab;   // [PAT_CLASSES] classes, then an int: more classes than the table holds
    unsigned int *patmm;     // [min, max] of the off-diagonal value bits
    long long pat_cap;       // capacity of `pcol` in words
    float offc;
    int pat_on;
    int pat_shared;          // identical compact slices share one stored copy (LS_PCG_PATSHARE=0 keeps one copy per slice)
    int pat_stored;          // slices stored (distinct, plus the ones never shared)
    int pat_words;           // words of `pcol` in use
    // fused two-synchronisation solver (ls_pcg_fused.cuh): the default; one configuration for K = 3 (k = 1..3) and one for K = 4
    lsf::GridBar *gbar;      // grid barrier counter
    double *partials;        // fenced all-reduce partials, [2][NVMAX][grid]
    long long *dbg;          // LS_PCG_PROFILE cycle counters
    unsigned long long *ring;   // fast all-reduce slots
    int ring_slots;
    float *pv;               // owner copy of p, k_max planes
    float *z2, *cy, *cd;     // Chebyshev preconditioner: second published row buffer, iterate and direction planes
    int cheb_m;              // 0 / 1: Jacobi only; m >= 2: polynomial of degree m - 1 (precond = 2)
    float cheb_c0, cheb_c1[8], cheb_c2[8];
    float *gersh;            // [1] max_i sum_j |a_ij| / a_ii
    struct FusedCfg : FusedPlan {
        int pat;
        const void *fn, *fn_prof;
    } fused[2];
    int max_smem_optin;
    int refine;              // max restarts from the true residual per solve
    float theta;
    int sell_tma;            // stand-alone SpMM: TMA-staged variant (0 = register-prefetch kernel)
    int sell_pf;             // ... halo (rows) of its bulk L2 prefetch of the gathered vector, 0 = off
    // graphs, one per K
    cudaGraphExec_t graph[KMAX + 1];
    cudaStream_t cap_stream;
    int *pinned_done;        // 2 ints, host pinned
    cudaEvent_t ev[2];
    size_t ws_bytes;
    struct Span {
        char *at;
        size_t bytes;
    } zeroed[2];             // workspace regions ls_pcg_create zeroes (carve_handle)
};

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
    h.part = c.take<int>(grid_cap + 1);
    h.desc = c.take<int4>((size_t)grid_cap * lsk::SPMM_BMAX);
    h.desc_cnt = c.take<int>(grid_cap);
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

// upper bound on the graph-mode kernels' grids (workspace sizing of their partials and SpMM descriptors; 132 SMs on H100 SXM).
// The fused solver's grid is at most 255 CTAs: its partials are carved for 256.
constexpr int GRID_CAP = 132 * 8 * 2;

// ---- setup kernels --------------------------------------------------------------------------------
__global__ void k_pad_tail(int *rowptr, int *col, float *val, int64_t V, int64_t nnz) {
    int t = threadIdx.x;
    if (t < 8) {
        rowptr[V + 1 + t] = (int)nnz;
        col[nnz + t] = 0;
        val[nnz + t] = 0.f;
    }
}

__global__ void k_dinv(int64_t V, int64_t Vp, const int *__restrict__ rowptr, const int *__restrict__ col,
                       const float *__restrict__ val, int precond, float *__restrict__ dinv, int *__restrict__ flags) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Vp) return;
    if (i >= V) {
        dinv[i] = 0.f;
        return;
    }
    float d = 0.f;
    bool found = false;
    int s = rowptr[i], e = rowptr[i + 1];
    if (e < s) atomicOr(flags, 4);
    for (int j = s; j < e; ++j) {
        int c = col[j];
        if (c < 0 || c >= V) atomicOr(flags, 1);
        if (c == (int)i) {
            d += val[j];
            found = true;
        }
    }
    if (!found || !(d > 0.f)) atomicOr(flags, 2);
    dinv[i] = precond ? (1.0f / d) : 1.0f;
}

// Gershgorin bound of lambda_max(D^-1 A): max_i sum_j |a_ij| / a_ii   (positive floats order like their bit patterns)
__global__ void k_gershgorin(int64_t V, const int *__restrict__ rowptr, const int *__restrict__ col, const float *__restrict__ val,
                             float *__restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    float g = 0.f;
    if (i < V) {
        float d = 0.f, sabs = 0.f;
        for (int j = rowptr[i]; j < rowptr[i + 1]; ++j) {
            const float a = val[j];
            sabs += fabsf(a);
            if (col[j] == (int)i) d += a;
        }
        g = d > 0.f ? sabs / d : 0.f;
    }
    g = fmaxf(g, 0.f);
    unsigned int b = __float_as_uint(g);
    b = __reduce_max_sync(0xffffffffu, b);
    if ((threadIdx.x & 31) == 0 && b) atomicMax(reinterpret_cast<unsigned int *>(out), b);
}

// ---- permuted copy  A' = P A P^T  (perm[new] = old) ------------------------------------------------
__global__ void k_perm_inv_len(int64_t V, const int *__restrict__ perm, const int *__restrict__ rowptr,
                               int *__restrict__ inv, int *__restrict__ len, int *__restrict__ flags) {
    int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= V) return;
    const int o = perm[n];
    if (o < 0 || o >= V) {
        atomicOr(flags, 8);
        len[n] = 0;
        return;
    }
    inv[o] = (int)n;
    len[n] = rowptr[o + 1] - rowptr[o];
}
// one thread per new row: copy the old row with renumbered columns, then insertion-sort it by new column
__global__ void k_perm_rows(int64_t V, const int *__restrict__ perm, const int *__restrict__ inv,
                            const int *__restrict__ rowptr, const int *__restrict__ col, const float *__restrict__ val,
                            const int *__restrict__ rowptr_new, int *__restrict__ col_new, float *__restrict__ val_new,
                            int *__restrict__ flags) {
    int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= V) return;
    const int o = perm[n];
    if (o < 0 || o >= V) return;
    const int s = rowptr[o], e = rowptr[o + 1];
    const int d = rowptr_new[n];
    for (int j = s; j < e; ++j) {
        int c = col[j];
        if (c < 0 || c >= V) {
            atomicOr(flags, 1);
            c = o;
        }
        const int cn = inv[c];
        const float w = val[j];
        int a = d + (j - s) - 1;
        while (a >= d && col_new[a] > cn) {
            col_new[a + 1] = col_new[a];
            val_new[a + 1] = val_new[a];
            --a;
        }
        col_new[a + 1] = cn;
        val_new[a + 1] = w;
    }
}
__global__ void k_perm_check(int64_t V, const int *__restrict__ perm, const int *__restrict__ inv, int *__restrict__ flags) {
    int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= V) return;
    const int o = perm[n];
    if (o >= 0 && o < V && inv[o] != (int)n) atomicOr(flags, 8);   // not a permutation (duplicate target)
}

// Gather-locality score of a row order: number of (row, slot) pairs whose column is NOT within 8 entries of the
// same slot's column in the previous row (adjacent rows are adjacent lanes of a warp, 8 float4 rows of p = one 128-byte
// line).  Lower is better; used to decide whether the Morton re-ordering actually helps (a row-major grid is already
// perfectly coalesced, a scanner mesh or a shuffled numbering is not).
__global__ void k_locality_score(int64_t V, const int *__restrict__ rowptr, const int *__restrict__ col,
                                 unsigned long long *__restrict__ score) {
    unsigned int bad = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < V; i += (int64_t)gridDim.x * blockDim.x) {
        if ((i & 31) == 0) continue;   // first lane of a warp has no left neighbour
        const int s = rowptr[i], e = rowptr[i + 1], sp = rowptr[i - 1], ep = rowptr[i];
        const int n = min(e - s, ep - sp);
        for (int j = 0; j < n; ++j) {
            const int d = col[s + j] - col[sp + j];
            bad += (d < -8 || d > 8) ? 1u : 0u;
        }
        bad += (unsigned int)((e - s) - n);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) bad += __shfl_xor_sync(0xffffffffu, bad, o);
    if ((threadIdx.x & 31) == 0 && bad) atomicAdd(score, (unsigned long long)bad);
}

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
    s.stages = h->cfg.stages;
    s.cap = h->cfg.cap;
    s.hint = h->cfg.hint;
    s.debug = h->cfg.debug;
    s.desc = h->planned ? h->desc : nullptr;
    s.desc_cnt = h->desc_cnt;
    s.rowptr = h->rowptr;
    s.col = h->col;
    s.val = h->val;
    s.x = h->p;
    s.y = h->Ap;
    s.ldx = (K == 1) ? 1 : (K == 2 ? 2 : 4);   // p rows
    s.ldy = h->Vp;
    s.part = h->part;
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
    lc.numAttrs = (h->sell_tma >= 10) ? 0 : 1;   // LS_SELL_TMA >= 10: same kernels without PDL (A/B)
    LS_CUDA_TRY(cudaLaunchKernelEx(&lc, lsk::spmm_sell_tma_kernel<K, DOT, NW, DEPTH, MINB>, a));
    g_ls_launches.fetch_add(1, std::memory_order_relaxed);
    return LS_OK;
}
template <int K, bool DOT = true>
int launch_sell_tma(PcgHandle *h, const lsk::SellArgs &a, cudaStream_t s) {
    if constexpr (K == 3) {
        switch (h->sell_tma % 10) {
            case 2: return launch_sell_tma_t<K, DOT, 24, 4, 1>(h, a, s);
            case 4: return launch_sell_tma_t<K, DOT, 16, 6, 1>(h, a, s);
            case 5: return launch_sell_tma_t<K, DOT, 16, 3, 2>(h, a, s);   // two CTAs per SM: the next launch's prefetch overlaps this one's tail
            case 6: return launch_sell_tma_t<K, DOT, 24, 2, 2>(h, a, s);
            case 7: return launch_sell_tma_t<K, DOT, 16, 2, 2>(h, a, s);   // 2 x 66 KB of rings: ~95 KB of L1 left for the gathers
            default: break;
        }
    }
    if (h->sell_tma % 10 == 1) return launch_sell_tma_t<K, DOT, 32, 3, 1>(h, a, s);
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
    a.pf_halo = h->sell_pf;
    return a;
}

template <int K>
int launch_spmm(PcgHandle *h, bool with_done, cudaStream_t s) {
    if (h->sell_on) {
        const lsk::SellArgs a = sell_args(h, with_done);
        if (h->sell_tma) return launch_sell_tma<K>(h, a, s);
        lsk::spmm_sell_kernel<K, true><<<h->sell_grid, lsk::SELL_THREADS, 0, s>>>(a);
        LS_LAUNCH_CHECK();
        return LS_OK;
    }
    return lsk::spmm_launch(K, true, h->cfg, spmm_args(h, K, with_done), h->spmm_grid, s);
}

template <int K>
int launch_iteration(PcgHandle *h, cudaStream_t s) {
    int rc = launch_spmm<K>(h, true, s);
    if (rc) return rc;
    k_update_cs<K><<<h->vec_grid, VEC_THREADS, 0, s>>>(vec_args(h, 1));
    LS_LAUNCH_CHECK();
    k_pupdate<K><<<h->vec_grid, VEC_THREADS, 0, s>>>(vec_args(h, 1));
    LS_LAUNCH_CHECK();
    return LS_OK;
}

// host-side resources only the graph-mode solver needs: created on its first use (they cost ~0.3 ms at handle creation)
int graph_host_resources(PcgHandle *h) {
    if (h->cap_stream) return LS_OK;
    LS_CUDA_TRY(cudaStreamCreateWithFlags(&h->cap_stream, cudaStreamNonBlocking));
    LS_CUDA_TRY(cudaEventCreateWithFlags(&h->ev[0], cudaEventDisableTiming));
    LS_CUDA_TRY(cudaEventCreateWithFlags(&h->ev[1], cudaEventDisableTiming));
    LS_CUDA_TRY(cudaMallocHost((void **)&h->pinned_done, 64));
    return LS_OK;
}

template <int K>
int build_graph(PcgHandle *h) {
    if (h->graph[K]) return LS_OK;
    {
        const int rc0 = graph_host_resources(h);
        if (rc0) return rc0;
    }
    cudaGraph_t g = nullptr;
    LS_CUDA_TRY(cudaStreamBeginCapture(h->cap_stream, cudaStreamCaptureModeThreadLocal));
    int rc = LS_OK;
    for (int i = 0; i < CHUNK && rc == LS_OK; ++i) rc = launch_iteration<K>(h, h->cap_stream);
    cudaError_t e = cudaStreamEndCapture(h->cap_stream, &g);
    if (rc) {
        if (g) cudaGraphDestroy(g);
        return rc;
    }
    LS_CUDA_TRY(e);
    // launches recorded during capture were counted once; replays are counted in solve
    e = cudaGraphInstantiate(&h->graph[K], g, 0);
    cudaGraphDestroy(g);
    LS_CUDA_TRY(e);
    return LS_OK;
}

int finish_info(PcgHandle *h, float rtol, int maxit, float *info_src, float *info_host, cudaStream_t stream) {
    if (!info_host) return LS_OK;
    LS_CUDA_TRY(cudaMemcpyAsync(info_host, info_src, 8 * sizeof(float), cudaMemcpyDefault, stream));
    LS_CUDA_TRY(cudaStreamSynchronize(stream));
    const int st = (int)info_host[1];
    if (st == 3) {
        ls_set_error("CG breakdown after %d iterations (matrix not SPD or NaN in the right-hand side)", (int)info_host[0]);
        return LS_ERR_BREAKDOWN;
    }
    if (st == 2) {
        ls_set_error("PCG did not reach rtol=%g within maxit=%d (relres %g %g %g %g)", (double)rtol, maxit,
                     (double)info_host[2], (double)info_host[3], (double)info_host[4], (double)info_host[5]);
        return LS_ERR_NOT_CONVERGED;
    }
    return LS_OK;
}

// ---- fused two-synchronisation solver (ls_pcg_fused.cuh) ------------------------------------------------------------
// instantiation table: (K, RES, NW, PAT, SYNC, PROF, CHEB) -> kernel, or NULL when that combination is not built.  The
// instantiations live in three translation units (ls_fused_a/b/c.cu) so that they compile in parallel.
const void *fused_fn(int K, int res, int nw, int pat, int sync, int prof, int cheb = 0) {
    if (cheb) return (K == 3 && !prof) ? ls_fused_fn_cheb(res, nw, pat, sync) : nullptr;
    if (K == 3 && !prof) return ls_fused_fn_jacobi(res, nw, pat, sync);
    return ls_fused_fn_misc(K, res, nw, pat, sync, prof);
}

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

// The environment switches of the fused solver's launch plan (DESIGN 4.6), read once per ls_pcg_create / ls_pcg_plan.
struct PlanEnv {
    int graph;       // LS_PCG_MODE=graph: no fused solver
    int cluster;     // LS_PCG_CLUSTER: -1 auto, 0 never one CTA or cluster, N a cluster of N CTAs
    int res;         // LS_PCG_RES: cap on the residency level, -1 none
    int onecta;      // LS_PCG_ONECTA: largest mesh (slices) on one CTA
    int clres;       // LS_PCG_CLRES: largest mesh (slices) on one cluster of CLRES_CS CTAs at RES 4
    int small_cta;   // 256-thread CTAs where they apply (LS_PCG_SMALLCTA=0: never)
};

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

// The environment switches of the matrix copies and the handle's defaults (DESIGN 4.6), read once per ls_pcg_create.
struct CreateEnv {
    int force_reorder;   // LS_FORCE_REORDER set: use the caller's permutation without comparing gather locality
    int pattern;         // pattern-only copy where every off-diagonal value is equal (LS_PCG_PATTERN=0: never)
    int patshare;        // ... with identical slices stored once (LS_PCG_PATSHARE=0: one copy per slice)
    int csr;             // LS_SPMM_ENGINE=csr: the TMA-staged CSR engine even when the SELL-32 copy fits
    int cheb_m;          // LS_PCG_CHEB_M: Chebyshev steps, 2..8
    int refine;          // LS_PCG_REFINE: restarts from the true residual per solve
    int sell_tma;        // LS_SELL_TMA: stand-alone SpMM variant (3: 32 warps x 2 slots of 2 KB)
    int sell_pf;         // LS_SELL_PF: halo (rows) of its L2 prefetch
};

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

// slices per CTA that fit in max_smem bytes of shared memory at residency level res (sync = 1: the one-CTA / cluster layout)
int slices_per_cta(int K, int res, int pat, int cheb, int sync, int max_smem) {
    if (res == 0) return 1 << 30;
    int n = 0;
    while (lsf::fused_smem_bytes(K, res, n + 1, pat, cheb, sync) <= (size_t)max_smem) ++n;
    return n;
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

int solve_fused(PcgHandle *h, const float *b, float *x, const float *x0, int k, float rtol, int maxit, float *info_dev,
                float *info_host, cudaStream_t stream) {
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
    a.info = info_dev ? info_dev : h->info;
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
    return finish_info(h, rtol, maxit, a.info, info_host, stream);
}

template <int K>
int solve_k(PcgHandle *h, const float *b, float *x, const float *x0, float rtol, int maxit, float *info_dev,
            float *info_host, cudaStream_t stream) {
    if (h->fused[K == 4 ? 1 : 0].on) {
        const int frc = solve_fused(h, b, x, x0, K, rtol, maxit, info_dev, info_host, stream);
        if (frc != -1) return frc;     // -1: launch refused, fall through to the graph-mode solver
    }
    int occ;
    int rc = lsk::spmm_prepare(K, true, h->cfg, &occ);
    if (rc) return rc;
    rc = build_graph<K>(h);
    if (rc) return rc;
    VecArgs va = vec_args(h, 1);
    if (x0) {
        k_warm_load<K><<<h->vec_grid, VEC_THREADS, 0, stream>>>(va, x0);
        LS_LAUNCH_CHECK();
        rc = launch_spmm<K>(h, false, stream);
        if (rc) return rc;
        k_init<K, true><<<h->vec_grid, VEC_THREADS, 0, stream>>>(va, b, rtol, maxit, 0);
        LS_LAUNCH_CHECK();
        k_init<K, false><<<h->vec_grid, VEC_THREADS, 0, stream>>>(va, b, rtol, maxit, 1);   // runs only if `restart`
        LS_LAUNCH_CHECK();
    } else {
        k_init<K, false><<<h->vec_grid, VEC_THREADS, 0, stream>>>(va, b, rtol, maxit, 0);
        LS_LAUNCH_CHECK();
    }
    // iterate: replay the CHUNK-iteration graph; the device `done` flag of chunk c-1 is checked while chunk c runs
    // (kernels of a chunk enqueued after convergence see `done` and return immediately).
    int launched = 0, nq = 0;
    bool finished = false;
    while (!finished) {
        LS_CUDA_TRY(cudaGraphLaunch(h->graph[K], stream));
        g_ls_launches.fetch_add(3 * CHUNK, std::memory_order_relaxed);
        LS_CUDA_TRY(cudaMemcpyAsync(&h->pinned_done[nq & 1], &h->ctrl->done, sizeof(int), cudaMemcpyDeviceToHost, stream));
        LS_CUDA_TRY(cudaEventRecord(h->ev[nq & 1], stream));
        ++nq;
        launched += CHUNK;
        if (nq >= 2) {
            LS_CUDA_TRY(cudaEventSynchronize(h->ev[(nq - 2) & 1]));
            if (h->pinned_done[(nq - 2) & 1] != 0) finished = true;
        }
        if (!finished && launched >= maxit) {   // every iteration maxit allows is enqueued: drain
            LS_CUDA_TRY(cudaEventSynchronize(h->ev[(nq - 1) & 1]));
            finished = true;
        }
    }
    float *info = info_dev ? info_dev : h->info;
    k_final<K><<<h->vec_grid, VEC_THREADS, 0, stream>>>(va, x, info);
    LS_LAUNCH_CHECK();
    return finish_info(h, rtol, maxit, info, info_host, stream);
}

// ---- the stages of ls_pcg_create, in the order it runs them: each returns an LS_* status ------------------------------------

// The solver's CSR copy: A' = P A P^T with rows re-sorted by new column when a permutation is given and it gathers more
// coherently than the caller's numbering (LS_FORCE_REORDER: always), else the caller's CSR as it is; then its padding tail and
// dinv.  Up to two host round trips, for the locality scores.
int copy_matrix(PcgHandle *h, const int *rowptr, const int *col, const float *val, const int *perm, int force_reorder,
                cudaStream_t stream) {
    const int64_t V = h->V, nnz = h->nnz;
    const unsigned gb = (unsigned)((V + 255) / 256), gs = gb > 2048 ? 2048 : gb;
    unsigned long long *sc = reinterpret_cast<unsigned long long *>(h->part_vec);   // scratch, zeroed by the create
    if (perm && !force_reorder) {
        // a numbering whose neighbouring rows already gather from neighbouring columns (a grid, a remesher's output) is kept
        // without ever building the permuted copy: fewer than 1 in 8 (row, slot) pairs break the coalescing
        k_locality_score<<<gs, 256, 0, stream>>>(V, rowptr, col, sc);
        LS_LAUNCH_CHECK();
        unsigned long long hs0 = 0;
        LS_CUDA_TRY(cudaMemcpyAsync(&hs0, sc, sizeof(hs0), cudaMemcpyDeviceToHost, stream));
        LS_CUDA_TRY(cudaStreamSynchronize(stream));
        if (hs0 * 8ull <= (unsigned long long)nnz) {
            perm = nullptr;
            LS_CUDA_TRY(cudaMemsetAsync(sc, 0, 16, stream));
        }
        // otherwise the score of the permuted order needs the permuted CSR: build it, score it, then decide
    }
    h->has_perm = perm ? 1 : 0;
    if (perm) {
        LS_CUDA_TRY(cudaMemcpyAsync(h->perm, perm, (size_t)V * 4, cudaMemcpyDeviceToDevice, stream));
        LS_CUDA_TRY(cudaMemsetAsync(h->inv, 0xff, (size_t)V * 4, stream));
        k_perm_inv_len<<<gb, 256, 0, stream>>>(V, h->perm, rowptr, h->inv, h->rowptr, h->flags);
        LS_LAUNCH_CHECK();
        k_perm_check<<<gb, 256, 0, stream>>>(V, h->perm, h->inv, h->flags);
        LS_LAUNCH_CHECK();
        const int rc = ls_exclusive_scan_i32(h->rowptr, h->rowptr, V, h->scan, stream);
        if (rc) return rc;
        k_perm_rows<<<gb, 256, 0, stream>>>(V, h->perm, h->inv, rowptr, col, val, h->rowptr, h->col, h->val, h->flags);
        LS_LAUNCH_CHECK();
        if (!force_reorder) {
            k_locality_score<<<gs, 256, 0, stream>>>(V, h->rowptr, h->col, sc + 1);
            LS_LAUNCH_CHECK();
            unsigned long long hs[2] = {0, 0};
            LS_CUDA_TRY(cudaMemcpyAsync(hs, sc, sizeof(hs), cudaMemcpyDeviceToHost, stream));
            LS_CUDA_TRY(cudaStreamSynchronize(stream));
            LS_CUDA_TRY(cudaMemsetAsync(sc, 0, sizeof(hs), stream));
            if (hs[0] <= hs[1]) h->has_perm = 0;   // native order is at least as good: drop the permutation
        }
    }
    if (!h->has_perm) {
        LS_CUDA_TRY(cudaMemcpyAsync(h->rowptr, rowptr, (size_t)(V + 1) * 4, cudaMemcpyDeviceToDevice, stream));
        LS_CUDA_TRY(cudaMemcpyAsync(h->col, col, (size_t)nnz * 4, cudaMemcpyDeviceToDevice, stream));
        LS_CUDA_TRY(cudaMemcpyAsync(h->val, val, (size_t)nnz * 4, cudaMemcpyDeviceToDevice, stream));
    }
    k_pad_tail<<<1, 32, 0, stream>>>(h->rowptr, h->col, h->val, V, nnz);
    LS_LAUNCH_CHECK();
    // (precond 3 is still unresolved here: dinv only tells precond 0 from the others)
    k_dinv<<<(unsigned)((h->Vp + 255) / 256), 256, 0, stream>>>(V, h->Vp, h->rowptr, h->col, h->val, h->precond, h->dinv, h->flags);
    LS_LAUNCH_CHECK();
    return LS_OK;
}

// The graph-mode solver's launch geometry: the CSR engine's grid, its nnz-balanced row partition and block plan (every CTA's
// block boundaries, so the producer warp never chases rowptr at run time), and the vector kernels' grid.
int graph_geometry(PcgHandle *h, cudaStream_t stream) {
    lsk::spmm_config(&h->cfg);
    int occ = 1;
    const int rc = lsk::spmm_prepare(3, true, h->cfg, &occ);
    if (rc) return rc;
    h->spmm_grid = lsk::spmm_grid_for(h->V, h->sm_count, occ);
    if (h->spmm_grid > GRID_CAP) h->spmm_grid = GRID_CAP;
    int64_t vg = (h->Vp / 4 + VEC_THREADS - 1) / VEC_THREADS;   // one float4 per thread per column
    if (vg > GRID_CAP) vg = GRID_CAP;                           // beyond that the kernels grid-stride
    if (vg < 1) vg = 1;
    h->vec_grid = (int)vg;
    k_partition<<<(h->spmm_grid + 1 + 127) / 128, 128, 0, stream>>>(h->V, h->rowptr, h->spmm_grid, h->part);
    LS_LAUNCH_CHECK();
    return lsk::spmm_plan(h->rowptr, h->part, h->spmm_grid, h->cfg.cap, h->desc, h->desc_cnt, h->flags + 1, stream);
}

}  // namespace

namespace lsk {

// ---- SELL build (from the solver's CSR copy; the layout and the SpMM kernels that read it: ls_sell_kernel.cuh) ----------
// widths: one warp per slice, w = max row length; cnt[s] = 32 w
static __global__ void sell_width_kernel(int V, int nslices, const int *__restrict__ rowptr, int *__restrict__ cnt) {
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (gw >= nslices) return;
    const int row = gw * 32 + lane;
    int len = (row < V) ? rowptr[row + 1] - rowptr[row] : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) len = max(len, __shfl_xor_sync(0xffffffffu, len, o));
    if (lane == 0) cnt[gw] = 32 * len;
}
static __global__ void sell_fill_kernel(int V, int nslices, const int *__restrict__ rowptr, const int *__restrict__ col,
                                        const float *__restrict__ val, const int *__restrict__ soff,
                                        int2 *__restrict__ ent, long long cap_entries) {
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (gw >= nslices) return;
    const int o0 = soff[gw], o1 = soff[gw + 1];
    if ((long long)o1 > cap_entries) return;   // over capacity: the caller falls back to the CSR engine
    const int w = (o1 - o0) >> 5;
    const int row = gw * 32 + lane;
    int j0 = 0, len = 0;
    if (row < V) {
        j0 = rowptr[row];
        len = rowptr[row + 1] - j0;
    }
    for (int j = 0; j < w; ++j) {
        int2 v = make_int2(row, 0);                         // padding: own row (inside the padded planes), weight 0
        if (j < len) v = make_int2(col[j0 + j], __float_as_int(val[j0 + j]));
        ent[(size_t)o0 + (size_t)j * 32 + lane] = v;
    }
}

// ---- pattern-only copy build (the layout: ls_sell_kernel.cuh "PAT") ---------------------------------------------------
static __global__ void pat_detect_kernel(int V, const int *__restrict__ rowptr, const int *__restrict__ col,
                                         const float *__restrict__ val, unsigned int *__restrict__ mm /* [min, max] */) {
    const int row = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned int mn = 0xffffffffu, mx = 0u;
    if (row < V) {
        for (int j = rowptr[row]; j < rowptr[row + 1]; ++j)
            if (col[j] != row) {
                const unsigned int b = __float_as_uint(val[j]);
                mn = min(mn, b);
                mx = max(mx, b);
            }
    }
    mn = __reduce_min_sync(0xffffffffu, mn);
    mx = __reduce_max_sync(0xffffffffu, mx);
    if ((threadIdx.x & 31) == 0) {
        if (mn != 0xffffffffu) atomicMin(mm, mn);
        if (mx != 0u) atomicMax(mm + 1, mx);
    }
}
// one warp per slice: pairs per row (ceil(max off-diagonal row length / 2)) and whether every offset fits 16 bits
__device__ __forceinline__ void pat_slice_shape(int V, int row, const int *__restrict__ rowptr, const int *__restrict__ col,
                                                int &w2, bool &wide) {
    int len = 0, far = 0;
    if (row < V)
        for (int j = rowptr[row]; j < rowptr[row + 1]; ++j) {
            const int c = col[j];
            if (c != row) {
                ++len;
                far |= (c - row > 32767 || row - c > 32767) ? 1 : 0;
            }
        }
    w2 = (__reduce_max_sync(0xffffffffu, len) + 1) >> 1;
    wide = __any_sync(0xffffffffu, far) != 0;
}
// widths: cnt[s] = words of slice s (32 per pair compact, 64 wide)
static __global__ void pat_width_kernel(int V, int nslices, const int *__restrict__ rowptr, const int *__restrict__ col,
                                        int *__restrict__ cnt) {
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (gw >= nslices) return;
    int w2;
    bool wide;
    pat_slice_shape(V, gw * 32 + lane, rowptr, col, w2, wide);
    if (lane == 0) cnt[gw] = (wide ? 64 : 32) * w2;
}
// the row's diagonal class: slot of (dinv, d') in the open-addressing table tab, *over = 1 when the table is full
__device__ __forceinline__ int pat_class(unsigned long long *tab, unsigned long long key, int *over) {
    unsigned int h = (unsigned int)((key * 0x9E3779B97F4A7C15ull) >> 56);
    if (key != PAT_EMPTY)
        for (int n = 0; n < PAT_CLASSES; ++n, h = (h + 1) & (PAT_CLASSES - 1)) {
            unsigned long long k = *reinterpret_cast<volatile unsigned long long *>(tab + h);
            if (k == PAT_EMPTY) k = atomicCAS(tab + h, PAT_EMPTY, key);
            if (k == PAT_EMPTY || k == key) return (int)h;
        }
    atomicOr(over, 1);
    return 0;
}
// poff (scanned word counts) -> pairs, the low bits of the slice's offset (pat_word), classes (cls, tab: PAT_EMPTY-filled, over:
// 0 on entry)
static __global__ void pat_fill_kernel(int V, int nslices, const int *__restrict__ rowptr, const int *__restrict__ col,
                                       const float *__restrict__ val, const float *__restrict__ dinv, int *__restrict__ poff,
                                       unsigned int *__restrict__ pc, long long cap_words, float offc, unsigned char *__restrict__ cls,
                                       unsigned long long *__restrict__ tab, int *__restrict__ over) {
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (gw >= nslices) return;
    const int row = gw * 32 + lane;
    int w2;
    bool wide;
    pat_slice_shape(V, row, rowptr, col, w2, wide);
    const int o0 = poff[gw] & ~31;   // (lane 0 sets the low bits below)
    if ((long long)o0 + (wide ? 64 : 32) * w2 > cap_words) return;
    float d = 0.f;
    int j = 0;
    auto put = [&](int slot, int c) {
        if (wide) pc[(size_t)o0 + 2 * ((size_t)(slot >> 1) * 32 + lane) + (slot & 1)] = (unsigned int)c;
        else reinterpret_cast<unsigned short *>(pc)[2 * ((size_t)o0 + (size_t)(slot >> 1) * 32 + lane) + (slot & 1)] = (unsigned short)(c - row);
    };
    if (row < V)
        for (int e = rowptr[row]; e < rowptr[row + 1]; ++e) {
            const int c = col[e];
            if (c == row) {
                d = val[e];
            } else {
                put(j, c);
                ++j;
            }
        }
    const int used = j;
    for (; j < 2 * w2; ++j) put(j, row);   // unused slot: the row itself
    const float di = (row < V) ? dinv[row] : 0.f, dp = (row < V) ? fmaf(-offc, (float)(2 * w2 - used), d) : 0.f;
    cls[row] = (unsigned char)pat_class(tab, ((unsigned long long)__float_as_uint(di) << 32) | __float_as_uint(dp), over);
    if (lane == 0) atomicOr(poff + gw, pat_word(0, w2, wide));
}

// ---- shared slices: store each distinct compact slice once ---------------------------------------------------------------
// Run after pat_fill_kernel on the unshared layout.  Scratch (ints): slot[n], off[n + 1], npoff[n + 1], stats[2] = {stored
// slices, 0}, tab[mask + 1] (PAT_SLOT_EMPTY-filled, mask + 1 >= 2 n a power of two); words: scr[cap_scr].
// The representative of a group of identical slices is its lowest slice index (atomicMin over the group's table slot), so
// the layout does not depend on scheduling.  Stored slices keep their order, so the slice after an escape slice -- never
// shared -- still starts where the escape slice ends.
constexpr unsigned int PAT_SLOT_EMPTY = 0xffffffffu;

__device__ __forceinline__ bool pat_shareable(const int *poff, int s) {
    const PatSlice ps = pat_slice(poff + s);
    return !ps.wide && ps.w2 < PAT_W2_ESC && !(s > 0 && pat_slice(poff + s - 1).w2 >= PAT_W2_ESC);
}
// one warp per slice: hash the slice's w2 and words, find or claim its group's slot (full comparison of the words)
static __global__ void pat_hash_kernel(int nslices, const int *__restrict__ poff, const unsigned int *__restrict__ pc,
                                       unsigned int *__restrict__ tab, unsigned int mask, int *__restrict__ slot) {
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (gw >= nslices) return;
    if (!pat_shareable(poff, gw)) {
        if (lane == 0) slot[gw] = -1;
        return;
    }
    const PatSlice ps = pat_slice(poff + gw);
    unsigned int h = 2166136261u ^ (unsigned int)lane;
    for (int m = 0; m < ps.w2; ++m) h = (h ^ pc[ps.o0 + m * 32 + lane]) * 16777619u;
    h = __reduce_add_sync(0xffffffffu, h * (2u * lane + 1u)) + (unsigned int)ps.w2 * 0x9E3779B9u;
    h ^= h >> 15;
    h *= 0x2C1B3C6Du;
    h ^= h >> 13;
    unsigned int i = h & mask;
    for (unsigned int n = 0; n <= mask; ++n, i = (i + 1) & mask) {
        unsigned int t = 0;
        if (lane == 0) {
            t = *reinterpret_cast<volatile unsigned int *>(tab + i);
            if (t == PAT_SLOT_EMPTY) t = atomicCAS(tab + i, PAT_SLOT_EMPTY, (unsigned int)gw);
        }
        t = __shfl_sync(0xffffffffu, t, 0);
        if (t == PAT_SLOT_EMPTY) break;   // claimed
        // a slot's group never changes once claimed: compare with the slice that claimed it (or any member since)
        const PatSlice pt = pat_slice(poff + t);
        bool same = pt.w2 == ps.w2;
        if (same)
            for (int m = 0; m < ps.w2; ++m) same &= pc[pt.o0 + m * 32 + lane] == pc[ps.o0 + m * 32 + lane];
        if (__all_sync(0xffffffffu, same)) {
            if (lane == 0) atomicMin(tab + i, (unsigned int)gw);
            break;
        }
    }
    if (lane == 0) slot[gw] = (int)i;
}
// one thread per slice: slot -> representative; off[s] = words the slice stores (its own copy or none), stats[0] += stored
static __global__ void pat_owner_kernel(int nslices, const int *__restrict__ poff, const unsigned int *__restrict__ tab,
                                        int *__restrict__ slot, int *__restrict__ off, int *__restrict__ stats) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= nslices) return;
    const int rep = slot[s] < 0 ? s : (int)tab[slot[s]];
    slot[s] = rep;
    const PatSlice ps = pat_slice(poff + s);
    off[s] = rep == s ? ps.w2 * (ps.wide ? 64 : 32) : 0;
    if (rep == s) atomicAdd(stats, 1);
}
// one warp per slice, after the scan of off[]: sharing pays (pat_share_on) -> copy the stored slices to scr at their new
// offsets; npoff[] = the new offsets (the old ones with sharing off)
static __global__ void pat_share_kernel(int nslices, const int *__restrict__ poff, const unsigned int *__restrict__ pc,
                                        const int *__restrict__ rep, const int *__restrict__ off, const int *__restrict__ stats,
                                        int *__restrict__ npoff, unsigned int *__restrict__ scr, long long cap_scr) {
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (gw >= nslices) return;
    const bool share = pat_share_on(nslices, stats[0], off[nslices], cap_scr);
    const PatSlice ps = pat_slice(poff + gw);
    const int r = rep[gw];
    if (share && r == gw) {
        const int nw = ps.w2 * (ps.wide ? 64 : 32);
        for (int j = lane; j < nw; j += 32) scr[off[gw] + j] = pc[ps.o0 + j];
    }
    if (lane == 0) {
        npoff[gw] = (share ? off[r] : ps.o0) | (poff[gw] & 31);
        if (gw == nslices - 1) npoff[nslices] = share ? off[nslices] : poff[nslices];
    }
}
// grid-stride: poff[] = npoff[], and with sharing on the stored slices back to the front of pc
static __global__ void pat_share_copy_kernel(int nslices, int *__restrict__ poff, unsigned int *__restrict__ pc,
                                             const int *__restrict__ npoff, const unsigned int *__restrict__ scr,
                                             const int *__restrict__ off, const int *__restrict__ stats, long long cap_scr) {
    const bool share = pat_share_on(nslices, stats[0], off[nslices], cap_scr);
    const long long n = share ? max((long long)off[nslices], (long long)nslices + 1) : (long long)nslices + 1;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        if (i <= nslices) poff[i] = npoff[i];
        if (share && i < off[nslices]) pc[i] = scr[i];
    }
}

}  // namespace lsk

namespace {

// SELL-32 copy of the solver's CSR (the fast SpMM engine's and the fused solver's), and its stand-alone kernel's grid.  Whether
// it is used depends on its padded size, which the readback brings.
int sell_copy(PcgHandle *h, cudaStream_t stream) {
    const unsigned wb = (unsigned)(((int64_t)h->nslices * 32 + 255) / 256);
    lsk::sell_width_kernel<<<wb, 256, 0, stream>>>((int)h->V, h->nslices, h->rowptr, h->soff);
    LS_LAUNCH_CHECK();
    const int rc = ls_exclusive_scan_i32(h->soff, h->soff, h->nslices, h->scan, stream);
    if (rc) return rc;
    lsk::sell_fill_kernel<<<wb, 256, 0, stream>>>((int)h->V, h->nslices, h->rowptr, h->col, h->val, h->soff, h->ent, h->sell_cap);
    LS_LAUNCH_CHECK();
    int socc = 0;
    LS_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&socc, lsk::spmm_sell_kernel<3, true>, lsk::SELL_THREADS, 0));
    if (socc < 1) socc = 1;
    int64_t sg = ((int64_t)h->nslices + lsk::SELL_WARPS - 1) / lsk::SELL_WARPS;   // >= one slice per warp
    if (sg > (int64_t)h->sm_count * socc) sg = (int64_t)h->sm_count * socc;
    if (sg > GRID_CAP) sg = GRID_CAP;
    if (sg < 1) sg = 1;
    h->sell_grid = (int)sg;
    return LS_OK;
}

// What create needs from the device, brought back in one round trip
struct Readback {
    int flags[2];          // the CSR checks' bits (k_dinv, the permuted copy); the block plan's overflow
    unsigned int mm[2];    // [min, max] of the off-diagonal value bits (equal: a pattern-only matrix)
    float gersh;           // Gershgorin bound of lambda_max(D^-1 A) (precond 2 only)
};

// The one shared readback; it decides the engine: SELL-32 unless its padding blew past the buffer (very long rows) or
// LS_SPMM_ENGINE=csr.
int read_back(PcgHandle *h, const CreateEnv &ce, Readback &rb, cudaStream_t stream) {
    const unsigned gv = (unsigned)((h->V + 255) / 256);
    rb = {{0, 0}, {0xffffffffu, 0u}, 0.f};
    if (ce.pattern) {
        LS_CUDA_TRY(cudaMemsetAsync(h->patmm, 0xff, 4, stream));
        LS_CUDA_TRY(cudaMemsetAsync(h->patmm + 1, 0, 4, stream));
        lsk::pat_detect_kernel<<<gv, 256, 0, stream>>>((int)h->V, h->rowptr, h->col, h->val, h->patmm);
        LS_LAUNCH_CHECK();
        LS_CUDA_TRY(cudaMemcpyAsync(rb.mm, h->patmm, sizeof(rb.mm), cudaMemcpyDeviceToHost, stream));
    }
    if (h->precond == 2) {
        LS_CUDA_TRY(cudaMemsetAsync(h->gersh, 0, 64, stream));
        k_gershgorin<<<gv, 256, 0, stream>>>(h->V, h->rowptr, h->col, h->val, h->gersh);
        LS_LAUNCH_CHECK();
        LS_CUDA_TRY(cudaMemcpyAsync(&rb.gersh, h->gersh, sizeof(float), cudaMemcpyDeviceToHost, stream));
    }
    int sell_total = 0;
    LS_CUDA_TRY(cudaMemcpyAsync(rb.flags, h->flags, sizeof(rb.flags), cudaMemcpyDeviceToHost, stream));
    LS_CUDA_TRY(cudaMemcpyAsync(&sell_total, h->soff + h->nslices, sizeof(int), cudaMemcpyDeviceToHost, stream));
    LS_CUDA_TRY(cudaStreamSynchronize(stream));
    h->planned = (rb.flags[1] == 0) ? 1 : 0;
    h->sell_entries = sell_total;
    h->sell_on = (!ce.csr && sell_total > 0 && (long long)sell_total <= h->sell_cap) ? 1 : 0;
    return LS_OK;
}

// Pattern-only copy of a matrix whose off-diagonal entries all carry the value with bits `offc_bits`: the column-only copy (its
// padded size is bounded by the general SELL copy's, which fits) and the diagonal classes, with identical compact slices
// stored once unless `share` is 0.  One host round trip tells whether the classes fit the table and what sharing saved.
int build_pattern_copy(PcgHandle *h, unsigned int offc_bits, int share, cudaStream_t stream) {
    memcpy(&h->offc, &offc_bits, 4);
    const int ns = h->nslices;
    const unsigned wb = (unsigned)(((int64_t)ns * 32 + 255) / 256);
    int *over = reinterpret_cast<int *>(h->pcls_tab + lsk::PAT_CLASSES);
    LS_CUDA_TRY(cudaMemsetAsync(h->pcls_tab, 0xff, (size_t)lsk::PAT_CLASSES * 8, stream));
    LS_CUDA_TRY(cudaMemsetAsync(over, 0, sizeof(int), stream));
    lsk::pat_width_kernel<<<wb, 256, 0, stream>>>((int)h->V, ns, h->rowptr, h->col, h->poff);
    LS_LAUNCH_CHECK();
    int rc = ls_exclusive_scan_i32(h->poff, h->poff, ns, h->scan, stream);
    if (rc) return rc;
    lsk::pat_fill_kernel<<<wb, 256, 0, stream>>>((int)h->V, ns, h->rowptr, h->col, h->val, h->dinv, h->poff, h->pcol, h->pat_cap,
                                                  h->offc, h->pcls, h->pcls_tab, over);
    LS_LAUNCH_CHECK();
    // Sharing borrows the solve's r planes (ints) and p rows (words) as scratch.  The graph-mode solver relies on their padding
    // rows being zero, so both are cleared again below.
    const long long cap_scr = share ? h->Vp * 4 : 0;
    int *slot = reinterpret_cast<int *>(h->r), *soff2 = slot + ns, *npoff = soff2 + ns + 1, *stats = npoff + ns + 1;
    unsigned int *ptab = reinterpret_cast<unsigned int *>(stats + 2);
    unsigned int pmask = 1;
    while (pmask + 1 < 2u * (unsigned)ns) pmask = 2 * pmask + 1;
    if (share) {
        LS_CUDA_TRY(cudaMemsetAsync(stats, 0, 2 * sizeof(int), stream));
        LS_CUDA_TRY(cudaMemsetAsync(ptab, 0xff, (size_t)(pmask + 1) * 4, stream));
        lsk::pat_hash_kernel<<<wb, 256, 0, stream>>>(ns, h->poff, h->pcol, ptab, pmask, slot);
        LS_LAUNCH_CHECK();
        lsk::pat_owner_kernel<<<(unsigned)((ns + 255) / 256), 256, 0, stream>>>(ns, h->poff, ptab, slot, soff2, stats);
        LS_LAUNCH_CHECK();
        rc = ls_exclusive_scan_i32(soff2, soff2, ns, h->scan, stream);
        if (rc) return rc;
        lsk::pat_share_kernel<<<wb, 256, 0, stream>>>(ns, h->poff, h->pcol, slot, soff2, stats, npoff,
                                                      reinterpret_cast<unsigned int *>(h->p), cap_scr);
        LS_LAUNCH_CHECK();
        lsk::pat_share_copy_kernel<<<2 * h->sm_count, 256, 0, stream>>>(ns, h->poff, h->pcol, npoff,
                                                                         reinterpret_cast<const unsigned int *>(h->p), soff2, stats, cap_scr);
        LS_LAUNCH_CHECK();
    }
    int hover = 1, hst[2] = {ns, 0}, hwords = 0;
    LS_CUDA_TRY(cudaMemcpyAsync(&hover, over, sizeof(int), cudaMemcpyDeviceToHost, stream));
    if (share) {
        LS_CUDA_TRY(cudaMemcpyAsync(hst, stats, sizeof(int), cudaMemcpyDeviceToHost, stream));
        LS_CUDA_TRY(cudaMemcpyAsync(&hst[1], soff2 + ns, sizeof(int), cudaMemcpyDeviceToHost, stream));
    }
    LS_CUDA_TRY(cudaMemcpyAsync(&hwords, h->poff + ns, sizeof(int), cudaMemcpyDeviceToHost, stream));
    LS_CUDA_TRY(cudaStreamSynchronize(stream));
    const bool shared = share && lsk::pat_share_on(ns, hst[0], hst[1], cap_scr);
    h->pat_on = hover ? 0 : 1;
    h->pat_shared = (h->pat_on && shared) ? 1 : 0;
    h->pat_stored = h->pat_shared ? hst[0] : ns;
    h->pat_words = hwords;
    if (share) {
        LS_CUDA_TRY(cudaMemsetAsync(h->r, 0, (size_t)((char *)(ptab + pmask + 1) - (char *)h->r), stream));
        if (shared) LS_CUDA_TRY(cudaMemsetAsync(h->p, 0, (size_t)hst[1] * 4, stream));
    }
    return LS_OK;
}

// Chebyshev semi-iteration for D^-1 A on [b/30, b], b = 1.02 x the Gershgorin bound: theta, delta, sigma = theta/delta,
// rho_0 = 1/sigma;  d_0 = g/theta;  rho_j = 1/(2 sigma - rho_{j-1});  d_j = rho_j rho_{j-1} d_{j-1} + 2 rho_j/delta (g - B y_j)
void chebyshev_coefficients(float gersh, int m, float &c0, float (&c1)[8], float (&c2)[8]) {
    const double b = 1.02 * (double)gersh, a = b / 30.0;
    const double th = 0.5 * (b + a), de = 0.5 * (b - a), sg = th / de;
    double rho = 1.0 / sg;
    c0 = (float)(1.0 / th);
    for (int j = 1; j < m; ++j) {
        const double rn = 1.0 / (2.0 * sg - rho);
        c1[j - 1] = (float)(rn * rho);
        c2[j - 1] = (float)(2.0 * rn / de);
        rho = rn;
    }
}

// The CSR checks' flag bits -> error code and message, the most fundamental first
int flag_error(int flags) {
    if (flags & 8) {
        ls_set_error("perm_new2old is not a permutation of [0, V)");
        return LS_ERR_BAD_ARG;
    }
    if (flags & (1 | 4)) {
        ls_set_error("CSR is malformed (column index out of range or decreasing rowptr)");
        return LS_ERR_INDEX_RANGE;
    }
    if (flags & 2) {
        ls_set_error("matrix has a missing or non-positive diagonal entry: not SPD");
        return LS_ERR_BREAKDOWN;
    }
    return LS_OK;
}

// Everything ls_pcg_create does once the handle is carved.  Host round trips: at most two in copy_matrix, one in read_back and one
// in build_pattern_copy.  Flag errors are reported last, after the fused solver is configured.
int build_solver(PcgHandle *h, const int *rowptr, const int *col, const float *val, const int *perm, const LsDevInfo &di,
                 cudaStream_t stream) {
    const PlanEnv env = plan_env();
    const CreateEnv ce = create_env();
    h->refine = ce.refine;
    h->sell_tma = ce.sell_tma;
    h->sell_pf = ce.sell_pf;
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
    switch (k) {
        case 1: return solve_k<1>(h, b, x, x0, rtol, maxit, info_dev, info_host, stream);
        case 2: return solve_k<2>(h, b, x, x0, rtol, maxit, info_dev, info_host, stream);
        case 3: return solve_k<3>(h, b, x, x0, rtol, maxit, info_dev, info_host, stream);
        default: return solve_k<4>(h, b, x, x0, rtol, maxit, info_dev, info_host, stream);
    }
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
    for (int k = 0; k <= KMAX; ++k)
        if (h->graph[k]) cudaGraphExecDestroy(h->graph[k]);
    if (h->ev[0]) cudaEventDestroy(h->ev[0]);
    if (h->ev[1]) cudaEventDestroy(h->ev[1]);
    if (h->cap_stream) cudaStreamDestroy(h->cap_stream);
    if (h->pinned_done) cudaFreeHost(h->pinned_done);
    delete h;
    return LS_OK;
}

extern "C" int ls_pcg_bench_spmm(void *handle, int k, int launches, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    PcgHandle *h = (PcgHandle *)handle;
    LS_REQUIRE(h != nullptr, "handle is NULL");
    LS_REQUIRE(k >= 1 && k <= h->k_max, "k out of range for this handle");
    int occ;
    int rc = lsk::spmm_prepare(k, true, h->cfg, &occ);
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

namespace {
template <int K>
int bench_one(PcgHandle *h, int which, cudaStream_t stream) {
    if (which == 4 && K == 3 && h->sell_on && h->sell_tma)   // pure y = A p, no dot-product epilogue (the SpMV of BASELINE's metric)
        return launch_sell_tma<3, false>(h, sell_args(h, false), stream);
    return launch_spmm<K>(h, false, stream);
}
}  // namespace

extern "C" int ls_pcg_bench(void **handles, int n_handles, int k, int which, int launches, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    LS_REQUIRE(handles != nullptr && n_handles >= 1, "no handles");
    LS_REQUIRE(which == 0 || which == 4, "which: 0 SpMM+dot, 4 SpMM without the dot epilogue");
    for (int i = 0; i < n_handles; ++i) {
        PcgHandle *h = (PcgHandle *)handles[i];
        LS_REQUIRE(h != nullptr, "NULL handle");
        LS_REQUIRE(k >= 1 && k <= h->k_max, "k out of range for this handle");
        int occ;
        int rc = lsk::spmm_prepare(k, true, h->cfg, &occ);
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

// ---- stand-alone SpMM input / output (diagnostics: the tests read what ls_pcg_bench / ls_pcg_bench_spmm compute) ----------
namespace {
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
    out8[2] = h->sell_on ? h->sell_grid : h->spmm_grid;
    out8[3] = h->vec_grid;
    out8[4] = 0;                          // mode: graph of 3 kernels (1 and 2 are retired, 10 + RES is the fused solver)
    out8[5] = 0;
    out8[6] = h->planned;
    out8[7] = h->has_perm;
    return LS_OK;
}

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

extern "C" int ls_pcg_pattern_copy(void *handle, int64_t *info4, int32_t *poff, uint32_t *words, void *stream_) {
    PcgHandle *h = (PcgHandle *)handle;
    LS_REQUIRE(h != nullptr && info4 != nullptr, "NULL pointer");
    info4[0] = h->pat_on;
    info4[1] = h->nslices;
    info4[2] = h->pat_on ? h->pat_stored : 0;
    info4[3] = h->pat_on ? h->pat_words : 0;
    if (h->pat_on && poff != nullptr && words != nullptr) {
        cudaStream_t stream = (cudaStream_t)stream_;
        LS_CUDA_TRY(cudaMemcpyAsync(poff, h->poff, (size_t)(h->nslices + 1) * 4, cudaMemcpyDeviceToHost, stream));
        LS_CUDA_TRY(cudaMemcpyAsync(words, h->pcol, (size_t)h->pat_words * 4, cudaMemcpyDeviceToHost, stream));
        LS_CUDA_TRY(cudaStreamSynchronize(stream));
    }
    return LS_OK;
}

extern "C" int64_t ls_pcg_spmm_bytes(void *handle, int k) {
    PcgHandle *h = (PcgHandle *)handle;
    if (!h) return 0;
    return 8 * h->nnz + 4 * (h->V + 1) + 8 * (int64_t)k * h->V;
}

// ---- batches: many independent meshes per launch, one thread-block cluster per mesh (ls_pcg_fused.cuh, BATCH) -----------
namespace {
constexpr int BATCH_CS_MAX = 16;

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

extern "C" int ls_pcg_batch_plan(int n, const int32_t *nslices, const int32_t *pat, int max_smem, int32_t *cluster,
                                 int32_t *res, int32_t *group, int32_t *n_groups) {
    return ls_pcg_batch_plan_ex(n, nslices, pat, nullptr, max_smem, cluster, res, group, n_groups);
}

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
    if (!info_host) return LS_OK;
    LS_CUDA_TRY(cudaMemcpyAsync(info_host, info, 8 * sizeof(float) * (size_t)B->n, cudaMemcpyDefault, stream));
    LS_CUDA_TRY(cudaStreamSynchronize(stream));
    for (int i = 0; i < B->n; ++i) {
        if ((int)info_host[8 * i + 1] == 3) {
            ls_set_error("mesh %d: CG breakdown after %d iterations (matrix not SPD or NaN in the right-hand side)", i, (int)info_host[8 * i]);
            return LS_ERR_BREAKDOWN;
        }
    }
    for (int i = 0; i < B->n; ++i) {
        const float *r = info_host + 8 * i;
        if ((int)r[1] == 2) {
            ls_set_error("mesh %d: PCG did not reach rtol=%g within maxit=%d (relres %g %g %g)", i, (double)rtol, maxit,
                         (double)r[2], (double)r[3], (double)r[4]);
            return LS_ERR_NOT_CONVERGED;
        }
    }
    return LS_OK;
}

extern "C" int ls_pcg_batch_destroy(void *batch) {
    batch_free((PcgBatch *)batch);
    return LS_OK;
}
