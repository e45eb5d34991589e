// ls_pcg_persistent.cuh -- the whole Jacobi-PCG solve as ONE persistent cooperative kernel (sm_90a).
//
// Why: at V = 1e6 every kernel boundary of the 3-kernel iteration costs microseconds of launch latency, ramp and drain,
// and r / Ap make a round trip through HBM between kernels although only their owner thread ever touches them.
//
// Structure: one CTA of 768 threads per SM (256 when a CTA owns <= 16 slices), launched cooperatively so that all CTAs
// are co-resident.  CTA c owns a contiguous range of SELL-32 slices; warp w of the CTA owns slices s_begin + w + NW i,
// lane l the row 32 s + l -- the SAME thread in every phase.  Per iteration:
//   phase A   Ap = A p for the owned rows (SELL entries streamed from HBM with register prefetch, p rows gathered
//             through L1), p.Ap partial                                      -> grid all-reduce #1  (alpha)
//   phase B   r -= alpha Ap (shared memory only), r.D^-1 r and r.r partials    -> grid all-reduce #2  (beta, convergence)
//   phase C   x += alpha p (owner-only, global), p = D^-1 r + beta p (p is the only vector other CTAs read)
//                                                                           -> grid barrier   #3  (p visible)
// r, Ap and D^-1 live in SHARED MEMORY for the whole solve when the CTA's rows fit (RES = 1: 28 B/row, 6784 rows/SM at
// V = 1e6 = 190 KB of the 227 KB); otherwise (RES = 0) they stay in global memory.
// The two all-reduces are one 64-bit fixed-point atomic per value (fast_allreduce below): integer sums do not depend on
// the arrival order, so the scalars are bit-identical on every CTA and run to run, and all CTAs take the same
// convergence decision without another exchange.  The fallback (grid_allreduce: per-CTA partials, a fenced barrier, a
// fixed-order re-reduction) has the same property and is used at start-up and whenever a partial does not fit the
// fixed-point window.  The grid barrier is a monotone arrival counter (release add / acquire poll).
#pragma once
#include <type_traits>
#include "ls_common.cuh"
#include "ls_sell_kernel.cuh"

namespace lsp {

#ifndef LS_PT
#define LS_PT 768
#endif
constexpr int PT = LS_PT;   // 24 warps: 85 registers per thread (1024 threads forced spills into the SpMM loop)
constexpr int PWARPS = PT / 32;
constexpr int PT_SMALL = 256;   // CTAs that own <= 16 slices (mid-size meshes): cheaper CTA barriers, no spills
constexpr int NVMAX = 16;   // values per all-reduce (the fused kernel reduces 4 K <= 16 at a restart)

struct GridBar {
    unsigned int count;
    unsigned int gen;
};

struct PersistArgs {
    int V;
    long long Vp;
    int nslices;
    int nsl_max;            // max slices per CTA (shared-memory sizing)
    const int *soff;
    const int2 *ent;
    const float *dinv;
    float *x;               // K planes of Vp
    float *r;               // K planes of Vp   (RES = 0 only)
    float *Ap;              // K planes of Vp   (RES = 0 only)
    float *p;               // rows of 4 floats
    const float *b;         // (V,K) caller layout
    float *out;             // (V,K) caller layout
    const int *perm;        // new -> old row, or NULL
    float rtol;
    int maxit;
    GridBar *bar;
    double *partials;       // [2][NVMAX][gridDim.x]
    // resume mode (warm start): x, r (planes) and p (rows) were initialised by the graph-mode kernels; scalars come from here
    const double *resume_rz, *resume_rr, *resume_bb;   // [4] each, or NULL for a cold start
    const int *resume_conv, *resume_done;
    unsigned long long *ring;   // fast all-reduce slots, 8 words each, zeroed by the host before the launch
    int ring_slots;
    float *info;            // 8 floats
    long long *dbg;         // optional [8] cycle counters of CTA 0: A, reduce1, B, reduce2, C, barrier3, init, iterations
};

__device__ __forceinline__ unsigned int ld_acquire(const unsigned int *p) {
    unsigned int v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ float4 ld_coherent4(const float *p) {   // plain (coherent after a fence), never the .nc path
    float4 v;
    asm volatile("ld.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
    return v;
}

// Grid barrier on a monotonically increasing arrival counter (reset to 0 by the host before every launch):
// barrier number n (1-based) is complete when count >= n * G.  It is split into arrive and wait so that loads which
// do not depend on other CTAs (the next phase's matrix entries, the owner's own vector rows) are issued in between and
// their latency overlaps the barrier's (store drain + atomic round trip + poll).
// One thread per CTA arrives / polls; the CTA barrier publishes the result to the rest of the CTA (the pattern
// cooperative-groups grid.sync uses), so ordinary loads after it see every other CTA's earlier writes.
__device__ __forceinline__ void grid_arrive(GridBar *gb, unsigned int &gen, int G = 2) {
    __syncthreads();
    gen += 1u;
    if (G == 1) return;            // single-CTA solve: the CTA barrier is the grid barrier
    if (threadIdx.x == 0) {
        // release: every write this CTA made before the CTA barrier above is visible to whoever acquires the counter.
        // (a plain __threadfence() here is a sequentially-consistent fence plus an L1 invalidate the arriving side has no use for)
        asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(&gb->count), "r"(1u) : "memory");
    }
}
__device__ __forceinline__ void grid_wait(GridBar *gb, unsigned int gen, int G) {
    if (G == 1) return;
    if (threadIdx.x == 0) {
        const unsigned int target = gen * (unsigned int)G;
        // the acquire load pairs with the release above and invalidates this SM's L1 (CCTL.IVALL), so the plain loads the
        // other threads issue after the CTA barrier below miss L1 and read the other CTAs' rows from L2
        while ((int)(ld_acquire(&gb->count) - target) < 0) {
        }
    }
    __syncthreads();
}
__device__ __forceinline__ void grid_barrier(GridBar *gb, unsigned int &gen, int G) {
    grid_arrive(gb, gen, G);
    grid_wait(gb, gen, G);
}

// deterministic all-reduce of NV doubles per thread across the whole grid, in two halves around one grid barrier
template <int NV>
__device__ __forceinline__ void allreduce_arrive(double (&v)[NV], double *partials, GridBar *gb, unsigned int &gen,
                                                 unsigned int parity, double *red /* >= NV*32 + NV doubles */, int G) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const double s = ls_warp_sum(v[i]);
        if (lane == 0) red[i * 32 + warp] = s;
    }
    __syncthreads();
    double *mine = partials + (size_t)parity * NVMAX * G;
    if (warp == 0) {
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const double s = ls_warp_sum(lane < (int)(blockDim.x >> 5) ? red[i * 32 + lane] : 0.0);
            if (lane == 0) mine[(size_t)i * G + blockIdx.x] = s;
        }
    }
    grid_arrive(gb, gen, G);
}
template <int NV>
__device__ __forceinline__ void allreduce_finish(double (&v)[NV], double *partials, GridBar *gb, unsigned int gen,
                                                 unsigned int &parity, double *red, int G) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    grid_wait(gb, gen, G);
    const double *mine = partials + (size_t)parity * NVMAX * G;
    for (int i = warp; i < NV; i += (int)(blockDim.x >> 5)) {
        const double *src = mine + (size_t)i * G;
        double s = 0.0;
        for (int c0 = 0; c0 < G; c0 += 256) {
            double t[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int c = c0 + j * 32 + lane;
                t[j] = (c < G) ? __ldcg(src + c) : 0.0;
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) s += t[j];
        }
        s = ls_warp_sum(s);
        if (lane == 0) red[NV * 32 + i] = s;
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < NV; ++i) v[i] = red[NV * 32 + i];
    parity ^= 1u;
    __syncthreads();   // red[] is reused by the next reduction
}
template <int NV>
__device__ __forceinline__ void grid_allreduce(double (&v)[NV], double *partials, GridBar *gb, unsigned int &gen,
                                               unsigned int &parity, double *red, int G) {
    allreduce_arrive<NV>(v, partials, gb, gen, parity, red, G);
    allreduce_finish<NV>(v, partials, gb, gen, parity, red, G);
}

struct Scal {                 // CTA-uniform solver scalars, kept in shared memory (identical on every CTA)
    double rz[4], bb[4], rr[4];
    float alpha[4], beta[4];
    int conv[4];
    int it, status, stop;
    int e_pAp[4];              // exponent references for the fixed-point all-reduce
    int e_rzrr[8];             // [rz | rr]
    int skipA[4], skipB[8];    // frozen columns contribute nothing
    int nslot;
    int poison;
};

// ---- fast deterministic all-reduce: one 64-bit atomic per value, no fences, no second pass ------------------------------
// The slow all-reduce above is a chain of ~6 dependent L2 round trips (partial store -> fence -> arrive -> poll -> fence ->
// re-read), a large share of an iteration.  Integer addition is associative, so a fixed-point sum is
// deterministic no matter in which order the CTAs' atomics land.  Word layout:  [63:16] signed fixed-point sum,
// [15:8] number of CTAs whose partial did not fit ("poison"), [7:0] arrival count.  The scale of value i is taken from
// the exponent `eref[i]` of the same quantity one iteration earlier (identical on every CTA): a partial must be finite and
// below 2^(eref+3); 2^-35 relative resolution, far below the fp32 noise of the dot products themselves.  The CTA that adds
// and the CTAs that poll touch only that word, so nothing needs a fence: r, Ap and x are owner-only, and the only vector
// other CTAs read (p) is published by the full barrier after phase C.  If any CTA poisons a value, every CTA sees the same
// poison count and the whole grid repeats that reduction through the slow path.
// binary exponent of a positive double straight from its bits (ilogb() is a function call); denormals / inf land outside
// +-900 and are clamped by the user
__device__ __forceinline__ int exp2_of(double d) { return (int)((__double_as_longlong(d) >> 52) & 0x7ff) - 1023; }

// value `off + lane` of a register array without turning the array into an indexed (local-memory) one
template <int KCOL, int N>
__device__ __forceinline__ double pick_lane(const double (&v)[N], int off, int lane) {
    double d = 0.0;
#pragma unroll
    for (int i = 0; i < KCOL; ++i) {
        double t = v[off + i];
        asm volatile("" : "+d"(t));
        if (lane == i) d = t;
    }
    return d;
}

template <int NV, int KCOL, typename Post>
__device__ __forceinline__ bool fast_allreduce(double (&v)[NV], const int *eref /* smem [NV] */, const int *skip /* smem [NV] */,
                                               unsigned long long *slot, double *red, int *poison_flag /* smem */, int G, Post post) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const double s = ls_warp_sum(v[i]);
        if (lane == 0) red[i * 32 + warp] = s;
    }
    __syncthreads();
    if (warp == 0) {
        double val = 0.0;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const double s = ls_warp_sum(lane < (int)(blockDim.x >> 5) ? red[i * 32 + lane] : 0.0);
            if (lane == i) val = s;
        }
        unsigned int pois = 0u;
        if (G > 1 && lane < NV) {
            // powers of two built from their bit patterns (ldexp() is a function call on the critical path); the exponent
            // reference is clamped so that 2^(35-e) and 2^(e-35) stay normal numbers (-1000 marks "previous value was 0")
            const int e = min(max(eref[lane], -900), 900);
            const double up = __longlong_as_double((long long)(1023 + 35 - e) << 52);     // 2^(35-e)
            const double down = __longlong_as_double((long long)(1023 + e - 35) << 52);   // 2^(e-35)
            unsigned long long word = 1ull;
            if (!skip[lane]) {
                const bool fits = (val == val) && (fabs(val) * up < 274877906944.0 /* 2^38 */);
                if (fits) word += ((unsigned long long)__double2ll_rn(val * up)) << 16;
                else word += 1ull << 8;
            }
            atomicAdd(slot + lane, word);
            unsigned long long w;
            do {
                asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(w) : "l"(slot + lane) : "memory");
            } while ((int)(w & 0xffull) != G);
            val = (double)((long long)w >> 16) * down;
            pois = (unsigned int)((w >> 8) & 0xffull);
        }
        // the scalar bookkeeping that follows every reduction runs right here, on the warp that already holds the sums
        // (one lane per column), instead of after another shared-memory round trip and two more CTA barriers
        const bool poison = __any_sync(0xffffffffu, pois != 0u);
        __syncwarp();   // lanes >= KCOL read eref[] / skip[] entries that post() rewrites from lanes < KCOL (racecheck)
        const double val2 = (NV > KCOL) ? __shfl_down_sync(0xffffffffu, val, KCOL) : 0.0;   // lane k: values k and KCOL + k
        if (!poison) post(val, val2);
        if (lane == 0) *poison_flag = poison ? 1 : 0;
    }
    __syncthreads();
    return *poison_flag == 0;
}

template <int K, int RES, bool PROF, int NW>
__global__ void __launch_bounds__(NW * 32, 1) pcg_persistent_kernel(const PersistArgs a) {
    static_assert(K == 3 || K == 4, "persistent kernel is instantiated for float4 p rows");
    constexpr int PWARPS = NW;   // warps per CTA: 24 for large meshes, 8 when a CTA owns only a handful of slices
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double *red = reinterpret_cast<double *>(smem_raw);                 // NV*32 + NV doubles (NV <= 8)
    Scal *S = reinterpret_cast<Scal *>(smem_raw + 3072);
    float *fs = reinterpret_cast<float *>(smem_raw + 4096);
    const int nsl_max = a.nsl_max;
    float *r_s = fs;                                                    // [nsl_max][K][32]
    float *q_s = r_s + (size_t)nsl_max * K * 32;                        // Ap
    float *d_s = q_s + (size_t)nsl_max * K * 32;                        // dinv [nsl_max][32]

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int G = gridDim.x, cta = blockIdx.x;
    const int s_begin = (int)((long long)a.nslices * cta / G);
    const int s_end = (int)((long long)a.nslices * (cta + 1) / G);
    const long long Vp = a.Vp;
    constexpr int U = 8;   // matrix entries a lane holds in registers (8 gathers in flight)
#ifndef LS_UBC
#define LS_UBC 1   // A/B: larger values keep more loads in flight but spill at 4
#endif
    constexpr int UBC = LS_UBC;    // owned slices whose global loads are in flight together in phase C
#ifndef LS_PREFC
#define LS_PREFC 0   // A/B: the live registers across the reduction cost more (spills) than the overlap gains
#endif
    constexpr bool PREFC = (LS_PREFC != 0);   // prefetch phase C's first batch across all-reduce 2

    unsigned int gen = 0, parity = 0;   // gen = number of grid barriers passed (the host zeroes the counter per launch)
    const long long ent_limit = a.soff[a.nslices];

    auto R = [&](int li, int k, int row) -> float & {
        return RES ? r_s[((size_t)li * K + k) * 32 + lane] : a.r[(size_t)k * Vp + row];
    };
    auto Q = [&](int li, int k, int row) -> float & {
        return RES ? q_s[((size_t)li * K + k) * 32 + lane] : a.Ap[(size_t)k * Vp + row];
    };
    long long tA = 0, tR1 = 0, tB = 0, tR2 = 0, tC = 0, tB3 = 0, t0 = 0;
    const bool prof = PROF && (a.dbg != nullptr) && tid == 0;   // every CTA's thread 0 (per-CTA skew table)

    // ------------------------------------------------------------------ resume (warm start): state is in global memory
    if (a.resume_rz != nullptr) {
        for (int s = s_begin + warp; s < s_end; s += PWARPS) {
            const int li = s - s_begin, row = s * 32 + lane;
            if (RES) {
                d_s[(size_t)li * 32 + lane] = a.dinv[row];
#pragma unroll
                for (int k = 0; k < K; ++k) r_s[((size_t)li * K + k) * 32 + lane] = a.r[(size_t)k * Vp + row];
            }
        }
        if (tid == 0) {
            int all = 1;
            for (int k = 0; k < K; ++k) {
                const double rz = a.resume_rz[k], rr = a.resume_rr[k], bb = a.resume_bb[k];
                S->rz[k] = rz;
                S->rr[k] = rr;
                S->bb[k] = bb;
                S->conv[k] = a.resume_conv[k];
                all &= S->conv[k];
                const int erz = (rz > 0.0 && rz == rz) ? ilogb(rz) : -1000;
                const int err = (rr > 0.0 && rr == rr) ? ilogb(rr) : -1000;
                S->e_pAp[k] = erz + 1;
                S->e_rzrr[k] = erz;
                S->e_rzrr[K + k] = err;
                S->skipA[k] = S->conv[k];
                S->skipB[k] = S->skipB[K + k] = S->conv[k];
            }
            S->nslot = 0;
            S->it = 0;
            S->status = (all || *a.resume_done == 1) ? 1 : (a.maxit <= 0 ? 2 : 0);
            S->stop = S->status != 0;
        }
        __syncthreads();
    } else
    // ------------------------------------------------------------------ init: x = 0, r = b, p = z = D^-1 r
    {
        double acc2[2 * K];
#pragma unroll
        for (int i = 0; i < 2 * K; ++i) acc2[i] = 0.0;
        for (int s = s_begin + warp; s < s_end; s += PWARPS) {
            const int li = s - s_begin, row = s * 32 + lane;
            float di = 0.f, bv[K];
#pragma unroll
            for (int k = 0; k < K; ++k) bv[k] = 0.f;
            if (row < a.V) {
                di = a.dinv[row];
                const long long io = a.perm ? a.perm[row] : row;
#pragma unroll
                for (int k = 0; k < K; ++k) bv[k] = a.b[io * K + k];
            }
            if (RES) d_s[(size_t)li * 32 + lane] = di;
            float z[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int k = 0; k < K; ++k) {
                z[k] = di * bv[k];
                R(li, k, row) = bv[k];
                a.x[(size_t)k * Vp + row] = 0.f;
                acc2[k] += (double)bv[k] * (double)z[k];
                acc2[K + k] += (double)bv[k] * (double)bv[k];
            }
            *reinterpret_cast<float4 *>(a.p + 4 * (size_t)row) = make_float4(z[0], z[1], z[2], z[3]);
        }
        grid_allreduce<2 * K>(acc2, a.partials, a.bar, gen, parity, red, G);
        if (tid == 0) {
            const double rtol2 = (double)a.rtol * (double)a.rtol;
            int all = 1;
            for (int k = 0; k < K; ++k) {
                S->rz[k] = acc2[k];
                S->bb[k] = acc2[K + k];
                S->rr[k] = acc2[K + k];
                S->conv[k] = acc2[K + k] <= rtol2 * acc2[K + k];   // only an all-zero column is converged at entry
                all &= S->conv[k];
            }
            for (int k = 0; k < K; ++k) {
                const int erz = (acc2[k] > 0.0 && acc2[k] == acc2[k]) ? ilogb(acc2[k]) : -1000;
                const int ebb = (acc2[K + k] > 0.0 && acc2[K + k] == acc2[K + k]) ? ilogb(acc2[K + k]) : -1000;
                S->e_pAp[k] = erz + 1;          // p = z at entry and lambda_max(D^-1 M) <= 2 for these matrices
                S->e_rzrr[k] = erz;
                S->e_rzrr[K + k] = ebb;
                S->skipA[k] = S->conv[k];
                S->skipB[k] = S->skipB[K + k] = S->conv[k];
            }
            S->nslot = 0;
            S->it = 0;
            S->status = all ? 1 : (a.maxit <= 0 ? 2 : 0);
            S->stop = S->status != 0;
        }
        __syncthreads();
    }

    // the matrix never changes: the entries of this warp's first slice are (re)loaded BEFORE waiting on the barrier
    // that ends the previous iteration, so their HBM latency hides under the barrier
    int o0 = 0, o1 = 0;
    int2 nv[U];
    auto prologue = [&]() {
        const int s = s_begin + warp;
        if (s < s_end) {
            o0 = a.soff[s];
            o1 = a.soff[s + 1];
            const int w = (o1 - o0) >> 5;
            const int2 *e = a.ent + o0 + lane;
#pragma unroll
            for (int u = 0; u < U; ++u) nv[u] = (u < w) ? lsk::ld_entry(e + u * 32) : make_int2(s * 32 + lane, 0);
        }
    };
    prologue();

    // ------------------------------------------------------------------ iterations
    while (!S->stop) {
        // ---------------- phase A: Ap = A p (owned rows), p.Ap
        if (prof) t0 = clock64();
        {
            double dacc[K];
#pragma unroll
            for (int k = 0; k < K; ++k) dacc[k] = 0.0;
            {
                int s = s_begin + warp;
                while (s < s_end) {
                    const int li = s - s_begin, row = s * 32 + lane;
                    const int w = (o1 - o0) >> 5;
                    const int2 *e = a.ent + o0 + lane;
                    int2 cv[U];
    #pragma unroll
                    for (int u = 0; u < U; ++u) cv[u] = nv[u];
                    const int sn = s + PWARPS;
                    int n0 = 0, n1 = 0;
                    if (sn < s_end) {
                        n0 = a.soff[sn];
                        n1 = a.soff[sn + 1];
                        if (sn + PWARPS < s_end) lsk::prefetch_entries_l2(a.ent, (long long)n0 + (n0 - o0), ent_limit, lane);
                    }
                    float acc[K];
    #pragma unroll
                    for (int k = 0; k < K; ++k) acc[k] = 0.f;
                    float4 po = make_float4(0.f, 0.f, 0.f, 0.f);   // own row of p: it is one of the gathered rows (diagonal entry)
                    {
                        float4 xv[U];
    #pragma unroll
                        for (int u = 0; u < U; ++u) xv[u] = ld_coherent4(a.p + 4 * (size_t)cv[u].x);
                        if (sn < s_end) {
                            const int wn = (n1 - n0) >> 5;
                            const int2 *en = a.ent + n0 + lane;
    #pragma unroll
                            for (int u = 0; u < U; ++u)
                                nv[u] = (u < wn) ? lsk::ld_entry(en + u * 32) : make_int2(sn * 32 + lane, 0);
                        }
    #pragma unroll
                        for (int u = 0; u < U; ++u) {
                            const float wv = __int_as_float(cv[u].y);
                            const float xk[4] = {xv[u].x, xv[u].y, xv[u].z, xv[u].w};
                            if (cv[u].x == row) po = xv[u];
    #pragma unroll
                            for (int k = 0; k < K; ++k) acc[k] = fmaf(wv, xk[k], acc[k]);
                        }
                    }
                    for (int j = U; j < w; j += U) {
    #pragma unroll
                        for (int u = 0; u < U; ++u) cv[u] = (j + u < w) ? lsk::ld_entry(e + (j + u) * 32) : make_int2(row, 0);
                        float4 xv[U];
    #pragma unroll
                        for (int u = 0; u < U; ++u) xv[u] = ld_coherent4(a.p + 4 * (size_t)cv[u].x);
    #pragma unroll
                        for (int u = 0; u < U; ++u) {
                            const float wv = __int_as_float(cv[u].y);
                            const float xk[4] = {xv[u].x, xv[u].y, xv[u].z, xv[u].w};
                            if (cv[u].x == row) po = xv[u];
    #pragma unroll
                            for (int k = 0; k < K; ++k) acc[k] = fmaf(wv, xk[k], acc[k]);
                        }
                    }
                    const float pk[4] = {po.x, po.y, po.z, po.w};
    #pragma unroll
                    for (int k = 0; k < K; ++k) {
                        Q(li, k, row) = acc[k];
                        dacc[k] += (double)pk[k] * (double)acc[k];
                    }
                    s = sn;
                    o0 = n0;
                    o1 = n1;
                }
            }
            if (prof) { const long long t1 = clock64(); tA += t1 - t0; t0 = t1; }
            {
                // alpha_k = rz_k / pAp_k, one lane per column (executed by warp 0 only, with the full sums in t[])
                auto postA = [&](const double d, const double) {
                    bool bad = false;
                    if (lane < K) {
                        const bool conv = S->conv[lane] != 0, ok = d > 0.0;
                        if (!conv && ok) S->e_pAp[lane] = exp2_of(d);
                        bad = !conv && !ok;      // not SPD / NaN: finish this iteration's update with alpha = 0, then stop
                        S->alpha[lane] = (conv || !ok) ? 0.f : (float)(S->rz[lane] / d);
                    }
                    const bool anybad = __any_sync(0xffffffffu, bad);
                    if (lane == 0) {
                        S->nslot += 1;
                        if (anybad) S->status = 3;
                    }
                };
                const int ns = S->nslot;
                bool ok = false;
                if (ns < a.ring_slots)
                    ok = fast_allreduce<K, K>(dacc, S->e_pAp, S->skipA, a.ring + 8 * (size_t)ns, red, &S->poison, G, postA);
                if (!ok) {
                    grid_allreduce<K>(dacc, a.partials, a.bar, gen, parity, red, G);
                    if (warp == 0) postA(pick_lane<K>(dacc, 0, lane), 0.0);
                    __syncthreads();
                }
            }
            if (prof) { const long long t1 = clock64(); tR1 += t1 - t0; t0 = t1; }
        }
        // ---------------- phase B: r -= alpha Ap, r.z, r.r   (x += alpha p is folded into phase C)
        float4 pc0[UBC];
        float xc0[UBC][K];
        {
            float alpha[K];
#pragma unroll
            for (int k = 0; k < K; ++k) alpha[k] = S->alpha[k];
            double acc2[2 * K];
#pragma unroll
            for (int i = 0; i < 2 * K; ++i) acc2[i] = 0.0;
            // r, Ap and D^-1 are in shared memory (RES = 1): this phase touches no global memory at all; the x update
            // that belongs here is done in phase C, which reads the owner's p row anyway
            for (int s = s_begin + warp; s < s_end; s += PWARPS) {
                const int li = s - s_begin, row = s * 32 + lane;
                const float di = RES ? d_s[(size_t)li * 32 + lane] : a.dinv[row];
#pragma unroll
                for (int k = 0; k < K; ++k) {
                    const float rn = fmaf(-alpha[k], Q(li, k, row), R(li, k, row));
                    R(li, k, row) = rn;
                    const float r2 = rn * rn;
                    acc2[k] += (double)(di * r2);
                    acc2[K + k] += (double)r2;
                }
            }
            if (prof) { const long long t1 = clock64(); tB += t1 - t0; t0 = t1; }
            // phase C's first batch of global loads (own p rows and x) depends on neither alpha nor beta: issue it now so
            // that its latency overlaps the all-reduce
#pragma unroll
            for (int j = 0; j < UBC; ++j) {
                const int s = s_begin + warp + j * PWARPS;
                if (PREFC && s < s_end) {
                    const int row = s * 32 + lane;
                    pc0[j] = ld_coherent4(a.p + 4 * (size_t)row);
#pragma unroll
                    for (int k = 0; k < K; ++k) xc0[j][k] = a.x[(size_t)k * Vp + row];
                }
            }
            {
                // beta_k, convergence and the stop decision; one lane per column, lane 0 combines
                auto postB = [&](const double rzn, const double rrn) {
                    bool bad = false, cvk = true;
                    if (lane < K) {
                        if (S->conv[lane]) {
                            S->beta[lane] = 0.f;
                        } else {
                            if (rzn > 0.0) S->e_rzrr[lane] = exp2_of(rzn);
                            if (rrn > 0.0) S->e_rzrr[K + lane] = exp2_of(rrn);
                            if (!(rzn == rzn)) bad = true;
                            const double rz_old = S->rz[lane];
                            float be = (rz_old > 0.0) ? (float)(rzn / rz_old) : 0.f;
                            S->rz[lane] = rzn;
                            S->rr[lane] = rrn;
                            const double rtol2 = (double)a.rtol * (double)a.rtol;
                            const bool cv = rrn <= rtol2 * S->bb[lane];
                            S->conv[lane] = cv ? 1 : 0;
                            if (cv) {
                                be = 0.f;
                                S->skipA[lane] = 1;
                                S->skipB[lane] = S->skipB[K + lane] = 1;
                            }
                            S->beta[lane] = be;
                            cvk = cv;
                        }
                    }
                    const bool all = __all_sync(0xffffffffu, cvk);
                    const bool anybad = __any_sync(0xffffffffu, bad);
                    if (lane == 0) {
                        S->nslot += 1;
                        const int it = S->it + 1;
                        S->it = it;
                        if (anybad || S->status == 3) S->status = 3;
                        else if (all) S->status = 1;
                        else if (it >= a.maxit) S->status = 2;
                        S->stop = S->status != 0;
                    }
                };
                const int ns = S->nslot;
                bool ok = false;
                if (ns < a.ring_slots)
                    ok = fast_allreduce<2 * K, K>(acc2, S->e_rzrr, S->skipB, a.ring + 8 * (size_t)ns, red, &S->poison, G, postB);
                if (!ok) {
                    grid_allreduce<2 * K>(acc2, a.partials, a.bar, gen, parity, red, G);
                    if (warp == 0) postB(pick_lane<K>(acc2, 0, lane), pick_lane<K>(acc2, K, lane));
                    __syncthreads();
                }
            }
            if (prof) { const long long t1 = clock64(); tR2 += t1 - t0; t0 = t1; }
        }
        if (S->stop) break;
        // ---------------- phase C: p = D^-1 r + beta p, then make p visible
        {
            float beta[K], alpha[K];
#pragma unroll
            for (int k = 0; k < K; ++k) {
                beta[k] = S->beta[k];
                alpha[k] = S->alpha[k];
            }
            for (int sb = s_begin + warp; sb < s_end; sb += UBC * PWARPS) {
                float4 po[UBC];
                float xo[UBC][K];
                if (PREFC && sb == s_begin + warp) {          // first batch was loaded before the all-reduce
#pragma unroll
                    for (int j = 0; j < UBC; ++j) {
                        po[j] = pc0[j];
#pragma unroll
                        for (int k = 0; k < K; ++k) xo[j][k] = xc0[j][k];
                    }
                } else {
#pragma unroll
                    for (int j = 0; j < UBC; ++j) {      // all global loads of UBC owned slices in flight together
                        const int s = sb + j * PWARPS;
                        if (s < s_end) {
                            const int row = s * 32 + lane;
                            po[j] = ld_coherent4(a.p + 4 * (size_t)row);
#pragma unroll
                            for (int k = 0; k < K; ++k) xo[j][k] = a.x[(size_t)k * Vp + row];
                        }
                    }
                }
#pragma unroll
                for (int j = 0; j < UBC; ++j) {
                    const int s = sb + j * PWARPS;
                    if (s < s_end) {
                        const int li = s - s_begin, row = s * 32 + lane;
                        const float di = RES ? d_s[(size_t)li * 32 + lane] : a.dinv[row];
                        float pn[4] = {po[j].x, po[j].y, po[j].z, po[j].w};
#pragma unroll
                        for (int k = 0; k < K; ++k) {
                            a.x[(size_t)k * Vp + row] = fmaf(alpha[k], pn[k], xo[j][k]);     // x += alpha p (this iteration's p)
                            pn[k] = fmaf(beta[k], pn[k], di * R(li, k, row));               // p = D^-1 r + beta p
                        }
                        *reinterpret_cast<float4 *>(a.p + 4 * (size_t)row) = make_float4(pn[0], pn[1], pn[2], pn[3]);
                    }
                }
            }
            if (prof) { const long long t1 = clock64(); tC += t1 - t0; t0 = t1; }
            grid_arrive(a.bar, gen, G);
            prologue();                      // next iteration's first matrix entries fly while the barrier completes
            grid_wait(a.bar, gen, G);
            if (prof) { const long long t1 = clock64(); tB3 += t1 - t0; t0 = t1; }
        }
    }
    if (prof) {
        if (cta == 0) {
            a.dbg[0] = tA; a.dbg[1] = tR1; a.dbg[2] = tB; a.dbg[3] = tR2; a.dbg[4] = tC; a.dbg[5] = tB3; a.dbg[6] = 0; a.dbg[7] = S->it;
        }
        long long *row = a.dbg + 8 + 8 * (size_t)cta;   // per-CTA table
        unsigned int smid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        row[0] = tA; row[1] = tR1; row[2] = tB; row[3] = tR2; row[4] = tC; row[5] = tB3; row[6] = smid; row[7] = S->it;
    }

    // ------------------------------------------------------------------ result: x (planes) -> caller layout
    // the last iteration's x += alpha p is still pending (it lives in phase C, which the stopping iteration skips)
    {
        const bool pending = S->it > 0;
        float alpha[K];
#pragma unroll
        for (int k = 0; k < K; ++k) alpha[k] = pending ? S->alpha[k] : 0.f;
        for (int s = s_begin + warp; s < s_end; s += PWARPS) {
            const int row = s * 32 + lane;
            if (row < a.V) {
                const long long io = a.perm ? a.perm[row] : row;
                const float4 po = ld_coherent4(a.p + 4 * (size_t)row);
                const float pk[4] = {po.x, po.y, po.z, po.w};
#pragma unroll
                for (int k = 0; k < K; ++k) a.out[io * K + k] = fmaf(alpha[k], pk[k], a.x[(size_t)k * Vp + row]);
            }
        }
    }
    if (cta == 0 && tid == 0 && a.info) {
        a.info[0] = (float)S->it;
        a.info[1] = (float)S->status;
        for (int k = 0; k < 4; ++k) a.info[2 + k] = (k < K && S->bb[k] > 0.0) ? (float)sqrt(S->rr[k] / S->bb[k]) : 0.f;
        a.info[6] = a.info[7] = 0.f;
    }
}

inline size_t persist_smem_bytes(int K, int res, int nsl_max) {
    return 4096 + (res ? (size_t)nsl_max * 32 * 4 * (2 * K + 1) : 0);
}

}  // namespace lsp
