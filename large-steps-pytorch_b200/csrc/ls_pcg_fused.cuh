// ls_pcg_fused.cuh -- two-synchronisation Jacobi-PCG: the whole solve as ONE persistent kernel (sm_90a), round 2.
//
// What round 1's kernel (three grid synchronisations per iteration: p.Ap all-reduce, r.z / r.r all-reduce, p barrier) taught us:
//   * with the pattern-only matrix copy the V = 1e6 solve is mostly L2-resident: nothing is HBM-bound;
//   * every phase is a chain of dependent L2 round trips: the slice offsets were loaded from global memory right before
//     the entries that need them (two round trips per slice in the SpMV phase), and the p-update phase paid one more
//     round trip per slice for the owner's p and x rows;
//   * a grid-wide all-reduce costs thousands of cycles of pure mechanics (no skew) and there were three per iteration.
//
// This kernel restructures the iteration so that there are TWO grid synchronisations and ONE round of global loads:
//   phase B   r -= alpha s,  z = D^-1 r  (shared memory only; z rows are the one vector other CTAs read: stored to global),
//             gamma' = r.z, rr = r.r                      -> all-reduce #1, which is also the barrier that publishes z
//             beta = gamma'/gamma, convergence per column, stop decision
//   phase A   w = A z (gathered), and in the same pass, with the owner's rows loaded next to the gathers:
//             x += alpha_prev p,  p = z + beta p,  s = w + beta s,  delta = p.s   -> all-reduce #2:  alpha = gamma/delta
// s = A p is carried by its recurrence (as in Chronopoulos-Gear CG) but delta is a directly computed dot product.  In exact
// arithmetic this is classical PCG.  In fp32 the recurrence lets the recursive residual drift from b - A x over long runs
// (rel-L2 error vs a direct solve: 6e-7 after 100 iterations, 1.7e-5 after 620 on the alpha = 0.999 plane; numpy model in
// DESIGN.md), so the solve ends with a check of the TRUE residual, accumulated in fp64 (restart_from_x below): if it sits
// more than `theta` times above the fp32 representation floor eps * || |A| |x| || the iteration restarts from that
// residual (at most `refine` times).  The same routine implements the warm start of the reference's CG plug-in
// (solvers.py:102-110): x0 is loaded, the true residual computed in-kernel, and a guess worse than zero is dropped.
//
// Data placement (per row, K = 3): r, s, D^-1 in shared memory (RES >= 1: 28 B/row; pattern copy: a 1-byte diagonal class instead
// of D^-1, 25 B/row, plus the two class tables), additionally x and the owner's p
// (RES = 2: 52 B/row, mid-size meshes); z rows (16 B) and, below RES = 2, x / p planes in global memory (L2-resident).
// Slice offsets of the CTA's own slices are copied to shared memory once.
// RES = 4 (one cluster, meshes of a few thousand vertices): every vector in shared memory INCLUDING the published rows, which the
// other CTAs of the cluster gather through distributed shared memory (mapa + ld.shared::cluster) -- inside the iteration nothing
// but the (read-only) matrix entries comes from global memory and a synchronisation is one barrier.cluster.
// Synchronisation: SYNC = 0 the whole grid (fixed-point single-atomic all-reduce, release/acquire where it publishes z),
// SYNC = 1 one thread-block cluster (<= 16 CTAs: partials exchanged through distributed shared memory + barrier.cluster),
// for meshes small enough that 16 SMs hold them -- a bare cluster barrier is an order of magnitude cheaper than a grid all-reduce.
#pragma once
#include <cuda_bf16.h>
#include <type_traits>
#include "ls_common.cuh"
#include "ls_sell_kernel.cuh"

namespace lsf {

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

struct FusedArgs {
    int V;
    long long Vp;
    int nslices;
    int nsl_max;
    int kb;                 // columns of b / out (<= K)
    const int *soff;        // general SELL-32 copy (always present: the true-residual pass uses it even when PAT)
    const int2 *ent;
    const int *poff;        // pattern-only copy (ls_sell_kernel.cuh): slice offsets in words, bit 0 = wide slice
    const unsigned int *pcol;
    const unsigned char *pcls;                 // diagonal class per row
    const unsigned long long *pcls_tab;        // [PAT_CLASSES] class -> (D^-1 bits << 32) | corrected diagonal bits
    float offc;
    int pat_l1;             // pattern copy shared (a few KB read by every CTA): its columns are cached in L1
    const float *dinv;
    float *x;               // K planes of Vp            (RES < 2)
    float *pv;              // owner copy of p, K planes (RES < 2)
    float *r;               // K planes                  (RES = 0)
    float *s;               // K planes                  (RES = 0)
    float *z;               // published rows of 4 floats
    float *z2;              // second row buffer (Chebyshev steps ping-pong between the two; ZH: holds the bf16 rows, 8 bytes each)
    float *cy, *cd;         // Chebyshev iterate and direction, K planes each (owner-only)
    int cheb_m;             // polynomial degree + 1 (<= 1: plain Jacobi);  z = q(D^-1 A) D^-1 r with m - 1 extra SpMVs
    float cheb_c0;          // 1 / theta
    float cheb_c1[8], cheb_c2[8];
    const float *b;         // (V,kb) caller layout
    float *out;             // (V,kb)
    const float *x0;        // warm start (V,kb) or NULL
    const int *perm;
    float rtol;
    int maxit;
    int refine;             // max restarts from the true residual
    float theta;            // restart if ||b - A x|| > theta * eps32 * || |A||x| ||  (and > rtol ||b||)
    GridBar *bar;
    double *partials;       // [2][NVMAX][G]
    unsigned long long *ring;
    int ring_slots;
    float *info;
    long long *dbg;
};

struct Scal {
    double gam[4], bb[4], rr[4];
    float alpha[4], beta[4];
    int conv[4];
    int it, status, stop, restarts, checks;
    int e_dl[4];
    int e_grr[8];
    int skipA[4], skipB[8];
    int nslot;
    int poison;
    int cold;       // warm start rejected: redo the initialisation from x = 0
};

__device__ __forceinline__ unsigned long long ld_acquire64(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

// ---- synchronisation policies ---------------------------------------------------------------------------------------
// Both expose:  barrier()                      everything written before it is visible to every CTA after it
//               allreduce<NV,KCOL,PUB>(v, eref, skip, post)   deterministic sum over all CTAs, then post(val, val2) on warp 0
//                                              (one lane per column); PUB: the reduction also acts as barrier()
struct GridSync {
    GridBar *bar;
    double *partials;
    unsigned long long *ring;
    int ring_slots;
    unsigned int gen, parity;
    int G;
    double *red;
    Scal *S;

    __device__ __forceinline__ void barrier() { grid_barrier(bar, gen, G); }

    // Fast path: one 64-bit atomic per value into a fresh ring slot, no second pass.  The fenced path (grid_allreduce) is a
    // chain of ~6 dependent L2 round trips (partial store -> fence -> arrive -> poll -> fence -> re-read).  Integer addition
    // is associative, so a fixed-point sum is deterministic no matter in which order the CTAs' atomics land.  Word layout:
    // [63:16] signed fixed-point sum, [15:8] number of CTAs whose partial did not fit ("poison"), [7:0] arrival count.  The
    // scale of value i is taken from the exponent `eref[i]` of the same quantity one iteration earlier (identical on every
    // CTA): a partial must be finite and below 2^(eref+3); 2^-35 relative resolution, far below the fp32 noise of the dot
    // products themselves.  If any CTA poisons a value, every CTA sees the same poison count and the whole grid repeats that
    // reduction through the fenced path.
    template <int NV, int KCOL, bool PUB, typename Post>
    __device__ __forceinline__ void allreduce(double (&v)[NV], const int *eref, const int *skip, bool allow_fast, Post post) {
        const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
        const int ns = S->nslot;
        bool ok = false;
        if (allow_fast && ns < ring_slots && G <= 255) {
            unsigned long long *slot = ring + 8 * (size_t)ns;
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
                    const int e = min(max(eref[lane], -900), 900);
                    const double up = __longlong_as_double((long long)(1023 + 35 - e) << 52);
                    const double down = __longlong_as_double((long long)(1023 + e - 35) << 52);
                    unsigned long long word = 1ull;
                    if (!skip[lane]) {
                        const bool fits = (val == val) && (fabs(val) * up < 274877906944.0 /* 2^38 */);
                        if (fits) word += ((unsigned long long)__double2ll_rn(val * up)) << 16;
                        else word += 1ull << 8;
                    }
                    unsigned long long w;
                    if (PUB) {
                        // release: the z rows every thread of this CTA stored before the CTA barrier above are visible to
                        // whoever acquires this word; the acquire below invalidates L1 so the gathers that follow miss it
                        asm volatile("red.release.gpu.global.add.u64 [%0], %1;" ::"l"(slot + lane), "l"(word) : "memory");
                        do {
                            w = ld_acquire64(slot + lane);
                        } while ((int)(w & 0xffull) != G);
                    } else {
                        atomicAdd(slot + lane, word);
                        do {
                            asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(w) : "l"(slot + lane) : "memory");
                        } while ((int)(w & 0xffull) != G);
                    }
                    val = (double)((long long)w >> 16) * down;
                    pois = (unsigned int)((w >> 8) & 0xffull);
                }
                const bool poison = __any_sync(0xffffffffu, pois != 0u);
                __syncwarp();
                const double val2 = (NV > KCOL) ? __shfl_down_sync(0xffffffffu, val, KCOL) : 0.0;
                if (!poison) post(val, val2);
                if (lane == 0) {
                    S->poison = poison ? 1 : 0;
                    S->nslot = ns + 1;
                }
            }
            __syncthreads();
            ok = S->poison == 0;
        }
        if (!ok) {
            // fenced path: per-CTA partials, a full grid barrier, a fixed-order re-reduction (also publishes everything)
            grid_allreduce<NV>(v, partials, bar, gen, parity, red, G);
            if (warp == 0) post(pick_lane<KCOL>(v, 0, lane), (NV > KCOL) ? pick_lane<KCOL>(v, NV > KCOL ? KCOL : 0, lane) : 0.0);
            __syncthreads();
        }
    }

    // plain deterministic sum of NV values, result in v[] on every thread (used by the init / restart paths)
    template <int NV>
    __device__ __forceinline__ void allreduce_slow(double (&v)[NV]) {
        grid_allreduce<NV>(v, partials, bar, gen, parity, red, G);
    }
};

// one thread-block cluster: partial sums are pushed into every CTA's shared memory (DSMEM), one cluster barrier later
// every CTA adds the CS partials in rank order -- bit-identical on all CTAs and run to run
struct ClusterSync {
    double *cl;            // shared: [2][NVMAX][16]
    unsigned int parity;
    int G;                 // cluster size (1 .. 16)
    double *red;
    Scal *S;

    __device__ __forceinline__ static unsigned int rank() {
        unsigned int r;
        asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
        return r;
    }
    __device__ __forceinline__ void barrier() {
        if (G == 1) {
            __syncthreads();
            return;
        }
        asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
        asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
    }
    template <int NV>
    __device__ __forceinline__ void exchange(double (&v)[NV]) {   // on return red[NV*32 + i] holds the cluster-wide sum i
        const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const double s = ls_warp_sum(v[i]);
            if (lane == 0) red[i * 32 + warp] = s;
        }
        __syncthreads();
        double *mine = cl + (size_t)parity * NVMAX * 16;
        if (warp == 0) {
            double val = 0.0;
#pragma unroll
            for (int i = 0; i < NV; ++i) {
                const double s = ls_warp_sum(lane < (int)(blockDim.x >> 5) ? red[i * 32 + lane] : 0.0);
                if (lane == i) val = s;
            }
            if (lane < NV) {
                const unsigned int me = (G > 1) ? rank() : 0u;
                const unsigned int local = ls_smem_u32(mine + lane * 16 + me);
                if (G == 1) {
                    mine[lane * 16] = val;
                } else {
                    for (int c = 0; c < G; ++c) {
                        unsigned int remote;
                        asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local), "r"(c));
                        asm volatile("st.shared::cluster.f64 [%0], %1;" ::"r"(remote), "d"(val) : "memory");
                    }
                }
            }
        }
        barrier();
        if (warp == 0 && lane < NV) {
            double t = 0.0;
            for (int c = 0; c < G; ++c) t += mine[lane * 16 + c];
            red[NV * 32 + lane] = t;
        }
        parity ^= 1u;
        __syncthreads();
    }
    template <int NV, int KCOL, bool PUB, typename Post>
    __device__ __forceinline__ void allreduce(double (&v)[NV], const int *, const int *, bool, Post post) {
        exchange<NV>(v);
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        if (warp == 0) {
            const double val = (lane < NV) ? red[NV * 32 + lane] : 0.0;
            const double val2 = (NV > KCOL) ? __shfl_down_sync(0xffffffffu, val, KCOL) : 0.0;
            post(val, val2);
        }
        __syncthreads();
    }
    template <int NV>
    __device__ __forceinline__ void allreduce_slow(double (&v)[NV]) {
        exchange<NV>(v);
#pragma unroll
        for (int i = 0; i < NV; ++i) v[i] = red[NV * 32 + i];
        __syncthreads();
    }
};

// entry loads: the grid kernel streams them past L1 (the gathers own it); a cluster / single CTA keeps them cached
template <bool KEEP>
__device__ __forceinline__ int2 ld_ent(const int2 *p) {
    if (KEEP) {
        int2 r;
        asm volatile("ld.global.nc.v2.s32 {%0, %1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
        return r;
    }
    return lsk::ld_entry(p);
}

// ---- the published preconditioned residual in bfloat16 (template flag ZH) ----------------------------------------------------
// z = D^-1 r is the one vector every CTA gathers (6-7 times per row) and stores each iteration.  CG does not need it exactly: if
// the SAME rounded vector z~ is used for the SpMV, for p = z~ + beta p and for gamma = r.z~, the recurrences s = A p, r = b - A x
// stay exact and only the preconditioner is perturbed by <= 2^-9 relative -- iteration counts and final accuracy are unchanged
// (numpy model and GPU tests: 99 / 124 / 537 -> 99 / 124 / 541 iterations, errors equal or smaller).  Rows of 4 x bf16 = 8 bytes
// halve the store and gather traffic of the published vector.  Anything that needs full precision (the x rows of the
// true-residual pass, the Chebyshev iterates) keeps using the fp32 row buffer.
__device__ __forceinline__ uint2 pack_bf16_row(float a, float b, float c) {
    const __nv_bfloat162 lo = __floats2bfloat162_rn(a, b), hi = __floats2bfloat162_rn(c, 0.f);
    return make_uint2(*reinterpret_cast<const unsigned int *>(&lo), *reinterpret_cast<const unsigned int *>(&hi));
}
__device__ __forceinline__ float4 unpack_bf16_row(const uint2 w) {
    return make_float4(__uint_as_float(w.x << 16), __uint_as_float(w.x & 0xffff0000u), __uint_as_float(w.y << 16), 0.f);
}
// x and the owner's p (RES < 2: planes in global memory, 24 MB at V = 1e6, K = 3) are read and written once per iteration, by
// their owner only, in phase A.  L1::no_allocate keeps them from evicting the published rows the gathers re-use from L1, and an
// L2 evict_last policy keeps them resident in L2 against the matrix and published-row traffic of the same pass.
__device__ __forceinline__ unsigned long long l2_evict_last_policy() {
    unsigned long long pol;
    asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ float ld_owned_f32(const float *p, unsigned long long pol) {
    float v;
    asm volatile("ld.global.L1::no_allocate.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(v) : "l"(p), "l"(pol) : "memory");
    return v;
}
__device__ __forceinline__ void st_owned_f32(float *p, float v, unsigned long long pol) {
    asm volatile("st.global.L1::no_allocate.L2::cache_hint.f32 [%0], %1, %2;" ::"l"(p), "f"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ uint2 ld_coherent_u2(const uint2 *p) {
    uint2 v;
    asm volatile("ld.global.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
    return v;
}

// ---- batches: many independent meshes per launch, one thread-block cluster per mesh (template flag BATCH) ----------------------
// Each mesh keeps its own handle (matrix copies, workspace); its FusedArgs are written once, when the batch is created, into a
// device table indexed by %clusterid.  A launch passes only what changes per call: the packed (sum V_i, kb) right-hand side,
// solution and warm start, the info records and the solve parameters.  The clusters never wait on each other: each mesh
// iterates, checks its true residual and stops on its own.  A Chebyshev mesh (its own instantiations, RES 2) finds its polynomial
// (cheb_m, cheb_c0, cheb_c1, cheb_c2) in its table entry; its steps synchronise its own cluster only, with a bare cluster barrier.
struct BatchEntry {
    FusedArgs a;            // the mesh's arguments; b, out, x0, info, kb, rtol and maxit come from BatchParams
    long long row0;         // first row of the mesh in the packed layout
    int mesh;               // index of the mesh in the batch: its info record is info + 8 * mesh
};
struct BatchParams {
    const BatchEntry *tab;  // one entry per cluster of this launch
    const float *b;         // packed (sum V_i, kb)
    float *out;
    const float *x0;        // or NULL
    float *info;            // 8 floats per mesh
    int kb;
    float rtol;
    int maxit;
};
template <bool BATCH> struct FusedParam { using type = FusedArgs; };
template <> struct FusedParam<true> { using type = BatchParams; };

__device__ __forceinline__ unsigned int cluster_nctarank() {
    unsigned int r;
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ unsigned int cluster_id_x() {
    unsigned int r;
    asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(r));
    return r;
}
// the single-mesh kernel reads its arguments from the parameter space as before
__device__ __forceinline__ const FusedArgs &kernel_args(const FusedArgs &p, unsigned char *) { return p; }
// batch: this cluster's table entry -> shared memory (`where`, in the header), completed with the per-call fields
__device__ __forceinline__ const FusedArgs &kernel_args(const BatchParams &p, unsigned char *where) {
    FusedArgs *a = reinterpret_cast<FusedArgs *>(where);
    const BatchEntry *e = p.tab + cluster_id_x();
    static_assert(sizeof(FusedArgs) % 8 == 0, "copied as 8-byte words");
    const unsigned long long *src = reinterpret_cast<const unsigned long long *>(&e->a);
    unsigned long long *dst = reinterpret_cast<unsigned long long *>(a);
    for (int i = threadIdx.x; i < (int)(sizeof(FusedArgs) / 8); i += blockDim.x) dst[i] = src[i];
    __syncthreads();
    if (threadIdx.x == 0) {
        const long long o = e->row0 * p.kb;
        a->b = p.b + o;
        a->out = p.out + o;
        a->x0 = p.x0 ? p.x0 + o : nullptr;
        a->info = p.info + 8 * (size_t)e->mesh;
        a->kb = p.kb;
        a->rtol = p.rtol;
        a->maxit = p.maxit;
    }
    __syncthreads();
    return *a;
}

constexpr size_t FUSED_SMEM_HDR = 4096 + 1024;   // reduction scratch + scalars, then the cluster exchange area
constexpr size_t FUSED_BATCH_ARGS = 4352 + 320;  // BATCH: the cluster's FusedArgs, between the scalars and the exchange area
__host__ __device__ inline size_t fused_off_bytes(int nsl_max) { return ((size_t)(2 * (nsl_max + 1)) * 4 + 127) / 128 * 128; }

// bytes per row kept in shared memory: RES 1: r, s, D^-1;  RES 2: + x, p;  RES 3 (single CTA) and 4 (cluster): + the z rows (4 floats);
// cheb (RES 2): + the Chebyshev iterate and direction.  Pattern copy: a 1-byte diagonal class instead of D^-1 (and the class
// tables, fused_tab_bytes, once per CTA)
__host__ __device__ inline int fused_row_bytes(int K, int res, int pat, int cheb = 0) {
    if (res == 0) return 0;
    return 4 * ((res == 1 ? 2 * K : (res == 2 ? 4 * K : 4 * K + 4)) + ((cheb && res == 2) ? 2 * K : 0)) + (pat ? 1 : 4);
}
__host__ __device__ inline size_t fused_tab_bytes(int pat) { return pat ? (size_t)lsk::PAT_CLASSES * 8 : 0; }   // D^-1, corrected diagonal
// the cluster exchange area exists only in the cluster instantiations: on the grid its 4 KB decide whether the V = 1e6 kernel fits
// the 196 KB shared-memory carve-out (and leaves 60 KB of L1) or needs the 228 KB one (28 KB of L1)
__host__ __device__ inline size_t fused_cl_bytes(int sync) { return sync == 1 ? (size_t)(2 * NVMAX * 16 * 8) : 0; }
inline size_t fused_smem_bytes(int K, int res, int nsl_max, int pat, int cheb, int sync) {
    return FUSED_SMEM_HDR + fused_cl_bytes(sync) + fused_off_bytes(nsl_max) + fused_tab_bytes(pat) + (size_t)nsl_max * 32u * fused_row_bytes(K, res, pat, cheb);
}

template <int K, int RES, int NW, bool PAT, int SYNC, bool PROF, bool CHEB = false, bool ZH = false, bool BATCH = false>
__global__ void __launch_bounds__(NW * 32, 1) pcg_fused_kernel(const typename FusedParam<BATCH>::type prm) {
    static_assert(K == 3 || K == 4, "z rows are float4");
    static_assert(!ZH || (K == 3 && !CHEB && RES != 3), "bf16 rows: 3 columns, Jacobi, published through global or distributed shared memory");
    static_assert(RES != 4 || (SYNC == 1 && !CHEB), "cluster-resident rows: one cluster, Jacobi");
    static_assert(!BATCH || (K == 3 && SYNC == 1 && !PROF && (RES == 2 || (RES == 3 && !CHEB))),
                  "batch: one cluster per mesh, 3 columns; Jacobi at RES 3 or 2, Chebyshev at RES 2");
    static_assert(sizeof(Scal) <= FUSED_BATCH_ARGS - 4352 && FUSED_BATCH_ARGS + sizeof(FusedArgs) <= FUSED_SMEM_HDR, "header layout");
    constexpr bool KEEP = (SYNC == 1);
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const FusedArgs &a = kernel_args(prm, smem_raw + FUSED_BATCH_ARGS);
    const bool pkeep = KEEP || (PAT && a.pat_l1 != 0);   // pattern columns: cached in L1 on the grid too when the copy is shared
    double *red = reinterpret_cast<double *>(smem_raw);                       // NV*32 + NV doubles, NV <= 16  (<= 4224 B)
    Scal *S = reinterpret_cast<Scal *>(smem_raw + 4352);
    double *cl = reinterpret_cast<double *>(smem_raw + FUSED_SMEM_HDR);       // [2][NVMAX][16]
    int *off_s = reinterpret_cast<int *>(smem_raw + FUSED_SMEM_HDR + fused_cl_bytes(SYNC));   // [nsl_max + 1] general, then [nsl_max + 1] pattern
    const int nsl_max = a.nsl_max;
    int *poff_s = off_s + (nsl_max + 1);
    float *tab_d = reinterpret_cast<float *>(reinterpret_cast<unsigned char *>(off_s) + fused_off_bytes(nsl_max));   // PAT: [PAT_CLASSES] D^-1
    float *tab_p = tab_d + lsk::PAT_CLASSES;                                  // PAT: [PAT_CLASSES] corrected diagonal
    float *r_s = tab_d + (PAT ? 2 * lsk::PAT_CLASSES : 0);                   // [nsl_max][K][32]
    float *s_s = r_s + (size_t)nsl_max * K * 32;
    float *d_s = s_s + (size_t)nsl_max * K * 32;                              // [nsl_max][32] D^-1, or (PAT) the class bytes
    unsigned char *c_s = reinterpret_cast<unsigned char *>(d_s);
    float *x_s = d_s + (size_t)(RES >= 1 ? nsl_max : 0) * (PAT ? 8 : 32);     // RES >= 2
    float *p_s = x_s + (size_t)nsl_max * K * 32;
    float *z_s = p_s + (size_t)nsl_max * K * 32;                              // RES = 3: rows of 4 floats, the "published" vector never leaves the SM
    float *cy_s = z_s;                                                        // CHEB && RES == 2: [nsl_max][K][32] each
    float *cd_s = cy_s + (size_t)nsl_max * K * 32;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // batch: the mesh's CTAs are the cluster's
    const int G = BATCH ? (int)cluster_nctarank() : (int)gridDim.x, cta = BATCH ? (int)ClusterSync::rank() : (int)blockIdx.x;
    // RES = 4: uniform blocks of nsl_max slices, so that the owner of a gathered row is a division by a constant
    const int s_begin = (RES == 4) ? min(cta * nsl_max, a.nslices) : (int)((long long)a.nslices * cta / G);
    const int s_end = (RES == 4) ? min(s_begin + nsl_max, a.nslices) : (int)((long long)a.nslices * (cta + 1) / G);
    const long long Vp = a.Vp;
    const int kb = a.kb;
    constexpr int U = PAT ? 4 : 8;

    typename std::conditional<SYNC == 1, ClusterSync, GridSync>::type sync;
    if constexpr (SYNC == 1) {
        sync.cl = cl;
        sync.parity = 0;
        sync.G = G;
        sync.red = red;
        sync.S = S;
    } else {
        sync.bar = a.bar;
        sync.partials = a.partials;
        sync.ring = a.ring;
        sync.ring_slots = a.ring_slots;
        sync.gen = 0;
        sync.parity = 0;
        sync.G = G;
        sync.red = red;
        sync.S = S;
    }

    auto R = [&](int li, int k, int row) -> float & { return RES ? r_s[((size_t)li * K + k) * 32 + lane] : a.r[(size_t)k * Vp + row]; };
    auto Sv = [&](int li, int k, int row) -> float & { return RES ? s_s[((size_t)li * K + k) * 32 + lane] : a.s[(size_t)k * Vp + row]; };
    auto X = [&](int li, int k, int row) -> float & { return RES >= 2 ? x_s[((size_t)li * K + k) * 32 + lane] : a.x[(size_t)k * Vp + row]; };
    auto P = [&](int li, int k, int row) -> float & { return RES >= 2 ? p_s[((size_t)li * K + k) * 32 + lane] : a.pv[(size_t)k * Vp + row]; };
    // the row's diagonal class (pattern copy): owned rows in shared memory, RES = 0 global memory
    auto Cls = [&](int li, int row) -> int { return RES ? c_s[(size_t)li * 32 + lane] : a.pcls[row]; };
    auto Dv = [&](int li, int row) -> float {
        if constexpr (PAT) return tab_d[Cls(li, row)];
        else return RES ? d_s[(size_t)li * 32 + lane] : a.dinv[row];
    };
    // Chebyshev iterate (own rows) and direction: shared memory at RES = 2, else the direction lives in global planes and the
    // own row of the iterate is read back from its published copy
    auto CY = [&](int li, int k) -> float & { return cy_s[((size_t)li * K + k) * 32 + lane]; };
    auto CD = [&](int li, int k, int row) -> float & { return (CHEB && RES == 2) ? cd_s[((size_t)li * K + k) * 32 + lane] : a.cd[(size_t)k * Vp + row]; };

    float *zcur = a.z, *zalt = a.z2;   // the published vector lives in zcur; Chebyshev steps write the next iterate to zalt and swap
    const int cheb_m = CHEB ? a.cheb_m : 0;   // the polynomial preconditioner is compiled into its own instantiations only
    // the published rows: global memory, or (RES = 3, one CTA owns every row) shared memory
    // RES = 4: row `col` lives in the shared memory of CTA (col / 32) / nsl_max of the cluster, at the same offset in every CTA.
    // The division is a multiplication: exact for slice < 16 nsl_max when nsl_max < 64 (s e < 2^16 with e = M nsl_max - 2^16 <= nsl_max).
    const unsigned int dsm_base = ls_smem_u32(z_s);
    const unsigned int dsm_magic = 65536u / (unsigned int)max(nsl_max, 1) + 1u;
    const unsigned int dsm_rows = (unsigned int)nsl_max * 32u;
    auto dsm_addr = [&](int col, unsigned int rowbytes) -> unsigned int {
        const unsigned int own = (((unsigned int)col >> 5) * dsm_magic) >> 16;
        const unsigned int lr = (unsigned int)col - own * dsm_rows;
        unsigned int ra;
        asm("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(dsm_base + lr * rowbytes), "r"(own));
        return ra;
    };
    auto Zld = [&](int col) -> float4 {
        if constexpr (RES == 3) return *reinterpret_cast<const float4 *>(z_s + 4 * (size_t)col);
        else if constexpr (RES == 4) {
            float4 v;
            asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(dsm_addr(col, 16u)) : "memory");
            return v;
        } else return ld_coherent4(zcur + 4 * (size_t)col);
    };
    auto Zst = [&](int row_, const float4 v_) {
        if constexpr (RES == 3) *reinterpret_cast<float4 *>(z_s + 4 * (size_t)row_) = v_;
        else if constexpr (RES == 4) *reinterpret_cast<float4 *>(z_s + 4 * (size_t)(row_ - s_begin * 32)) = v_;
        else *reinterpret_cast<float4 *>(zcur + 4 * (size_t)row_) = v_;
    };
    // the published PRECONDITIONED RESIDUAL (phase B -> phase A): bf16 rows when ZH, else the same fp32 rows as above
    // (RES = 4: the bf16 rows alias the fp32 row area -- the two uses are always separated by a cluster barrier)
    uint2 *zh = (RES == 4) ? reinterpret_cast<uint2 *>(z_s) - (size_t)s_begin * 32 : reinterpret_cast<uint2 *>(a.z2);
    auto ZldP = [&](int col) -> float4 {
        if constexpr (ZH && RES == 4) {
            uint2 w;
            asm volatile("ld.shared::cluster.v2.u32 {%0, %1}, [%2];" : "=r"(w.x), "=r"(w.y) : "r"(dsm_addr(col, 8u)) : "memory");
            return unpack_bf16_row(w);
        } else if constexpr (ZH) return unpack_bf16_row(ld_coherent_u2(zh + col));
        else return Zld(col);
    };
    // rounds zz[] to what the other CTAs will see, stores the row; the caller keeps using the rounded zz[] (consistency)
    auto ZstP = [&](int row_, float (&zz)[4]) {
        if constexpr (ZH) {
            const uint2 w = pack_bf16_row(zz[0], zz[1], zz[2]);
            const float4 q = unpack_bf16_row(w);
            zz[0] = q.x;
            zz[1] = q.y;
            zz[2] = q.z;
            zh[row_] = w;
        } else {
            Zst(row_, make_float4(zz[0], zz[1], zz[2], zz[3]));
        }
    };

    // sum += row_a + row_b of two gathered rows
    auto acc_pair = [&](float (&sum)[K], const float4 &ga, const float4 &gb) {
        const float xk[4] = {ga.x + gb.x, ga.y + gb.y, ga.z + gb.z, ga.w + gb.w};
#pragma unroll
        for (int k = 0; k < K; ++k) sum[k] += xk[k];
    };

    long long tA = 0, tS2 = 0, tB = 0, tS1 = 0, tX = 0, t0 = 0;
    const bool prof = PROF && (a.dbg != nullptr) && tid == 0;

    // slice offsets of the owned slices -> shared memory (they sat on the critical path of every slice as global loads)
    for (int i = tid; i <= s_end - s_begin; i += NW * 32) {
        off_s[i] = a.soff[s_begin + i];
        if (PAT) poff_s[i] = a.poff[s_begin + i];
    }
    if constexpr (PAT) {
        for (int i = tid; i < lsk::PAT_CLASSES; i += NW * 32) {
            const unsigned long long e = a.pcls_tab[i];
            tab_d[i] = __uint_as_float((unsigned int)(e >> 32));
            tab_p[i] = __uint_as_float((unsigned int)e);
        }
        if (RES)
            for (int i = tid; i < (s_end - s_begin) * 32; i += NW * 32) c_s[i] = a.pcls[(size_t)s_begin * 32 + i];
    }
    if (tid == 0) {
        S->nslot = 0;
        S->it = 0;
        S->checks = 0;
        S->restarts = 0;
        S->poison = 0;
        S->cold = 0;
    }
    // cluster: no CTA may write into another's shared memory before that CTA has started (compute-sanitizer flagged exactly that)
    if constexpr (SYNC == 1) sync.barrier();
    else __syncthreads();

    auto set_exponents = [&](int k, double gam, double rr) {   // thread 0
        const int eg = (gam > 0.0 && gam == gam) ? ilogb(gam) : -1000;
        const int er = (rr > 0.0 && rr == rr) ? ilogb(rr) : -1000;
        S->e_dl[k] = eg + 1;          // delta = z.Az <= lambda_max(D^-1 A) gamma <= 2 gamma at a (re)start
        S->e_grr[k] = eg;
        S->e_grr[K + k] = er;
        S->skipA[k] = S->conv[k];
        S->skipB[k] = S->skipB[K + k] = S->conv[k];
    };

    // matrix entries of this warp's first slice, (re)loaded before each wait so their latency hides under the barrier
    int2 nv[U];
    auto prologue = [&]() {
        const int s = s_begin + warp;
        if (s < s_end) {
            const int li = s - s_begin;
            if constexpr (PAT) {
                const lsk::PatSlice ps = lsk::pat_slice(poff_s + li);
#pragma unroll
                for (int u = 0; u < U; ++u) nv[u] = lsk::pat_load(a.pcol, ps, u, s * 32 + lane, lane, pkeep);
            } else {
                const int o0 = off_s[li], w = (off_s[li + 1] - o0) >> 5;
                const int2 *e = a.ent + o0 + lane;
#pragma unroll
                for (int u = 0; u < U; ++u) nv[u] = (u < w) ? ld_ent<KEEP>(e + u * 32) : make_int2(s * 32 + lane, 0);
            }
        }
    };

    // ---------------------------------------------------------------- one gather pass over the owned slices
    // For every owned slice: t = (A y)(row) with y the published vector (zcur rows), gathered through the prefetched entries
    // (`nv`: this slice's were loaded while the previous one was in flight; prologue() loads the first slice's before a barrier).
    //   pre(li,row)  issues the caller's own loads right behind the gathers (same latency window),
    //   own(li,row)  the caller's copy of row `row` of y (pattern copy only: the general copy gets it from the diagonal gather),
    //   epi(li,row,t,yown)  consumes the result.
    auto spmv_pass = [&](auto &&pre, auto &&own, auto &&epi) {
        for (int s = s_begin + warp; s < s_end; s += NW) {
            const int li = s - s_begin, row = s * 32 + lane;
            const int sn = s + NW;
            int2 cv[U];
#pragma unroll
            for (int u = 0; u < U; ++u) cv[u] = nv[u];
            float w_[K];
            float4 zo = make_float4(0.f, 0.f, 0.f, 0.f);
            if constexpr (PAT) {
                const lsk::PatSlice ps = lsk::pat_slice(poff_s + li);
                const int w2 = ps.w2;
                float sum[K];
#pragma unroll
                for (int k = 0; k < K; ++k) sum[k] = 0.f;
                float dp;
                auto body = [&](auto ub_tag) {
                    constexpr int UB = decltype(ub_tag)::value;
                    float4 xa[UB], xb[UB];
#pragma unroll
                    for (int u = 0; u < UB; ++u) {
                        const int2 c = lsk::pat_cols(cv[u], ps.wide, row);
                        xa[u] = ZldP(c.x);
                        xb[u] = ZldP(c.y);
                    }
                    zo = own(li, row);
                    dp = tab_p[Cls(li, row)];
                    pre(li, row);
                    if (sn < s_end) {
                        const lsk::PatSlice pn = lsk::pat_slice(poff_s + li + NW);
#pragma unroll
                        for (int u = 0; u < U; ++u) nv[u] = lsk::pat_load(a.pcol, pn, u, sn * 32 + lane, lane, pkeep);
                    }
#pragma unroll
                    for (int u = 0; u < UB; ++u) acc_pair(sum, xa[u], xb[u]);
                    const int extra = 2 * (UB - min(w2, UB));
                    dp = fmaf(-a.offc, (float)extra, dp);
                };
                if (w2 <= 3) body(std::integral_constant<int, 3>());
                else body(std::integral_constant<int, 4>());
                for (int j = U; j < w2; j += U) {
#pragma unroll
                    for (int u = 0; u < U; ++u) cv[u] = lsk::pat_load(a.pcol, ps, j + u, row, lane, pkeep);
                    float4 xa[U], xb[U];
#pragma unroll
                    for (int u = 0; u < U; ++u) {
                        const int2 c = lsk::pat_cols(cv[u], ps.wide, row);
                        xa[u] = ZldP(c.x);
                        xb[u] = ZldP(c.y);
                    }
#pragma unroll
                    for (int u = 0; u < U; ++u) acc_pair(sum, xa[u], xb[u]);
                    const int extra = 2 * max(0, j + U - w2);
                    dp = fmaf(-a.offc, (float)extra, dp);
                }
                const float zk[4] = {zo.x, zo.y, zo.z, zo.w};
#pragma unroll
                for (int k = 0; k < K; ++k) w_[k] = fmaf(dp, zk[k], a.offc * sum[k]);
            } else {
                const int o0 = off_s[li], w = (off_s[li + 1] - o0) >> 5;
                const int2 *e = a.ent + o0 + lane;
#pragma unroll
                for (int k = 0; k < K; ++k) w_[k] = 0.f;
                {
                    float4 xv[U];
#pragma unroll
                    for (int u = 0; u < U; ++u) xv[u] = ZldP(cv[u].x);
                    pre(li, row);
                    if (sn < s_end) {
                        const int n0 = off_s[li + NW], wn = (off_s[li + NW + 1] - n0) >> 5;
                        const int2 *en = a.ent + n0 + lane;
#pragma unroll
                        for (int u = 0; u < U; ++u) nv[u] = (u < wn) ? ld_ent<KEEP>(en + u * 32) : make_int2(sn * 32 + lane, 0);
                    }
#pragma unroll
                    for (int u = 0; u < U; ++u) {
                        const float wv = __int_as_float(cv[u].y);
                        const float xk[4] = {xv[u].x, xv[u].y, xv[u].z, xv[u].w};
                        if (cv[u].x == row) zo = xv[u];
#pragma unroll
                        for (int k = 0; k < K; ++k) w_[k] = fmaf(wv, xk[k], w_[k]);
                    }
                }
                for (int j = U; j < w; j += U) {
#pragma unroll
                    for (int u = 0; u < U; ++u) cv[u] = (j + u < w) ? ld_ent<KEEP>(e + (j + u) * 32) : make_int2(row, 0);
                    float4 xv[U];
#pragma unroll
                    for (int u = 0; u < U; ++u) xv[u] = ZldP(cv[u].x);
#pragma unroll
                    for (int u = 0; u < U; ++u) {
                        const float wv = __int_as_float(cv[u].y);
                        const float xk[4] = {xv[u].x, xv[u].y, xv[u].z, xv[u].w};
                        if (cv[u].x == row) zo = xv[u];
#pragma unroll
                        for (int k = 0; k < K; ++k) w_[k] = fmaf(wv, xk[k], w_[k]);
                    }
                }
            }
            epi(li, row, w_, zo);
        }
    };

    // the owner's row of the published vector for phase A (pattern copy): Jacobi: D^-1 r recomputed exactly as phase B stored
    // it; Chebyshev: the final iterate (shared memory at RES = 2, else its published row)
    auto own_z = [&](int li, int row) -> float4 {
        if constexpr (CHEB) {
            if constexpr (RES == 2) return make_float4(CY(li, 0), CY(li, 1), CY(li, 2), K > 3 ? CY(li, K > 3 ? 3 : 0) : 0.f);
            else return Zld(row);
        } else if constexpr (RES >= 1) {
            const float di_ = Dv(li, row);
            if constexpr (ZH) return unpack_bf16_row(pack_bf16_row(di_ * R(li, 0, row), di_ * R(li, 1, row), di_ * R(li, 2, row)));
            else return make_float4(di_ * R(li, 0, row), di_ * R(li, 1, row), di_ * R(li, 2, row), K > 3 ? di_ * R(li, K > 3 ? 3 : 0, row) : 0.f);
        } else {
            return ZldP(row);
        }
    };

    // ---------------------------------------------------------------- Chebyshev polynomial preconditioner (precond = 2)
    // z = q_{m-1}(D^-1 A) D^-1 r by the Chebyshev semi-iteration on [lambda_max / 30, lambda_max] (Gershgorin bound), y_1 = g / theta:
    //   d_j = c1_j d_{j-1} + c2_j D^-1 (r - A y_j),  y_{j+1} = y_j + d_j .   Each step gathers the published iterate, so it costs one
    // grid barrier but NO reduction: 2 all-reduces + (m - 1) barriers per m SpMVs instead of 2 all-reduces per SpMV.
    // cheb_first: y_1 (from the residual already in R) -> zcur rows, cy / cd planes.   cheb_steps: the m - 1 gather steps; the last
    // one accumulates r.z and r.r.  The caller's all-reduce publishes the final iterate.
    auto cheb_first = [&]() {
        for (int s = s_begin + warp; s < s_end; s += NW) {
            const int li = s - s_begin, row = s * 32 + lane;
            const float di = Dv(li, row) * a.cheb_c0;
            float yy[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int k = 0; k < K; ++k) {
                yy[k] = di * R(li, k, row);
                if constexpr (RES == 2) CY(li, k) = yy[k];
                CD(li, k, row) = yy[k];
            }
            Zst(row, make_float4(yy[0], yy[1], yy[2], yy[3]));
        }
    };
    auto cheb_steps = [&](double (&acc2)[2 * K]) {
        for (int j = 1; j < cheb_m; ++j) {
            prologue();                           // first slice's entries fly while the barrier completes
            sync.barrier();                       // iterate j is visible everywhere
            const float c1 = a.cheb_c1[j - 1], c2 = a.cheb_c2[j - 1];
            const bool last = (j == cheb_m - 1);
            float dprev[K];
            spmv_pass(
                [&](int li, int row) {
#pragma unroll
                    for (int k = 0; k < K; ++k) dprev[k] = CD(li, k, row);
                },
                [&](int li, int row) -> float4 {
                    if constexpr (RES == 2) return make_float4(CY(li, 0), CY(li, 1), CY(li, 2), K > 3 ? CY(li, K > 3 ? 3 : 0) : 0.f);
                    else return Zld(row);
                },
                [&](int li, int row, const float (&t)[K], const float4 &yo) {
                    const float di = Dv(li, row);
                    const float yk[4] = {yo.x, yo.y, yo.z, yo.w};
                    float yy[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                    for (int k = 0; k < K; ++k) {
                        const float rk = R(li, k, row);
                        const float dn = fmaf(c1, dprev[k], c2 * (di * (rk - t[k])));
                        yy[k] = yk[k] + dn;
                        CD(li, k, row) = dn;
                        if constexpr (RES == 2) CY(li, k) = yy[k];
                        if (last) {
                            acc2[k] += (double)rk * (double)yy[k];
                            acc2[K + k] += (double)rk * (double)rk;
                        }
                    }
                    *reinterpret_cast<float4 *>(zalt + 4 * (size_t)row) = make_float4(yy[0], yy[1], yy[2], yy[3]);
                });
            float *tz = zcur;
            zcur = zalt;
            zalt = tz;
        }
    };

    // ---------------------------------------------------------------- cold start: x = 0, r = b, z = D^-1 b, p = s = 0
    auto cold_init = [&]() {
        double acc[2 * K];
#pragma unroll
        for (int i = 0; i < 2 * K; ++i) acc[i] = 0.0;
        for (int s = s_begin + warp; s < s_end; s += NW) {
            const int li = s - s_begin, row = s * 32 + lane;
            float di = 0.f, bv[K];
#pragma unroll
            for (int k = 0; k < K; ++k) bv[k] = 0.f;
            if (row < a.V) {
                di = a.dinv[row];
                const long long io = a.perm ? a.perm[row] : row;
#pragma unroll
                for (int k = 0; k < K; ++k)
                    if (k < kb) bv[k] = a.b[io * kb + k];
            }
            if (RES && !PAT) d_s[(size_t)li * 32 + lane] = di;
            float zz[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int k = 0; k < K; ++k) zz[k] = di * bv[k];
            ZstP(row, zz);                 // (rounds zz to the published values when ZH)
#pragma unroll
            for (int k = 0; k < K; ++k) {
                R(li, k, row) = bv[k];
                Sv(li, k, row) = 0.f;
                X(li, k, row) = 0.f;
                P(li, k, row) = 0.f;
                acc[k] += (double)bv[k] * (double)zz[k];
                acc[K + k] += (double)bv[k] * (double)bv[k];
            }
        }
        if constexpr (CHEB) {
            if (cheb_m > 1) {     // gamma = r . q(D^-1 A) D^-1 r instead of r . D^-1 r
                double a2[2 * K];
#pragma unroll
                for (int i = 0; i < 2 * K; ++i) a2[i] = 0.0;
                cheb_first();
                cheb_steps(a2);
#pragma unroll
                for (int k = 0; k < K; ++k) acc[k] = a2[k];
            }
        }
        sync.template allreduce_slow<2 * K>(acc);     // fenced: also publishes z
        if (tid == 0) {
            int all = 1;
            for (int k = 0; k < K; ++k) {
                S->gam[k] = acc[k];
                S->bb[k] = acc[K + k];
                S->rr[k] = acc[K + k];
                S->conv[k] = !(acc[K + k] > 0.0);       // only an all-zero column is converged at entry (NaN: not converged)
                if (acc[K + k] != acc[K + k]) S->conv[k] = 0;
                S->alpha[k] = 0.f;
                S->beta[k] = 0.f;
                all &= S->conv[k];
                set_exponents(k, acc[k], acc[K + k]);
            }
            S->status = all ? 1 : (a.maxit <= 0 ? 2 : 0);
            S->stop = S->status != 0;
        }
        __syncthreads();
    };

    // ---------------------------------------------------------------- restart from the current x (warm start / refinement)
    // x (complete, no pending update) -> rows in the z buffer -> barrier -> r = b - A x with fp64 accumulation over the
    // general SELL copy, floor = |A||x| -> decide -> z = D^-1 r published, p and s restart through beta = 0.
    auto restart_from_x = [&](bool warm) {
        for (int s = s_begin + warp; s < s_end; s += NW) {
            const int li = s - s_begin, row = s * 32 + lane;
            float xv[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int k = 0; k < K; ++k) xv[k] = X(li, k, row);
            Zst(row, make_float4(xv[0], xv[1], xv[2], xv[3]));
        }
        sync.barrier();
        double acc[4 * K];   // [gamma | rr | floor^2 | bb]
#pragma unroll
        for (int i = 0; i < 4 * K; ++i) acc[i] = 0.0;
        for (int s = s_begin + warp; s < s_end; s += NW) {
            const int li = s - s_begin, row = s * 32 + lane;
            const int o0 = off_s[li], w = (off_s[li + 1] - o0) >> 5;
            const int2 *e = a.ent + o0 + lane;
            double ax[K];
            float fl[K];
#pragma unroll
            for (int k = 0; k < K; ++k) {
                ax[k] = 0.0;
                fl[k] = 0.f;
            }
            for (int j = 0; j < w; j += 4) {
                int2 cv[4];
                float4 xg[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) cv[u] = (j + u < w) ? ld_ent<KEEP>(e + (j + u) * 32) : make_int2(row, 0);
#pragma unroll
                for (int u = 0; u < 4; ++u) xg[u] = Zld(cv[u].x);
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const float wv = __int_as_float(cv[u].y);
                    const float xk[4] = {xg[u].x, xg[u].y, xg[u].z, xg[u].w};
#pragma unroll
                    for (int k = 0; k < K; ++k) {
                        ax[k] = fma((double)wv, (double)xk[k], ax[k]);
                        fl[k] = fmaf(fabsf(wv), fabsf(xk[k]), fl[k]);
                    }
                }
            }
            float di = 0.f, bv[K];
#pragma unroll
            for (int k = 0; k < K; ++k) bv[k] = 0.f;
            if (row < a.V) {
                di = a.dinv[row];
                const long long io = a.perm ? a.perm[row] : row;
#pragma unroll
                for (int k = 0; k < K; ++k)
                    if (k < kb) bv[k] = a.b[io * kb + k];
            }
            if (RES && !PAT) d_s[(size_t)li * 32 + lane] = di;
#pragma unroll
            for (int k = 0; k < K; ++k) {
                const float rv = (float)((double)bv[k] - ax[k]);
                R(li, k, row) = rv;
                float zz = di * rv;
                if constexpr (ZH) zz = __bfloat162float(__float2bfloat16_rn(zz));   // gamma = r . z~ with the z~ that gets published below
                acc[k] += (double)rv * (double)zz;
                acc[K + k] += (double)rv * (double)rv;
                acc[2 * K + k] += (double)fl[k] * (double)fl[k];
                acc[3 * K + k] += (double)bv[k] * (double)bv[k];
            }
        }
        if constexpr (CHEB) {
            if (cheb_m > 1) {     // preconditioned residual norm of the new residual (the gathers of the x rows end at the first barrier inside)
                double a2[2 * K];
#pragma unroll
                for (int i = 0; i < 2 * K; ++i) a2[i] = 0.0;
                sync.barrier();
                cheb_first();
                cheb_steps(a2);
#pragma unroll
                for (int k = 0; k < K; ++k) acc[k] = a2[k];
            }
        }
        sync.template allreduce_slow<4 * K>(acc);   // every CTA has finished gathering x rows once this returns
        if (tid == 0) {
            const double rtol2 = (double)a.rtol * (double)a.rtol;
            const double th = (double)a.theta * 5.9604644775390625e-08;   // theta * 2^-24
            int all = 1, worse = 0, bad = 0;
            for (int k = 0; k < K; ++k) {
                const double gam = acc[k], rr = acc[K + k], fl2 = acc[2 * K + k], bb = acc[3 * K + k];
                if (warm) {
                    S->bb[k] = bb;
                    if (rr > bb) worse = 1;               // guess worse than x = 0 (also caps fp32 accuracy): cold start instead
                    S->conv[k] = rr <= rtol2 * bb;
                } else {
                    const bool need = (rr > rtol2 * S->bb[k]) && (rr > th * th * fl2) && !(S->bb[k] == 0.0) && (S->restarts < a.refine);
                    S->conv[k] = need ? 0 : 1;
                }
                if (rr != rr) {
                    bad = 1;
                    S->conv[k] = 0;
                }
                S->gam[k] = gam;
                S->rr[k] = rr;
                S->alpha[k] = 0.f;
                S->beta[k] = 0.f;
                all &= S->conv[k];
                set_exponents(k, gam, rr);
            }
            S->cold = (warm && worse) ? 1 : 0;
            if (!warm) {
                S->checks += 1;
                if (!all && !bad) S->restarts += 1;
            }
            if (bad) S->status = 3;
            else if (all) S->status = 1;
            else if (S->it >= a.maxit) S->status = 2;
            else S->status = 0;
            S->stop = S->status != 0;
        }
        __syncthreads();
        if (S->cold) return;
        if (!S->stop) {
            for (int s = s_begin + warp; s < s_end; s += NW) {
                const int li = s - s_begin, row = s * 32 + lane;
                const float di = Dv(li, row);
                float zz[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                for (int k = 0; k < K; ++k) {
                    zz[k] = di * R(li, k, row);
                    if (warm) {
                        Sv(li, k, row) = 0.f;
                        P(li, k, row) = 0.f;
                    }
                }
                if (cheb_m <= 1)      // (Chebyshev: the preconditioned residual is already published in zcur)
                    ZstP(row, zz);
            }
            sync.barrier();
        }
    };

    // ---------------------------------------------------------------- entry
    if (a.x0 != nullptr) {
        for (int s = s_begin + warp; s < s_end; s += NW) {
            const int li = s - s_begin, row = s * 32 + lane;
            float xv[K];
#pragma unroll
            for (int k = 0; k < K; ++k) xv[k] = 0.f;
            if (row < a.V) {
                const long long io = a.perm ? a.perm[row] : row;
#pragma unroll
                for (int k = 0; k < K; ++k)
                    if (k < kb) xv[k] = a.x0[io * kb + k];
            }
#pragma unroll
            for (int k = 0; k < K; ++k) X(li, k, row) = xv[k];
        }
        restart_from_x(true);
        if (S->cold) {
            sync.barrier();      // every CTA is done with the z buffer (x rows) before cold_init overwrites it
            cold_init();
        }
    } else {
        cold_init();
    }

    for (;;) {   // episodes: iterate to convergence, check the true residual, maybe restart
        prologue();
        while (!S->stop) {
            // ------------------------------------------------ phase A: w = A z; x += alpha_prev p; p = z + beta p; s = w + beta s; p.s
            if (prof) t0 = clock64();
            {
                // per-thread partial of p.s in fp32 (a thread owns a few dozen rows at most), fp64 across threads; alpha_prev and
                // beta are read from shared memory where they are used: both keep registers out of the gather loop
                float dacc_f[K];
#pragma unroll
                for (int k = 0; k < K; ++k) dacc_f[k] = 0.f;
                float po[K], xo[K];
                const unsigned long long xp_pol = RES < 2 ? l2_evict_last_policy() : 0ull;
                spmv_pass(
                    [&](int li, int row) {
#pragma unroll
                        for (int k = 0; k < K; ++k) {
                            if constexpr (RES < 2) {
                                po[k] = ld_owned_f32(&P(li, k, row), xp_pol);
                                xo[k] = ld_owned_f32(&X(li, k, row), xp_pol);
                            } else {
                                po[k] = P(li, k, row);
                                xo[k] = X(li, k, row);
                            }
                        }
                    },
                    own_z,
                    [&](int li, int row, const float (&w_)[K], const float4 &zo) {
                        const float zk[4] = {zo.x, zo.y, zo.z, zo.w};
                        float xn[4] = {0.f, 0.f, 0.f, 0.f}, pn4[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                        for (int k = 0; k < K; ++k) {
                            const float al = S->alpha[k], be = S->beta[k];
                            xn[k] = fmaf(al, po[k], xo[k]);                         // x += alpha_prev p   (the previous iteration's pair)
                            const float pn = fmaf(be, po[k], zk[k]);                // p = z + beta p
                            const float sn_ = fmaf(be, Sv(li, k, row), w_[k]);      // s = A z + beta s  (= A p)
                            pn4[k] = pn;
                            Sv(li, k, row) = sn_;
                            dacc_f[k] = fmaf(pn, sn_, dacc_f[k]);
                        }
#pragma unroll
                        for (int k = 0; k < K; ++k) {
                            if constexpr (RES < 2) {
                                st_owned_f32(&X(li, k, row), xn[k], xp_pol);
                                st_owned_f32(&P(li, k, row), pn4[k], xp_pol);
                            } else {
                                X(li, k, row) = xn[k];
                                P(li, k, row) = pn4[k];
                            }
                        }
                    });
                double dacc[K];
#pragma unroll
                for (int k = 0; k < K; ++k) dacc[k] = (double)dacc_f[k];
                if (prof) { const long long t1 = clock64(); tA += t1 - t0; t0 = t1; }
                auto postA = [&](const double d, const double) {   // alpha_k = gamma_k / delta_k, one lane per column
                    bool bad = false;
                    if (lane < K) {
                        const bool conv = S->conv[lane] != 0, ok = d > 0.0;
                        if (!conv && ok) S->e_dl[lane] = exp2_of(d);
                        bad = !conv && !ok;      // not SPD / NaN: finish the update with alpha = 0, then stop
                        S->alpha[lane] = (conv || !ok) ? 0.f : (float)(S->gam[lane] / d);
                    }
                    const bool anybad = __any_sync(0xffffffffu, bad);
                    if (lane == 0 && anybad) S->status = 3;
                };
                sync.template allreduce<K, K, false>(dacc, S->e_dl, S->skipA, true, postA);
                if (prof) { const long long t1 = clock64(); tS2 += t1 - t0; t0 = t1; }
            }
            // ------------------------------------------------ phase B: r -= alpha s; z = D^-1 r (published); r.z, r.r
            {
                float alpha[K];
#pragma unroll
                for (int k = 0; k < K; ++k) alpha[k] = S->alpha[k];
                double acc2[2 * K];
#pragma unroll
                for (int i = 0; i < 2 * K; ++i) acc2[i] = 0.0;
                bool preconditioned = false;
                if constexpr (CHEB) {
                    if (cheb_m > 1) {
                        for (int s = s_begin + warp; s < s_end; s += NW) {
                            const int li = s - s_begin, row = s * 32 + lane;
#pragma unroll
                            for (int k = 0; k < K; ++k) R(li, k, row) = fmaf(-alpha[k], Sv(li, k, row), R(li, k, row));
                        }
                        __syncwarp();
                        cheb_first();
                        cheb_steps(acc2);
                        preconditioned = true;
                    }
                }
                if (!preconditioned)
                for (int s = s_begin + warp; s < s_end; s += NW) {
                    const int li = s - s_begin, row = s * 32 + lane;
                    const float di = Dv(li, row);
                    float zz[4] = {0.f, 0.f, 0.f, 0.f}, rn[K];
#pragma unroll
                    for (int k = 0; k < K; ++k) {
                        rn[k] = fmaf(-alpha[k], Sv(li, k, row), R(li, k, row));
                        R(li, k, row) = rn[k];
                        zz[k] = di * rn[k];
                    }
                    ZstP(row, zz);             // (rounds zz to the published values when ZH)
#pragma unroll
                    for (int k = 0; k < K; ++k) {
                        acc2[k] += (double)(rn[k] * zz[k]);
                        acc2[K + k] += (double)(rn[k] * rn[k]);
                    }
                }
                if (prof) { const long long t1 = clock64(); tB += t1 - t0; t0 = t1; }
                auto postB = [&](const double gn, const double rrn) {   // beta, convergence, stop decision
                    bool bad = false, cvk = true;
                    if (lane < K) {
                        if (S->conv[lane]) {
                            S->beta[lane] = 0.f;
                        } else {
                            if (gn > 0.0) S->e_grr[lane] = exp2_of(gn);
                            if (rrn > 0.0) S->e_grr[K + lane] = exp2_of(rrn);
                            if (!(gn == gn)) bad = true;
                            const double g_old = S->gam[lane];
                            float be = (g_old > 0.0) ? (float)(gn / g_old) : 0.f;
                            S->gam[lane] = gn;
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
                        const int it = S->it + 1;
                        S->it = it;
                        if (anybad || S->status == 3) S->status = 3;
                        else if (all) S->status = 1;
                        else if (it >= a.maxit) S->status = 2;
                        S->stop = S->status != 0;
                    }
                };
                prologue();   // next phase A's first entries fly while the all-reduce completes
                sync.template allreduce<2 * K, K, true>(acc2, S->e_grr, S->skipB, true, postB);
                if (prof) { const long long t1 = clock64(); tS1 += t1 - t0; t0 = t1; }
            }
        }
        // ---------------------------------------------------------------- the last iteration's x += alpha p is still pending
        if (prof) t0 = clock64();
        {
            const bool pending = S->it > 0;
            float alpha[K];
#pragma unroll
            for (int k = 0; k < K; ++k) alpha[k] = pending ? S->alpha[k] : 0.f;
            for (int s = s_begin + warp; s < s_end; s += NW) {
                const int li = s - s_begin, row = s * 32 + lane;
#pragma unroll
                for (int k = 0; k < K; ++k) X(li, k, row) = fmaf(alpha[k], P(li, k, row), X(li, k, row));
            }
        }
        __syncthreads();
        const bool check = (S->status == 1) && (a.refine > 0) && (S->checks <= a.refine) && (S->it > 0);
        if (!check) break;
        sync.barrier();           // all gathers of z are over before the buffer is reused for the x rows
        restart_from_x(false);
        if (prof) { const long long t1 = clock64(); tX += t1 - t0; t0 = t1; }
        if (S->stop) break;
    }

    if (prof) {
        if (cta == 0) {
            a.dbg[0] = tA; a.dbg[1] = tS2; a.dbg[2] = tB; a.dbg[3] = tS1; a.dbg[4] = tX; a.dbg[5] = 0; a.dbg[6] = S->restarts; a.dbg[7] = S->it;
        }
        long long *rowd = a.dbg + 8 + 8 * (size_t)cta;
        unsigned int smid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        rowd[0] = tA; rowd[1] = tS2; rowd[2] = tB; rowd[3] = tS1; rowd[4] = tX; rowd[5] = 0; rowd[6] = smid; rowd[7] = S->it;
    }

    // ---------------------------------------------------------------- result: x -> caller layout
    for (int s = s_begin + warp; s < s_end; s += NW) {
        const int li = s - s_begin, row = s * 32 + lane;
        if (row < a.V) {
            const long long io = a.perm ? a.perm[row] : row;
#pragma unroll
            for (int k = 0; k < K; ++k)
                if (k < kb) a.out[io * kb + k] = X(li, k, row);
        }
    }
    if (cta == 0 && tid == 0 && a.info) {
        a.info[0] = (float)S->it;
        a.info[1] = (float)S->status;
        for (int k = 0; k < 4; ++k) a.info[2 + k] = (k < K && S->bb[k] > 0.0) ? (float)sqrt(S->rr[k] / S->bb[k]) : 0.f;
        a.info[6] = (float)S->restarts;
        a.info[7] = 0.f;
    }
    if constexpr (SYNC == 1) sync.barrier();   // no CTA of the cluster may exit while another can still write into its shared memory
}

#ifndef LS_ZH
#define LS_ZH 1   // publish the preconditioned residual as bf16 rows ("ZH" above); -DLS_ZH=0 builds the fp32-row variant for A/B
#endif
// The instantiation rule of pcg_fused_kernel, for every ls_fused_*.cu: ZH for the 3-column Jacobi instantiations that publish
// through global or distributed shared memory.  Chebyshev keeps fp32 rows (its iterates need full precision), and so does RES 3,
// whose one CTA keeps its rows in its own shared memory.
template <int K, int RES, int NW, bool PAT, int SYNC, bool PROF, bool CHEB = false, bool BATCH = false>
const void *fused_fn() {
    constexpr bool ZH = (LS_ZH != 0) && K == 3 && !CHEB && RES != 3;
    return (const void *)pcg_fused_kernel<K, RES, NW, PAT, SYNC, PROF, CHEB, ZH, BATCH>;
}

}  // namespace lsf
