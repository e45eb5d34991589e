// ls_sell_kernel.cuh -- in-solver SpMM engine on a SELL-32 copy of the CSR (sm_90a).
//
// Why a second engine: ncu + a gather-less diagnostic showed the TMA-staged CSR kernel is *instruction-issue bound*
// (253 instructions per 7-entry row: per-lane row-length predication, two LDS and three 64-bit address computations +
// three LDG per non-zero), not memory bound.
//
// SELL-32 ("sliced ELLPACK", slice height 32 = one warp): the rows of a slice are padded to the slice's longest row
// and stored column-major, entry (j, lane) at ent[soff[s] + 32 j + lane] as an int2 {col, val bits}.  Consequences:
//   * the row loop is warp-uniform (no per-lane predication); padded entries are {own row, 0.0f};
//   * one coalesced 8-byte load per entry (256 B per warp per slot), streamed with L1::no_allocate;
//   * the gathered vector p is stored as rows of PW floats (float4 for K=3,4): one LDG.128 and one address per entry
//     instead of three of each;  ~75 instructions per row instead of 253.
// The next slice's entries are prefetched into registers while the current slice's gathers are in flight.
// Bytes streamed per launch: 8 nnz_padded + 4 (V/32+1) + 4 PW V (gather, once) + 4 K V (y) -- within a few % of the
// CSR algorithmic bytes (padding is ~0.2 % on the plane, <= 15 % on irregular meshes; above 1.5x the CSR engine is used).
#pragma once
#include "ls_common.cuh"

namespace lsk {

#ifndef LS_SELL_THREADS
#define LS_SELL_THREADS 768
#endif
constexpr int SELL_THREADS = LS_SELL_THREADS;   // one CTA per SM, 24 warps, <= 85 registers (same shape as the persistent solver's phase A)
constexpr int SELL_WARPS = SELL_THREADS / 32;

struct SellArgs {
    int V;
    int nslices;
    const int *soff;        // [nslices + 1] entry offsets (multiples of 32)
    const int2 *ent;        // [soff[nslices]] {col, float bits}
    const float *p;         // gathered vector, rows of PW floats
    float *y;               // K planes of ldy floats (SoA)
    long long ldy;
    const int *done;        // optional early-exit flag
    double *partials;       // [K][gridDim.x]
    unsigned int *ticket;
    double *dot_out;        // [K]
    int pf_halo;            // TMA kernel: rows of p beyond the CTA's own range to pull into L2 with a bulk prefetch (0 = off)
};

template <int K> struct PRow;
template <> struct PRow<1> { typedef float T; static constexpr int PW = 1; };
template <> struct PRow<2> { typedef float2 T; static constexpr int PW = 2; };
template <> struct PRow<3> { typedef float4 T; static constexpr int PW = 4; };
template <> struct PRow<4> { typedef float4 T; static constexpr int PW = 4; };

__device__ __forceinline__ void prow_get(const float &v, float (&o)[1]) { o[0] = v; }
__device__ __forceinline__ void prow_get(const float2 &v, float (&o)[2]) { o[0] = v.x; o[1] = v.y; }
__device__ __forceinline__ void prow_get(const float4 &v, float (&o)[3]) { o[0] = v.x; o[1] = v.y; o[2] = v.z; }
__device__ __forceinline__ void prow_get(const float4 &v, float (&o)[4]) { o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w; }

// streaming 8-byte load of a matrix entry: read-only path, do not allocate in L1 (the gathers own L1)
__device__ __forceinline__ int2 ld_entry(const int2 *p) {
    int2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.s32 {%0, %1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
    return r;
}

// L2 prefetch of the entries two slices ahead of this warp (the register prefetch covers one slice ahead): costs no
// registers, turns the register prefetch's HBM miss into an L2 hit.  The address is extrapolated from the last two slice
// offsets (slices of a mesh have near-constant width); a wrong guess only prefetches a neighbouring line.
#ifndef LS_PF2
#define LS_PF2 0   // A/B: no gain HBM-cold for the stand-alone kernel, and a slower persistent solve (more spills)
#endif
__device__ __forceinline__ void prefetch_entries_l2(const int2 *ent, long long off, long long limit, int lane) {
    if (LS_PF2 && off >= 0 && off + 256 <= limit) {
#pragma unroll
        for (int u = 0; u < 8; ++u) asm volatile("prefetch.global.L2 [%0];" ::"l"(ent + off + u * 32 + lane));
    }
}

template <int K, bool DOT>
__global__ void __launch_bounds__(SELL_THREADS, 1) spmm_sell_kernel(const SellArgs a) {
    typedef typename PRow<K>::T PT;
    constexpr int U = 8;
    __shared__ double red[K * 32 + K + 1];
    if (a.done != nullptr && *reinterpret_cast<const volatile int *>(a.done) != 0) return;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int G = gridDim.x, cta = blockIdx.x;
    // contiguous chunk of slices per CTA; its warps interleave over the chunk
    const int s_begin = (int)((long long)a.nslices * cta / G);
    const int s_end = (int)((long long)a.nslices * (cta + 1) / G);
    const PT *__restrict__ prow = reinterpret_cast<const PT *>(a.p);
    const long long limit = a.soff[a.nslices];

    double dacc[K];
#pragma unroll
    for (int k = 0; k < K; ++k) dacc[k] = 0.0;

    int s = s_begin + warp;
    int o0 = 0, o1 = 0;
    int2 nv[U];
    if (s < s_end) {
        o0 = a.soff[s];
        o1 = a.soff[s + 1];
        const int w = (o1 - o0) >> 5;
        const int2 *e = a.ent + o0 + lane;
#pragma unroll
        for (int u = 0; u < U; ++u) nv[u] = (u < w) ? ld_entry(e + u * 32) : make_int2(s * 32 + lane, 0);
    }
    while (s < s_end) {
        const int row = s * 32 + lane;
        const int w = (o1 - o0) >> 5;
        const int2 *e = a.ent + o0 + lane;
        int2 cv[U];
#pragma unroll
        for (int u = 0; u < U; ++u) cv[u] = nv[u];
        // prefetch the first U entries of this warp's next slice
        const int sn = s + SELL_WARPS;
        int n0 = 0, n1 = 0;
        if (sn < s_end) {
            n0 = a.soff[sn];
            n1 = a.soff[sn + 1];
            if (sn + SELL_WARPS < s_end) prefetch_entries_l2(a.ent, (long long)n0 + (n0 - o0), limit, lane);
        }
        float acc[K];
#pragma unroll
        for (int k = 0; k < K; ++k) acc[k] = 0.f;
        // first pass uses the prefetched entries
        {
            PT xv[U];
#pragma unroll
            for (int u = 0; u < U; ++u) xv[u] = prow[cv[u].x];
            if (sn < s_end) {
                const int wn = (n1 - n0) >> 5;
                const int2 *en = a.ent + n0 + lane;
#pragma unroll
                for (int u = 0; u < U; ++u) nv[u] = (u < wn) ? ld_entry(en + u * 32) : make_int2(sn * 32 + lane, 0);
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                float xk[K];
                prow_get(xv[u], xk);
                const float wv = __int_as_float(cv[u].y);
#pragma unroll
                for (int k = 0; k < K; ++k) acc[k] = fmaf(wv, xk[k], acc[k]);
            }
        }
        // slices wider than U (rare on meshes): remaining passes load their entries directly
        for (int j = U; j < w; j += U) {
#pragma unroll
            for (int u = 0; u < U; ++u) cv[u] = (j + u < w) ? ld_entry(e + (j + u) * 32) : make_int2(row, 0);
            PT xv[U];
#pragma unroll
            for (int u = 0; u < U; ++u) xv[u] = prow[cv[u].x];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                float xk[K];
                prow_get(xv[u], xk);
                const float wv = __int_as_float(cv[u].y);
#pragma unroll
                for (int k = 0; k < K; ++k) acc[k] = fmaf(wv, xk[k], acc[k]);
            }
        }
#pragma unroll
        for (int k = 0; k < K; ++k) a.y[(size_t)k * a.ldy + row] = acc[k];   // planes are padded to 32: no guard
        if (DOT) {
            float xr[K];
            prow_get(prow[row], xr);
#pragma unroll
            for (int k = 0; k < K; ++k) dacc[k] += (double)xr[k] * (double)acc[k];
        }
        s = sn;
        o0 = n0;
        o1 = n1;
    }
    if (DOT) {
        double tot[K];
        const bool last = ls_grid_reduce<K>(dacc, tot, a.partials, a.ticket, red, tid, SELL_THREADS, 1, cta, G);
        if (last && tid == 0) {
#pragma unroll
            for (int k = 0; k < K; ++k) a.dot_out[k] = tot[k];
        }
    }
}

// ---- TMA-staged variant: the entry stream goes HBM -> shared memory through per-warp rings of 1-D bulk copies ----------
// The register-prefetch kernel above keeps 24 warps x 2 KB of matrix stream in flight per SM and spends 16 registers per
// thread on it; it is latency-bound (ncu at V = 1e6: warps active 37 %, long-scoreboard 16 stalls/issue, DRAM 58 % busy).
// Here every warp owns a private ring of DEPTH slots of 2 KB in shared memory.  Lane 0 issues one cp.async.bulk per slice
// (the first <= 8 entry columns of a slice are 256 w contiguous bytes) DEPTH slices ahead; completion is counted on one
// mbarrier per slot.  Only the owning warp ever touches its slots, so there is no CTA-level synchronisation and no
// "empty" barrier: a slot is refilled by the same warp right after it has issued the gathers that consumed its column
// indices (those gathers cannot issue before the LDS results exist).  NW x DEPTH x 2 KB = 192 KB of matrix stream in
// flight per SM, no prefetch registers, so 32 warps fit.  Columns beyond the 8th of a wide slice (rare on meshes) are read
// straight from global memory as before.  The kernel is PDL-aware: it lets the next kernel of the stream start its own
// matrix prefetch early (griddepcontrol.launch_dependents) and touches the vectors only after griddepcontrol.wait.
constexpr int SELL_SLOT_BYTES = 2048;   // 8 entry columns x 32 lanes x 8 bytes

inline size_t sell_tma_smem_bytes(int nw, int depth) {
    return (size_t)nw * depth * SELL_SLOT_BYTES + (size_t)nw * depth * 8 + 2048;   // rings, mbarriers, reduction scratch
}

template <int K, bool DOT, int NW, int DEPTH, int MINB = 1>
__global__ void __launch_bounds__(NW * 32, MINB) spmm_sell_tma_kernel(const SellArgs a) {
    typedef typename PRow<K>::T PT;
    constexpr int U = 8;
    extern __shared__ __align__(128) unsigned char sm_raw[];
    int2 *ring = reinterpret_cast<int2 *>(sm_raw);                                         // [NW][DEPTH][256]
    uint64_t *bars = reinterpret_cast<uint64_t *>(sm_raw + (size_t)NW * DEPTH * SELL_SLOT_BYTES);   // [NW][DEPTH]
    double *red = reinterpret_cast<double *>(sm_raw + (size_t)NW * DEPTH * SELL_SLOT_BYTES + (size_t)NW * DEPTH * 8);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int G = gridDim.x, cta = blockIdx.x;
    const int s_begin = (int)((long long)a.nslices * cta / G);
    const int s_end = (int)((long long)a.nslices * (cta + 1) / G);
    const PT *__restrict__ prow = reinterpret_cast<const PT *>(a.p);
    int2 *myring = ring + (size_t)warp * DEPTH * 256;
    uint64_t *mybar = bars + warp * DEPTH;

    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    if (lane == 0) {
#pragma unroll
        for (int d = 0; d < DEPTH; ++d) ls_mbar_init(mybar + d, 1);
    }
    ls_fence_mbar_init();
    __syncwarp();

    // this warp's slices: s_begin + warp + i NW, i = 0 .. n - 1
    const int n = (s_end - s_begin - warp + NW - 1) / NW;   // may be <= 0
    // slice offsets, 32 slices at a time: lane l holds soff of slice i0 + l and of its successor
    int win_i0 = 0, so0 = 0, so1 = 0;
    auto load_window = [&](int i0) {
        const int i = i0 + lane;
        if (i < n) {
            const int s = s_begin + warp + i * NW;
            so0 = a.soff[s];
            so1 = a.soff[s + 1];
        } else {
            so0 = so1 = 0;
        }
        win_i0 = i0;
    };
    uint64_t policy = ls_policy_evict_first();
    auto issue = [&](int i) {   // warp-uniform; window must cover i
        const int o0 = __shfl_sync(0xffffffffu, so0, i - win_i0), o1 = __shfl_sync(0xffffffffu, so1, i - win_i0);
        const int w = (o1 - o0) >> 5;
        const int cw = w < U ? w : U;
        if (lane == 0) {
            uint64_t *bar = mybar + (i % DEPTH);
            ls_mbar_expect_tx(bar, (uint32_t)(cw * 256));
            if (cw > 0) ls_bulk_g2s_hint(myring + (size_t)(i % DEPTH) * 256, a.ent + o0, (uint32_t)(cw * 256), bar, policy);
        }
    };
    if (n > 0) {
        load_window(0);
#pragma unroll
        for (int d = 0; d < DEPTH; ++d)
            if (d < n) issue(d);
    }
    // the matrix never changes between launches; the vectors do: wait for the previous kernel before touching them
    asm volatile("griddepcontrol.wait;" ::: "memory");
    if (a.pf_halo > 0 && warp < 8) {
        // HBM-cold launches: every slice's gathers used to wait a full DRAM round trip for the first touch of its p lines
        // (~2 us x 6.6 slices per warp).  The rows this CTA gathers are its own range plus a halo: pull them into L2 with a
        // handful of bulk prefetches (UBLKPF.L2) so that the gathers that follow hit L2.
        const long long r0 = max(0LL, (long long)s_begin * 32 - a.pf_halo), r1 = min((long long)a.nslices * 32, (long long)s_end * 32 + a.pf_halo);
        const long long bytes = (r1 - r0) * (long long)sizeof(PT);
        const char *base = reinterpret_cast<const char *>(a.p) + r0 * (long long)sizeof(PT);
        constexpr int CH = 16384;
        for (long long off = (long long)warp * CH; off < bytes; off += 8LL * CH) {
            const unsigned int nb = (unsigned int)min((long long)CH, bytes - off) & ~15u;
            if (lane == 0 && nb > 0) asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(base + off), "r"(nb) : "memory");
        }
    }
    if (a.done != nullptr && *reinterpret_cast<const volatile int *>(a.done) != 0) {
        // converged earlier in this graph chunk: nothing to do, but the bulk copies already in flight must land before the
        // CTA (and its shared memory) goes away
#pragma unroll
        for (int d = 0; d < DEPTH; ++d)
            if (d < n) ls_mbar_wait(mybar + d, 0u);
        return;
    }

    double dacc[K];
#pragma unroll
    for (int k = 0; k < K; ++k) dacc[k] = 0.0;

    // consumer side needs the offsets of slice i (window A) while the producer side runs DEPTH ahead (window B = so0/so1)
    int c_i0 = 0, c0 = 0, c1 = 0;
    auto load_cwindow = [&](int i0) {
        const int i = i0 + lane;
        if (i < n) {
            const int s = s_begin + warp + i * NW;
            c0 = a.soff[s];
            c1 = a.soff[s + 1];
        } else {
            c0 = c1 = 0;
        }
        c_i0 = i0;
    };
    if (n > 0) load_cwindow(0);
    for (int i = 0; i < n; ++i) {
        if (i - c_i0 >= 32) load_cwindow(i);
        const int s = s_begin + warp + i * NW;
        const int row = s * 32 + lane;
        const int o0 = __shfl_sync(0xffffffffu, c0, i - c_i0), o1 = __shfl_sync(0xffffffffu, c1, i - c_i0);
        const int w = (o1 - o0) >> 5;
        const int slot = i % DEPTH;
        ls_mbar_wait(mybar + slot, (uint32_t)((i / DEPTH) & 1));
        const int2 *e_s = myring + (size_t)slot * 256 + lane;
        int2 cv[U];
#pragma unroll
        for (int u = 0; u < U; ++u) cv[u] = (u < w) ? e_s[u * 32] : make_int2(row, 0);
        float acc[K];
#pragma unroll
        for (int k = 0; k < K; ++k) acc[k] = 0.f;
        {
            PT xv[U];
#pragma unroll
            for (int u = 0; u < U; ++u) xv[u] = prow[cv[u].x];
            // the gathers above could only issue once every LDS of this slot had returned: the slot is free, refill it
            __syncwarp();
            if (i + DEPTH < n) {
                if (i + DEPTH - win_i0 >= 32) load_window(i + DEPTH);
                issue(i + DEPTH);
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                float xk[K];
                prow_get(xv[u], xk);
                const float wv = __int_as_float(cv[u].y);
#pragma unroll
                for (int k = 0; k < K; ++k) acc[k] = fmaf(wv, xk[k], acc[k]);
            }
        }
        const int2 *e = a.ent + o0 + lane;
        for (int j = U; j < w; j += U) {   // wide slices: remaining columns straight from global memory
#pragma unroll
            for (int u = 0; u < U; ++u) cv[u] = (j + u < w) ? ld_entry(e + (j + u) * 32) : make_int2(row, 0);
            PT xv[U];
#pragma unroll
            for (int u = 0; u < U; ++u) xv[u] = prow[cv[u].x];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                float xk[K];
                prow_get(xv[u], xk);
                const float wv = __int_as_float(cv[u].y);
#pragma unroll
                for (int k = 0; k < K; ++k) acc[k] = fmaf(wv, xk[k], acc[k]);
            }
        }
#pragma unroll
        for (int k = 0; k < K; ++k) a.y[(size_t)k * a.ldy + row] = acc[k];
        if (DOT) {
            float xr[K];
            prow_get(prow[row], xr);
#pragma unroll
            for (int k = 0; k < K; ++k) dacc[k] += (double)xr[k] * (double)acc[k];
        }
    }
    if (DOT) {
        double tot[K];
        const bool last = ls_grid_reduce<K>(dacc, tot, a.partials, a.ticket, red, tid, NW * 32, 1, cta, G);
        if (last && tid == 0) {
#pragma unroll
            for (int k = 0; k < K; ++k) a.dot_out[k] = tot[k];
        }
    }
}

// ---- pattern-only SELL-32 ("PAT"): matrices whose off-diagonal entries all carry the same value ---------------------
// M = I + lambda L with the uniform (combinatorial) Laplacian -- the reference's default, geometry.py:112-133 -- has
// M_ij = -lambda for every edge: only the diagonal differs from row to row.  For such matrices the solver streams column
// indices alone and leaves the diagonal out of the gather list (the owner loads its own p row anyway):
//   (M p)_i = d'_i p_i + c * sum_{j in slots(i)} p_j .
// Layout: pc is an array of 32-bit words; slice s starts at word poff[s] & ~31 and holds w2 "pairs" per row (slots 2m and
// 2m+1 of row 32 s + lane), pair (m, lane) read by one load per lane:
//   compact slice (bit 0 of poff[s] clear): one word per pair, two signed 16-bit offsets from the row, col = row + (int16)half;
//   wide slice (bit 0 set, some |col - row| > 32767): two words per pair, the columns themselves (8-byte aligned: every slice
//   is a multiple of 32 words long).
// Bits 1-4 of poff[s] hold w2; the value PAT_W2_ESC means "w2 >= 15: the slice ends where poff[s + 1] starts".  So a slice's
// width does not depend on where the next slice lies, and compact slices with identical words share one stored copy
// (ls_pcg_copies.cu, pat_hash_kernel .. pat_share_copy_kernel): a mesh in native order has a handful of distinct slices (12 of 31 250 on the
// 1000 x 1000 plane), which then stay in L1 instead of streaming ~12 MB through L2 per gather pass.  Wide slices, escape
// slices and the slice after an escape slice (whose offset ends the escape slice) always keep their own copy.
// Meshes in native order are compact throughout (a plane of n x n vertices has |col - row| <= n + 1); a reordered large mesh
// keeps wide pairs only on the slices whose neighbours lie far away.  Unused slots point at the row itself (offset 0) and are
// paid back in the diagonal: d'_i = M_ii - c * (unused slots of row i), so the inner loop has no per-lane predicate.
// Diagonal classes: a row's (D^-1_ii, d'_i) is one of a few pairs (a function of valence and slice padding), so the solver
// keeps a 1-byte class per row and a table of at most PAT_CLASSES pairs, keyed on their bit patterns (the exact floats: the
// arithmetic does not change).  More classes than that: the matrix takes the general copy.
// On by default since round 2 (LS_PCG_PATTERN=0 keeps the general copy); detection is exact (bitwise equality of all off-diagonal values).
constexpr int PAT_CLASSES = 256;
constexpr unsigned long long PAT_EMPTY = ~0ull;   // unused table slot (bits of two NaNs no matrix of ours produces: such a row overflows)

constexpr int PAT_W2_ESC = 15;   // bits 1-4 of a slice offset: w2, or this value for w2 >= 15

struct PatSlice {
    int o0;      // first word
    int w2;      // pairs per row
    bool wide;   // two words per pair (columns) instead of one (16-bit offsets)
};
__host__ __device__ __forceinline__ int pat_word(int o0, int w2, bool wide) {
    return o0 | ((w2 < PAT_W2_ESC ? w2 : PAT_W2_ESC) << 1) | (wide ? 1 : 0);
}
// slice at po[0]; po[1] is read only for an escape slice (w2 >= 15), whose next slice always starts right after it
__host__ __device__ __forceinline__ PatSlice pat_slice(const int *po) {
    const int p0 = po[0], p1 = po[1];
    const bool wide = (p0 & 1) != 0;
    const int o0 = p0 & ~31, f = (p0 >> 1) & 15;
    return {o0, f < PAT_W2_ESC ? f : ((p1 & ~31) - o0) >> (wide ? 6 : 5), wide};
}
// pair m of the row `row` as stored (compact: the word in .x), {0, 0} / {row, row} past the slice width.  The caller keeps it
// raw until the gathers need the columns (pat_cols), so that the load stays in flight.  keep: cache in L1 (single CTA / cluster,
// or a shared copy whose few KB every CTA reads over and over); else stream past L1, which the gathers own.
__device__ __forceinline__ int2 pat_load(const unsigned int *pc, const PatSlice &ps, int m, int row, int lane, bool keep) {
    int2 r = ps.wide ? make_int2(row, row) : make_int2(0, 0);
    if (m < ps.w2) {
        if (ps.wide) {
            const int2 *p = reinterpret_cast<const int2 *>(pc + ps.o0) + m * 32 + lane;
            if (keep) asm volatile("ld.global.nc.v2.s32 {%0, %1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
            else asm volatile("ld.global.nc.L1::no_allocate.v2.s32 {%0, %1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
        } else {
            const unsigned int *p = pc + ps.o0 + m * 32 + lane;
            if (keep) asm volatile("ld.global.nc.s32 %0, [%1];" : "=r"(r.x) : "l"(p));
            else asm volatile("ld.global.nc.L1::no_allocate.s32 %0, [%1];" : "=r"(r.x) : "l"(p));
        }
    }
    return r;
}
__device__ __forceinline__ int2 pat_cols(const int2 raw, bool wide, int row) {
    return wide ? raw : make_int2(row + (int)(short)raw.x, row + (raw.x >> 16));
}

// sharing pays (fewer slices stored) and fits the scratch: decided alike by the build kernels and by the host that reads
// back what they stored
__host__ __device__ __forceinline__ bool pat_share_on(int nslices, int stored, int words, long long cap_scr) {
    return stored < nslices && (long long)words <= cap_scr;
}

}  // namespace lsk
