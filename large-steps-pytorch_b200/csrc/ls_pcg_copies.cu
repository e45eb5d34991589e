// ls_pcg_copies.cu -- the solver's matrix copies, built by ls_pcg_create (build_solver) from the caller's CSR: the CSR copy, optionally
// re-ordered P A P^T, with its padding and dinv; the SELL-32 copy; the pattern-only copy of a matrix with one off-diagonal value;
// the Gershgorin bound and the Chebyshev coefficients.  The formats, and the kernels that read them, are in ls_sell_kernel.cuh.
#include <string.h>
#include "ls_pcg_handle.h"

using namespace lspcg;

namespace {

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

namespace lspcg {

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

// SELL-32 copy of the solver's CSR (the fast SpMM engine's and the fused solver's).  Whether it is used depends on its padded
// size, which the readback brings.
int sell_copy(PcgHandle *h, cudaStream_t stream) {
    const unsigned wb = (unsigned)(((int64_t)h->nslices * 32 + 255) / 256);
    lsk::sell_width_kernel<<<wb, 256, 0, stream>>>((int)h->V, h->nslices, h->rowptr, h->soff);
    LS_LAUNCH_CHECK();
    const int rc = ls_exclusive_scan_i32(h->soff, h->soff, h->nslices, h->scan, stream);
    if (rc) return rc;
    lsk::sell_fill_kernel<<<wb, 256, 0, stream>>>((int)h->V, h->nslices, h->rowptr, h->col, h->val, h->soff, h->ent, h->sell_cap);
    LS_LAUNCH_CHECK();
    return LS_OK;
}

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

}  // namespace lspcg

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
