// ls_common.cuh -- shared helpers for libls_b200 (sm_90a: H100).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include "../../include/largesteps_b200.h"
#include "../../include/largesteps_b200_diag.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libls_b200 is written for sm_90a (Hopper H100) only"
#endif

// ---- host-side error plumbing ---------------------------------------------------------------------
void ls_set_error(const char *fmt, ...);
extern std::atomic<uint64_t> g_ls_launches;

#define LS_CUDA_TRY(expr)                                                                          \
    do {                                                                                           \
        cudaError_t _e = (expr);                                                                   \
        if (_e != cudaSuccess) {                                                                   \
            ls_set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return LS_ERR_CUDA;                                                                    \
        }                                                                                          \
    } while (0)

#define LS_REQUIRE(cond, msg)                                                                      \
    do {                                                                                           \
        if (!(cond)) {                                                                             \
            ls_set_error("bad argument: %s  [%s] (%s:%d)", msg, #cond, __FILE__, __LINE__);        \
            return LS_ERR_BAD_ARG;                                                                 \
        }                                                                                          \
    } while (0)

// count + check a kernel launch
#define LS_LAUNCH_CHECK()                                                                          \
    do {                                                                                           \
        g_ls_launches.fetch_add(1, std::memory_order_relaxed);                                     \
        LS_CUDA_TRY(cudaGetLastError());                                                           \
    } while (0)

static inline size_t ls_align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Correctly rounded float32 operations that nvcc cannot contract into an FMA, for bodies that repeat a reference's float32
// operation order.  On the host (the CPU test harnesses) they are the plain operators.
__host__ __device__ __forceinline__ float add_rn(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}
__host__ __device__ __forceinline__ float sub_rn(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fsub_rn(a, b);
#else
    return a - b;
#endif
}
__host__ __device__ __forceinline__ float mul_rn(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ __forceinline__ float sqrt_rn(float a) {
#ifdef __CUDA_ARCH__
    return __fsqrt_rn(a);
#else
    return sqrtf(a);
#endif
}

// device properties cached per process (current device)
struct LsDevInfo {
    int device;
    int sm_count;
    int max_smem_optin;
    int cc_major;
};
int ls_dev_info(LsDevInfo *out);

// exclusive prefix sum over int32 (n elements, out[n] receives the total): host launcher
// scratch: device ints, >= ls_scan_scratch_elems(n)
size_t ls_scan_scratch_elems(int64_t n);
int ls_exclusive_scan_i32(const int *in, int *out, int64_t n, int *scratch, cudaStream_t stream);

// ls_face_incidence on int32 faces without its read-back: rows with a negative index are skipped, not flagged.  workspace:
// ls_bucket_workspace_bytes(V) (ls_glue.cu)
int ls_face_buckets_i32_async(const int32_t *faces, int64_t F, int64_t V, int32_t *inc_ptr, int32_t *inc, void *workspace,
                              cudaStream_t stream);

// the same without a read-back for int32 / int64 keys (key_bytes 4 or 8): per_face = 1 buckets the 3F corners of faces by
// vertex (items 4 f + c, as ls_face_incidence), per_face = 0 the positions of an index vector by key (as ls_index_buckets).
// Keys outside [0, nkeys) are skipped.  workspace: ls_bucket_workspace_bytes(nkeys) (ls_glue.cu)
int ls_buckets_async(const void *keys, int key_bytes, int64_t n, int64_t nkeys, int per_face, int32_t *ptr, int32_t *items,
                     void *workspace, cudaStream_t stream);

// ls_order_morton over B segments of the points at once (offsets: B + 1 device int64, NULL when B == 1): each segment is
// ordered along the Morton curve of its own bounding box, the segments one after the other; B == 1 is ls_order_morton.
// workspace: ls_order_seg_workspace_bytes(V, B) (ls_order.cu)
#define LS_ORDER_MAX_SEGMENTS (1 << 24)
int ls_order_seg_workspace_bytes(int64_t V, int64_t B, size_t *bytes_out);
int ls_order_morton_seg(const float *points, int64_t V, const int64_t *offsets, int64_t B, int32_t *perm_new2old,
                        void *workspace, size_t workspace_bytes, cudaStream_t stream);

// after ls_order_morton_seg(points, V, ..., B, ..., workspace, ...): each point's bucket s * 8^bits + Morton cell code, indexed
// by point id, and the segments' bounding boxes in ls_morton.cuh's f2ord encoding, lo [3B] then hi [3B] (ls_order.cu)
void ls_order_views(const void *workspace, int64_t V, int64_t B, const unsigned int **code, const unsigned int **bbox);

// ---- device helpers -------------------------------------------------------------------------------
#ifdef __CUDACC__

__device__ __forceinline__ uint32_t ls_smem_u32(const void *p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// mbarrier + 1-D TMA bulk copy (cp.async.bulk -> SASS UBLKCP)
__device__ __forceinline__ void ls_mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(ls_smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void ls_fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void ls_mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(ls_smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void ls_mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(ls_smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool ls_mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(ls_smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void ls_mbar_wait(uint64_t *bar, uint32_t parity) {
    while (!ls_mbar_try_wait(bar, parity)) {
    }
}
// global -> shared bulk copy, completion counted in bytes on `bar`.  dst/src 16-byte aligned, bytes % 16 == 0.
__device__ __forceinline__ void ls_bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     ls_smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(ls_smem_u32(bar))
                 : "memory");
}
// same with an L2 cache-policy operand
__device__ __forceinline__ void ls_bulk_g2s_hint(void *dst_smem, const void *src_gmem, uint32_t bytes,
                                                 uint64_t *bar, uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::
            "r"(ls_smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(ls_smem_u32(bar)), "l"(policy)
        : "memory");
}
__device__ __forceinline__ uint64_t ls_policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t ls_policy_evict_last() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ void ls_named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

__device__ __forceinline__ double ls_warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Deterministic grid-wide sum of NV doubles per CTA.
//   Every CTA: block-reduce its per-thread values (fixed order), write them to partials[v][cta], take a ticket.
//   The CTA that draws the last ticket re-reduces all partials in a fixed order, so the result does not depend
//   on CTA completion order (bit-reproducible CG trajectories), and resets the ticket for the next launch.
//   The re-reduction is spread over the warps of that CTA (one value per warp) with 8 independent L2 loads in
//   flight per lane: ~3 L2 round trips instead of one per partial (a serial loop here cost 17-25 us per kernel).
//   Returns true (uniformly across the calling threads) in the last CTA, with the totals in `tot[NV]` valid
//   for ALL threads of the group.  `nthreads` threads (multiple of 32, ids tid in [0,nthreads)) must call it
//   together; `bar_id` is the named barrier they may use; red_smem: >= (NV*32 + NV + 1) doubles.
//   partials: >= NV * ncta doubles, layout [v][cta].
template <int NV>
__device__ __forceinline__ bool ls_grid_reduce(double (&v)[NV], double (&tot)[NV], double *partials,
                                               unsigned int *ticket, double *red_smem, int tid, int nthreads,
                                               int bar_id, int cta, int ncta) {
    const int lane = tid & 31, warp = tid >> 5, nwarp = nthreads >> 5;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        double s = ls_warp_sum(v[i]);
        if (lane == 0) red_smem[i * 32 + warp] = s;
    }
    ls_named_bar_sync(bar_id, nthreads);
    int *flag = reinterpret_cast<int *>(red_smem + NV * 32 + NV);
    if (warp == 0) {
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            double s = (lane < nwarp) ? red_smem[i * 32 + lane] : 0.0;
            s = ls_warp_sum(s);
            if (lane == 0) partials[(size_t)i * ncta + cta] = s;
        }
        if (lane == 0) {
            __threadfence();
            const unsigned int t = atomicAdd(ticket, 1u);
            const int last = (t == (unsigned int)(ncta - 1));
            if (last) {
                __threadfence();
                *ticket = 0u;
            }
            *flag = last;
        }
    }
    ls_named_bar_sync(bar_id, nthreads);
    const bool is_last = (*flag != 0);
    if (is_last) {
        for (int i = warp; i < NV; i += nwarp) {
            const double *src = partials + (size_t)i * ncta;
            double s = 0.0;
            for (int c0 = 0; c0 < ncta; c0 += 256) {
                double t[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int c = c0 + j * 32 + lane;
                    t[j] = (c < ncta) ? __ldcg(src + c) : 0.0;
                }
#pragma unroll
                for (int j = 0; j < 8; ++j) s += t[j];
            }
            s = ls_warp_sum(s);
            if (lane == 0) red_smem[NV * 32 + i] = s;
        }
        ls_named_bar_sync(bar_id, nthreads);
#pragma unroll
        for (int i = 0; i < NV; ++i) tot[i] = red_smem[NV * 32 + i];
    }
    return is_last;
}

#endif  // __CUDACC__
