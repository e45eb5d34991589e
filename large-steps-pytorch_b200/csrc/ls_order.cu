// ls_order.cu -- locality-improving vertex order for the solver's internal matrix copy (sm_90a).
//
// Why: the SpMM gathers p[col] through L1.  With the mesh's native vertex numbering (e.g. a row-major grid) the
// three gather bands of a 256-row block do not stay in L1, so p crosses the L2->SM fabric several times per SpMM.
// Sorting the vertices along a Morton (Z-order) curve of their positions makes every block of
// consecutive rows a compact patch of the surface whose neighbours are mostly inside the patch.
//
// Deterministic counting sort, same bucket machinery as the assembly: cell code per vertex (isotropic grid of
// 2^bits cells per axis over the bounding box, bits interleaved) -> histogram -> scan -> scatter -> per-bucket
// sort by vertex id.  perm[new] = old.
//
// Segmented form (ls_order_morton_seg, the distance BVHs of a packed batch): B runs of points, each with its own bounding
// box and grid; the bucket of point i in segment s is s * 8^bits + its cell, so the order is by (segment, cell, point) in
// one pass for any B.  ls_order_morton is B = 1.
#include "ls_morton.cuh"

namespace {

// one point per thread; mm holds the B boxes as lo [3B] then hi [3B] (f2ord).  A block whose points share a segment (always,
// when B == 1) folds its box first and issues one atomic per coordinate, as few as a grid-stride loop over a capped grid
// would; otherwise each warp whose points share a segment folds its own.  min and max are exact, so the box does not depend
// on the order of the atomics.
__global__ void __launch_bounds__(256) k_bbox(const float *__restrict__ verts, int64_t V, const int64_t *__restrict__ off, int B,
                                              unsigned int *__restrict__ mm) {
    __shared__ float red[2][3][8];
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    float lo[3] = {3.4e38f, 3.4e38f, 3.4e38f}, hi[3] = {-3.4e38f, -3.4e38f, -3.4e38f};
    if (i < V) {
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            float x = verts[3 * i + d];
            if (x == x) {   // ignore NaN
                lo[d] = x;
                hi[d] = x;
            }
        }
    }
    const int s = ls_segment_of(off, B, i < V ? i : V - 1, 0);
    const int s_block = ls_segment_of(off, B, (int64_t)blockIdx.x * blockDim.x, 0);
    const bool block_uniform = __syncthreads_and(s == s_block);
    const bool uniform = block_uniform || __all_sync(0xffffffffu, s == __shfl_sync(0xffffffffu, s, 0));
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        if (uniform) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                lo[d] = fminf(lo[d], __shfl_xor_sync(0xffffffffu, lo[d], o));
                hi[d] = fmaxf(hi[d], __shfl_xor_sync(0xffffffffu, hi[d], o));
            }
        }
        if (block_uniform) {
            if (lane == 0) {
                red[0][d][warp] = lo[d];
                red[1][d][warp] = hi[d];
            }
        } else if (!uniform || lane == 0) {
            atomicMin(&mm[3 * s + d], f2ord(lo[d]));
            atomicMax(&mm[3 * B + 3 * s + d], f2ord(hi[d]));
        }
    }
    if (block_uniform) {
        __syncthreads();
        if (threadIdx.x < 3) {
            const int d = threadIdx.x;
            float l = red[0][d][0], h = red[1][d][0];
            for (int w = 1; w < (int)(blockDim.x >> 5); ++w) {
                l = fminf(l, red[0][d][w]);
                h = fmaxf(h, red[1][d][w]);
            }
            atomicMin(&mm[3 * s + d], f2ord(l));
            atomicMax(&mm[3 * B + 3 * s + d], f2ord(h));
        }
    }
}

__global__ void k_code_count(const float *__restrict__ verts, int64_t V, const int64_t *__restrict__ off, int B,
                             const unsigned int *__restrict__ mm, int bits, unsigned int *__restrict__ code,
                             int *__restrict__ cnt) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < V; i += (int64_t)gridDim.x * blockDim.x) {
        const int s = ls_segment_of(off, B, i, 0);
        unsigned int c = ((unsigned int)s << (3 * bits)) + cell_code(verts, i, mm + 3 * s, mm + 3 * B + 3 * s, bits);
        code[i] = c;
        atomicAdd(&cnt[c], 1);
    }
}

__global__ void k_scatter(int64_t V, const unsigned int *__restrict__ code, const int *__restrict__ start,
                          int *__restrict__ cursor, int *__restrict__ perm) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < V; i += (int64_t)gridDim.x * blockDim.x) {
        unsigned int c = code[i];
        int p = start[c] + atomicAdd(&cursor[c], 1);
        perm[p] = (int)i;
    }
}

// buckets hold a few dozen vertices: per-bucket insertion sort by vertex id makes the order deterministic
__global__ void k_sort_buckets(int64_t nb, const int *__restrict__ start, int *__restrict__ perm) {
    int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    int s = start[b], e = start[b + 1];
    // shell sort (a cell that catches 1e5 coincident or outlier-squeezed vertices must not cost 1e10 operations)
    const int n = e - s;
    for (int gap = n >> 1; gap > 0; gap >>= 1)
        for (int a = s + gap; a < e; ++a) {
            int v = perm[a];
            int j = a - gap;
            while (j >= s && perm[j] > v) {
                perm[j + gap] = perm[j];
                j -= gap;
            }
            perm[j + gap] = v;
        }
}

struct OrderWs {
    unsigned int *mm;     // 6B: the boxes, lo [3B] then hi [3B]
    unsigned int *code;   // V
    int *cnt;             // nb + 1 (-> starts)
    int *cursor;          // nb
    int *scan;
    size_t total;
};

void carve(OrderWs &w, char *base, int64_t V, int64_t B, int64_t nb) {
    size_t off = 0;
    auto take = [&](size_t bytes) {
        size_t o = off;
        off = ls_align_up(off + bytes, 256);
        return o;
    };
    size_t o_mm = take((size_t)B * 24);
    size_t o_code = take((size_t)V * 4);
    size_t o_cnt = take((size_t)(nb + 1) * 4);
    size_t o_cur = take((size_t)(nb + 1) * 4);
    size_t o_scan = take(ls_scan_scratch_elems(nb + 1) * 4);
    w.total = off;
    if (base) {
        w.mm = (unsigned int *)(base + o_mm);
        w.code = (unsigned int *)(base + o_code);
        w.cnt = (int *)(base + o_cnt);
        w.cursor = (int *)(base + o_cur);
        w.scan = (int *)(base + o_scan);
    }
}

int pick_bits(int64_t V) {
    // ~32 vertices per occupied cell of a 2-D surface: 4^bits ~ V / 32
    int bits = 1;
    while (bits < 7 && ((int64_t)32 << (2 * (bits + 1))) <= V * 2) ++bits;
    return bits;
}

// B segments of V points in all: the grid of the mean segment, coarsened to at most 2^24 buckets in all, or 8B (bits = 1)
// when B > 2^21 (B = 1: pick_bits(V)).  A segment far above the mean gets cells of more points than the mean grid targets.
int seg_bits(int64_t V, int64_t B) {
    int bits = pick_bits((V + B - 1) / B);
    while (bits > 1 && (B << (3 * bits)) > ((int64_t)1 << 24)) --bits;
    return bits;
}

}  // namespace

int ls_order_morton_seg(const float *verts, int64_t V, const int64_t *off, int64_t B, int32_t *perm_new2old, void *workspace,
                        size_t workspace_bytes, cudaStream_t stream) {
    LS_REQUIRE(V >= 0 && V < (int64_t)0x7ffffff0, "V out of range");
    LS_REQUIRE(B >= 1 && B <= LS_ORDER_MAX_SEGMENTS, "B out of range");
    if (V == 0) return LS_OK;
    LS_REQUIRE(verts && perm_new2old && workspace, "NULL pointer");
    LS_REQUIRE(B == 1 || off, "NULL offsets");
    const int bits = seg_bits(V, B);
    const int64_t nb = B << (3 * bits);
    OrderWs w;
    carve(w, (char *)workspace, V, B, nb);
    if (workspace_bytes < w.total) {
        ls_set_error("order workspace too small: %zu < %zu", workspace_bytes, w.total);
        return LS_ERR_WORKSPACE;
    }
    LsDevInfo di;
    int rc = ls_dev_info(&di);
    if (rc) return rc;
    LS_CUDA_TRY(cudaMemsetAsync(w.mm, 0xff, (size_t)B * 12, stream));           // lo = f2ord(+max), hi = f2ord(-max)
    LS_CUDA_TRY(cudaMemsetAsync(w.mm + 3 * B, 0, (size_t)B * 12, stream));
    LS_CUDA_TRY(cudaMemsetAsync(w.cnt, 0, (size_t)(nb + 1) * 4, stream));
    LS_CUDA_TRY(cudaMemsetAsync(w.cursor, 0, (size_t)(nb + 1) * 4, stream));
    int64_t g = (V + 255) / 256;
    k_bbox<<<(unsigned)g, 256, 0, stream>>>(verts, V, off, (int)B, w.mm);
    LS_LAUNCH_CHECK();
    if (g > (int64_t)di.sm_count * 8) g = (int64_t)di.sm_count * 8;
    k_code_count<<<(unsigned)g, 256, 0, stream>>>(verts, V, off, (int)B, w.mm, bits, w.code, w.cnt);
    LS_LAUNCH_CHECK();
    rc = ls_exclusive_scan_i32(w.cnt, w.cnt, nb, w.scan, stream);
    if (rc) return rc;
    k_scatter<<<(unsigned)g, 256, 0, stream>>>(V, w.code, w.cnt, w.cursor, perm_new2old);
    LS_LAUNCH_CHECK();
    k_sort_buckets<<<(unsigned)((nb + 127) / 128), 128, 0, stream>>>(nb, w.cnt, perm_new2old);
    LS_LAUNCH_CHECK();
    return LS_OK;
}

int ls_order_seg_workspace_bytes(int64_t V, int64_t B, size_t *bytes_out) {
    LS_REQUIRE(bytes_out != nullptr, "bytes_out is NULL");
    LS_REQUIRE(V >= 0 && V < (int64_t)0x7ffffff0, "V out of range");
    LS_REQUIRE(B >= 1 && B <= LS_ORDER_MAX_SEGMENTS, "B out of range");
    OrderWs w;
    carve(w, nullptr, V, B, B << (3 * seg_bits(V, B)));
    *bytes_out = w.total;
    return LS_OK;
}

extern "C" int ls_order_workspace_bytes(int64_t V, size_t *bytes_out) { return ls_order_seg_workspace_bytes(V, 1, bytes_out); }

void ls_order_views(const void *workspace, int64_t V, int64_t B, const unsigned int **code, const unsigned int **bbox) {
    OrderWs w;
    carve(w, (char *)workspace, V, B, B << (3 * seg_bits(V, B)));
    *code = w.code;
    *bbox = w.mm;
}

extern "C" int ls_order_morton(const float *verts, int64_t V, int32_t *perm_new2old, void *workspace,
                               size_t workspace_bytes, void *stream_) {
    return ls_order_morton_seg(verts, V, nullptr, 1, perm_new2old, workspace, workspace_bytes, (cudaStream_t)stream_);
}
