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
#include "ls_morton.cuh"

namespace {

__global__ void k_bbox(const float *__restrict__ verts, int64_t V, unsigned int *__restrict__ mm) {
    float lo[3] = {3.4e38f, 3.4e38f, 3.4e38f}, hi[3] = {-3.4e38f, -3.4e38f, -3.4e38f};
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < V; i += (int64_t)gridDim.x * blockDim.x) {
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            float x = verts[3 * i + d];
            if (x == x) {   // ignore NaN
                lo[d] = fminf(lo[d], x);
                hi[d] = fmaxf(hi[d], x);
            }
        }
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo[d] = fminf(lo[d], __shfl_xor_sync(0xffffffffu, lo[d], o));
            hi[d] = fmaxf(hi[d], __shfl_xor_sync(0xffffffffu, hi[d], o));
        }
        if ((threadIdx.x & 31) == 0) {
            atomicMin(&mm[d], f2ord(lo[d]));
            atomicMax(&mm[3 + d], f2ord(hi[d]));
        }
    }
}

__global__ void k_code_count(const float *__restrict__ verts, int64_t V, const unsigned int *__restrict__ mm, int bits,
                             unsigned int *__restrict__ code, int *__restrict__ cnt) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < V; i += (int64_t)gridDim.x * blockDim.x) {
        unsigned int c = cell_code(verts, i, mm, bits);
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
    unsigned int *mm;     // 6
    unsigned int *code;   // V
    int *cnt;             // nb + 1 (-> starts)
    int *cursor;          // nb
    int *scan;
    size_t total;
};

void carve(OrderWs &w, char *base, int64_t V, int64_t nb) {
    size_t off = 0;
    auto take = [&](size_t bytes) {
        size_t o = off;
        off = ls_align_up(off + bytes, 256);
        return o;
    };
    size_t o_mm = take(64);
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

}  // namespace

extern "C" int ls_order_workspace_bytes(int64_t V, size_t *bytes_out) {
    LS_REQUIRE(bytes_out != nullptr, "bytes_out is NULL");
    LS_REQUIRE(V >= 0 && V < (int64_t)0x7ffffff0, "V out of range");
    OrderWs w;
    carve(w, nullptr, V, (int64_t)1 << (3 * pick_bits(V)));
    *bytes_out = w.total;
    return LS_OK;
}

// what ls_order_morton(points, V, ..., workspace, ...) left in `workspace`: each point's cell code (indexed by point id) and
// the bounding box of the points as f2ord-encoded [lo x, y, z, hi x, y, z]
void ls_order_views(const void *workspace, int64_t V, const unsigned int **code, const unsigned int **bbox) {
    OrderWs w;
    carve(w, (char *)workspace, V, (int64_t)1 << (3 * pick_bits(V)));
    *code = w.code;
    *bbox = w.mm;
}

extern "C" int ls_order_morton(const float *verts, int64_t V, int32_t *perm_new2old, void *workspace,
                               size_t workspace_bytes, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    LS_REQUIRE(V >= 0 && V < (int64_t)0x7ffffff0, "V out of range");
    if (V == 0) return LS_OK;
    LS_REQUIRE(verts && perm_new2old && workspace, "NULL pointer");
    const int bits = pick_bits(V);
    const int64_t nb = (int64_t)1 << (3 * bits);
    OrderWs w;
    carve(w, (char *)workspace, V, nb);
    if (workspace_bytes < w.total) {
        ls_set_error("order workspace too small: %zu < %zu", workspace_bytes, w.total);
        return LS_ERR_WORKSPACE;
    }
    LsDevInfo di;
    int rc = ls_dev_info(&di);
    if (rc) return rc;
    unsigned int init[8] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u, 0u, 0u};
    LS_CUDA_TRY(cudaMemcpyAsync(w.mm, init, sizeof(init), cudaMemcpyHostToDevice, stream));
    LS_CUDA_TRY(cudaMemsetAsync(w.cnt, 0, (size_t)(nb + 1) * 4, stream));
    LS_CUDA_TRY(cudaMemsetAsync(w.cursor, 0, (size_t)(nb + 1) * 4, stream));
    int64_t g = (V + 255) / 256;
    if (g > (int64_t)di.sm_count * 8) g = (int64_t)di.sm_count * 8;
    k_bbox<<<(unsigned)g, 256, 0, stream>>>(verts, V, w.mm);
    LS_LAUNCH_CHECK();
    k_code_count<<<(unsigned)g, 256, 0, stream>>>(verts, V, w.mm, bits, w.code, w.cnt);
    LS_LAUNCH_CHECK();
    rc = ls_exclusive_scan_i32(w.cnt, w.cnt, nb, w.scan, stream);
    if (rc) return rc;
    k_scatter<<<(unsigned)g, 256, 0, stream>>>(V, w.code, w.cnt, w.cursor, perm_new2old);
    LS_LAUNCH_CHECK();
    k_sort_buckets<<<(unsigned)((nb + 127) / 128), 128, 0, stream>>>(nb, w.cnt, perm_new2old);
    LS_LAUNCH_CHECK();
    return LS_OK;
}
