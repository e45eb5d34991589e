// ls_assemble.cu -- on-device assembly of M = shift*I + scale*L from triangle faces (sm_90a).
//
// Replaces largesteps/geometry.py:3-133 (laplacian_cot / laplacian_uniform / compute_matrix), which in the
// reference is torch.unique(dim=1) + two coalesce() sorts over 2x12M int64 indices at 1M vertices.
//
// Sort-free design: every face emits its 6 directed edges into per-row buckets (row degree is known from a
// counting pass + prefix scan), each row then sorts and de-duplicates its own ~2*valence entries in place.
// The output is therefore born row-major sorted and coalesced, in both layouts at once:
//   * the int64 COO triplets torch.sparse_coo_tensor(...).coalesce() would hold (geometry.py:133), and
//   * the int32 CSR the solver streams.
// Semantics follow the reference exactly, including its corner cases: duplicate directed edges are de-duplicated
// for the uniform Laplacian (geometry.py:82) but summed for the cotangent one (coalesce), isolated vertices get a
// pure identity row, and right-angle cotangents are kept as explicit ~0 entries.
#include "ls_common.cuh"

namespace {

struct AsmWs {
    int *cnt;      // V+1   bucket sizes -> bucket starts (exclusive scan, in place)
    int *cursor;   // V     fill cursors
    int *ucnt;     // V+1   unique entries per row (+1 diagonal) -> rowptr
    int *bcol;     // 6F    bucket: neighbour column
    int *bsrc;     // 6F    bucket: 3*face + which cotangent
    float *cot;    // 3F    per-face cotangents / 4
    int *scan;     // scan scratch
    int *flags;    // [0] index-range error
    size_t total;
};

static int carve(AsmWs &w, void *base, int64_t F, int64_t V) {
    size_t off = 0;
    auto take = [&](size_t bytes) {
        size_t o = off;
        off = ls_align_up(off + bytes, 256);
        return o;
    };
    char *b = static_cast<char *>(base);
    size_t o_cnt = take((V + 1) * sizeof(int));
    size_t o_cur = take((V + 1) * sizeof(int));
    size_t o_ucnt = take((V + 1) * sizeof(int));
    size_t o_bcol = take((size_t)6 * F * sizeof(int) + 16);
    size_t o_bsrc = take((size_t)6 * F * sizeof(int) + 16);
    size_t o_cot = take((size_t)3 * F * sizeof(float) + 16);
    size_t o_scan = take(ls_scan_scratch_elems(V + 1) * sizeof(int));
    size_t o_flags = take(64);
    w.total = off;
    if (b) {
        w.cnt = (int *)(b + o_cnt);
        w.cursor = (int *)(b + o_cur);
        w.ucnt = (int *)(b + o_ucnt);
        w.bcol = (int *)(b + o_bcol);
        w.bsrc = (int *)(b + o_bsrc);
        w.cot = (float *)(b + o_cot);
        w.scan = (int *)(b + o_scan);
        w.flags = (int *)(b + o_flags);
    }
    return LS_OK;
}

template <typename IdxT>
__device__ __forceinline__ bool load_face(const IdxT *faces, int64_t f, int64_t V, int (&v)[3]) {
    long long a = faces[3 * f + 0], b = faces[3 * f + 1], c = faces[3 * f + 2];
    v[0] = (int)a;
    v[1] = (int)b;
    v[2] = (int)c;
    return a >= 0 && b >= 0 && c >= 0 && a < V && b < V && c < V;
}

// pass 1: each vertex of a face is the row of two directed edges
template <typename IdxT>
__global__ void k_count(const IdxT *__restrict__ faces, int64_t F, int64_t V, int *__restrict__ cnt,
                        int *__restrict__ flags) {
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += (int64_t)gridDim.x * blockDim.x) {
        int v[3];
        if (!load_face(faces, f, V, v)) {
            atomicOr(&flags[0], 1);
            continue;
        }
        atomicAdd(&cnt[v[0]], 2);
        atomicAdd(&cnt[v[1]], 2);
        atomicAdd(&cnt[v[2]], 2);
    }
}

// pass 2: drop the 6 directed edges of each face into the row buckets.
//   reference: ii = faces[:, [1,2,0]], jj = faces[:, [2,0,1]]  (geometry.py:47-48, 80-81)
//   edge e (0..2): (ii,jj) = (v1,v2) carries cot a, (v2,v0) cot b, (v0,v1) cot c; plus the transposed entry.
template <typename IdxT>
__global__ void k_fill_buckets(const IdxT *__restrict__ faces, int64_t F, int64_t V, const int *__restrict__ bstart,
                               int *__restrict__ cursor, int *__restrict__ bcol, int *__restrict__ bsrc) {
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += (int64_t)gridDim.x * blockDim.x) {
        int v[3];
        if (!load_face(faces, f, V, v)) continue;
#pragma unroll
        for (int e = 0; e < 3; ++e) {
            int i = v[(e + 1) % 3], j = v[(e + 2) % 3];
            int src = (int)(3 * f + e);
            int p = bstart[i] + atomicAdd(&cursor[i], 1);
            bcol[p] = j;
            bsrc[p] = src;
            int q = bstart[j] + atomicAdd(&cursor[j], 1);
            bcol[q] = i;
            bsrc[q] = src;
        }
    }
}

// pass 3: per row, sort the bucket by (col, src) in place and count the distinct off-diagonal columns.
// Buckets are tiny (2 x valence), one thread per row with an insertion sort is the right tool.
__global__ void k_sort_rows(int64_t V, const int *__restrict__ bstart, int *__restrict__ bcol, int *__restrict__ bsrc,
                            int *__restrict__ ucnt) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= V) return;
    int s = bstart[i], e = bstart[i + 1];
    // shell sort by (col, src): for the ~12-entry buckets of a mesh row this is the insertion sort it always was (one pass with
    // gap 1 after a few trivial ones); for a hub of valence 1e4-1e5 it is O(n^1.3) instead of O(n^2) -- no watchdog cliff
    const int n = e - s;
    for (int gap = n >> 1; gap > 0; gap >>= 1)
        for (int a = s + gap; a < e; ++a) {
            int c = bcol[a], r = bsrc[a];
            int b = a - gap;
            while (b >= s && (bcol[b] > c || (bcol[b] == c && bsrc[b] > r))) {
                bcol[b + gap] = bcol[b];
                bsrc[b + gap] = bsrc[b];
                b -= gap;
            }
            bcol[b + gap] = c;
            bsrc[b + gap] = r;
        }
    int u = 1;  // the diagonal is always present (the identity term, geometry.py:124-128)
    int prev = -1;
    for (int a = s; a < e; ++a) {
        int c = bcol[a];
        if (c != prev && c != (int)i) ++u;
        prev = c;
    }
    ucnt[i] = u;
}

// One face's cotangent chain, in geometry.py:20-41's fp32 operation order (no FMA contraction; `/` is the correctly rounded
// division on the device too).  k_cot writes its weights; the assembly backward and the product backward recompute it for the
// gradient.
struct CotFace {
    float e[3][3];   // e0 = p1 - p2, e1 = p0 - p2, e2 = p0 - p1
    float l[3];      // A = |e0|, B = |e1|, C = |e2|                                geometry.py:25-27
    float s, t[3];   // s = 0.5 ((A + B) + C),  t_k = s - l_k                       geometry.py:30
    float P, area;   // Heron's product ((s t0) t1) t2 before the clamp,  area = sqrt(max(P, 1e-12))   geometry.py:33
    float num[3];    // (B2 + C2) - A2,  (A2 + C2) - B2,  (A2 + B2) - C2
    float q[3];      // num_k / area                                                geometry.py:37-39
};
__host__ __device__ __forceinline__ void cot_face(const float (&p)[3][3], CotFace &c) {
    const int a[3] = {1, 0, 0}, b[3] = {2, 2, 1};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
#pragma unroll
        for (int d = 0; d < 3; ++d) c.e[k][d] = sub_rn(p[a[k]][d], p[b[k]][d]);
        const float s2 = add_rn(add_rn(mul_rn(c.e[k][0], c.e[k][0]), mul_rn(c.e[k][1], c.e[k][1])), mul_rn(c.e[k][2], c.e[k][2]));
        c.l[k] = sqrt_rn(s2);
    }
    c.s = mul_rn(0.5f, add_rn(add_rn(c.l[0], c.l[1]), c.l[2]));
    c.P = c.s;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        c.t[k] = sub_rn(c.s, c.l[k]);
        c.P = mul_rn(c.P, c.t[k]);
    }
    c.area = sqrt_rn(fmaxf(c.P, 1e-12f));
    const float sq[3] = {mul_rn(c.l[0], c.l[0]), mul_rn(c.l[1], c.l[1]), mul_rn(c.l[2], c.l[2])};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        c.num[k] = sub_rn(add_rn(sq[(k + 1) % 3], sq[(k + 2) % 3]), sq[k]);
        c.q[k] = c.num[k] / c.area;
    }
}

// per-face cotangents: the weight k is q_k / 4 (geometry.py:41)
template <typename IdxT>
__global__ void k_cot(const IdxT *__restrict__ faces, const float *__restrict__ verts, int64_t F, int64_t V,
                      float *__restrict__ cot) {
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += (int64_t)gridDim.x * blockDim.x) {
        int v[3];
        if (!load_face(faces, f, V, v)) continue;
        float p[3][3];
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int d = 0; d < 3; ++d) p[a][d] = verts[3 * (int64_t)v[a] + d];
        CotFace c;
        cot_face(p, c);
#pragma unroll
        for (int k = 0; k < 3; ++k) cot[3 * f + k] = __fdiv_rn(c.q[k], 4.0f);
    }
}

// pass 4: write each row: sorted unique columns with the diagonal merged in at its sorted position.
//   uniform (geometry.py:82-94,128): off = scale * (-1);  diag = shift + scale * deg,  deg = #distinct neighbours
//   cotan   (geometry.py:47-62,128): off = sum_e scale * (-w_e); diag = shift + scale * (sum of all w in the row)
//                                    (+ scale * (-w) for degenerate self-edges, which coalesce onto the diagonal)
__global__ void k_write_rows(int64_t V, int cotan, float shift, float scale, const int *__restrict__ bstart,
                             const int *__restrict__ bcol, const int *__restrict__ bsrc, const float *__restrict__ cot,
                             const int *__restrict__ rowptr, int64_t *__restrict__ coo_row,
                             int64_t *__restrict__ coo_col, float *__restrict__ coo_val, int *__restrict__ csr_rowptr,
                             int *__restrict__ csr_col, float *__restrict__ csr_val) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i > V) return;
    if (i == V) {
        if (csr_rowptr) csr_rowptr[V] = rowptr[V];
        return;
    }
    int s = bstart[i], e = bstart[i + 1];
    int o = rowptr[i];
    if (csr_rowptr) csr_rowptr[i] = o;
    // diagonal first (needs the whole row), then stream the row out
    float dsum = 0.f, dself = 0.f;
    int deg = 0, prev = -1;
    for (int a = s; a < e; ++a) {
        int c = bcol[a];
        if (cotan) {
            float w = cot[bsrc[a]];
            dsum = __fadd_rn(dsum, w);
            if (c == (int)i) dself = __fadd_rn(dself, __fmul_rn(scale, -w));
        } else if (c != prev && c != (int)i) {
            ++deg;
        }
        prev = c;
    }
    float diag = cotan ? __fadd_rn(__fadd_rn(shift, __fmul_rn(scale, dsum)), dself)
                       : __fadd_rn(shift, __fmul_rn(scale, (float)deg));
    auto emit = [&](int c, float v) {
        if (coo_row) {
            coo_row[o] = i;
            coo_col[o] = c;
            coo_val[o] = v;
        }
        if (csr_col) {
            csr_col[o] = c;
            csr_val[o] = v;
        }
        ++o;
    };
    bool diag_done = false;
    int a = s;
    while (a < e) {
        int c = bcol[a];
        float acc = 0.f;
        int b = a;
        while (b < e && bcol[b] == c) {
            if (cotan) acc = __fadd_rn(acc, __fmul_rn(scale, -cot[bsrc[b]]));
            ++b;
        }
        if (!cotan) acc = __fmul_rn(scale, -1.0f);
        a = b;
        if (c == (int)i) continue;  // self-edges were folded into the diagonal
        if (!diag_done && c > (int)i) {
            emit((int)i, diag);
            diag_done = true;
        }
        emit(c, acc);
    }
    if (!diag_done) emit((int)i, diag);
}

__global__ void k_coo_rowptr(const int64_t *__restrict__ rows, const int64_t *__restrict__ cols, int64_t nnz, int64_t V,
                             int *__restrict__ rowptr, int *__restrict__ col32, int *__restrict__ flags) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    // rowptr[i] = lower_bound(rows, i)
    for (int64_t i = t; i <= V; i += stride) {
        int64_t lo = 0, hi = nnz;
        while (lo < hi) {
            int64_t mid = (lo + hi) >> 1;
            if (rows[mid] < i) lo = mid + 1;
            else hi = mid;
        }
        rowptr[i] = (int)lo;
    }
    for (int64_t j = t; j < nnz; j += stride) {
        int64_t r = rows[j], c = cols[j];
        if (r < 0 || r >= V || c < 0 || c >= V) atomicOr(&flags[0], 1);
        if (j > 0 && rows[j - 1] > r) atomicOr(&flags[0], 2);
        col32[j] = (int)c;
    }
}

inline unsigned grid_for(int64_t n, int threads, int cap = 132 * 16) {   // 132 SMs (H100 SXM) x 16
    int64_t g = (n + threads - 1) / threads;
    if (g < 1) g = 1;
    if (g > cap) g = cap;
    return (unsigned)g;
}

// ---- backward of the cotangent assembly ---------------------------------------------------------------------------------
// Gbar is the gradient of M's (nnz,) values in their row-major order.  The weight w of a face on edge (i, j) (w_a on (v1, v2),
// w_b on (v2, v0), w_c on (v0, v1): k_fill_buckets) adds scale w to M_ii and M_jj and -scale w to M_ij and M_ji
// (k_write_rows), so its gradient is
//     wbar = scale (Gbar_ii + Gbar_jj - Gbar_ij - Gbar_ji),   and 0 on a self-edge (i = j), whose contributions cancel.
// Pass 1, one thread per face: the four entries of each edge by binary search in M's CSR rows, wbar -> scratch (3F floats).
// Pass 2, one thread per vertex: each incident face is recomputed as k_cot computes it and its chain is followed back to the
// corner node for node as torch's autograd of geometry.py:20-41 runs it, summed in face order over the incidence list.  No
// atomics, so the gradient is bit-reproducible.  The bodies are __host__ __device__ so that a CPU test can run them.
// Gradient of sum_k wbar_k w_k w.r.t. the three edge vectors.  As torch's backward nodes: `cot /= 4` passes wbar / 4, the
// division num / area gives g / area to num and -g ((num / area) / area) to area, sqrt gives g / (2 area), the clamp passes
// the gradient only where P >= 1e-12 (an exact 0 elsewhere, and for a NaN P), and the 2-norm gives g (e / l) with e / l set
// to 0 where l = 0.
__host__ __device__ __forceinline__ void cot_face_grad(const CotFace &c, const float (&wbar)[3], float (&ge)[3][3]) {
    float gsq[3] = {0.f, 0.f, 0.f}, garea = 0.f;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float gw = wbar[k] / 4.0f;
        const float gnum = gw / c.area;
        garea -= gw * ((c.num[k] / c.area) / c.area);
        gsq[(k + 1) % 3] += gnum;
        gsq[(k + 2) % 3] += gnum;
        gsq[k] -= gnum;
    }
    float gl[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) gl[k] = gsq[k] * c.l[k] + gsq[k] * c.l[k];   // l_k^2 = l_k * l_k
    const float gP = c.P >= 1e-12f ? garea / (2.f * c.area) : 0.f;
    const float q1 = c.s * c.t[0], q2 = q1 * c.t[1];                       // P = ((s t0) t1) t2
    const float gt2 = gP * q2, gq2 = gP * c.t[2];
    const float gt1 = gq2 * q1, gq1 = gq2 * c.t[1];
    const float gt0 = gq1 * c.s;
    const float gs = gq1 * c.t[0] + gt0 + gt1 + gt2;                        // t_k = s - l_k
    gl[0] += 0.5f * gs - gt0;                                                // s = 0.5 ((A + B) + C)
    gl[1] += 0.5f * gs - gt1;
    gl[2] += 0.5f * gs - gt2;
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
        for (int d = 0; d < 3; ++d) ge[k][d] = gl[k] * (c.l[k] == 0.f ? 0.f : c.e[k][d] / c.l[k]);
}
// position of column j in CSR row i (present by construction; the row's end if it is not)
__host__ __device__ __forceinline__ int csr_find(const int *rowptr, const int *col, int i, int j) {
    int lo = rowptr[i], hi = rowptr[i + 1];
    const int end = hi;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (col[mid] < j) lo = mid + 1;
        else hi = mid;
    }
    return lo < end && col[lo] == j ? lo : -1;
}
__host__ __device__ __forceinline__ float gval_at(const int *rowptr, const int *col, const float *gval, int i, int j) {
    const int p = csr_find(rowptr, col, i, j);
    return p >= 0 ? gval[p] : 0.f;
}
template <typename I>
__host__ __device__ __forceinline__ void cot_face_wbar(const I *faces, int64_t f, float scale, const int *rowptr, const int *col,
                                                       const float *gval, float (&wbar)[3]) {
    const int v[3] = {(int)faces[3 * f], (int)faces[3 * f + 1], (int)faces[3 * f + 2]};
    const float gd[3] = {gval_at(rowptr, col, gval, v[0], v[0]), gval_at(rowptr, col, gval, v[1], v[1]),
                         gval_at(rowptr, col, gval, v[2], v[2])};
#pragma unroll
    for (int e = 0; e < 3; ++e) {
        const int a = (e + 1) % 3, b = (e + 2) % 3, i = v[a], j = v[b];
        wbar[e] = i == j ? 0.f
                         : scale * (((gd[a] + gd[b]) - gval_at(rowptr, col, gval, i, j)) - gval_at(rowptr, col, gval, j, i));
    }
}
template <typename I>
__host__ __device__ __forceinline__ void cot_vertex_grad(const float *verts, const I *faces, const int *ptr, const int *inc,
                                                         const float *wbar, int64_t v, float (&acc)[3]) {
    acc[0] = acc[1] = acc[2] = 0.f;
    for (int j = ptr[v]; j < ptr[v + 1]; ++j) {
        const int code = inc[j];
        const int64_t f = code >> 2;
        const int me = code & 3;
        float p[3][3];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const int64_t id = (int64_t)faces[3 * f + a];
#pragma unroll
            for (int d = 0; d < 3; ++d) p[a][d] = verts[3 * id + d];
        }
        CotFace c;
        cot_face(p, c);
        const float wb[3] = {wbar[3 * f], wbar[3 * f + 1], wbar[3 * f + 2]};
        float ge[3][3];
        cot_face_grad(c, wb, ge);
        // e0 = p1 - p2, e1 = p0 - p2, e2 = p0 - p1
#pragma unroll
        for (int d = 0; d < 3; ++d)
            acc[d] += me == 0 ? ge[1][d] + ge[2][d] : (me == 1 ? ge[0][d] - ge[2][d] : -ge[0][d] - ge[1][d]);
    }
}
template <typename I>
__global__ void k_cot_wbar(const I *__restrict__ faces, int64_t F, float scale, const int *__restrict__ rowptr,
                           const int *__restrict__ col, const float *__restrict__ gval, float *__restrict__ wbar) {
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += (int64_t)gridDim.x * blockDim.x) {
        float w[3];
        cot_face_wbar(faces, f, scale, rowptr, col, gval, w);
        wbar[3 * f] = w[0];
        wbar[3 * f + 1] = w[1];
        wbar[3 * f + 2] = w[2];
    }
}
template <typename I>
__global__ void k_cot_vertex_grad(const float *__restrict__ verts, const I *__restrict__ faces, int64_t V,
                                  const int *__restrict__ ptr, const int *__restrict__ inc, const float *__restrict__ wbar,
                                  float *__restrict__ gverts) {
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    float acc[3];
    cot_vertex_grad(verts, faces, ptr, inc, wbar, v, acc);
    gverts[3 * v] = acc[0];
    gverts[3 * v + 1] = acc[1];
    gverts[3 * v + 2] = acc[2];
}

// ---- matrix-free product y = L x with the cotangent Laplacian -------------------------------------------------------------
// L = diag(colsum W) - W, so (L x)_i = sum over the edges (i, j) of the faces at i of w (x_i - x_j): no matrix is needed, only
// the three weights per face that k_cot writes.  One thread per vertex walks the incidence list in its sorted order (corners in
// face order, then the corner's two edges in edge order), so the sum order is fixed and y bit-reproducible.  A self-edge adds
// nothing (it cancels in L), a duplicated face adds twice, a vertex in no face gets 0.  Columns go in chunks of four: one walk
// of the list per chunk.
template <typename I>
__host__ __device__ __forceinline__ void cot_product_row(const I *faces, const int *ptr, const int *inc, const float *w,
                                                         const float *x, int k, int c0, int64_t v, float (&acc)[4]) {
    const int nc = k - c0 < 4 ? k - c0 : 4;
    float xi[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        acc[q] = 0.f;
        xi[q] = q < nc ? x[v * k + c0 + q] : 0.f;
    }
    for (int p = ptr[v]; p < ptr[v + 1]; ++p) {
        const int code = inc[p];
        const int64_t f = code >> 2;
        const int me = code & 3;
        // edge e joins corners (e + 1) % 3 and (e + 2) % 3: the corner's edges are the other two, in increasing e
        const int e0 = me == 0 ? 1 : 0, e1 = me == 2 ? 1 : 2;
#pragma unroll
        for (int t = 0; t < 2; ++t) {
            const int e = t == 0 ? e0 : e1;
            const int64_t j = (int64_t)faces[3 * f + (3 - me - e)];
            if (j == v) continue;
            const float we = w[3 * f + e];
#pragma unroll
            for (int q = 0; q < 4; ++q)
                if (q < nc) acc[q] = add_rn(acc[q], mul_rn(we, sub_rn(xi[q], x[j * k + c0 + q])));
        }
    }
}
// wbar_e = d(gy . L x) / d w_e = sum_q (gy_i,q - gy_j,q)(x_i,q - x_j,q) for edge e = (i, j), q in order; exactly 0 on a self-edge
template <typename I>
__host__ __device__ __forceinline__ void cot_product_face_wbar(const I *faces, int64_t f, const float *x, const float *gy, int k,
                                                               float (&wbar)[3]) {
    const int64_t v[3] = {(int64_t)faces[3 * f], (int64_t)faces[3 * f + 1], (int64_t)faces[3 * f + 2]};
#pragma unroll
    for (int e = 0; e < 3; ++e) {
        const int64_t i = v[(e + 1) % 3], j = v[(e + 2) % 3];
        float s = 0.f;
        if (i != j)
            for (int q = 0; q < k; ++q)
                s = add_rn(s, mul_rn(sub_rn(gy[i * k + q], gy[j * k + q]), sub_rn(x[i * k + q], x[j * k + q])));
        wbar[e] = s;
    }
}
template <typename I>
__global__ void k_cot_product(const I *__restrict__ faces, int64_t V, const int *__restrict__ ptr, const int *__restrict__ inc,
                              const float *__restrict__ w, const float *__restrict__ x, int k, float *__restrict__ y) {
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    for (int c0 = 0; c0 < k; c0 += 4) {
        float acc[4];
        cot_product_row(faces, ptr, inc, w, x, k, c0, v, acc);
#pragma unroll
        for (int q = 0; q < 4; ++q)
            if (c0 + q < k) y[v * k + c0 + q] = acc[q];
    }
}
template <typename I>
__global__ void k_cot_product_wbar(const I *__restrict__ faces, int64_t F, const float *__restrict__ x,
                                   const float *__restrict__ gy, int k, float *__restrict__ wbar) {
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += (int64_t)gridDim.x * blockDim.x) {
        float wb[3];
        cot_product_face_wbar(faces, f, x, gy, k, wb);
        wbar[3 * f] = wb[0];
        wbar[3 * f + 1] = wb[1];
        wbar[3 * f + 2] = wb[2];
    }
}

}  // namespace

extern "C" int ls_assemble_workspace_bytes(int64_t F, int64_t V, size_t *bytes_out) {
    LS_REQUIRE(bytes_out != nullptr, "bytes_out is NULL");
    LS_REQUIRE(F >= 0 && V >= 0, "negative size");
    LS_REQUIRE(6 * F < (int64_t)0x7fffffff && V < (int64_t)0x7ffffff0, "mesh too large for int32 bucket offsets");
    AsmWs w;
    carve(w, nullptr, F, V);
    *bytes_out = w.total;
    return LS_OK;
}

extern "C" int ls_assemble_count(const void *faces, int idx_bytes, int64_t F, int64_t V, void *workspace,
                                 size_t workspace_bytes, int64_t *nnz_out, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    LS_REQUIRE(nnz_out != nullptr, "nnz_out is NULL");
    LS_REQUIRE(idx_bytes == 4 || idx_bytes == 8, "idx_bytes must be 4 or 8");
    LS_REQUIRE(F >= 0 && V >= 0, "negative size");
    LS_REQUIRE(F == 0 || faces != nullptr, "faces is NULL");
    LS_REQUIRE(workspace != nullptr && ((uintptr_t)workspace & 15) == 0, "workspace NULL or misaligned");
    LS_REQUIRE(6 * F < (int64_t)0x7fffffff && V < (int64_t)0x7ffffff0, "mesh too large for int32 bucket offsets");
    LsDevInfo di;
    int rc = ls_dev_info(&di);
    if (rc) return rc;
    AsmWs w;
    carve(w, workspace, F, V);
    if (workspace_bytes < w.total) {
        ls_set_error("assembly workspace too small: %zu < %zu", workspace_bytes, w.total);
        return LS_ERR_WORKSPACE;
    }
    LS_CUDA_TRY(cudaMemsetAsync(w.cnt, 0, (V + 1) * sizeof(int), stream));
    LS_CUDA_TRY(cudaMemsetAsync(w.cursor, 0, (V + 1) * sizeof(int), stream));
    LS_CUDA_TRY(cudaMemsetAsync(w.flags, 0, 64, stream));
    if (F > 0) {
        if (idx_bytes == 4) k_count<int><<<grid_for(F, 256), 256, 0, stream>>>((const int *)faces, F, V, w.cnt, w.flags);
        else k_count<long long><<<grid_for(F, 256), 256, 0, stream>>>((const long long *)faces, F, V, w.cnt, w.flags);
        LS_LAUNCH_CHECK();
    }
    rc = ls_exclusive_scan_i32(w.cnt, w.cnt, V, w.scan, stream);   // cnt[0..V] = bucket starts, cnt[V] = 6F'
    if (rc) return rc;
    if (F > 0) {
        if (idx_bytes == 4)
            k_fill_buckets<int><<<grid_for(F, 256), 256, 0, stream>>>((const int *)faces, F, V, w.cnt, w.cursor, w.bcol, w.bsrc);
        else
            k_fill_buckets<long long><<<grid_for(F, 256), 256, 0, stream>>>((const long long *)faces, F, V, w.cnt, w.cursor, w.bcol, w.bsrc);
        LS_LAUNCH_CHECK();
    }
    if (V > 0) {
        k_sort_rows<<<(unsigned)((V + 127) / 128), 128, 0, stream>>>(V, w.cnt, w.bcol, w.bsrc, w.ucnt);
        LS_LAUNCH_CHECK();
    }
    rc = ls_exclusive_scan_i32(w.ucnt, w.ucnt, V, w.scan, stream);  // ucnt[0..V] = rowptr
    if (rc) return rc;
    int h[2] = {0, 0};
    LS_CUDA_TRY(cudaMemcpyAsync(&h[0], w.ucnt + V, sizeof(int), cudaMemcpyDeviceToHost, stream));
    LS_CUDA_TRY(cudaMemcpyAsync(&h[1], w.flags, sizeof(int), cudaMemcpyDeviceToHost, stream));
    LS_CUDA_TRY(cudaStreamSynchronize(stream));
    if (h[1] != 0) {
        ls_set_error("face index outside [0, V=%lld)", (long long)V);
        return LS_ERR_INDEX_RANGE;
    }
    *nnz_out = h[0];
    return LS_OK;
}

extern "C" int ls_assemble_fill(const void *faces, int idx_bytes, const float *verts, int64_t F, int64_t V, int cotan,
                                float diag_shift, float scale, void *workspace, size_t workspace_bytes, int64_t nnz,
                                int64_t *coo_row, int64_t *coo_col, float *coo_val, int32_t *csr_rowptr,
                                int32_t *csr_col, float *csr_val, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    LS_REQUIRE(idx_bytes == 4 || idx_bytes == 8, "idx_bytes must be 4 or 8");
    LS_REQUIRE(workspace != nullptr, "workspace is NULL");
    LS_REQUIRE(!cotan || verts != nullptr || F == 0, "verts required for the cotangent Laplacian");
    LS_REQUIRE((coo_row == nullptr) == (coo_col == nullptr) && (coo_row == nullptr) == (coo_val == nullptr),
               "COO outputs must be all set or all NULL");
    LS_REQUIRE((csr_col == nullptr) == (csr_val == nullptr), "CSR col/val must be both set or both NULL");
    LS_REQUIRE(nnz >= V, "nnz smaller than V: was ls_assemble_count run on this workspace?");
    AsmWs w;
    carve(w, workspace, F, V);
    if (workspace_bytes < w.total) {
        ls_set_error("assembly workspace too small: %zu < %zu", workspace_bytes, w.total);
        return LS_ERR_WORKSPACE;
    }
    if (cotan && F > 0) {
        if (idx_bytes == 4) k_cot<int><<<grid_for(F, 256), 256, 0, stream>>>((const int *)faces, verts, F, V, w.cot);
        else k_cot<long long><<<grid_for(F, 256), 256, 0, stream>>>((const long long *)faces, verts, F, V, w.cot);
        LS_LAUNCH_CHECK();
    }
    k_write_rows<<<(unsigned)((V + 1 + 127) / 128), 128, 0, stream>>>(V, cotan, diag_shift, scale, w.cnt, w.bcol, w.bsrc,
                                                                    w.cot, w.ucnt, coo_row, coo_col, coo_val,
                                                                    csr_rowptr, csr_col, csr_val);
    LS_LAUNCH_CHECK();
    return LS_OK;
}

extern "C" int ls_coo_to_csr(const int64_t *coo_row, const int64_t *coo_col, int64_t nnz, int64_t V,
                             int32_t *csr_rowptr, int32_t *csr_col, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    LS_REQUIRE(nnz >= 0 && V >= 0 && nnz < (int64_t)0x7ffffff0 && V < (int64_t)0x7ffffff0, "size out of int32 range");
    LS_REQUIRE(csr_rowptr != nullptr && (nnz == 0 || (coo_row && coo_col && csr_col)), "NULL pointer");
    int *flags = nullptr;
    LS_CUDA_TRY(cudaMallocAsync((void **)&flags, 64, stream));
    LS_CUDA_TRY(cudaMemsetAsync(flags, 0, 64, stream));
    int64_t work = nnz > V + 1 ? nnz : V + 1;
    k_coo_rowptr<<<grid_for(work, 256), 256, 0, stream>>>(coo_row, coo_col, nnz, V, csr_rowptr, csr_col, flags);
    LS_LAUNCH_CHECK();
    int h = 0;
    LS_CUDA_TRY(cudaMemcpyAsync(&h, flags, sizeof(int), cudaMemcpyDeviceToHost, stream));
    LS_CUDA_TRY(cudaFreeAsync(flags, stream));
    LS_CUDA_TRY(cudaStreamSynchronize(stream));
    if (h & 1) {
        ls_set_error("COO index outside [0, V=%lld)", (long long)V);
        return LS_ERR_INDEX_RANGE;
    }
    if (h & 2) {
        ls_set_error("COO rows are not sorted (matrix must be coalesced)");
        return LS_ERR_INDEX_RANGE;
    }
    return LS_OK;
}

extern "C" int ls_laplacian_cot_bwd_scratch_bytes(int64_t F, size_t *bytes_out) {
    LS_REQUIRE(bytes_out != nullptr, "bytes_out is NULL");
    LS_REQUIRE(F >= 0 && 3 * F < (int64_t)0x7fffffff, "F out of range");
    *bytes_out = ls_align_up((size_t)3 * F * sizeof(float) + 16, 256);
    return LS_OK;
}

extern "C" int ls_laplacian_cot_bwd_f32(const float *verts, const void *faces, int idx_bytes, int64_t F, int64_t V, float scale,
                                        const int32_t *rowptr, const int32_t *col, const float *gval, const int32_t *inc_ptr,
                                        const int32_t *inc, void *scratch, size_t scratch_bytes, float *gverts, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    LS_REQUIRE(idx_bytes == 4 || idx_bytes == 8, "idx_bytes must be 4 or 8");
    LS_REQUIRE(F >= 0 && V >= 0 && V < (int64_t)0x7ffffff0, "bad size");
    size_t need = 0;
    int rc = ls_laplacian_cot_bwd_scratch_bytes(F, &need);
    if (rc) return rc;
    if (V == 0) return LS_OK;
    LS_REQUIRE(verts && (faces || F == 0) && rowptr && col && gval && inc_ptr && inc && gverts, "NULL pointer");
    LS_REQUIRE(scratch != nullptr && scratch_bytes >= need, "scratch NULL or smaller than ls_laplacian_cot_bwd_scratch_bytes(F)");
    float *wbar = (float *)scratch;
    if (F > 0) {
        if (idx_bytes == 4)
            k_cot_wbar<int><<<grid_for(F, 256), 256, 0, stream>>>((const int *)faces, F, scale, rowptr, col, gval, wbar);
        else
            k_cot_wbar<long long><<<grid_for(F, 256), 256, 0, stream>>>((const long long *)faces, F, scale, rowptr, col, gval, wbar);
        LS_LAUNCH_CHECK();
    }
    const unsigned gv = (unsigned)((V + 127) / 128);
    if (idx_bytes == 4)
        k_cot_vertex_grad<int><<<gv, 128, 0, stream>>>(verts, (const int *)faces, V, inc_ptr, inc, wbar, gverts);
    else
        k_cot_vertex_grad<long long><<<gv, 128, 0, stream>>>(verts, (const long long *)faces, V, inc_ptr, inc, wbar, gverts);
    LS_LAUNCH_CHECK();
    return LS_OK;
}

extern "C" int ls_cot_laplacian_product_scratch_bytes(int64_t F, size_t *bytes_out) {
    return ls_laplacian_cot_bwd_scratch_bytes(F, bytes_out);   // the same 3F-float wbar buffer
}

extern "C" int ls_cot_laplacian_product_f32(const float *verts, const void *faces, int idx_bytes, int64_t F, int64_t V,
                                            const int32_t *inc_ptr, const int32_t *inc, const float *x, int k, float *y,
                                            float *w_out, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    LS_REQUIRE(idx_bytes == 4 || idx_bytes == 8, "idx_bytes must be 4 or 8");
    LS_REQUIRE(F >= 0 && V >= 0 && V < (int64_t)0x7ffffff0 && 3 * F < (int64_t)0x1ffffff0, "bad size");
    LS_REQUIRE(k >= 1, "k must be >= 1");
    if (V == 0) return LS_OK;
    LS_REQUIRE((F == 0 || (verts && faces && w_out)) && inc_ptr && inc && x && y, "NULL pointer");
    if (F > 0) {
        if (idx_bytes == 4) k_cot<int><<<grid_for(F, 256), 256, 0, stream>>>((const int *)faces, verts, F, V, w_out);
        else k_cot<long long><<<grid_for(F, 256), 256, 0, stream>>>((const long long *)faces, verts, F, V, w_out);
        LS_LAUNCH_CHECK();
    }
    const unsigned gv = (unsigned)((V + 127) / 128);
    if (idx_bytes == 4) k_cot_product<int><<<gv, 128, 0, stream>>>((const int *)faces, V, inc_ptr, inc, w_out, x, k, y);
    else k_cot_product<long long><<<gv, 128, 0, stream>>>((const long long *)faces, V, inc_ptr, inc, w_out, x, k, y);
    LS_LAUNCH_CHECK();
    return LS_OK;
}

extern "C" int ls_cot_laplacian_product_bwd_f32(const float *verts, const void *faces, int idx_bytes, int64_t F, int64_t V,
                                                const int32_t *inc_ptr, const int32_t *inc, const float *w, const float *x, int k,
                                                const float *gy, float *gx, float *gverts, void *scratch, size_t scratch_bytes,
                                                void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    LS_REQUIRE(idx_bytes == 4 || idx_bytes == 8, "idx_bytes must be 4 or 8");
    LS_REQUIRE(F >= 0 && V >= 0 && V < (int64_t)0x7ffffff0 && 3 * F < (int64_t)0x1ffffff0, "bad size");
    LS_REQUIRE(k >= 1, "k must be >= 1");
    if (V == 0 || (gx == nullptr && gverts == nullptr)) return LS_OK;
    LS_REQUIRE((F == 0 || faces) && inc_ptr && inc && gy, "NULL pointer");
    const unsigned gv = (unsigned)((V + 127) / 128);
    if (gx) {   // L is symmetric: the adjoint is the same gather, on gy
        LS_REQUIRE(F == 0 || w, "w is NULL");
        if (idx_bytes == 4) k_cot_product<int><<<gv, 128, 0, stream>>>((const int *)faces, V, inc_ptr, inc, w, gy, k, gx);
        else k_cot_product<long long><<<gv, 128, 0, stream>>>((const long long *)faces, V, inc_ptr, inc, w, gy, k, gx);
        LS_LAUNCH_CHECK();
    }
    if (gverts) {
        size_t need = 0;
        int rc = ls_cot_laplacian_product_scratch_bytes(F, &need);
        if (rc) return rc;
        LS_REQUIRE(verts && x, "NULL pointer");
        LS_REQUIRE(scratch != nullptr && scratch_bytes >= need,
                   "scratch NULL or smaller than ls_cot_laplacian_product_scratch_bytes(F)");
        float *wbar = (float *)scratch;
        if (F > 0) {
            if (idx_bytes == 4)
                k_cot_product_wbar<int><<<grid_for(F, 256), 256, 0, stream>>>((const int *)faces, F, x, gy, k, wbar);
            else
                k_cot_product_wbar<long long><<<grid_for(F, 256), 256, 0, stream>>>((const long long *)faces, F, x, gy, k, wbar);
            LS_LAUNCH_CHECK();
        }
        if (idx_bytes == 4)
            k_cot_vertex_grad<int><<<gv, 128, 0, stream>>>(verts, (const int *)faces, V, inc_ptr, inc, wbar, gverts);
        else
            k_cot_vertex_grad<long long><<<gv, 128, 0, stream>>>(verts, (const long long *)faces, V, inc_ptr, inc, wbar, gverts);
        LS_LAUNCH_CHECK();
    }
    return LS_OK;
}
