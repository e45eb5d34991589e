// ls_distance.cu -- point-to-mesh squared distances and the mesh Hausdorff distance (sm_90a): the figure scripts'
// igl.point_mesh_squared_distance and igl.hausdorff on the device.
//
// BVH: a linear BVH over the triangles.  The centroids are put in Morton order by ls_order_morton_seg (ls_order.cu), whose
// cells hold ~32 centroids on a surface (~120 at F = 2e6) in face-index order; each cell is then re-sorted along the
// 10-bit-per-axis Morton curve of the same box, so that the leaves follow the surface inside a cell too, whatever the
// face numbering.  The binary radix tree over the keys (cell code << 32 | sorted position) is built with one thread per internal node (Karras
// 2012), so the keys are unique even where faces coincide and a root-to-leaf path has at most 64 - 11 + 1 nodes (the
// codes have at most 21 bits).  The boxes are refitted bottom-up, one thread per leaf, with an arrival counter per node:
// they are min / max of fp32 corners, so they are exact whatever order the threads arrive in.
//
// Query: one thread per point, the points in Morton order, a 64-entry stack, the nearer child first.  The leaf test is
// the closest point on the triangle in fp64 from the exact fp32 corners (Ericson, Real-Time Collision Detection 5.1.5).
// A box is pruned only when its lower bound exceeds the best distance so far by more than the leaf test's rounding
// error, so no face whose computed distance is <= the best is ever skipped: the answer is the lowest-index face among
// those at the least computed fp64 distance, whatever order the tree is walked in.
//
// Batches (the _batch entry points): the BVHs of B packed meshes are one forest, built in the same launches as one BVH.  Each
// mesh's faces are ordered along the Morton curve of its own centroid box (ls_order_morton_seg), each mesh has its own
// radix tree over its own leaf range (the key comparisons end at the mesh's range; its internal nodes are
// [fo[b] - b, fo[b+1] - b - 1)) and its own header, so its prune slack and NaN rule are its own.  The points of a query are
// ordered by (segment, Morton cell), and each starts at its own mesh's root.  The answer of a point does not depend on the
// tree (above), so it is bitwise what a BVH of its mesh alone gives.  A single mesh is the batch B = 1.
//
// Backward (ls_distance_grad_f32): from the query's face and closest point, grad P in one streaming kernel and grad V as a
// per-vertex gather over the queries bucketed by face (ls_glue.cu's buckets), in fp64 without atomics.  It does not touch
// the BVH or the query kernel.
#include <float.h>
#include <math.h>
#include "ls_morton.cuh"

// ---- per-query bodies (__host__ __device__: tests/test_distance_host.py and test_distance_grad_host.py run them on the CPU)

// a triangle whose squared sine at corner a is below this (|ab x ac|^2 <= 2^-36 |ab|^2 |ac|^2, collinear corners or a
// zero-length edge) is treated as its three segments: Ericson's barycentrics lose ~eps / sin^2 there, while the segments
// are within the triangle's squared in-radius (<= sin^2 |ab|^2) of the exact distance
#define LS_DIST_DEGENERATE 0x1p-36

__host__ __device__ __forceinline__ double ls_dot3(const double *u, const double *v) {
    return u[0] * v[0] + u[1] * v[1] + u[2] * v[2];
}

// closest point to p on the segment [a, b]; returns its squared distance (and with W, the point's parameter t on [a, b])
template <bool W>
__host__ __device__ __forceinline__ double ls_closest_on_segment_body(const double *p, const double *a, const double *b,
                                                                      double *out, double *t_out) {
    double ab[3], ap[3];
    for (int d = 0; d < 3; ++d) {
        ab[d] = b[d] - a[d];
        ap[d] = p[d] - a[d];
    }
    const double den = ls_dot3(ab, ab);
    double t = den > 0.0 ? ls_dot3(ap, ab) / den : 0.0;
    t = t < 0.0 ? 0.0 : (t > 1.0 ? 1.0 : t);
    if (W) *t_out = t;
    double s = 0.0;
    for (int d = 0; d < 3; ++d) {
        out[d] = a[d] + t * ab[d];
        const double e = p[d] - out[d];
        s += e * e;
    }
    return s;
}

__host__ __device__ __forceinline__ double ls_closest_on_segment(const double *p, const double *a, const double *b,
                                                                 double *out) {
    return ls_closest_on_segment_body<false>(p, a, b, out, nullptr);
}

// closest point to p on the triangle (a, b, c), all in fp64 (the corners are exact fp32 values); returns |p - out|^2.
// With W, also beta[3]: the point's weights on (a, b, c), out = beta_a a + beta_b b + beta_c c up to rounding, from the same
// Voronoi region (face (1 - v - t, v, t), vertex one-hot, edge (1 - v, v) on its ends, a degenerate triangle (1 - t, t) on
// the segment it picked).  W = false is ls_closest_on_triangle, which the query kernel calls; the W branches compile out.
template <bool W>
__host__ __device__ __forceinline__ double ls_closest_on_triangle_body(const double *p, const double *a, const double *b,
                                                                       const double *c, double *out, double *beta) {
    double ab[3], ac[3], ap[3], bp[3], cp[3], n[3];
    for (int d = 0; d < 3; ++d) {
        ab[d] = b[d] - a[d];
        ac[d] = c[d] - a[d];
        ap[d] = p[d] - a[d];
        bp[d] = p[d] - b[d];
        cp[d] = p[d] - c[d];
    }
    n[0] = ab[1] * ac[2] - ab[2] * ac[1];
    n[1] = ab[2] * ac[0] - ab[0] * ac[2];
    n[2] = ab[0] * ac[1] - ab[1] * ac[0];
    double w[3];
    int region = 0;   // 0 face, 1 a, 2 b, 3 c, 4 ab, 5 ac, 6 bc, 7 degenerate
    double v = 0.0, t = 0.0;
    if (ls_dot3(n, n) <= LS_DIST_DEGENERATE * ls_dot3(ab, ab) * ls_dot3(ac, ac)) {
        region = 7;
    } else {
        const double d1 = ls_dot3(ab, ap), d2 = ls_dot3(ac, ap);
        const double d3 = ls_dot3(ab, bp), d4 = ls_dot3(ac, bp);
        const double d5 = ls_dot3(ab, cp), d6 = ls_dot3(ac, cp);
        const double vc = d1 * d4 - d3 * d2, vb = d5 * d2 - d1 * d6, va = d3 * d6 - d5 * d4;
        if (d1 <= 0.0 && d2 <= 0.0) {
            region = 1;
        } else if (d3 >= 0.0 && d4 <= d3) {
            region = 2;
        } else if (d6 >= 0.0 && d5 <= d6) {
            region = 3;
        } else if (vc <= 0.0 && d1 >= 0.0 && d3 <= 0.0) {
            region = 4;
            v = d1 / (d1 - d3);
        } else if (vb <= 0.0 && d2 >= 0.0 && d6 <= 0.0) {
            region = 5;
            v = d2 / (d2 - d6);
        } else if (va <= 0.0 && d4 - d3 >= 0.0 && d5 - d6 >= 0.0) {
            region = 6;
            v = (d4 - d3) / ((d4 - d3) + (d5 - d6));
        } else {
            const double den = 1.0 / (va + vb + vc);
            v = vb * den;
            t = vc * den;
        }
    }
    if (region == 7) {
        double q[3], t0 = 0.0, t1 = 0.0, t2 = 0.0;
        double best = ls_closest_on_segment_body<W>(p, a, b, out, &t0);
        int seg = 0;
        double s = ls_closest_on_segment_body<W>(p, b, c, q, &t1);
        if (s < best) {
            best = s;
            seg = 1;
            for (int d = 0; d < 3; ++d) out[d] = q[d];
        }
        s = ls_closest_on_segment_body<W>(p, c, a, q, &t2);
        if (s < best) {
            best = s;
            seg = 2;
            for (int d = 0; d < 3; ++d) out[d] = q[d];
        }
        if (W) {
            // segment ab: a + t0 (b - a); bc: b + t1 (c - b); ca: c + t2 (a - c)
            beta[0] = seg == 0 ? 1.0 - t0 : (seg == 2 ? t2 : 0.0);
            beta[1] = seg == 0 ? t0 : (seg == 1 ? 1.0 - t1 : 0.0);
            beta[2] = seg == 1 ? t1 : (seg == 2 ? 1.0 - t2 : 0.0);
        }
        return best;
    }
    if (W) {
        switch (region) {
            case 0: beta[0] = 1.0 - v - t; beta[1] = v; beta[2] = t; break;
            case 1: beta[0] = 1.0; beta[1] = 0.0; beta[2] = 0.0; break;
            case 2: beta[0] = 0.0; beta[1] = 1.0; beta[2] = 0.0; break;
            case 3: beta[0] = 0.0; beta[1] = 0.0; beta[2] = 1.0; break;
            case 4: beta[0] = 1.0 - v; beta[1] = v; beta[2] = 0.0; break;
            case 5: beta[0] = 1.0 - v; beta[1] = 0.0; beta[2] = v; break;
            default: beta[0] = 0.0; beta[1] = 1.0 - v; beta[2] = v; break;
        }
    }
    for (int d = 0; d < 3; ++d) {
        switch (region) {
            case 0: w[d] = a[d] + ab[d] * v + ac[d] * t; break;
            case 1: w[d] = a[d]; break;
            case 2: w[d] = b[d]; break;
            case 3: w[d] = c[d]; break;
            case 4: w[d] = a[d] + v * ab[d]; break;
            case 5: w[d] = a[d] + v * ac[d]; break;
            default: w[d] = b[d] + v * (c[d] - b[d]); break;
        }
    }
    double s = 0.0;
    for (int d = 0; d < 3; ++d) {
        out[d] = w[d];
        const double e = p[d] - w[d];
        s += e * e;
    }
    return s;
}

__host__ __device__ __forceinline__ double ls_closest_on_triangle(const double *p, const double *a, const double *b,
                                                                  const double *c, double *out) {
    return ls_closest_on_triangle_body<false>(p, a, b, c, out, nullptr);
}

// ls_closest_on_triangle plus the weights beta[3] of its point on (a, b, c): the backward's body
__host__ __device__ __forceinline__ double ls_closest_on_triangle_w(const double *p, const double *a, const double *b,
                                                                    const double *c, double *out, double *beta) {
    return ls_closest_on_triangle_body<true>(p, a, b, c, out, beta);
}

// A lower bound of the squared distance from p (fp32 coordinates held in fp64) to the box [lo, hi].  Every gap is a
// difference of two fp32 values, so it is >= 2^-149 when non-zero and its square is a normal fp64 number: the five
// roundings stay within a relative 5 * 2^-53, and the factor 1 - 2^-50 takes the result below the exact value.
__host__ __device__ __forceinline__ double ls_box_lower_bound(const double *p, const float *lo, const float *hi) {
    double s = 0.0;
    for (int d = 0; d < 3; ++d) {
        const double l = lo[d], h = hi[d];
        const double g = p[d] < l ? l - p[d] : (p[d] > h ? p[d] - h : 0.0);
        s += g * g;
    }
    return s * (1.0 - 0x1p-50);
}

// How far the leaf test's result may fall below the exact distance: its closest point is a convex combination of the
// corners up to a few roundings, so the error is a small multiple of 2^-53 (|p| + max|corner|)^2.  2^-40 leaves a margin
// of 2^13; pruning only boxes beyond best + slack costs nothing measurable and keeps every tie.
__host__ __device__ __forceinline__ double ls_prune_slack(double pmax, double corner_max) {
    const double r = pmax + corner_max;
    return 0x1p-40 * r * r;
}

namespace {

constexpr int DIST_STACK = 64;
constexpr int DIST_THREADS = 128;

struct BvhHeader {           // one per mesh at the start of the BVH, then the face offsets (B > 1)
    unsigned int nonfinite;  // a corner of some face of the mesh is NaN or infinite: every query answers NaN / -1
    unsigned int max_abs;    // bits of the largest |corner coordinate| (a non-negative float orders as its bits)
};

// 64 bytes: both children's boxes and references (ref >= 0: internal node, ~ref: leaf); parent and arrivals serve the build
struct __align__(16) Node {
    float lo0[3], hi0[3], lo1[3], hi1[3];
    int child[2];
    int parent;
    unsigned int arrivals;
};
static_assert(sizeof(Node) == 64, "one node is 64 bytes");

// 48 bytes: the corners in leaf order; a.w = face index, b.w = parent node (build), c.w = Morton cell code (build)
struct __align__(16) Leaf {
    float4 a, b, c;
};

struct DistRecord {          // the first 256 bytes of a query workspace
    double max;              // max of sqrD over the queries folded in (NaN-propagating; atomicMax of its bits)
    unsigned int overflow;   // a traversal stack overflowed
};

struct BvhWs {
    BvhHeader *hdr;          // B
    int64_t *fo;             // B + 1 face offsets (read when B > 1)
    Leaf *leaves;
    Node *nodes;             // F - B internal nodes; before the tree exists this region holds the build scratch below
    float *cent;             // 3F centroids
    int *perm;               // F: sorted position -> face
    unsigned int *fine;      // F: the fine Morton code at each sorted position
    char *order_ws;
    size_t order_bytes;
    size_t total;
};

void carve_bvh(BvhWs &w, char *base, int64_t F, int64_t B) {
    size_t order_bytes = 0;
    ls_order_seg_workspace_bytes(F, B, &order_bytes);
    const size_t o_fo = (size_t)B * sizeof(BvhHeader);
    const size_t o_leaf = ls_align_up(o_fo + (size_t)(B + 1) * 8, 256);   // 256 for one mesh
    const size_t o_node = ls_align_up(o_leaf + (size_t)F * sizeof(Leaf), 256);
    const size_t o_perm = ls_align_up((size_t)F * 12, 256);
    const size_t o_fine = o_perm + ls_align_up((size_t)F * 4, 256);
    const size_t o_ows = o_fine + ls_align_up((size_t)F * 4, 256);
    const size_t scratch = o_ows + order_bytes;
    const size_t nodes = (size_t)(F - B) * sizeof(Node);
    w.total = o_node + (scratch > nodes ? scratch : nodes);
    w.order_bytes = order_bytes;
    if (base) {
        w.hdr = (BvhHeader *)base;
        w.fo = (int64_t *)(base + o_fo);
        w.leaves = (Leaf *)(base + o_leaf);
        w.nodes = (Node *)(base + o_node);
        w.cent = (float *)(base + o_node);
        w.perm = (int *)(base + o_node + o_perm);
        w.fine = (unsigned int *)(base + o_node + o_fine);
        w.order_ws = base + o_node + o_ows;
    }
}

struct QueryWs {
    DistRecord *rec;
    int *perm;               // n: sorted position -> query
    char *order_ws;
    size_t order_bytes;
    size_t total;
};

void carve_query(QueryWs &w, char *base, int64_t n, int64_t S) {
    size_t order_bytes = 0;
    ls_order_seg_workspace_bytes(n, S, &order_bytes);
    const size_t o_perm = 256;
    const size_t o_ows = ls_align_up(o_perm + (size_t)n * 4, 256);
    w.total = o_ows + order_bytes;
    w.order_bytes = order_bytes;
    if (base) {
        w.rec = (DistRecord *)base;
        w.perm = (int *)(base + o_perm);
        w.order_ws = base + o_ows;
    }
}

__device__ __forceinline__ void face_corners(const float *__restrict__ verts, const void *__restrict__ faces, int idx_bytes,
                                             int64_t f, float (&x)[9]) {
    int64_t i[3];
#pragma unroll
    for (int k = 0; k < 3; ++k)
        i[k] = idx_bytes == 4 ? (int64_t)((const int32_t *)faces)[3 * f + k] : ((const int64_t *)faces)[3 * f + k];
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
        for (int d = 0; d < 3; ++d) x[3 * k + d] = verts[3 * i[k] + d];
}

// the NaN-propagating maximum of the non-negative doubles of a warp's lanes by segment, folded into out[s] as ordered bits
// (a non-negative double orders as its bits, and the NaN the query writes, 0x7ff8..., above +inf): atomicMax in any order gives
// the same result.  A warp whose lanes share one segment folds first.  Lanes with s < 0 take no part.
__device__ __forceinline__ void seg_max_fold(unsigned long long *out, int s, double v) {
    unsigned long long m = s >= 0 ? (unsigned long long)__double_as_longlong(v) : 0ull;
    const int s0 = __shfl_sync(0xffffffffu, s, 0);
    if (__all_sync(0xffffffffu, s == s0 || s < 0)) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long x = __shfl_xor_sync(0xffffffffu, m, o);
            m = x > m ? x : m;
        }
        if ((threadIdx.x & 31) == 0 && s0 >= 0) atomicMax(out + s0, m);
    } else if (s >= 0) {
        atomicMax(out + s, m);
    }
}

__global__ void k_face_centroids(const float *__restrict__ verts, const void *__restrict__ faces, int idx_bytes, int64_t F,
                                 const int64_t *__restrict__ fo, int B, float *__restrict__ cent, BvhHeader *__restrict__ hdr) {
    const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    float m = 0.f;
    bool finite = true;
    if (f < F) {
        float x[9];
        face_corners(verts, faces, idx_bytes, f, x);
#pragma unroll
        for (int k = 0; k < 9; ++k) {
            const float a = fabsf(x[k]);
            finite &= a <= FLT_MAX;
            m = fmaxf(m, a);
        }
#pragma unroll
        for (int d = 0; d < 3; ++d) cent[3 * f + d] = (x[d] + x[3 + d] + x[6 + d]) * (1.f / 3.f);
    }
    const int b = ls_segment_of(fo, B, f < F ? f : F - 1, 0);
    if (!finite) atomicOr(&hdr[b].nonfinite, 1u);
    if (__all_sync(0xffffffffu, b == __shfl_sync(0xffffffffu, b, 0))) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(&hdr[b].max_abs, __float_as_uint(m));
    } else if (m > 0.f) {
        atomicMax(&hdr[b].max_abs, __float_as_uint(m));
    }
}

constexpr int FINE_BITS = 10;

__global__ void k_fine_codes(const float *__restrict__ cent, int64_t F, const int64_t *__restrict__ fo, int B,
                             const int *__restrict__ perm, const unsigned int *__restrict__ bbox, unsigned int *__restrict__ fine) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= F) return;
    const int b = ls_segment_of(fo, B, i, 0);   // positions stay inside their mesh's range
    fine[i] = cell_code(cent, perm[i], bbox + 3 * b, bbox + 3 * B + 3 * b, FINE_BITS);
}

// One warp per 32 sorted positions; for each cell of ls_order_morton_seg (a run of equal codes, inside one mesh) that starts there, the warp
// sorts the run by (fine code, face): a rank sort in shared memory for runs of up to CELL_MAX, a shell sort by one lane
// beyond (coincident or outlier-squeezed centroids).  Other warps may read perm inside a run while it is being permuted;
// every entry of a run has the run's code, so what they read does not change their result.
constexpr int CELL_MAX = 256;

__global__ void __launch_bounds__(256) k_sort_cells(int64_t F, const unsigned int *__restrict__ code, int *perm,
                                                    unsigned int *fine) {
    __shared__ unsigned long long keys[8][CELL_MAX];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t base = ((int64_t)blockIdx.x * 8 + warp) * 32;
    if (base >= F) return;
    const int64_t p = base + lane;
    const bool start = p < F && (p == 0 || code[perm[p - 1]] != code[perm[p]]);
    unsigned int starts = __ballot_sync(0xffffffffu, start);
    unsigned long long *k = keys[warp];
    while (starts) {
        const int64_t s = base + __ffs(starts) - 1;
        starts &= starts - 1;
        const unsigned int c = code[perm[s]];
        int64_t e = F;
        for (int64_t j0 = s + 1; j0 < F; j0 += 32) {
            const int64_t j = j0 + lane;
            const unsigned int in = __ballot_sync(0xffffffffu, j < F && code[perm[j]] == c);
            if (in != 0xffffffffu) {
                e = j0 + __ffs(~in) - 1;
                break;
            }
        }
        const int64_t n = e - s;
        if (n <= CELL_MAX) {
            for (int64_t a = lane; a < n; a += 32) k[a] = ((unsigned long long)fine[s + a] << 32) | (unsigned int)perm[s + a];
            __syncwarp();
            for (int64_t a = lane; a < n; a += 32) {
                const unsigned long long key = k[a];
                int r = 0;
                for (int b = 0; b < n; ++b) r += k[b] < key;
                perm[s + r] = (int)(unsigned int)key;
                fine[s + r] = (unsigned int)(key >> 32);
            }
        } else if (lane == 0) {
            for (int64_t gap = n >> 1; gap > 0; gap >>= 1)
                for (int64_t a = s + gap; a < e; ++a) {
                    const int f = perm[a];
                    const unsigned int kf = fine[a];
                    int64_t j = a - gap;
                    while (j >= s && (fine[j] > kf || (fine[j] == kf && perm[j] > f))) {
                        perm[j + gap] = perm[j];
                        fine[j + gap] = fine[j];
                        j -= gap;
                    }
                    perm[j + gap] = f;
                    fine[j + gap] = kf;
                }
        }
        __syncwarp();
    }
}

__global__ void k_leaves(const float *__restrict__ verts, const void *__restrict__ faces, int idx_bytes, int64_t F,
                         const int *__restrict__ perm, const unsigned int *__restrict__ code, Leaf *__restrict__ leaves) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= F) return;
    const int f = perm[i];
    float x[9];
    face_corners(verts, faces, idx_bytes, f, x);
    Leaf l;
    l.a = make_float4(x[0], x[1], x[2], __int_as_float(f));
    l.b = make_float4(x[3], x[4], x[5], __int_as_float(-1));
    l.c = make_float4(x[6], x[7], x[8], __uint_as_float(code[f]));
    leaves[i] = l;
}

// common-prefix length of the keys (code << 32 | position) at positions i and j of one mesh's leaves; -1 outside [0, n)
__device__ __forceinline__ int key_delta(const Leaf *leaves, int64_t n, int64_t i, uint64_t ki, int64_t j) {
    if (j < 0 || j >= n) return -1;
    const uint64_t kj = ((uint64_t)__float_as_uint(leaves[j].c.w) << 32) | (uint64_t)j;
    return __clzll(ki ^ kj);
}

// Karras, "Maximizing parallelism in the construction of BVHs, octrees, and k-d trees" (HPG 2012), section 4: one thread per
// internal node of the forest (F - B of them).  Mesh b's tree is built over its own leaves [fo[b], fo[b+1]) in positions local
// to the mesh, and its nodes are [fo[b] - b, fo[b+1] - b - 1), its root first.
__global__ void k_radix_tree(Leaf *all_leaves, int64_t F, const int64_t *__restrict__ fo, int B, Node *__restrict__ all_nodes) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= F - B) return;
    const int mb = ls_segment_of(fo, B, t, 1);
    const int64_t f0 = fo ? fo[mb] : 0;
    const int64_t n = (fo ? fo[mb + 1] : F) - f0;
    Leaf *leaves = all_leaves + f0;
    Node *nodes = all_nodes + (f0 - mb);
    const int64_t i = t - (f0 - mb);
    const uint64_t ki = ((uint64_t)__float_as_uint(leaves[i].c.w) << 32) | (uint64_t)i;
    const int d = key_delta(leaves, n, i, ki, i + 1) > key_delta(leaves, n, i, ki, i - 1) ? 1 : -1;
    const int dmin = key_delta(leaves, n, i, ki, i - d);
    int64_t lmax = 2;
    while (key_delta(leaves, n, i, ki, i + lmax * d) > dmin) lmax *= 2;
    int64_t l = 0;
    for (int64_t t = lmax / 2; t >= 1; t /= 2)
        if (key_delta(leaves, n, i, ki, i + (l + t) * d) > dmin) l += t;
    const int64_t j = i + l * d;
    const int dnode = key_delta(leaves, n, i, ki, j);
    int64_t s = 0;
    for (int64_t div = 2;; div *= 2) {
        const int64_t t = (l + div - 1) / div;
        if (key_delta(leaves, n, i, ki, i + (s + t) * d) > dnode) s += t;
        if (t <= 1) break;
    }
    const int64_t g = i + s * d + (d < 0 ? -1 : 0);
    const int64_t lo = i < j ? i : j, hi = i < j ? j : i;
    Node &nd = nodes[i];
    const int self = (int)t, nbase = (int)(f0 - mb), lbase = (int)f0;   // forest indices
    if (lo == g) {
        nd.child[0] = ~(int)(lbase + g);
        leaves[g].b.w = __int_as_float(self);
    } else {
        nd.child[0] = (int)(nbase + g);
        nodes[g].parent = self;
    }
    if (hi == g + 1) {
        nd.child[1] = ~(int)(lbase + g + 1);
        leaves[g + 1].b.w = __int_as_float(self);
    } else {
        nd.child[1] = (int)(nbase + g + 1);
        nodes[g + 1].parent = self;
    }
    nd.arrivals = 0u;
    if (i == 0) nd.parent = -1;
}

__global__ void k_refit(const Leaf *__restrict__ leaves, int64_t n, Node *nodes) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Leaf l = leaves[i];
    float lo[3] = {fminf(fminf(l.a.x, l.b.x), l.c.x), fminf(fminf(l.a.y, l.b.y), l.c.y), fminf(fminf(l.a.z, l.b.z), l.c.z)};
    float hi[3] = {fmaxf(fmaxf(l.a.x, l.b.x), l.c.x), fmaxf(fmaxf(l.a.y, l.b.y), l.c.y), fmaxf(fmaxf(l.a.z, l.b.z), l.c.z)};
    int ref = ~(int)i;
    int p = __float_as_int(l.b.w);
    while (p >= 0) {
        volatile Node *nd = nodes + p;
        const int slot = nd->child[0] == ref ? 0 : 1;
        volatile float *mine_lo = slot ? nd->lo1 : nd->lo0, *mine_hi = slot ? nd->hi1 : nd->hi0;
        volatile float *other_lo = slot ? nd->lo0 : nd->lo1, *other_hi = slot ? nd->hi0 : nd->hi1;
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            mine_lo[d] = lo[d];
            mine_hi[d] = hi[d];
        }
        __threadfence();
        if (atomicAdd((unsigned int *)&nd->arrivals, 1u) == 0u) return;   // the sibling's thread carries on
        __threadfence();
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            lo[d] = fminf(lo[d], other_lo[d]);
            hi[d] = fmaxf(hi[d], other_hi[d]);
        }
        ref = p;
        p = nd->parent;
    }
}

__device__ __forceinline__ void leaf_test(const Leaf *__restrict__ leaves, int ref, const double *q, double &best, int &best_f,
                                          double *best_c) {
    const float4 *lp = reinterpret_cast<const float4 *>(leaves + ~ref);
    const float4 a = __ldg(lp), b = __ldg(lp + 1), c = __ldg(lp + 2);
    const double pa[3] = {a.x, a.y, a.z}, pb[3] = {b.x, b.y, b.z}, pc[3] = {c.x, c.y, c.z};
    double cl[3];
    const double s = ls_closest_on_triangle(q, pa, pb, pc, cl);
    const int f = __float_as_int(a.w);
    if (s < best || (s == best && f < best_f)) {
        best = s;
        best_f = f;
        best_c[0] = cl[0];
        best_c[1] = cl[1];
        best_c[2] = cl[2];
    }
}

// One thread per point in (segment, Morton) order; segment s of the points (po, S of them; NULL: one) is answered by mesh s of
// the forest, or by its only mesh when B == 1.  maxbits (S, nullable): seg_max_fold of sqrD per segment.
__global__ void __launch_bounds__(DIST_THREADS) k_distance_query(const BvhHeader *__restrict__ hdrs, const int64_t *__restrict__ fo,
                                                                 int B, const Node *__restrict__ nodes,
                                                                 const Leaf *__restrict__ leaves, int64_t F,
                                                                 const float *__restrict__ points, int64_t n,
                                                                 const int64_t *__restrict__ po, int S,
                                                                 const int *__restrict__ perm, double *__restrict__ sqrD,
                                                                 int64_t *__restrict__ face, double *__restrict__ closest,
                                                                 unsigned long long *__restrict__ maxbits,
                                                                 DistRecord *__restrict__ rec) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    double best = 0.0;
    int seg = -1;
    if (t < n) {
        const int64_t qi = perm[t];
        seg = ls_segment_of(po, S, qi, 0);
        const int mb = B == 1 ? 0 : seg;
        const BvhHeader *hdr = hdrs + mb;
        const int64_t f0 = fo ? fo[mb] : 0, nf = (fo ? fo[mb + 1] : F) - f0;
        const float px = points[3 * qi], py = points[3 * qi + 1], pz = points[3 * qi + 2];
        const double q[3] = {px, py, pz};
        int best_f = -1;
        double best_c[3];
        const bool finite = fabsf(px) <= FLT_MAX && fabsf(py) <= FLT_MAX && fabsf(pz) <= FLT_MAX;   // false on NaN
        const float pmax = fmaxf(fmaxf(fabsf(px), fabsf(py)), fabsf(pz));
        if (!finite || hdr->nonfinite) {
            best = __longlong_as_double(0x7ff8000000000000ll);
            best_c[0] = best_c[1] = best_c[2] = best;
        } else {
            best = __longlong_as_double(0x7ff0000000000000ll);   // +inf
            best_f = 0x7fffffff;
            const double slack = ls_prune_slack(pmax, __uint_as_float(hdr->max_abs));
            int stack[DIST_STACK];
            double stack_lb[DIST_STACK];
            int sp = 0;
            int node = nf > 1 ? (int)(f0 - mb) : ~(int)f0;   // the mesh's root
            bool overflow = false;
            while (true) {
                if (node < 0) {
                    leaf_test(leaves, node, q, best, best_f, best_c);
                } else {
                    const float4 *np = reinterpret_cast<const float4 *>(nodes + node);
                    const float4 r0 = __ldg(np), r1 = __ldg(np + 1), r2 = __ldg(np + 2), r3 = __ldg(np + 3);
                    const float lo0[3] = {r0.x, r0.y, r0.z}, hi0[3] = {r0.w, r1.x, r1.y};
                    const float lo1[3] = {r1.z, r1.w, r2.x}, hi1[3] = {r2.y, r2.z, r2.w};
                    const double b0 = ls_box_lower_bound(q, lo0, hi0), b1 = ls_box_lower_bound(q, lo1, hi1);
                    const int c0 = __float_as_int(r3.x), c1 = __float_as_int(r3.y);
                    const bool t0 = !(b0 > best + slack), t1 = !(b1 > best + slack);
                    if (t0 && t1) {
                        const bool first0 = b0 <= b1;
                        if (sp < DIST_STACK) {
                            stack[sp] = first0 ? c1 : c0;
                            stack_lb[sp] = first0 ? b1 : b0;
                            ++sp;
                        } else {
                            overflow = true;
                        }
                        node = first0 ? c0 : c1;
                        continue;
                    }
                    if (t0 || t1) {
                        node = t0 ? c0 : c1;
                        continue;
                    }
                }
                // pop the next subtree that can still hold a face at <= best
                bool found = false;
                while (sp > 0) {
                    --sp;
                    if (!(stack_lb[sp] > best + slack)) {
                        node = stack[sp];
                        found = true;
                        break;
                    }
                }
                if (!found) break;
            }
            if (overflow) atomicOr(&rec->overflow, 1u);
        }
        if (sqrD) sqrD[qi] = best;
        if (face) face[qi] = best_f;
        if (closest) {
            closest[3 * qi] = best_c[0];
            closest[3 * qi + 1] = best_c[1];
            closest[3 * qi + 2] = best_c[2];
        }
    }
    if (maxbits) seg_max_fold(maxbits, seg, best);
}

// out[s] = the sum of x[off[s] .. off[s+1]) in float64, one block per segment in a fixed order (per-thread strided sums, then a
// fixed tree): bitwise reproducible, no atomics.  The chamfer means of a batch.
__global__ void __launch_bounds__(256) k_segment_sum(const double *__restrict__ x, const int64_t *__restrict__ off,
                                                     double *__restrict__ out) {
    __shared__ double ws[8];
    const int64_t s = blockIdx.x, a = off[s], e = off[s + 1];
    double v = 0.0;
    for (int64_t i = a + threadIdx.x; i < e; i += blockDim.x) v += x[i];
    v = ls_warp_sum(v);
    if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double r = ws[0];
#pragma unroll
        for (int k = 1; k < 8; ++k) r += ws[k];
        out[s] = r;
    }
}

// ---- backward of sqrD (ls_distance_grad_f32) ---------------------------------------------------------------------------
// d sqrD[q] / d p_q = 2 (p_q - C_q) and d sqrD[q] / d V[k] = -2 beta_k (p_q - C_q) for the corners k of face I[q] (Danskin:
// only the active face counts).  C is the forward's; beta is recomputed from p and the corners by ls_closest_on_triangle_w.

// grad P: one thread per query, streaming; a row answered with face -1 gets NaN
__global__ void __launch_bounds__(256) k_distance_grad_points(const float *__restrict__ points, int64_t n,
                                                              const int64_t *__restrict__ face, const double *__restrict__ closest,
                                                              const double *__restrict__ gsq, float *__restrict__ gpoints) {
    const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n) return;
    if (face[q] < 0) {
        const float nan = __int_as_float(0x7fc00000);
        gpoints[3 * q] = gpoints[3 * q + 1] = gpoints[3 * q + 2] = nan;
        return;
    }
    const double g2 = 2.0 * gsq[q];
#pragma unroll
    for (int d = 0; d < 3; ++d) gpoints[3 * q + d] = (float)(g2 * ((double)points[3 * q + d] - closest[3 * q + d]));
}

// grad V: one thread per vertex, gathering over its corners 4 f + c (ascending, ls_face_incidence's buckets) and, per corner,
// over the queries whose face is f (ascending, qptr / qitems); fp64 sums in that fixed order, one rounding to float32.  No
// atomics: the result does not depend on the launch, the stream or the index type.
__global__ void __launch_bounds__(256) k_distance_grad_verts(const float *__restrict__ points, const float *__restrict__ verts,
                                                             const void *__restrict__ faces, int idx_bytes, int64_t V,
                                                             const double *__restrict__ closest, const double *__restrict__ gsq,
                                                             const int *__restrict__ inc_ptr, const int *__restrict__ inc,
                                                             const int *__restrict__ qptr, const int *__restrict__ qitems,
                                                             float *__restrict__ gverts) {
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    double acc[3] = {0.0, 0.0, 0.0};
    for (int e = inc_ptr[v], e1 = inc_ptr[v + 1]; e < e1; ++e) {
        const int item = inc[e];
        const int f = item >> 2, k = item & 3;
        const int j0 = qptr[f], j1 = qptr[f + 1];
        if (j0 == j1) continue;
        float x[9];
        face_corners(verts, faces, idx_bytes, f, x);
        const double a[3] = {x[0], x[1], x[2]}, b[3] = {x[3], x[4], x[5]}, c[3] = {x[6], x[7], x[8]};
        for (int j = j0; j < j1; ++j) {
            const int64_t q = qitems[j];
            const double p[3] = {points[3 * q], points[3 * q + 1], points[3 * q + 2]};
            double cl[3], beta[3];
            ls_closest_on_triangle_w(p, a, b, c, cl, beta);
            const double bk = k == 0 ? beta[0] : (k == 1 ? beta[1] : beta[2]);   // not beta[k]: keeps beta in registers
            const double w = -2.0 * gsq[q] * bk;
#pragma unroll
            for (int d = 0; d < 3; ++d) acc[d] += w * (p[d] - closest[3 * q + d]);
        }
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) gverts[3 * v + d] = (float)acc[d];
}

struct GradWs {
    int *qptr;               // F + 1: queries bucketed by their face
    int *qitems;             // n
    int *inc_ptr;            // V + 1: each vertex's corners
    int *inc;                // 3F
    char *bucket_ws;         // the two bucket builds, one after the other
    size_t total;
};

void carve_grad(GradWs &w, char *base, int64_t n, int64_t F, int64_t V) {
    size_t bf = 0, bv = 0;
    ls_bucket_workspace_bytes(F, &bf);
    ls_bucket_workspace_bytes(V, &bv);
    const size_t o_qitems = ls_align_up((size_t)(F + 1) * 4, 256);
    const size_t o_incptr = o_qitems + ls_align_up((size_t)n * 4, 256);
    const size_t o_inc = o_incptr + ls_align_up((size_t)(V + 1) * 4, 256);
    const size_t o_bws = o_inc + ls_align_up((size_t)F * 12, 256);
    w.total = o_bws + (bf > bv ? bf : bv);
    if (base) {
        w.qptr = (int *)base;
        w.qitems = (int *)(base + o_qitems);
        w.inc_ptr = (int *)(base + o_incptr);
        w.inc = (int *)(base + o_inc);
        w.bucket_ws = base + o_bws;
    }
}

int check_grad_sizes(int64_t n, int64_t F, int64_t V) {
    LS_REQUIRE(n >= 0 && n < (int64_t)0x7ffffff0, "n out of range");
    LS_REQUIRE(F >= 1 && 3 * F < (int64_t)0x1ffffff0, "F must be in [1, 0x1ffffff0 / 3)");
    LS_REQUIRE(V >= 1 && V < (int64_t)0x7ffffff0, "V out of range");
    return LS_OK;
}

int check_faces_f(int64_t F) {
    LS_REQUIRE(F >= 1 && F <= ((int64_t)1 << 30), "F must be in [1, 2^30]");
    return LS_OK;
}

int check_forest(int64_t F, int64_t B) {
    int rc = check_faces_f(F);
    if (rc) return rc;
    LS_REQUIRE(B >= 1 && B <= F && B <= LS_ORDER_MAX_SEGMENTS, "B must be in [1, min(F, 2^24)]");
    return LS_OK;
}

int check_points_n(int64_t n, int64_t S) {
    LS_REQUIRE(n >= 0 && n < (int64_t)0x7ffffff0, "n out of range");
    LS_REQUIRE(S >= 1 && S <= LS_ORDER_MAX_SEGMENTS, "the number of point segments must be in [1, 2^24]");
    return LS_OK;
}

// the forest of B meshes (fo: B + 1 device offsets, NULL when B == 1)
int build_forest(const float *verts, int64_t V, const void *faces, int idx_bytes, int64_t F, int64_t B, const int64_t *fo_in,
                 void *bvh, size_t bvh_bytes, cudaStream_t stream) {
    int rc = check_forest(F, B);
    if (rc) return rc;
    LS_REQUIRE(V >= 1 && V < (int64_t)0x7ffffff0, "V out of range");
    LS_REQUIRE(idx_bytes == 4 || idx_bytes == 8, "idx_bytes must be 4 or 8");
    LS_REQUIRE(verts && faces && bvh, "NULL pointer");
    LS_REQUIRE(B == 1 || fo_in, "NULL face_offsets");
    LS_REQUIRE(((uintptr_t)bvh & 255) == 0, "bvh must be 256-byte aligned");
    BvhWs w;
    carve_bvh(w, (char *)bvh, F, B);
    if (bvh_bytes < w.total) {
        ls_set_error("BVH buffer too small: %zu < %zu", bvh_bytes, w.total);
        return LS_ERR_WORKSPACE;
    }
    const int64_t *fo = B > 1 ? w.fo : nullptr;
    const unsigned int g = (unsigned int)((F + 255) / 256);
    LS_CUDA_TRY(cudaMemsetAsync(w.hdr, 0, (size_t)B * sizeof(BvhHeader), stream));
    if (fo) LS_CUDA_TRY(cudaMemcpyAsync(w.fo, fo_in, (size_t)(B + 1) * 8, cudaMemcpyDeviceToDevice, stream));
    k_face_centroids<<<g, 256, 0, stream>>>(verts, faces, idx_bytes, F, fo, (int)B, w.cent, w.hdr);
    LS_LAUNCH_CHECK();
    rc = ls_order_morton_seg(w.cent, F, fo, B, w.perm, w.order_ws, w.order_bytes, stream);
    if (rc) return rc;
    const unsigned int *code, *bbox;
    ls_order_views(w.order_ws, F, B, &code, &bbox);
    k_fine_codes<<<g, 256, 0, stream>>>(w.cent, F, fo, (int)B, w.perm, bbox, w.fine);
    LS_LAUNCH_CHECK();
    k_sort_cells<<<g, 256, 0, stream>>>(F, code, w.perm, w.fine);   // 8 warps x 32 positions per block
    LS_LAUNCH_CHECK();
    k_leaves<<<g, 256, 0, stream>>>(verts, faces, idx_bytes, F, w.perm, code, w.leaves);
    LS_LAUNCH_CHECK();
    if (F > B) {   // the scratch above lives where the nodes go: every reader of it has run by now
        k_radix_tree<<<(unsigned int)((F - B + 255) / 256), 256, 0, stream>>>(w.leaves, F, fo, (int)B, w.nodes);
        LS_LAUNCH_CHECK();
        k_refit<<<g, 256, 0, stream>>>(w.leaves, F, w.nodes);
        LS_LAUNCH_CHECK();
    }
    return LS_OK;
}

// the points in S segments (po: S + 1 device offsets, NULL when S == 1) against a forest of B meshes, S == B or B == 1.
// max_mode 1 / 2: maxout (S) is set to / folded with the segments' maxima (single-mesh calls pass the record's max).
int query_forest(const void *bvh, int64_t F, int64_t B, const float *points, int64_t n, int64_t S, const int64_t *po, double *sqrD,
                 int64_t *face, double *closest, double *maxout, int max_mode, void *workspace, size_t workspace_bytes,
                 cudaStream_t stream) {
    int rc = check_forest(F, B);
    if (rc) return rc;
    rc = check_points_n(n, S);
    if (rc) return rc;
    LS_REQUIRE(S == B || B == 1, "the points must have one segment per mesh, or the BVH one mesh");
    LS_REQUIRE(max_mode >= 0 && max_mode <= 2, "max_mode must be 0, 1 or 2");
    LS_REQUIRE(bvh && workspace, "NULL pointer");
    LS_REQUIRE(n == 0 || points, "NULL points");
    LS_REQUIRE(S == 1 || po, "NULL point_offsets");
    LS_REQUIRE(((uintptr_t)bvh & 255) == 0 && ((uintptr_t)workspace & 255) == 0, "bvh and workspace must be 256-byte aligned");
    QueryWs w;
    carve_query(w, (char *)workspace, n, S);
    if (workspace_bytes < w.total) {
        ls_set_error("query workspace too small: %zu < %zu", workspace_bytes, w.total);
        return LS_ERR_WORKSPACE;
    }
    BvhWs b;
    carve_bvh(b, (char *)bvh, F, B);
    if (!maxout) maxout = &w.rec->max;
    if (max_mode != 2) LS_CUDA_TRY(cudaMemsetAsync(w.rec, 0, sizeof(DistRecord), stream));
    if (max_mode == 1 && maxout != &w.rec->max) LS_CUDA_TRY(cudaMemsetAsync(maxout, 0, (size_t)S * 8, stream));
    if (n == 0) return LS_OK;
    rc = ls_order_morton_seg(points, n, S > 1 ? po : nullptr, S, w.perm, w.order_ws, w.order_bytes, stream);
    if (rc) return rc;
    const int64_t blocks = (n + DIST_THREADS - 1) / DIST_THREADS;
    k_distance_query<<<(unsigned int)blocks, DIST_THREADS, 0, stream>>>(
        b.hdr, B > 1 ? b.fo : nullptr, (int)B, b.nodes, b.leaves, F, points, n, S > 1 ? po : nullptr, (int)S, w.perm, sqrD, face,
        closest, max_mode ? (unsigned long long *)maxout : nullptr, w.rec);
    LS_LAUNCH_CHECK();
    return LS_OK;
}

}  // namespace

extern "C" int ls_distance_bvh_batch_bytes(int64_t F, int64_t B, size_t *bytes_out) {
    LS_REQUIRE(bytes_out != nullptr, "bytes_out is NULL");
    int rc = check_forest(F, B);
    if (rc) return rc;
    BvhWs w;
    carve_bvh(w, nullptr, F, B);
    *bytes_out = w.total;
    return LS_OK;
}

extern "C" int ls_distance_bvh_bytes(int64_t F, size_t *bytes_out) { return ls_distance_bvh_batch_bytes(F, 1, bytes_out); }

extern "C" int ls_distance_bvh_build(const float *verts, int64_t V, const void *faces, int idx_bytes, int64_t F, void *bvh,
                                     size_t bvh_bytes, void *stream) {
    return build_forest(verts, V, faces, idx_bytes, F, 1, nullptr, bvh, bvh_bytes, (cudaStream_t)stream);
}

extern "C" int ls_distance_bvh_batch_build(const float *verts, int64_t V, const void *faces, int idx_bytes, int64_t F, int64_t B,
                                           const int64_t *face_offsets, void *bvh, size_t bvh_bytes, void *stream) {
    LS_REQUIRE(face_offsets != nullptr, "NULL face_offsets");
    return build_forest(verts, V, faces, idx_bytes, F, B, face_offsets, bvh, bvh_bytes, (cudaStream_t)stream);
}

extern "C" int ls_distance_query_batch_workspace_bytes(int64_t n, int64_t S, size_t *bytes_out) {
    LS_REQUIRE(bytes_out != nullptr, "bytes_out is NULL");
    int rc = check_points_n(n, S);
    if (rc) return rc;
    QueryWs w;
    carve_query(w, nullptr, n, S);
    *bytes_out = w.total;
    return LS_OK;
}

extern "C" int ls_distance_query_workspace_bytes(int64_t n, size_t *bytes_out) {
    return ls_distance_query_batch_workspace_bytes(n, 1, bytes_out);
}

extern "C" int ls_distance_query(const void *bvh, int64_t F, const float *points, int64_t n, double *sqrD, int64_t *face,
                                 double *closest, int max_mode, void *workspace, size_t workspace_bytes, void *stream) {
    return query_forest(bvh, F, 1, points, n, 1, nullptr, sqrD, face, closest, nullptr, max_mode, workspace, workspace_bytes,
                        (cudaStream_t)stream);
}

extern "C" int ls_distance_query_batch(const void *bvh, int64_t F, int64_t B, const float *points, int64_t n, int64_t S,
                                       const int64_t *point_offsets, double *sqrD, int64_t *face, double *closest,
                                       double *max_out, int max_mode, void *workspace, size_t workspace_bytes, void *stream) {
    LS_REQUIRE(point_offsets != nullptr, "NULL point_offsets");
    LS_REQUIRE((max_mode == 0) == (max_out == nullptr), "max_out must be set exactly when max_mode is 1 or 2");
    return query_forest(bvh, F, B, points, n, S, point_offsets, sqrD, face, closest, max_out, max_mode, workspace,
                        workspace_bytes, (cudaStream_t)stream);
}

extern "C" int ls_distance_segment_sum_f64(const double *x, int64_t n, int64_t S, const int64_t *offsets, double *out,
                                           void *stream) {
    LS_REQUIRE(n >= 0 && S >= 1 && S < (int64_t)0x7fffffff, "n or S out of range");
    LS_REQUIRE(offsets && out && (n == 0 || x), "NULL pointer");
    k_segment_sum<<<(unsigned int)S, 256, 0, (cudaStream_t)stream>>>(x, offsets, out);
    LS_LAUNCH_CHECK();
    return LS_OK;
}

extern "C" int ls_distance_result(const void *workspace, double *max_host, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    LS_REQUIRE(workspace != nullptr, "NULL workspace");
    DistRecord r;
    LS_CUDA_TRY(cudaMemcpyAsync(&r, workspace, sizeof(r), cudaMemcpyDeviceToHost, stream));
    LS_CUDA_TRY(cudaStreamSynchronize(stream));
    if (max_host) *max_host = r.max;
    if (r.overflow) {
        ls_set_error("BVH traversal stack overflow (more than %d pending subtrees)", DIST_STACK);
        return LS_ERR_UNSUPPORTED;
    }
    return LS_OK;
}

extern "C" int ls_distance_grad_workspace_bytes(int64_t n, int64_t F, int64_t V, size_t *bytes_out) {
    LS_REQUIRE(bytes_out != nullptr, "bytes_out is NULL");
    int rc = check_grad_sizes(n, F, V);
    if (rc) return rc;
    GradWs w;
    carve_grad(w, nullptr, n, F, V);
    *bytes_out = w.total;
    return LS_OK;
}

extern "C" int ls_distance_grad_f32(const float *points, int64_t n, const float *verts, int64_t V, const void *faces, int idx_bytes,
                                    int64_t F, const int64_t *face, const double *closest, const double *grad_sqrD,
                                    float *grad_points, float *grad_verts, void *workspace, size_t workspace_bytes, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    int rc = check_grad_sizes(n, F, V);
    if (rc) return rc;
    LS_REQUIRE(idx_bytes == 4 || idx_bytes == 8, "idx_bytes must be 4 or 8");
    LS_REQUIRE(n == 0 || (points && face && closest && grad_sqrD), "NULL points, face, closest or grad_sqrD");
    GradWs w;
    if (grad_verts) {
        LS_REQUIRE(verts && faces, "grad_verts needs verts and faces");
        LS_REQUIRE(workspace != nullptr, "NULL workspace");
        LS_REQUIRE(((uintptr_t)workspace & 255) == 0, "workspace must be 256-byte aligned");
        carve_grad(w, (char *)workspace, n, F, V);
        if (workspace_bytes < w.total) {
            ls_set_error("gradient workspace too small: %zu < %zu", workspace_bytes, w.total);
            return LS_ERR_WORKSPACE;
        }
    }
    if (n == 0) {
        if (grad_verts) LS_CUDA_TRY(cudaMemsetAsync(grad_verts, 0, (size_t)V * 12, stream));
        return LS_OK;
    }
    if (grad_points) {
        k_distance_grad_points<<<(unsigned int)((n + 255) / 256), 256, 0, stream>>>(points, n, face, closest, grad_sqrD, grad_points);
        LS_LAUNCH_CHECK();
    }
    if (grad_verts) {
        // queries by face (rows answered with face -1 fall outside [0, F) and are skipped), then each vertex's corners
        rc = ls_buckets_async(face, 8, n, F, 0, w.qptr, w.qitems, w.bucket_ws, stream);
        if (rc) return rc;
        rc = ls_buckets_async(faces, idx_bytes, 3 * F, V, 1, w.inc_ptr, w.inc, w.bucket_ws, stream);
        if (rc) return rc;
        k_distance_grad_verts<<<(unsigned int)((V + 255) / 256), 256, 0, stream>>>(points, verts, faces, idx_bytes, V, closest,
                                                                                   grad_sqrD, w.inc_ptr, w.inc, w.qptr, w.qitems,
                                                                                   grad_verts);
        LS_LAUNCH_CHECK();
    }
    return LS_OK;
}
