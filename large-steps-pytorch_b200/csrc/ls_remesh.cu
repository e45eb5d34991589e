// ls_remesh.cu -- the Botsch-Kobbelt isotropic remesher of the reference loop (scripts/main.py:149, remesh_botsch) on the
// device: split, collapse, flip and tangential relaxation with projection, for closed, edge-manifold, consistently oriented
// triangle meshes.  The Python driver (largesteps_b200/remesh.py) runs the iterations and the rounds; each entry point below
// is one stage or one round on a caller-owned workspace, and reads back at most one set of counts.
//
// Topology, rebuilt at the start of every stage and round, from the faces alone (int32, a dead face is a row of -1):
//   inc_ptr / inc   vertex -> its corners 4 f + c, ascending (the buckets of ls_face_incidence, ls_glue.cu)
//   eptr / ev       edges (a, b), a < b, numbered by a, then b: the edges of a are eptr[a] .. eptr[a + 1]
//   ef              per edge, the face holding a -> b and the face holding b -> a
//   fe              per face, the edge of corners (k, k + 1)
// On a closed manifold every neighbour of a vertex is the next vertex of exactly one of its corners, so the one-ring is the
// corner list.  Collapse and flip rounds pick an independent set of local minima: every candidate writes its key into each
// vertex it depends on with atomicMin, and a candidate is applied only if it holds the minimum at all of them.  Two winners
// then share no vertex of their regions, so they read and write disjoint parts of the mesh and the result does not depend
// on the order in which threads run.  Eligibility and claims, the winner check and the rewrite are separate kernels.
//
// Predicates and positions are computed in float64 from the stored float32 coordinates; the file is built with
// -fmad=false, so every float64 expression rounds as written and tests/remesh_model.py repeats it bit for bit.
//
// Adaptive remeshing (the reference's remesh_botsch(V, F, target, iters, feature, project)) carries three per-vertex
// attributes in caller buffers of the vertices' capacity: the bounds vhigh = 1.4 t and vlow = 0.7 t, float64, and a feature
// flag, uint8.  An edge (a, b) is measured against the mean of its ends' bounds, a neighbour of a collapsing end x against
// x's own vhigh, and a feature vertex is never split, collapsed, flipped or moved.  The kernels take the three pointers and
// the scalar bounds; null pointers mean "every vertex has the scalar bound, no vertex is a feature", and since (x + x) / 2 == x
// in float64 a constant target gives the scalar call's result bit for bit.
#include <float.h>
#include <math.h>
#include "ls_common.cuh"

namespace {

constexpr int RT = 256;

enum : unsigned int {
    BAD_BOUNDARY = 1u,      // an edge with one face
    BAD_NONMANIFOLD = 2u,   // an edge with more than two faces
    BAD_ORIENTATION = 4u,   // a directed edge held by two faces
    BAD_DEGENERATE = 8u,    // a face that repeats a vertex
    BAD_INDEX = 16u,        // a face index outside [0, V)
};

struct Header {
    unsigned int flags;        // BAD_* bits of ls_remesh_check
    unsigned int count;        // winners of the last collapse or flip round
};

struct Ws {
    Header *hdr;
    int *inc_ptr, *inc, *eptr, *ev, *ef, *fe, *eflag, *vmap, *fmap, *ftmp, *scan;
    unsigned long long *ekey, *claim;
    float *vtmp;
    double *closest;
    char *bucket_ws, *query_ws;
    size_t query_bytes, total;
};

// Vc vertex slots, Fc face slots; edges: at most 3 Fc / 2 on a closed mesh
void carve(Ws &w, char *base, int64_t Vc, int64_t Fc) {
    const int64_t Ec = 3 * Fc / 2 + 1;
    size_t bucket_bytes = 0, query_bytes = 0;
    ls_bucket_workspace_bytes(Vc, &bucket_bytes);
    ls_distance_query_workspace_bytes(Vc, &query_bytes);
    int64_t nmax = Vc > Fc ? Vc : Fc;
    nmax = nmax > Ec ? nmax : Ec;
    size_t off = 256;
    auto take = [&](size_t bytes) {
        const size_t o = off;
        off = ls_align_up(off + bytes, 256);
        return o;
    };
    const size_t o_inc_ptr = take((size_t)(Vc + 1) * 4), o_inc = take((size_t)3 * Fc * 4 + 4);
    const size_t o_eptr = take((size_t)(Vc + 1) * 4), o_ev = take((size_t)2 * Ec * 4), o_ef = take((size_t)2 * Ec * 4);
    const size_t o_fe = take((size_t)3 * Fc * 4 + 4), o_eflag = take((size_t)(Ec + 1) * 4);
    const size_t o_vmap = take((size_t)(Vc + 1) * 4), o_fmap = take((size_t)(Fc + 1) * 4), o_ftmp = take((size_t)3 * Fc * 4 + 4);
    const size_t o_scan = take(ls_scan_scratch_elems(nmax + 1) * 4);
    const size_t o_ekey = take((size_t)Ec * 8), o_claim = take((size_t)Vc * 8);
    const size_t o_vtmp = take((size_t)3 * Vc * 4), o_closest = take((size_t)3 * Vc * 8);
    const size_t o_bucket = take(bucket_bytes), o_query = take(query_bytes);
    w.total = off;
    w.query_bytes = query_bytes;
    if (base) {
        w.hdr = (Header *)base;
        w.inc_ptr = (int *)(base + o_inc_ptr);
        w.inc = (int *)(base + o_inc);
        w.eptr = (int *)(base + o_eptr);
        w.ev = (int *)(base + o_ev);
        w.ef = (int *)(base + o_ef);
        w.fe = (int *)(base + o_fe);
        w.eflag = (int *)(base + o_eflag);
        w.vmap = (int *)(base + o_vmap);
        w.fmap = (int *)(base + o_fmap);
        w.ftmp = (int *)(base + o_ftmp);
        w.scan = (int *)(base + o_scan);
        w.ekey = (unsigned long long *)(base + o_ekey);
        w.claim = (unsigned long long *)(base + o_claim);
        w.vtmp = (float *)(base + o_vtmp);
        w.closest = (double *)(base + o_closest);
        w.bucket_ws = base + o_bucket;
        w.query_ws = base + o_query;
    }
}

unsigned int blocks(int64_t n) { return (unsigned int)((n + RT - 1) / RT); }

// ---- small float64 vector helpers --------------------------------------------------------------------------------------
struct D3 {
    double x, y, z;
};
__device__ __forceinline__ D3 ld(const float *v, int i) { return D3{(double)v[3 * i], (double)v[3 * i + 1], (double)v[3 * i + 2]}; }
__device__ __forceinline__ D3 sub(D3 a, D3 b) { return D3{a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ double dot(D3 a, D3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ D3 cross(D3 a, D3 b) { return D3{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
__device__ __forceinline__ double len2(D3 a) { return dot(a, a); }
// the float32 midpoint of two float32 points, held in float64
__device__ __forceinline__ D3 mid(D3 a, D3 b) {
    return D3{(double)(float)(0.5 * (a.x + b.x)), (double)(float)(0.5 * (a.y + b.y)), (double)(float)(0.5 * (a.z + b.z))};
}
// cos of the angle between the normals n and m; NaN when either is zero, which every caller rejects
__device__ __forceinline__ double cos_normals(D3 n, D3 m) { return dot(n, m) / (sqrt(len2(n)) * sqrt(len2(m))); }

// vertex i's own bound, or the scalar bound when there are no per-vertex bounds
__device__ __forceinline__ double own_bound(const double *per, double scalar, int i) { return per ? per[i] : scalar; }
// the bound of edge (a, b): the mean of its ends' bounds (split_edges_until_bound.cpp, collapse_edges.cpp)
__device__ __forceinline__ double edge_bound(const double *per, double scalar, int a, int b) {
    return per ? (per[a] + per[b]) / 2 : scalar;
}
__device__ __forceinline__ bool is_feature(const uint8_t *feat, int i) { return feat && feat[i]; }

__device__ __forceinline__ int corner_next(const int *faces, int item) {
    const int f = item >> 2, c = item & 3;
    return faces[3 * f + (c == 2 ? 0 : c + 1)];
}
__device__ __forceinline__ int corner_prev(const int *faces, int item) {
    const int f = item >> 2, c = item & 3;
    return faces[3 * f + (c == 0 ? 2 : c - 1)];
}

// ---- validation ----------------------------------------------------------------------------------------------------------
__global__ void k_check_faces(const int *__restrict__ faces, int64_t F, int64_t V, Header *hdr) {
    const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    const int a = faces[3 * f], b = faces[3 * f + 1], c = faces[3 * f + 2];
    unsigned int bad = 0;
    if (a < 0 || a >= V || b < 0 || b >= V || c < 0 || c >= V) bad |= BAD_INDEX;
    else if (a == b || b == c || c == a) bad |= BAD_DEGENERATE;
    if (bad) atomicOr(&hdr->flags, bad);
}

// per vertex a and each neighbour b: n_ab corners of a whose next is b (directed a -> b), n_ba whose previous is b
__global__ void k_check_edges(const int *__restrict__ faces, int64_t V, const int *__restrict__ inc_ptr, const int *__restrict__ inc,
                              Header *hdr) {
    const int64_t a = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= V) return;
    const int s = inc_ptr[a], e = inc_ptr[a + 1];
    unsigned int bad = 0;
    for (int i = s; i < e; ++i)
        for (int side = 0; side < 2; ++side) {
            const int b = side ? corner_prev(faces, inc[i]) : corner_next(faces, inc[i]);
            int n_ab = 0, n_ba = 0;
            for (int j = s; j < e; ++j) {
                n_ab += corner_next(faces, inc[j]) == b;
                n_ba += corner_prev(faces, inc[j]) == b;
            }
            if (n_ab + n_ba == 1) bad |= BAD_BOUNDARY;
            else if (n_ab + n_ba > 2) bad |= BAD_NONMANIFOLD;
            else if (n_ab != 1) bad |= BAD_ORIENTATION;
        }
    if (bad) atomicOr(&hdr->flags, bad);
}

// ---- topology ------------------------------------------------------------------------------------------------------------
__global__ void k_edge_count(const int *__restrict__ faces, int64_t V, const int *__restrict__ inc_ptr, const int *__restrict__ inc,
                             int *__restrict__ cnt) {
    const int64_t a = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= V) return;
    int n = 0;
    for (int i = inc_ptr[a]; i < inc_ptr[a + 1]; ++i) n += corner_next(faces, inc[i]) > a;
    cnt[a] = n;
}

__global__ void k_edge_fill(const int *__restrict__ faces, int64_t V, const int *__restrict__ inc_ptr, const int *__restrict__ inc,
                            const int *__restrict__ eptr, int *__restrict__ ev, int *__restrict__ ef) {
    const int64_t a = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= V) return;
    const int s = inc_ptr[a], e = inc_ptr[a + 1];
    for (int i = s; i < e; ++i) {
        const int b = corner_next(faces, inc[i]);
        if (b <= a) continue;
        int r = 0, back = -1;
        for (int j = s; j < e; ++j) {
            const int x = corner_next(faces, inc[j]);
            r += x > a && x < b;
            if (corner_prev(faces, inc[j]) == b) back = inc[j] >> 2;
        }
        const int id = eptr[a] + r;
        ev[2 * id] = (int)a;
        ev[2 * id + 1] = b;
        ef[2 * id] = inc[i] >> 2;
        ef[2 * id + 1] = back;
    }
}

__device__ __forceinline__ int edge_id(const int *__restrict__ eptr, const int *__restrict__ ev, int a, int b) {
    const int lo = a < b ? a : b, hi = a < b ? b : a;
    int l = eptr[lo], r = eptr[lo + 1] - 1;
    while (l < r) {
        const int m = (l + r) >> 1;
        if (ev[2 * m + 1] < hi) l = m + 1;
        else r = m;
    }
    return l;
}

__global__ void k_face_edges(const int *__restrict__ faces, int64_t F, const int *__restrict__ eptr, const int *__restrict__ ev,
                             int *__restrict__ fe) {
    const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F || faces[3 * f] < 0) return;
#pragma unroll
    for (int k = 0; k < 3; ++k) fe[3 * f + k] = edge_id(eptr, ev, faces[3 * f + k], faces[3 * f + (k + 1) % 3]);
}

int build_topology(const Ws &w, const int *faces, int64_t V, int64_t F, bool edges, cudaStream_t st) {
    int rc = ls_face_buckets_i32_async(faces, F, V, w.inc_ptr, w.inc, w.bucket_ws, st);
    if (rc || !edges) return rc;
    k_edge_count<<<blocks(V), RT, 0, st>>>(faces, V, w.inc_ptr, w.inc, w.eptr);
    LS_LAUNCH_CHECK();
    rc = ls_exclusive_scan_i32(w.eptr, w.eptr, V, w.scan, st);
    if (rc) return rc;
    k_edge_fill<<<blocks(V), RT, 0, st>>>(faces, V, w.inc_ptr, w.inc, w.eptr, w.ev, w.ef);
    LS_LAUNCH_CHECK();
    k_face_edges<<<blocks(F), RT, 0, st>>>(faces, F, w.eptr, w.ev, w.fe);
    LS_LAUNCH_CHECK();
    return LS_OK;
}

// ---- split ---------------------------------------------------------------------------------------------------------------
__global__ void k_split_mark(const float *__restrict__ verts, int64_t E, const int *__restrict__ ev, double high,
                             const double *__restrict__ vhigh, const uint8_t *__restrict__ feat, int *__restrict__ flag) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= E) return;
    const int a = ev[2 * e], b = ev[2 * e + 1];
    const double h = edge_bound(vhigh, high, a, b);
    flag[e] = !is_feature(feat, a) && !is_feature(feat, b) && len2(sub(ld(verts, a), ld(verts, b))) > h * h;
}

// the midpoint of a split edge takes the mean of its ends' bounds and is not a feature (split_edges.cpp)
__global__ void k_split_verts(float *__restrict__ verts, int64_t V, int64_t E, const int *__restrict__ ev, const int *__restrict__ rank,
                              double *__restrict__ vhigh, double *__restrict__ vlow, uint8_t *__restrict__ feat) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= E || rank[e + 1] == rank[e]) return;
    const int a = ev[2 * e], b = ev[2 * e + 1];
    const D3 m = mid(ld(verts, a), ld(verts, b));
    const int64_t n = V + rank[e];
    float *o = verts + 3 * n;
    o[0] = (float)m.x;
    o[1] = (float)m.y;
    o[2] = (float)m.z;
    if (vhigh) {
        vhigh[n] = (vhigh[a] + vhigh[b]) / 2;
        vlow[n] = (vlow[a] + vlow[b]) / 2;
        feat[n] = 0;
    }
}

// One thread per face: its triangles go to its own slot and, one per split edge in the order k = 0, 1, 2, to the slot
// F + 2 rank(e) + side of that edge (side 0 for the face holding a -> b); the new vertex of edge e is V + rank(e).
__global__ void k_split_faces(const float *__restrict__ verts, int *__restrict__ faces, int64_t V, int64_t F,
                              const int *__restrict__ fe, const int *__restrict__ ef, const int *__restrict__ rank) {
    const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    int v[3], m[3], slot[3], tri[4][3];
    int ns = 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        v[k] = faces[3 * f + k];
        const int e = fe[3 * f + k];
        m[k] = -1;
        if (rank[e + 1] != rank[e]) {
            m[k] = (int)V + rank[e];
            slot[ns++] = (int)F + 2 * rank[e] + (ef[2 * e] == (int)f ? 0 : 1);
        }
    }
    if (ns == 0) return;
    int nt = 0;
    auto put = [&](int a, int b, int c) {
        tri[nt][0] = a;
        tri[nt][1] = b;
        tri[nt][2] = c;
        ++nt;
    };
    if (ns == 1) {
        const int k = m[0] >= 0 ? 0 : (m[1] >= 0 ? 1 : 2);
        const int a = v[k], b = v[(k + 1) % 3], c = v[(k + 2) % 3];
        put(a, m[k], c);
        put(m[k], b, c);
    } else if (ns == 2) {
        const int u = m[0] < 0 ? 0 : (m[1] < 0 ? 1 : 2);   // the edge that is not split: (c, a)
        const int c = v[u], a = v[(u + 1) % 3], b = v[(u + 2) % 3];
        const int m0 = m[(u + 1) % 3], m1 = m[(u + 2) % 3];
        const D3 pa = ld(verts, a), pb = ld(verts, b), pc = ld(verts, c);
        const D3 q0 = mid(pa, pb), q1 = mid(pb, pc);
        put(m0, b, m1);
        if (len2(sub(pa, q1)) <= len2(sub(q0, pc))) {
            put(a, m0, m1);
            put(a, m1, c);
        } else {
            put(a, m0, c);
            put(m0, m1, c);
        }
    } else {
        put(m[0], m[1], m[2]);
        put(v[0], m[0], m[2]);
        put(m[0], v[1], m[1]);
        put(m[2], m[1], v[2]);
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) faces[3 * f + d] = tri[0][d];
    for (int t = 1; t < nt; ++t)
#pragma unroll
        for (int d = 0; d < 3; ++d) faces[3 * (int64_t)slot[t - 1] + d] = tri[t][d];
}

// ---- collapse ------------------------------------------------------------------------------------------------------------
constexpr unsigned long long NO_KEY = ~0ull;

// the faces around x other than the two of edge (x, y) keep their normal within 60 degrees when x moves to p
__device__ bool normals_keep(const float *verts, const int *faces, const int *inc_ptr, const int *inc, int x, int y, D3 p) {
    const D3 px = ld(verts, x);
    for (int i = inc_ptr[x]; i < inc_ptr[x + 1]; ++i) {
        const int n = corner_next(faces, inc[i]), q = corner_prev(faces, inc[i]);
        if (n == y || q == y) continue;
        const D3 pn = ld(verts, n), pq = ld(verts, q);
        const D3 before = cross(sub(pn, px), sub(pq, px)), after = cross(sub(pn, p), sub(pq, p));
        if (!(cos_normals(before, after) >= 0.5)) return false;
    }
    return true;
}

__device__ bool ring_within(const float *verts, const int *faces, const int *inc_ptr, const int *inc, int x, int y, D3 p, double high) {
    const double high2 = high * high;
    for (int i = inc_ptr[x]; i < inc_ptr[x + 1]; ++i) {
        const int n = corner_next(faces, inc[i]);
        if (n != y && len2(sub(ld(verts, n), p)) > high2) return false;
    }
    return true;
}

// claims x and its neighbours
__device__ void claim_ring(unsigned long long *claim, const int *faces, const int *inc_ptr, const int *inc, int x, unsigned long long key) {
    atomicMin(claim + x, key);
    for (int i = inc_ptr[x]; i < inc_ptr[x + 1]; ++i) atomicMin(claim + corner_next(faces, inc[i]), key);
}

__device__ bool holds_ring(const unsigned long long *claim, const int *faces, const int *inc_ptr, const int *inc, int x,
                           unsigned long long key) {
    if (claim[x] != key) return false;
    for (int i = inc_ptr[x]; i < inc_ptr[x + 1]; ++i)
        if (claim[corner_next(faces, inc[i])] != key) return false;
    return true;
}

__global__ void k_collapse_claim(const float *__restrict__ verts, const int *__restrict__ faces, int64_t E, const int *__restrict__ ev,
                                 const int *__restrict__ inc_ptr, const int *__restrict__ inc, double low, double high,
                                 const double *__restrict__ vhigh, const double *__restrict__ vlow, const uint8_t *__restrict__ feat,
                                 int allow, const int *__restrict__ ne, unsigned long long *__restrict__ key_out,
                                 unsigned long long *claim) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= *ne) return;
    const int a = ev[2 * e], b = ev[2 * e + 1];
    const D3 pa = ld(verts, a), pb = ld(verts, b);
    const double l2 = len2(sub(pa, pb)), lo = edge_bound(vlow, low, a, b);
    unsigned long long key = NO_KEY;
    if (allow && !is_feature(feat, a) && !is_feature(feat, b) && l2 < lo * lo) {
        const D3 p = mid(pa, pb);
        bool ok = ring_within(verts, faces, inc_ptr, inc, a, b, p, own_bound(vhigh, high, a)) &&
                  ring_within(verts, faces, inc_ptr, inc, b, a, p, own_bound(vhigh, high, b));
        // igl::edge_collapse_is_valid: an edge whose ends both have valence 3 is an edge of a lone tetrahedron (a closed
        // component of 4 vertices), which would fold into a doubled triangle
        ok = ok && !(inc_ptr[a + 1] - inc_ptr[a] == 3 && inc_ptr[b + 1] - inc_ptr[b] == 3);
        if (ok) {   // link condition: a and b share exactly the two opposite vertices
            int common = 0;
            for (int i = inc_ptr[a]; i < inc_ptr[a + 1]; ++i) {
                const int x = corner_next(faces, inc[i]);
                for (int j = inc_ptr[b]; j < inc_ptr[b + 1]; ++j) common += corner_next(faces, inc[j]) == x;
            }
            ok = common == 2;
        }
        ok = ok && normals_keep(verts, faces, inc_ptr, inc, a, b, p) && normals_keep(verts, faces, inc_ptr, inc, b, a, p);
        if (ok) key = ((unsigned long long)__float_as_uint((float)sqrt(l2)) << 32) | (unsigned long long)e;
    }
    key_out[e] = key;
    if (key != NO_KEY) {
        claim_ring(claim, faces, inc_ptr, inc, a, key);
        claim_ring(claim, faces, inc_ptr, inc, b, key);
    }
}

__global__ void k_round_check(const int *__restrict__ faces, int64_t E, const int *__restrict__ ev, const int *__restrict__ ef,
                              const int *__restrict__ inc_ptr, const int *__restrict__ inc, const unsigned long long *__restrict__ key_in,
                              const unsigned long long *__restrict__ claim, int flip, const int *__restrict__ ne,
                              int *__restrict__ win, Header *hdr) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= E) return;
    if (e >= *ne) {
        win[e] = 0;
        return;
    }
    const unsigned long long key = key_in[e];
    int w = 0;
    if (key != NO_KEY) {
        const int a = ev[2 * e], b = ev[2 * e + 1];
        if (flip) {
            int opp[2];
#pragma unroll
            for (int s = 0; s < 2; ++s) {
                const int f = ef[2 * e + s];
                const int x = faces[3 * f], y = faces[3 * f + 1], z = faces[3 * f + 2];
                opp[s] = (x != a && x != b) ? x : ((y != a && y != b) ? y : z);
            }
            w = claim[a] == key && claim[b] == key && claim[opp[0]] == key && claim[opp[1]] == key;
        } else {
            w = holds_ring(claim, faces, inc_ptr, inc, a, key) && holds_ring(claim, faces, inc_ptr, inc, b, key);
        }
    }
    win[e] = w;
    if (w) atomicAdd(&hdr->count, 1u);
}

// the winner (a, b) keeps a at the midpoint, and a keeps its own bounds; the two faces of the edge die, the other faces of b
// take a
__global__ void k_collapse_apply(float *__restrict__ verts, int *__restrict__ faces, int64_t E, const int *__restrict__ ev,
                                 const int *__restrict__ inc_ptr, const int *__restrict__ inc, const int *__restrict__ win) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= E || !win[e]) return;
    const int a = ev[2 * e], b = ev[2 * e + 1];
    const D3 p = mid(ld(verts, a), ld(verts, b));
    verts[3 * a] = (float)p.x;
    verts[3 * a + 1] = (float)p.y;
    verts[3 * a + 2] = (float)p.z;
    for (int i = inc_ptr[b]; i < inc_ptr[b + 1]; ++i) {
        const int f = inc[i] >> 2, c = inc[i] & 3;
        int *t = faces + 3 * (int64_t)f;
        if (t[0] == a || t[1] == a || t[2] == a) {
            t[0] = t[1] = t[2] = -1;
        } else {
            t[c] = a;
        }
    }
}

// ---- flip ----------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int third(const int *faces, int f, int a, int b) {
    const int x = faces[3 * f], y = faces[3 * f + 1], z = faces[3 * f + 2];
    return (x != a && x != b) ? x : ((y != a && y != b) ? y : z);
}
__device__ __forceinline__ int dev6(int v) { return v > 6 ? v - 6 : 6 - v; }

// edge (a, b) with faces (a, b, c) and (b, a, d) becomes (c, d) with faces (a, d, c) and (d, b, c)
__global__ void k_flip_claim(const float *__restrict__ verts, const int *__restrict__ faces, int64_t E, const int *__restrict__ ev,
                             const int *__restrict__ ef, const int *__restrict__ inc_ptr, const int *__restrict__ inc,
                             const uint8_t *__restrict__ feat, const int *__restrict__ ne, unsigned long long *__restrict__ key_out,
                             unsigned long long *claim) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= *ne) return;
    const int a = ev[2 * e], b = ev[2 * e + 1];
    const int c = third(faces, ef[2 * e], a, b), d = third(faces, ef[2 * e + 1], a, b);
    const int va = inc_ptr[a + 1] - inc_ptr[a], vb = inc_ptr[b + 1] - inc_ptr[b];
    const int vc = inc_ptr[c + 1] - inc_ptr[c], vd = inc_ptr[d + 1] - inc_ptr[d];
    const int gain = dev6(va) + dev6(vb) + dev6(vc) + dev6(vd) - (dev6(va - 1) + dev6(vb - 1) + dev6(vc + 1) + dev6(vd + 1));
    unsigned long long key = NO_KEY;
    bool ok = gain > 0 && c != d && !is_feature(feat, a) && !is_feature(feat, b) && !is_feature(feat, c) && !is_feature(feat, d);
    for (int i = inc_ptr[c]; ok && i < inc_ptr[c + 1]; ++i) ok = corner_next(faces, inc[i]) != d;
    if (ok) {
        const D3 pa = ld(verts, a), pb = ld(verts, b), pc = ld(verts, c), pd = ld(verts, d);
        const D3 n0 = cross(sub(pb, pa), sub(pc, pa)), n1 = cross(sub(pa, pb), sub(pd, pb));
        const D3 g0 = cross(sub(pd, pa), sub(pc, pa)), g1 = cross(sub(pb, pd), sub(pc, pd));
        ok = len2(g0) != 0.0 && len2(g1) != 0.0 && cos_normals(g0, n0) >= 0.5 && cos_normals(g0, n1) >= 0.5 &&
             cos_normals(g1, n0) >= 0.5 && cos_normals(g1, n1) >= 0.5;
    }
    if (ok) key = ((unsigned long long)(8 - gain) << 32) | (unsigned long long)e;
    key_out[e] = key;
    if (key != NO_KEY) {
        atomicMin(claim + a, key);
        atomicMin(claim + b, key);
        atomicMin(claim + c, key);
        atomicMin(claim + d, key);
    }
}

__global__ void k_flip_apply(int *__restrict__ faces, int64_t E, const int *__restrict__ ev, const int *__restrict__ ef,
                             const int *__restrict__ win) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= E || !win[e]) return;
    const int a = ev[2 * e], b = ev[2 * e + 1], f0 = ef[2 * e], f1 = ef[2 * e + 1];
    const int c = third(faces, f0, a, b), d = third(faces, f1, a, b);
    int *t0 = faces + 3 * (int64_t)f0, *t1 = faces + 3 * (int64_t)f1;
    t0[0] = a;
    t0[1] = d;
    t0[2] = c;
    t1[0] = d;
    t1[1] = b;
    t1[2] = c;
}

// ---- relax and project ---------------------------------------------------------------------------------------------------
// p = v - (I - n n^T)(v - q): q the mean of the neighbours, n the normalised sum of the faces' cross products (igl's default
// area-weighted vertex normal); every vertex reads the positions before the step.  A feature vertex stays where it is.
__global__ void k_relax(const float *__restrict__ verts, const int *__restrict__ faces, int64_t V, const int *__restrict__ inc_ptr,
                        const int *__restrict__ inc, const uint8_t *__restrict__ feat, float *__restrict__ out) {
    const int64_t a = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= V) return;
    const D3 pv = ld(verts, (int)a);
    const int s = inc_ptr[a], k = inc_ptr[a + 1] - s;
    D3 p = pv;
    if (k > 0 && !is_feature(feat, (int)a)) {
        D3 q{0.0, 0.0, 0.0}, n{0.0, 0.0, 0.0};
        for (int i = s; i < s + k; ++i) {
            const D3 x = ld(verts, corner_next(faces, inc[i]));
            q = D3{q.x + x.x, q.y + x.y, q.z + x.z};
            const int f = inc[i] >> 2;
            const D3 f0 = ld(verts, faces[3 * f]), f1 = ld(verts, faces[3 * f + 1]), f2 = ld(verts, faces[3 * f + 2]);
            const D3 c = cross(sub(f1, f0), sub(f2, f0));
            n = D3{n.x + c.x, n.y + c.y, n.z + c.z};
        }
        q = D3{q.x / k, q.y / k, q.z / k};
        const double nl = sqrt(len2(n));
        n = D3{n.x / nl, n.y / nl, n.z / nl};
        const D3 d = sub(pv, q);
        const double t = dot(n, d);
        p = sub(pv, D3{d.x - n.x * t, d.y - n.y * t, d.z - n.z * t});
    }
    out[3 * a] = (float)p.x;
    out[3 * a + 1] = (float)p.y;
    out[3 * a + 2] = (float)p.z;
}

// the projection of a feature vertex is not stored: it keeps its position bit for bit
__global__ void k_store_closest(const double *__restrict__ closest, int64_t n, const uint8_t *__restrict__ feat, float *__restrict__ verts) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && !is_feature(feat, (int)(i / 3))) verts[i] = (float)closest[i];
}

// ---- compaction ----------------------------------------------------------------------------------------------------------
__global__ void k_mark_live(const int *__restrict__ faces, int64_t F, int *__restrict__ vlive, int *__restrict__ flive) {
    const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    const bool live = faces[3 * f] >= 0;
    flive[f] = live;
    if (live)
#pragma unroll
        for (int k = 0; k < 3; ++k) vlive[faces[3 * f + k]] = 1;
}

// the positions go to out, the attributes (when vhigh is set) to out_high, out_low and out_feat
__global__ void k_compact_verts(const float *__restrict__ verts, int64_t V, const int *__restrict__ vmap, float *__restrict__ out,
                                const double *__restrict__ vhigh, const double *__restrict__ vlow, const uint8_t *__restrict__ feat,
                                double *__restrict__ out_high, double *__restrict__ out_low, uint8_t *__restrict__ out_feat) {
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V || vmap[v + 1] == vmap[v]) return;
    const int64_t o = vmap[v];
#pragma unroll
    for (int d = 0; d < 3; ++d) out[3 * o + d] = verts[3 * v + d];
    if (vhigh) {
        out_high[o] = vhigh[v];
        out_low[o] = vlow[v];
        out_feat[o] = feat[v];
    }
}

__global__ void k_compact_faces(const int *__restrict__ faces, int64_t F, const int *__restrict__ fmap, const int *__restrict__ vmap,
                                int *__restrict__ out) {
    const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F || fmap[f + 1] == fmap[f]) return;
#pragma unroll
    for (int k = 0; k < 3; ++k) out[3 * (int64_t)fmap[f] + k] = vmap[faces[3 * f + k]];
}

// ---- host helpers --------------------------------------------------------------------------------------------------------
int open_ws(Ws &w, const int *faces, int64_t V, int64_t F, int64_t Vc, int64_t Fc, void *ws, size_t bytes) {
    LS_REQUIRE(V >= 0 && F >= 0 && V <= Vc && F <= Fc && Vc < (int64_t)0x3ffffff0 && 3 * Fc < (int64_t)0x3ffffff0,
               "sizes out of range");
    LS_REQUIRE(faces != nullptr && ws != nullptr, "NULL pointer");
    LS_REQUIRE(F == 0 || V > 0, "faces without vertices");
    LS_REQUIRE(((uintptr_t)ws & 255) == 0, "workspace must be 256-byte aligned");
    carve(w, (char *)ws, Vc, Fc);
    if (bytes < w.total) {
        ls_set_error("remesh workspace too small: %zu < %zu", bytes, w.total);
        return LS_ERR_WORKSPACE;
    }
    return LS_OK;
}

int read_count(const Ws &w, int64_t *out, cudaStream_t st) {
    Header h;
    LS_CUDA_TRY(cudaMemcpyAsync(&h, w.hdr, sizeof(h), cudaMemcpyDeviceToHost, st));
    LS_CUDA_TRY(cudaStreamSynchronize(st));
    if (out) *out = h.count;
    return LS_OK;
}

// one collapse or flip round after the claims: check, apply, read the number of winners
int finish_round(const Ws &w, float *verts, int *faces, int64_t V, int64_t E, int flip, int64_t *count, cudaStream_t st) {
    k_round_check<<<blocks(E), RT, 0, st>>>(faces, E, w.ev, w.ef, w.inc_ptr, w.inc, w.ekey, w.claim, flip, w.eptr + V, w.eflag, w.hdr);
    LS_LAUNCH_CHECK();
    if (flip) k_flip_apply<<<blocks(E), RT, 0, st>>>(faces, E, w.ev, w.ef, w.eflag);
    else k_collapse_apply<<<blocks(E), RT, 0, st>>>(verts, faces, E, w.ev, w.inc_ptr, w.inc, w.eflag);
    LS_LAUNCH_CHECK();
    return read_count(w, count, st);
}

int begin_round(const Ws &w, const int *faces, int64_t V, int64_t F, int64_t *E, cudaStream_t st) {
    LS_CUDA_TRY(cudaMemsetAsync(w.hdr, 0, sizeof(Header), st));
    LS_CUDA_TRY(cudaMemsetAsync(w.claim, 0xff, (size_t)(V > 0 ? V : 1) * 8, st));
    int rc = build_topology(w, faces, V, F, true, st);
    *E = 3 * F / 2;   // a bound: the kernels read the number of edges of the live faces from eptr[V]
    return rc;
}

// the per-vertex attributes of the _v entry points: all NULL or all set
int check_attrs(const double *vhigh, const double *vlow, const uint8_t *feature) {
    LS_REQUIRE((vhigh == nullptr) == (vlow == nullptr) && (vhigh == nullptr) == (feature == nullptr),
               "vhigh, vlow and feature must be all NULL or all set");
    return LS_OK;
}

}  // namespace

extern "C" int ls_remesh_workspace_bytes(int64_t V, int64_t F, size_t *bytes_out) {
    LS_REQUIRE(bytes_out != nullptr, "bytes_out is NULL");
    LS_REQUIRE(V >= 0 && F >= 0 && V < (int64_t)0x3ffffff0 && 3 * F < (int64_t)0x3ffffff0, "sizes out of range");
    Ws w;
    carve(w, nullptr, V, F);
    *bytes_out = w.total;
    return LS_OK;
}

extern "C" int ls_remesh_check(const int32_t *faces, int64_t F, int64_t V, void *workspace, size_t workspace_bytes,
                               uint32_t *flags_out, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    LS_REQUIRE(flags_out != nullptr, "flags_out is NULL");
    LS_REQUIRE(F >= 1, "the mesh has no faces");
    if (V == 0) {   // every index is out of range
        ls_set_error("a face indexes a vertex outside [0, 0)");
        return LS_ERR_INDEX_RANGE;
    }
    Ws w;
    int rc = open_ws(w, faces, V, F, V, F, workspace, workspace_bytes);
    if (rc) return rc;
    LS_CUDA_TRY(cudaMemsetAsync(w.hdr, 0, sizeof(Header), st));
    k_check_faces<<<blocks(F), RT, 0, st>>>(faces, F, V, w.hdr);
    LS_LAUNCH_CHECK();
    rc = ls_face_buckets_i32_async(faces, F, V, w.inc_ptr, w.inc, w.bucket_ws, st);
    if (rc) return rc;
    k_check_edges<<<blocks(V), RT, 0, st>>>(faces, V, w.inc_ptr, w.inc, w.hdr);
    LS_LAUNCH_CHECK();
    Header h;
    LS_CUDA_TRY(cudaMemcpyAsync(&h, w.hdr, sizeof(h), cudaMemcpyDeviceToHost, st));
    LS_CUDA_TRY(cudaStreamSynchronize(st));
    *flags_out = h.flags;
    if (h.flags & BAD_INDEX) {
        ls_set_error("a face indexes a vertex outside [0, %lld)", (long long)V);
        return LS_ERR_INDEX_RANGE;
    }
    return LS_OK;
}

extern "C" int ls_remesh_split_v(float *verts, int32_t *faces, int64_t V, int64_t F, int64_t V_cap, int64_t F_cap, double high,
                                 double *vhigh, double *vlow, uint8_t *feature, void *workspace, size_t workspace_bytes,
                                 int64_t *n_split, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    LS_REQUIRE(n_split != nullptr && verts != nullptr, "NULL pointer");
    int rc = check_attrs(vhigh, vlow, feature);
    if (rc) return rc;
    LS_REQUIRE(vhigh || high > 0.0, "high must be positive");
    LS_REQUIRE(V_cap >= V + 3 * F / 2 && F_cap >= 4 * F, "capacity below V + E vertices and 4 F faces");
    Ws w;
    rc = open_ws(w, faces, V, F, V_cap, F_cap, workspace, workspace_bytes);
    if (rc) return rc;
    *n_split = 0;
    if (F == 0) return LS_OK;
    rc = build_topology(w, faces, V, F, true, st);
    if (rc) return rc;
    const int64_t E = 3 * F / 2;
    k_split_mark<<<blocks(E), RT, 0, st>>>(verts, E, w.ev, high, vhigh, feature, w.eflag);
    LS_LAUNCH_CHECK();
    rc = ls_exclusive_scan_i32(w.eflag, w.eflag, E, w.scan, st);
    if (rc) return rc;
    k_split_verts<<<blocks(E), RT, 0, st>>>(verts, V, E, w.ev, w.eflag, vhigh, vlow, feature);
    LS_LAUNCH_CHECK();
    k_split_faces<<<blocks(F), RT, 0, st>>>(verts, faces, V, F, w.fe, w.ef, w.eflag);
    LS_LAUNCH_CHECK();
    int total = 0;
    LS_CUDA_TRY(cudaMemcpyAsync(&total, w.eflag + E, sizeof(int), cudaMemcpyDeviceToHost, st));
    LS_CUDA_TRY(cudaStreamSynchronize(st));
    *n_split = total;
    return LS_OK;
}

extern "C" int ls_remesh_collapse_round_v(float *verts, int32_t *faces, int64_t V, int64_t F, int64_t V_live, double low, double high,
                                          double *vhigh, double *vlow, uint8_t *feature, void *workspace, size_t workspace_bytes,
                                          int64_t *n_collapsed, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    LS_REQUIRE(n_collapsed != nullptr && verts != nullptr, "NULL pointer");
    int rc = check_attrs(vhigh, vlow, feature);
    if (rc) return rc;
    LS_REQUIRE(vhigh || (low > 0.0 && high > low), "need 0 < low < high");
    Ws w;
    rc = open_ws(w, faces, V, F, V, F, workspace, workspace_bytes);
    if (rc) return rc;
    *n_collapsed = 0;
    if (F == 0) return LS_OK;
    int64_t E;
    rc = begin_round(w, faces, V, F, &E, st);
    if (rc) return rc;
    k_collapse_claim<<<blocks(E), RT, 0, st>>>(verts, faces, E, w.ev, w.inc_ptr, w.inc, low, high, vhigh, vlow, feature, V_live > 4,
                                               w.eptr + V, w.ekey, w.claim);
    LS_LAUNCH_CHECK();
    return finish_round(w, verts, faces, V, E, 0, n_collapsed, st);
}

extern "C" int ls_remesh_flip_round_v(const float *verts, int32_t *faces, int64_t V, int64_t F, double *vhigh, double *vlow,
                                      uint8_t *feature, void *workspace, size_t workspace_bytes, int64_t *n_flipped, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    LS_REQUIRE(n_flipped != nullptr && verts != nullptr, "NULL pointer");
    int rc = check_attrs(vhigh, vlow, feature);
    if (rc) return rc;
    Ws w;
    rc = open_ws(w, faces, V, F, V, F, workspace, workspace_bytes);
    if (rc) return rc;
    *n_flipped = 0;
    if (F == 0) return LS_OK;
    int64_t E;
    rc = begin_round(w, faces, V, F, &E, st);
    if (rc) return rc;
    k_flip_claim<<<blocks(E), RT, 0, st>>>(verts, faces, E, w.ev, w.ef, w.inc_ptr, w.inc, feature, w.eptr + V, w.ekey, w.claim);
    LS_LAUNCH_CHECK();
    return finish_round(w, (float *)verts, faces, V, E, 1, n_flipped, st);
}

// The attributes are staged in the `closest` region (24 bytes per vertex slot): vhigh, vlow, then the flags, 17 bytes per slot.
extern "C" int ls_remesh_compact_v(float *verts, int32_t *faces, int64_t V, int64_t F, double *vhigh, double *vlow, uint8_t *feature,
                                   void *workspace, size_t workspace_bytes, int64_t *V_out, int64_t *F_out, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    LS_REQUIRE(V_out && F_out && verts, "NULL pointer");
    int rc = check_attrs(vhigh, vlow, feature);
    if (rc) return rc;
    Ws w;
    rc = open_ws(w, faces, V, F, V, F, workspace, workspace_bytes);
    if (rc) return rc;
    *V_out = 0;   // no face: no vertex is referenced
    *F_out = 0;
    if (F == 0) return LS_OK;
    double *high_tmp = w.closest, *low_tmp = w.closest + V;
    uint8_t *feat_tmp = (uint8_t *)(w.closest + 2 * V);
    LS_CUDA_TRY(cudaMemsetAsync(w.vmap, 0, (size_t)(V + 1) * 4, st));
    k_mark_live<<<blocks(F), RT, 0, st>>>(faces, F, w.vmap, w.fmap);
    LS_LAUNCH_CHECK();
    rc = ls_exclusive_scan_i32(w.vmap, w.vmap, V, w.scan, st);
    if (rc) return rc;
    rc = ls_exclusive_scan_i32(w.fmap, w.fmap, F, w.scan, st);
    if (rc) return rc;
    k_compact_verts<<<blocks(V), RT, 0, st>>>(verts, V, w.vmap, w.vtmp, vhigh, vlow, feature, high_tmp, low_tmp, feat_tmp);
    LS_LAUNCH_CHECK();
    k_compact_faces<<<blocks(F), RT, 0, st>>>(faces, F, w.fmap, w.vmap, w.ftmp);
    LS_LAUNCH_CHECK();
    int nv = 0, nf = 0;
    LS_CUDA_TRY(cudaMemcpyAsync(&nv, w.vmap + V, sizeof(int), cudaMemcpyDeviceToHost, st));
    LS_CUDA_TRY(cudaMemcpyAsync(&nf, w.fmap + F, sizeof(int), cudaMemcpyDeviceToHost, st));
    LS_CUDA_TRY(cudaStreamSynchronize(st));
    if (nv > 0) LS_CUDA_TRY(cudaMemcpyAsync(verts, w.vtmp, (size_t)nv * 12, cudaMemcpyDeviceToDevice, st));
    if (nf > 0) LS_CUDA_TRY(cudaMemcpyAsync(faces, w.ftmp, (size_t)nf * 12, cudaMemcpyDeviceToDevice, st));
    if (nv > 0 && vhigh) {
        LS_CUDA_TRY(cudaMemcpyAsync(vhigh, high_tmp, (size_t)nv * 8, cudaMemcpyDeviceToDevice, st));
        LS_CUDA_TRY(cudaMemcpyAsync(vlow, low_tmp, (size_t)nv * 8, cudaMemcpyDeviceToDevice, st));
        LS_CUDA_TRY(cudaMemcpyAsync(feature, feat_tmp, (size_t)nv, cudaMemcpyDeviceToDevice, st));
    }
    *V_out = nv;
    *F_out = nf;
    return LS_OK;
}

extern "C" int ls_remesh_relax_v(float *verts, const int32_t *faces, int64_t V, int64_t F, const void *bvh, int64_t F0, double *vhigh,
                                 double *vlow, uint8_t *feature, void *workspace, size_t workspace_bytes, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    LS_REQUIRE(bvh != nullptr && verts != nullptr, "NULL pointer");
    int rc = check_attrs(vhigh, vlow, feature);
    if (rc) return rc;
    Ws w;
    rc = open_ws(w, faces, V, F, V, F, workspace, workspace_bytes);
    if (rc) return rc;
    if (V == 0) return LS_OK;
    rc = build_topology(w, faces, V, F, false, st);
    if (rc) return rc;
    k_relax<<<blocks(V), RT, 0, st>>>(verts, faces, V, w.inc_ptr, w.inc, feature, w.vtmp);
    LS_LAUNCH_CHECK();
    rc = ls_distance_query(bvh, F0, w.vtmp, V, nullptr, nullptr, w.closest, 0, w.query_ws, w.query_bytes, st);
    if (rc) return rc;
    k_store_closest<<<blocks(3 * V), RT, 0, st>>>(w.closest, 3 * V, feature, verts);
    LS_LAUNCH_CHECK();
    return LS_OK;
}

extern "C" int ls_remesh_split(float *verts, int32_t *faces, int64_t V, int64_t F, int64_t V_cap, int64_t F_cap, double high,
                               void *workspace, size_t workspace_bytes, int64_t *n_split, void *stream) {
    return ls_remesh_split_v(verts, faces, V, F, V_cap, F_cap, high, nullptr, nullptr, nullptr, workspace, workspace_bytes, n_split,
                             stream);
}

extern "C" int ls_remesh_collapse_round(float *verts, int32_t *faces, int64_t V, int64_t F, int64_t V_live, double low, double high,
                                        void *workspace, size_t workspace_bytes, int64_t *n_collapsed, void *stream) {
    return ls_remesh_collapse_round_v(verts, faces, V, F, V_live, low, high, nullptr, nullptr, nullptr, workspace, workspace_bytes,
                                      n_collapsed, stream);
}

extern "C" int ls_remesh_flip_round(const float *verts, int32_t *faces, int64_t V, int64_t F, void *workspace, size_t workspace_bytes,
                                    int64_t *n_flipped, void *stream) {
    return ls_remesh_flip_round_v(verts, faces, V, F, nullptr, nullptr, nullptr, workspace, workspace_bytes, n_flipped, stream);
}

extern "C" int ls_remesh_compact(float *verts, int32_t *faces, int64_t V, int64_t F, void *workspace, size_t workspace_bytes,
                                 int64_t *V_out, int64_t *F_out, void *stream) {
    return ls_remesh_compact_v(verts, faces, V, F, nullptr, nullptr, nullptr, workspace, workspace_bytes, V_out, F_out, stream);
}

extern "C" int ls_remesh_relax(float *verts, const int32_t *faces, int64_t V, int64_t F, const void *bvh, int64_t F0, void *workspace,
                               size_t workspace_bytes, void *stream) {
    return ls_remesh_relax_v(verts, faces, V, F, bvh, F0, nullptr, nullptr, nullptr, workspace, workspace_bytes, stream);
}
