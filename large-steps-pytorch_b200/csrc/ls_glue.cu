// ls_glue.cu -- the per-step glue either side of the solve (SURVEY 8 f2), on the device and differentiable:
//   v_opt = v_unique[duplicate_idx]                       scripts/main.py:176      (gather; backward = segmented sum)
//   compute_face_normals / compute_vertex_normals         scripts/geometry.py:91-147, main.py:177-180
// and the one operator of scripts/geometry.py the reference loop does not call:
//   massmatrix_voronoi (mixed Voronoi area per vertex)    scripts/geometry.py:35-89
// The reference runs ~40 eager kernels per step for these (index_select x6, cross, norms, acos, nine index_add_ calls with
// atomics, ...).  Here: one kernel per operator per direction.  Scatter-adds are turned into gathers over an incidence list
// built once per connectivity (vertex -> its (face, corner) pairs, sorted), so there are no atomics in the per-step
// kernels and results are bit-reproducible.
//
// compute_vertex_normals quirk reproduced on purpose (geometry.py:137-140): `d0 / torch.norm(d0)` divides by the Frobenius
// norm of the WHOLE (3,F) edge field, not per face, so every corner weight is acos(tiny) ~ pi/2 and its derivative couples
// all faces through three global scalars.  The backward below carries those terms.  The vertex-normal kernels take those
// scalars per mesh of a packed batch, so each mesh gets exactly what a call on it alone gives; a single mesh is a batch of one.
//
// The normals' per-face and per-vertex bodies are __host__ __device__ functions that the kernels call, so that
// tests/test_glue_host.py can run on a CPU the code the GPU runs, against the float64 model of tests/glue_model.py.
#include "ls_common.cuh"

namespace {

constexpr int GT = 256;

template <typename I>
__host__ __device__ __forceinline__ void face_ids(const I *faces, int64_t f, int (&id)[3]) {
    id[0] = (int)faces[3 * f];
    id[1] = (int)faces[3 * f + 1];
    id[2] = (int)faces[3 * f + 2];
}
__host__ __device__ __forceinline__ void ld3(const float *p, int64_t i, float (&o)[3]) {
    o[0] = p[3 * i];
    o[1] = p[3 * i + 1];
    o[2] = p[3 * i + 2];
}

// ---- buckets: items grouped by key, each bucket sorted by item ------------------------------------------------------
template <typename I>
__global__ void k_count_keys(const I *keys, int64_t n, int64_t nkeys, int *cnt, int *flags) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long long k = (long long)keys[i];
    if (k < 0 || k >= nkeys) {
        atomicOr(flags, 1);
        return;
    }
    atomicAdd(cnt + k, 1);
}
// item code: for faces (stride 3) the item is 4 * face + corner, for a plain index vector it is the position
template <typename I>
__global__ void k_fill_keys(const I *keys, int64_t n, int64_t nkeys, int per_face, const int *ptr, int *cursor, int *items) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long long k = (long long)keys[i];
    if (k < 0 || k >= nkeys) return;
    const int slot = ptr[k] + atomicAdd(cursor + k, 1);
    items[slot] = per_face ? (int)(4 * (i / 3) + (i % 3)) : (int)i;
}
// one thread per bucket: shell sort (gap sequence n/2, n/4, ... 1): O(n^1.3) even for a hub of valence 1e4
__global__ void k_sort_buckets_items(int64_t nkeys, const int *ptr, int *items) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nkeys) return;
    const int b = ptr[k], n = ptr[k + 1] - b;
    int *a = items + b;
    for (int gap = n >> 1; gap > 0; gap >>= 1)
        for (int i = gap; i < n; ++i) {
            const int t = a[i];
            int j = i;
            for (; j >= gap && a[j - gap] > t; j -= gap) a[j] = a[j - gap];
            a[j] = t;
        }
}

// the launches of build_buckets; keys outside [0, nkeys) are skipped and flagged in the workspace
template <typename I>
int launch_buckets(const I *keys, int64_t n, int64_t nkeys, int per_face, int *ptr, int *items, void *ws, cudaStream_t st) {
    int *cnt = (int *)ws;                          // nkeys + 1 counts, then cursor (nkeys), flags, scan scratch
    int *cursor = cnt + (nkeys + 8);
    int *flags = cursor + (nkeys + 8);
    int *scan = flags + 8;
    LS_CUDA_TRY(cudaMemsetAsync(ws, 0, (size_t)(2 * (nkeys + 8) + 8) * 4, st));
    const unsigned gb = (unsigned)((n + GT - 1) / GT), gk = (unsigned)((nkeys + GT - 1) / GT);
    if (n > 0) {
        k_count_keys<I><<<gb, GT, 0, st>>>(keys, n, nkeys, cnt, flags);
        LS_LAUNCH_CHECK();
    }
    int rc = ls_exclusive_scan_i32(cnt, ptr, nkeys, scan, st);
    if (rc) return rc;
    if (n > 0) {
        k_fill_keys<I><<<gb, GT, 0, st>>>(keys, n, nkeys, per_face, ptr, cursor, items);
        LS_LAUNCH_CHECK();
        k_sort_buckets_items<<<gk, GT, 0, st>>>(nkeys, ptr, items);
        LS_LAUNCH_CHECK();
    }
    return LS_OK;
}

template <typename I>
int build_buckets(const I *keys, int64_t n, int64_t nkeys, int per_face, int *ptr, int *items, void *ws, cudaStream_t st) {
    int rc = launch_buckets<I>(keys, n, nkeys, per_face, ptr, items, ws, st);
    if (rc) return rc;
    const int *flags = (const int *)ws + 2 * (nkeys + 8);
    int hflags = 0;
    LS_CUDA_TRY(cudaMemcpyAsync(&hflags, flags, sizeof(int), cudaMemcpyDeviceToHost, st));
    LS_CUDA_TRY(cudaStreamSynchronize(st));
    if (hflags) {
        ls_set_error("index outside [0, %lld)", (long long)nkeys);
        return LS_ERR_INDEX_RANGE;
    }
    return LS_OK;
}

// ---- gather rows and its adjoint -------------------------------------------------------------------------------------
template <typename I>
__global__ void k_gather_rows(const float *__restrict__ src, const I *__restrict__ idx, int64_t n, int k, float *__restrict__ dst) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n * k) return;
    const int64_t i = t / k;
    const int c = (int)(t - i * k);
    dst[t] = src[(int64_t)idx[i] * k + c];
}
__global__ void k_gather_rows_bwd(const float *__restrict__ g, const int *__restrict__ ptr, const int *__restrict__ items,
                                  int64_t V, int k, float *__restrict__ out) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= V * k) return;
    const int64_t v = t / k;
    const int c = (int)(t - v * k);
    float s = 0.f;
    for (int j = ptr[v]; j < ptr[v + 1]; ++j) s += g[(int64_t)items[j] * k + c];   // fixed order: items are sorted
    out[t] = s;
}

// ---- face normals (geometry.py:91-110): n = cross(v1 - v0, v2 - v0) / |.|, stored (3,F) -----------------------------
template <typename I>
__global__ void k_face_normals(const float *__restrict__ verts, const I *__restrict__ faces, int64_t F, float *__restrict__ n) {
    const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    int id[3];
    face_ids(faces, f, id);
    float a[3], b[3], c[3];
    ld3(verts, id[0], a);
    ld3(verts, id[1], b);
    ld3(verts, id[2], c);
    const float e1[3] = {b[0] - a[0], b[1] - a[1], b[2] - a[2]}, e2[3] = {c[0] - a[0], c[1] - a[1], c[2] - a[2]};
    const float cx = e1[1] * e2[2] - e1[2] * e2[1], cy = e1[2] * e2[0] - e1[0] * e2[2], cz = e1[0] * e2[1] - e1[1] * e2[0];
    const float len = sqrtf(cx * cx + cy * cy + cz * cz);
    n[f] = cx / len;
    n[F + f] = cy / len;
    n[2 * F + f] = cz / len;
}
// gradient w.r.t. the vertex at corner `corner` of face f, given g_n (3 floats)
__host__ __device__ __forceinline__ void face_normal_grad(const float (&p0)[3], const float (&p1)[3], const float (&p2)[3],
                                                 const float (&gn)[3], int corner, float (&out)[3]) {
    const float e1[3] = {p1[0] - p0[0], p1[1] - p0[1], p1[2] - p0[2]}, e2[3] = {p2[0] - p0[0], p2[1] - p0[1], p2[2] - p0[2]};
    const float c[3] = {e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0]};
    const float len = sqrtf(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]);
    const float inv = 1.0f / len;
    const float nn[3] = {c[0] * inv, c[1] * inv, c[2] * inv};
    const float dot = nn[0] * gn[0] + nn[1] * gn[1] + nn[2] * gn[2];
    const float gc[3] = {(gn[0] - nn[0] * dot) * inv, (gn[1] - nn[1] * dot) * inv, (gn[2] - nn[2] * dot) * inv};
    // c = e1 x e2:  g_e1 = e2 x g_c,  g_e2 = g_c x e1
    const float ge1[3] = {e2[1] * gc[2] - e2[2] * gc[1], e2[2] * gc[0] - e2[0] * gc[2], e2[0] * gc[1] - e2[1] * gc[0]};
    const float ge2[3] = {gc[1] * e1[2] - gc[2] * e1[1], gc[2] * e1[0] - gc[0] * e1[2], gc[0] * e1[1] - gc[1] * e1[0]};
#pragma unroll
    for (int d = 0; d < 3; ++d) out[d] = corner == 0 ? -(ge1[d] + ge2[d]) : (corner == 1 ? ge1[d] : ge2[d]);
}
// row v of the face-normal backward: the sum over v's incident corners, in incidence-list order
template <typename I>
__host__ __device__ __forceinline__ void face_normals_vertex_grad(const float *__restrict__ verts, const I *__restrict__ faces,
                                                                  int64_t F, const int *__restrict__ ptr, const int *__restrict__ inc,
                                                                  const float *__restrict__ gn, int64_t v, float *__restrict__ gverts) {
    float acc[3] = {0.f, 0.f, 0.f};
    for (int j = ptr[v]; j < ptr[v + 1]; ++j) {
        const int code = inc[j];
        const int64_t f = code >> 2;
        const int corner = code & 3;
        int id[3];
        face_ids(faces, f, id);
        float p0[3], p1[3], p2[3], g[3] = {gn[f], gn[F + f], gn[2 * F + f]}, o[3];
        ld3(verts, id[0], p0);
        ld3(verts, id[1], p1);
        ld3(verts, id[2], p2);
        face_normal_grad(p0, p1, p2, g, corner, o);
        acc[0] += o[0];
        acc[1] += o[1];
        acc[2] += o[2];
    }
    gverts[3 * v] = acc[0];
    gverts[3 * v + 1] = acc[1];
    gverts[3 * v + 2] = acc[2];
}
template <typename I>
__global__ void k_face_normals_bwd(const float *__restrict__ verts, const I *__restrict__ faces, int64_t F, int64_t V,
                                   const int *__restrict__ ptr, const int *__restrict__ inc, const float *__restrict__ gn,
                                   float *__restrict__ gverts) {
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    face_normals_vertex_grad(verts, faces, F, ptr, inc, gn, v, gverts);
}

// ---- vertex normals (geometry.py:115-147) ------------------------------------------------------------------------------
// corner i of a face: d0 = (v[i+1] - v[i]) / A_i, d1 = (v[i+2] - v[i]) / B_i with the global norms
//   i = 0: A = N01, B = N02;   i = 1: A = N12, B = N01;   i = 2: A = N02, B = N12
__host__ __device__ __forceinline__ void corner_norms(const float *nm, int i, float &A, float &B) {
    A = i == 0 ? nm[0] : (i == 1 ? nm[2] : nm[1]);
    B = i == 0 ? nm[1] : (i == 1 ? nm[0] : nm[2]);
}
__host__ __device__ __forceinline__ float corner_cos(const float (&pi)[3], const float (&pj)[3], const float (&pk)[3], float A, float B) {
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < 3; ++d) s += ((pj[d] - pi[d]) / A) * ((pk[d] - pi[d]) / B);
    return s;
}
__host__ __device__ __forceinline__ float safe_acosf(float x) { return acosf(fminf(fmaxf(x, -1.f), 1.f)); }

// row v: out = N_v / |N_v| and raw_len = |N_v|, N_v = sum of fn * theta over v's incident corners
template <typename I>
__host__ __device__ __forceinline__ void vertex_normal(const float *__restrict__ verts, const I *__restrict__ faces, int64_t F,
                                                      const int *__restrict__ ptr, const int *__restrict__ inc,
                                                      const float *__restrict__ fn, const float (&nm)[3], int64_t v,
                                                      float *__restrict__ out, float *__restrict__ raw_len) {
    float acc[3] = {0.f, 0.f, 0.f};
    for (int j = ptr[v]; j < ptr[v + 1]; ++j) {
        const int code = inc[j];
        const int64_t f = code >> 2;
        const int i = code & 3;
        int id[3];
        face_ids(faces, f, id);
        float p[3][3];
        ld3(verts, id[0], p[0]);
        ld3(verts, id[1], p[1]);
        ld3(verts, id[2], p[2]);
        float A, B;
        corner_norms(nm, i, A, B);
        const float th = safe_acosf(corner_cos(p[i], p[(i + 1) % 3], p[(i + 2) % 3], A, B));
        acc[0] += fn[f] * th;
        acc[1] += fn[F + f] * th;
        acc[2] += fn[2 * F + f] * th;
    }
    const float len = sqrtf(acc[0] * acc[0] + acc[1] * acc[1] + acc[2] * acc[2]);
    raw_len[v] = len;
    out[3 * v] = acc[0] / len;
    out[3 * v + 1] = acc[1] / len;
    out[3 * v + 2] = acc[2] / len;
}

// backward helpers.  g_N[v] = (g_out - out <out, g_out>) / |N_v| is recomputed where needed.
__host__ __device__ __forceinline__ void raw_grad(const float *out, const float *gout, const float *raw_len, int64_t v, float (&g)[3]) {
    const float o[3] = {out[3 * v], out[3 * v + 1], out[3 * v + 2]}, go[3] = {gout[3 * v], gout[3 * v + 1], gout[3 * v + 2]};
    const float dot = o[0] * go[0] + o[1] * go[1] + o[2] * go[2];
    const float inv = 1.0f / raw_len[v];
#pragma unroll
    for (int d = 0; d < 3; ++d) g[d] = (go[d] - o[d] * dot) * inv;
}
// face f's part of pass 1: the gradient reaching its face normal, gf, and its three terms g_q(f,i) q(f,i) added to acc[i]
template <typename I>
__host__ __device__ __forceinline__ void vertex_normals_face_grad(const float *__restrict__ verts, const I *__restrict__ faces, int64_t F,
                                                                  const float *__restrict__ fn, const float (&nm)[3],
                                                                  const float *__restrict__ out, const float *__restrict__ gout,
                                                                  const float *__restrict__ raw_len, int64_t f, float (&gf)[3],
                                                                  double (&acc)[3]) {
    int id[3];
    face_ids(faces, f, id);
    float p[3][3];
    ld3(verts, id[0], p[0]);
    ld3(verts, id[1], p[1]);
    ld3(verts, id[2], p[2]);
    const float n[3] = {fn[f], fn[F + f], fn[2 * F + f]};
    gf[0] = gf[1] = gf[2] = 0.f;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        float A, B, gN[3];
        corner_norms(nm, i, A, B);
        const float q = corner_cos(p[i], p[(i + 1) % 3], p[(i + 2) % 3], A, B);
        const float th = safe_acosf(q);
        raw_grad(out, gout, raw_len, id[i], gN);
        gf[0] += th * gN[0];
        gf[1] += th * gN[1];
        gf[2] += th * gN[2];
        const float gth = n[0] * gN[0] + n[1] * gN[1] + n[2] * gN[2];
        const float gq = (q > -1.f && q < 1.f) ? -gth / sqrtf(1.f - q * q) : 0.f;
        acc[i] += (double)gq * (double)q;
    }
}
// pass 2 (per vertex): position gradient.  For corner i of a face with a = v[i+1] - v[i], b = v[i+2] - v[i]:
//   g_a = g_q / (A B) b - T_i / A^2 a,   g_b = g_q / (A B) a - T_i / B^2 b;   v[i+1] += g_a, v[i+2] += g_b, v[i] -= g_a + g_b
// vertex_normals_vertex_grad sums these over the faces incident to v, in incidence-list order
template <typename I>
__host__ __device__ __forceinline__ void vertex_normals_vertex_grad(const float *__restrict__ verts, const I *__restrict__ faces, int64_t F,
                                                                    const int *__restrict__ ptr, const int *__restrict__ inc,
                                                                    const float *__restrict__ fn, const float (&nm)[3], const float (&Tg)[3],
                                                                    const float *__restrict__ out, const float *__restrict__ gout,
                                                                    const float *__restrict__ raw_len, int64_t v,
                                                                    float *__restrict__ gverts) {
    float acc[3] = {0.f, 0.f, 0.f};
    for (int j = ptr[v]; j < ptr[v + 1]; ++j) {
        const int code = inc[j];
        const int64_t f = code >> 2;
        const int me = code & 3;           // position of this vertex inside the face
        int id[3];
        face_ids(faces, f, id);
        float p[3][3];
        ld3(verts, id[0], p[0]);
        ld3(verts, id[1], p[1]);
        ld3(verts, id[2], p[2]);
        const float n[3] = {fn[f], fn[F + f], fn[2 * F + f]};
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            float A, B, gN[3];
            corner_norms(nm, i, A, B);
            const int i1 = (i + 1) % 3, i2 = (i + 2) % 3;
            const float q = corner_cos(p[i], p[i1], p[i2], A, B);
            raw_grad(out, gout, raw_len, id[i], gN);
            const float gth = n[0] * gN[0] + n[1] * gN[1] + n[2] * gN[2];
            const float gq = (q > -1.f && q < 1.f) ? -gth / sqrtf(1.f - q * q) : 0.f;
            const float cab = gq / (A * B), ca = Tg[i] / (A * A), cb = Tg[i] / (B * B);
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                const float a = p[i1][d] - p[i][d], b = p[i2][d] - p[i][d];
                const float ga = cab * b - ca * a, gb = cab * a - cb * b;
                acc[d] += (me == i1) ? ga : ((me == i2) ? gb : -(ga + gb));
            }
        }
    }
    gverts[3 * v] = acc[0];
    gverts[3 * v + 1] = acc[1];
    gverts[3 * v + 2] = acc[2];
}

// ---- Voronoi mass matrix (geometry.py:35-89) -----------------------------------------------------------------------------
// The mixed Voronoi area of each vertex.  The per-face values repeat the reference's float32 operations one for one: torch's
// CPU 2-norm of a 3-vector is sqrt(fma(z, z, fma(y, y, x * x))), the cosines come from the law of cosines, the area from
// Heron's formula with no clamp, and the obtuse override is three sequential torch.where's, so the last obtuse corner wins
// and a NaN cosine selects none.  mul_rn keeps nvcc from contracting a product into the add that follows it.
// The per-vertex bodies are __host__ __device__ so that tests/test_massmatrix_host.py can check them on a CPU.
struct MassFace {
    float e[3][3];       // e0 = p1 - p2, e1 = p2 - p0, e2 = p0 - p1
    float l[3];          // |e_k|
    float cs[3], den[3]; // cos_k = (l_{k+1}^2 + l_{k+2}^2 - l_k^2) / den_k,  den_k = 2 l_{k+1} l_{k+2}
    float b[3], S;       // b_k = cos_k l_k,  S = (b0 + b1) + b2;  barycentric weight bar_k = b_k / S
    float bar[3];
    float s[4], R, A;    // Heron: P = s0 s1 s2 s3, R = sqrt(P), A = R / 4
    int sel;             // the obtuse corner whose override the cells end with, or -1
};
__host__ __device__ __forceinline__ void mass_face(const float (&p)[3][3], MassFace &m) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
#pragma unroll
        for (int d = 0; d < 3; ++d) m.e[k][d] = p[(k + 1) % 3][d] - p[(k + 2) % 3][d];
        m.l[k] = sqrtf(fmaf(m.e[k][2], m.e[k][2], fmaf(m.e[k][1], m.e[k][1], mul_rn(m.e[k][0], m.e[k][0]))));
    }
    const float sq[3] = {mul_rn(m.l[0], m.l[0]), mul_rn(m.l[1], m.l[1]), mul_rn(m.l[2], m.l[2])};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int k1 = (k + 1) % 3, k2 = (k + 2) % 3;
        m.den[k] = mul_rn(2.f * m.l[k1], m.l[k2]);
        m.cs[k] = ((sq[k1] + sq[k2]) - sq[k]) / m.den[k];
        m.b[k] = mul_rn(m.cs[k], m.l[k]);
    }
    m.S = (m.b[0] + m.b[1]) + m.b[2];
#pragma unroll
    for (int k = 0; k < 3; ++k) m.bar[k] = m.b[k] / m.S;
    const float l0 = m.l[0], l1 = m.l[1], l2 = m.l[2];
    m.s[0] = (l0 + l1) + l2;
    m.s[1] = (l0 + l1) - l2;
    m.s[2] = (l0 - l1) + l2;
    m.s[3] = (-l0 + l1) + l2;
    m.R = sqrtf(mul_rn(mul_rn(mul_rn(m.s[0], m.s[1]), m.s[2]), m.s[3]));
    m.A = 0.25f * m.R;
    m.sel = m.cs[2] < 0.f ? 2 : (m.cs[1] < 0.f ? 1 : (m.cs[0] < 0.f ? 0 : -1));
}
// cell k: 0.5 (t_{k+1} + t_{k+2}) with t_j = A bar_j, or after an override 0.5 A at the obtuse corner and 0.25 A elsewhere
__host__ __device__ __forceinline__ float mass_cell(const MassFace &m, int k) {
    if (m.sel >= 0) return (k == m.sel ? 0.5f : 0.25f) * m.A;
    return 0.5f * (mul_rn(m.A, m.bar[(k + 1) % 3]) + mul_rn(m.A, m.bar[(k + 2) % 3]));
}
// Gradient of sum_k g_k cell_k w.r.t. the three edge vectors, following the reference's autograd graph node by node so that
// degenerate faces give non-finite gradients exactly where it does: a cell the override replaced passes an exact zero to
// its cell expression (0 * inf is still NaN below), and the 2-norm's backward is g * (e / l) with e / l set to 0 where l = 0.
__host__ __device__ __forceinline__ void mass_face_grad(const MassFace &m, const float (&g)[3], float (&ge)[3][3]) {
    float gA = 0.f, gc[3] = {g[0], g[1], g[2]};
    if (m.sel >= 0) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            gA += (k == m.sel ? 0.5f : 0.25f) * gc[k];
            gc[k] = 0.f;
        }
    }
    float gbar[3], gS = 0.f;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float gt = 0.5f * gc[(k + 1) % 3] + 0.5f * gc[(k + 2) % 3];   // t_k feeds cells k+1 and k+2
        gA += gt * m.bar[k];
        gbar[k] = gt * m.A;
        gS -= gbar[k] * (m.bar[k] / m.S);
    }
    float gb[3], gl[3], gsq[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        gb[k] = gbar[k] / m.S + gS;
        gl[k] = gb[k] * m.cs[k];
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float gcs = gb[k] * m.l[k];
        const float gnum = gcs / m.den[k], gden = -gcs * (m.cs[k] / m.den[k]);
        const int k1 = (k + 1) % 3, k2 = (k + 2) % 3;
        gsq[k1] += gnum;
        gsq[k2] += gnum;
        gsq[k] -= gnum;
        gl[k1] += 2.f * (gden * m.l[k2]);
        gl[k2] += gden * (2.f * m.l[k1]);
    }
    const float gP = (0.25f * gA) / (2.f * m.R);
    const float q01 = m.s[0] * m.s[1], q012 = q01 * m.s[2];
    const float g3 = gP * q012, gq012 = gP * m.s[3], g2 = gq012 * q01, gq01 = gq012 * m.s[2], g0 = gq01 * m.s[1],
                g1 = gq01 * m.s[0];
    gl[0] += gsq[0] * (2.f * m.l[0]) + (g0 + g1 + g2 - g3);
    gl[1] += gsq[1] * (2.f * m.l[1]) + (g0 + g1 - g2 + g3);
    gl[2] += gsq[2] * (2.f * m.l[2]) + (g0 - g1 + g2 + g3);
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
        for (int d = 0; d < 3; ++d) ge[k][d] = gl[k] * (m.l[k] == 0.f ? 0.f : m.e[k][d] / m.l[k]);
}
template <typename I>
__host__ __device__ __forceinline__ void load_face(const float *verts, const I *faces, int64_t f, int (&id)[3], float (&p)[3][3]) {
    face_ids(faces, f, id);
    ld3(verts, id[0], p[0]);
    ld3(verts, id[1], p[1]);
    ld3(verts, id[2], p[2]);
}
// m[v]: column j of the reference's scatter_add_ sums the corner-j cells in face order (the incidence list is sorted by
// 4 face + corner), then the three columns are summed as (c0 + c1) + c2
template <typename I>
__host__ __device__ __forceinline__ float mass_vertex(const float *verts, const I *faces, const int *ptr, const int *inc, int64_t v) {
    float c0 = 0.f, c1 = 0.f, c2 = 0.f;
    for (int j = ptr[v]; j < ptr[v + 1]; ++j) {
        const int code = inc[j];
        const int corner = code & 3;
        int id[3];
        float p[3][3];
        load_face(verts, faces, code >> 2, id, p);
        MassFace m;
        mass_face(p, m);
        const float c = mass_cell(m, corner);
        if (corner == 0) c0 += c;
        else if (corner == 1) c1 += c;
        else c2 += c;
    }
    return (c0 + c1) + c2;
}
template <typename I>
__host__ __device__ __forceinline__ void mass_vertex_grad(const float *verts, const I *faces, const int *ptr, const int *inc,
                                                          const float *gout, int64_t v, float (&acc)[3]) {
    acc[0] = acc[1] = acc[2] = 0.f;
    for (int j = ptr[v]; j < ptr[v + 1]; ++j) {
        const int code = inc[j];
        const int me = code & 3;
        int id[3];
        float p[3][3];
        load_face(verts, faces, code >> 2, id, p);
        const float g[3] = {gout[id[0]], gout[id[1]], gout[id[2]]};
        MassFace m;
        mass_face(p, m);
        float ge[3][3];
        mass_face_grad(m, g, ge);
        // corner c is the head of e_{c+2} and the tail of e_{c+1}
#pragma unroll
        for (int d = 0; d < 3; ++d)
            acc[d] += me == 0 ? ge[2][d] - ge[1][d] : (me == 1 ? ge[0][d] - ge[2][d] : ge[1][d] - ge[0][d]);
    }
}
template <typename I>
__global__ void k_massmatrix_voronoi(const float *__restrict__ verts, const I *__restrict__ faces, int64_t V,
                                     const int *__restrict__ ptr, const int *__restrict__ inc, float *__restrict__ out) {
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v < V) out[v] = mass_vertex(verts, faces, ptr, inc, v);
}
template <typename I>
__global__ void k_massmatrix_voronoi_bwd(const float *__restrict__ verts, const I *__restrict__ faces, int64_t V,
                                         const int *__restrict__ ptr, const int *__restrict__ inc, const float *__restrict__ gout,
                                         float *__restrict__ gverts) {
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    float acc[3];
    mass_vertex_grad(verts, faces, ptr, inc, gout, v, acc);
    gverts[3 * v] = acc[0];
    gverts[3 * v + 1] = acc[1];
    gverts[3 * v + 2] = acc[2];
}

inline unsigned grid_for(int64_t n) { return (unsigned)((n + GT - 1) / GT > 0 ? (n + GT - 1) / GT : 1); }
constexpr int RED_GRID_MAX = 132 * 4;   // 132 SMs (H100 SXM) x 4
__host__ __device__ inline unsigned red_grid(int64_t n) {
    int64_t g = (n + GT - 1) / GT;
    if (g > RED_GRID_MAX) g = RED_GRID_MAX;
    if (g < 1) g = 1;
    return (unsigned)g;
}

// ---- vertex-normal kernels, for B packed meshes (ls_vertex_normals_batch_*) or one mesh (ls_vertex_normals_*) ----------
// A single mesh is the batch B = 1 with null device offsets: faces [0, F), vertices [0, V).  The two per-face reductions
// run on a (max_i red_grid(F_i), B) grid: block row i is mesh i, and its first red_grid(F_i) blocks walk mesh i's faces
// (face f relative to the mesh's first face, stride red_grid(F_i) blocks), each into mesh i's own partials and ticket; the
// remaining blocks of the row exit at once.  So each mesh's norms, T, outputs and gradients are bitwise those of a call on
// that mesh alone.  The per-vertex kernels find their vertex's mesh by binary search.
struct MeshSlice {
    int64_t f0, F;    // first face and face count of the block row's mesh
    unsigned nb;      // red_grid(F): the blocks that walk the mesh's faces
};
__device__ __forceinline__ MeshSlice mesh_slice(const int64_t *face_offsets, int64_t F) {
    MeshSlice s;
    s.f0 = face_offsets ? face_offsets[blockIdx.y] : 0;
    s.F = face_offsets ? face_offsets[blockIdx.y + 1] - s.f0 : F;
    s.nb = red_grid(s.F);
    return s;
}
__device__ __forceinline__ int mesh_of(const int64_t *__restrict__ vert_offsets, int B, int64_t v) {
    int lo = 0, hi = B - 1;          // the last mesh whose first vertex is <= v (empty meshes are skipped); B = 1 reads nothing
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (vert_offsets[mid] <= v) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}
// scratch: partials [B][3][RED_GRID_MAX] doubles, then B tickets, then T [B][3] floats
constexpr size_t batch_partials_bytes(int B) { return (size_t)B * 3 * RED_GRID_MAX * 8; }
constexpr size_t batch_ticket_bytes(int B) { return ((size_t)B * 4 + 15) / 16 * 16; }

// pass 0: squared Frobenius norms of the three edge fields E01 = v1 - v0, E02 = v2 - v0, E12 = v2 - v1
template <typename I>
__global__ void __launch_bounds__(GT) k_edge_norms_batch(const float *__restrict__ verts, const I *__restrict__ faces, int64_t F,
                                                         const int64_t *__restrict__ face_offsets, double *partials,
                                                         unsigned int *tickets, float *norms /* [B][3] */) {
    const MeshSlice s = mesh_slice(face_offsets, F);
    if (blockIdx.x >= s.nb) return;
    faces += 3 * s.f0;
    __shared__ double red[3 * 32 + 3 + 1];
    double acc[3] = {0.0, 0.0, 0.0};
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < s.F; f += (int64_t)s.nb * blockDim.x) {
        int id[3];
        face_ids(faces, f, id);
        float a[3], b[3], c[3];
        ld3(verts, id[0], a);
        ld3(verts, id[1], b);
        ld3(verts, id[2], c);
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const float e01 = b[d] - a[d], e02 = c[d] - a[d], e12 = c[d] - b[d];
            acc[0] += (double)(e01 * e01);
            acc[1] += (double)(e02 * e02);
            acc[2] += (double)(e12 * e12);
        }
    }
    double tot[3];
    const bool last = ls_grid_reduce<3>(acc, tot, partials + (size_t)blockIdx.y * 3 * RED_GRID_MAX, tickets + blockIdx.y, red,
                                        threadIdx.x, GT, 1, blockIdx.x, s.nb);
    if (last && threadIdx.x == 0) {
        float *nm = norms + 3 * blockIdx.y;
        nm[0] = (float)sqrt(tot[0]);
        nm[1] = (float)sqrt(tot[1]);
        nm[2] = (float)sqrt(tot[2]);
    }
}

template <typename I>
__global__ void k_vertex_normals_batch(const float *__restrict__ verts, const I *__restrict__ faces, int64_t F, int64_t V,
                                       int B, const int64_t *__restrict__ vert_offsets, const int *__restrict__ ptr,
                                       const int *__restrict__ inc, const float *__restrict__ fn,
                                       const float *__restrict__ norms, float *__restrict__ out, float *__restrict__ raw_len) {
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    const float *mn = norms + 3 * mesh_of(vert_offsets, B, v);
    const float nm[3] = {mn[0], mn[1], mn[2]};
    vertex_normal(verts, faces, F, ptr, inc, fn, nm, v, out, raw_len);
}

// pass 1 (per face): gradient w.r.t. the face normal, and the three sums T_i = sum_f g_q(f,i) q(f,i) over the mesh's faces.
// At most 64 registers, so that 4 blocks fit on an SM and a row's RED_GRID_MAX = 132 x 4 blocks run in one wave.
template <typename I>
__global__ void __launch_bounds__(GT, 4) k_vertex_normals_batch_bwd1(const float *__restrict__ verts, const I *__restrict__ faces,
                                                                  int64_t F, const int64_t *__restrict__ face_offsets,
                                                                  const float *__restrict__ fn, const float *__restrict__ norms,
                                                                  const float *__restrict__ out, const float *__restrict__ gout,
                                                                  const float *__restrict__ raw_len, float *__restrict__ gfn,
                                                                  double *partials, unsigned int *tickets, float *T /* [B][3] */) {
    const MeshSlice s = mesh_slice(face_offsets, F);
    if (blockIdx.x >= s.nb) return;
    __shared__ double red[3 * 32 + 3 + 1];
    const float *mn = norms + 3 * blockIdx.y;
    const float nm[3] = {mn[0], mn[1], mn[2]};
    double acc[3] = {0.0, 0.0, 0.0};
    for (int64_t fl = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; fl < s.F; fl += (int64_t)s.nb * blockDim.x) {
        const int64_t f = s.f0 + fl;
        float gf[3];
        vertex_normals_face_grad(verts, faces, F, fn, nm, out, gout, raw_len, f, gf, acc);
        gfn[f] = gf[0];
        gfn[F + f] = gf[1];
        gfn[2 * F + f] = gf[2];
    }
    double tot[3];
    const bool last = ls_grid_reduce<3>(acc, tot, partials + (size_t)blockIdx.y * 3 * RED_GRID_MAX, tickets + blockIdx.y, red,
                                        threadIdx.x, GT, 1, blockIdx.x, s.nb);
    if (last && threadIdx.x == 0) {
        float *Tm = T + 3 * blockIdx.y;
        Tm[0] = (float)tot[0];
        Tm[1] = (float)tot[1];
        Tm[2] = (float)tot[2];
    }
}

template <typename I>
__global__ void k_vertex_normals_batch_bwd2(const float *__restrict__ verts, const I *__restrict__ faces, int64_t F, int64_t V,
                                            int B, const int64_t *__restrict__ vert_offsets, const int *__restrict__ ptr,
                                            const int *__restrict__ inc, const float *__restrict__ fn,
                                            const float *__restrict__ norms, const float *__restrict__ out,
                                            const float *__restrict__ gout, const float *__restrict__ raw_len,
                                            const float *__restrict__ T, float *__restrict__ gverts) {
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    const int m = mesh_of(vert_offsets, B, v);
    const float nm[3] = {norms[3 * m], norms[3 * m + 1], norms[3 * m + 2]}, Tg[3] = {T[3 * m], T[3 * m + 1], T[3 * m + 2]};
    vertex_normals_vertex_grad(verts, faces, F, ptr, inc, fn, nm, Tg, out, gout, raw_len, v, gverts);
}

}  // namespace

// scratch for the two reductions of a single mesh: the batch layout for B = 1 (partials [3][RED_GRID_MAX] doubles, a 16-byte
// ticket, T [3] floats)
static constexpr size_t GLUE_SCRATCH = 3 * RED_GRID_MAX * 8 + 64;
static_assert(GLUE_SCRATCH >= batch_partials_bytes(1) + batch_ticket_bytes(1) + 3 * 4, "single-mesh scratch holds B = 1");

extern "C" int ls_glue_scratch_bytes(size_t *bytes_out) {
    LS_REQUIRE(bytes_out != nullptr, "bytes_out is NULL");
    *bytes_out = GLUE_SCRATCH;
    return LS_OK;
}

extern "C" int ls_bucket_workspace_bytes(int64_t n_keys, size_t *bytes_out) {
    LS_REQUIRE(bytes_out != nullptr, "bytes_out is NULL");
    LS_REQUIRE(n_keys >= 0 && n_keys < (int64_t)0x7ffffff0, "n_keys out of range");
    *bytes_out = ((size_t)(2 * (n_keys + 8) + 8) + ls_scan_scratch_elems(n_keys + 1)) * 4;
    return LS_OK;
}

extern "C" int ls_face_incidence(const void *faces, int idx_bytes, int64_t F, int64_t V, int32_t *inc_ptr, int32_t *inc,
                                 void *workspace, size_t workspace_bytes, void *stream) {
    LS_REQUIRE(faces != nullptr || F == 0, "faces is NULL");
    LS_REQUIRE(inc_ptr && inc && workspace, "NULL output / workspace");
    LS_REQUIRE(idx_bytes == 4 || idx_bytes == 8, "idx_bytes must be 4 or 8");
    LS_REQUIRE(F >= 0 && V >= 0 && 3 * F < (int64_t)0x1ffffff0, "size out of range");
    size_t need;
    ls_bucket_workspace_bytes(V, &need);
    LS_REQUIRE(workspace_bytes >= need, "workspace too small");
    if (idx_bytes == 4) return build_buckets<int32_t>((const int32_t *)faces, 3 * F, V, 1, inc_ptr, inc, workspace, (cudaStream_t)stream);
    return build_buckets<int64_t>((const int64_t *)faces, 3 * F, V, 1, inc_ptr, inc, workspace, (cudaStream_t)stream);
}

int ls_face_buckets_i32_async(const int32_t *faces, int64_t F, int64_t V, int32_t *inc_ptr, int32_t *inc, void *workspace,
                              cudaStream_t stream) {
    return launch_buckets<int32_t>(faces, 3 * F, V, 1, inc_ptr, inc, workspace, stream);
}

int ls_buckets_async(const void *keys, int key_bytes, int64_t n, int64_t nkeys, int per_face, int32_t *ptr, int32_t *items,
                     void *workspace, cudaStream_t stream) {
    if (key_bytes == 4) return launch_buckets<int32_t>((const int32_t *)keys, n, nkeys, per_face, ptr, items, workspace, stream);
    return launch_buckets<int64_t>((const int64_t *)keys, n, nkeys, per_face, ptr, items, workspace, stream);
}

extern "C" int ls_index_buckets(const void *idx, int idx_bytes, int64_t n, int64_t V, int32_t *ptr, int32_t *items,
                                void *workspace, size_t workspace_bytes, void *stream) {
    LS_REQUIRE(idx != nullptr || n == 0, "idx is NULL");
    LS_REQUIRE(ptr && items && workspace, "NULL output / workspace");
    LS_REQUIRE(idx_bytes == 4 || idx_bytes == 8, "idx_bytes must be 4 or 8");
    LS_REQUIRE(n >= 0 && V >= 0 && n < (int64_t)0x7ffffff0, "size out of range");
    size_t need;
    ls_bucket_workspace_bytes(V, &need);
    LS_REQUIRE(workspace_bytes >= need, "workspace too small");
    if (idx_bytes == 4) return build_buckets<int32_t>((const int32_t *)idx, n, V, 0, ptr, items, workspace, (cudaStream_t)stream);
    return build_buckets<int64_t>((const int64_t *)idx, n, V, 0, ptr, items, workspace, (cudaStream_t)stream);
}

extern "C" int ls_gather_rows_f32(const float *src, const void *idx, int idx_bytes, int64_t n, int k, float *dst, void *stream) {
    LS_REQUIRE(idx_bytes == 4 || idx_bytes == 8, "idx_bytes must be 4 or 8");
    LS_REQUIRE(n >= 0 && k >= 1, "bad size");
    if (n == 0) return LS_OK;
    LS_REQUIRE(src && idx && dst, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    if (idx_bytes == 4) k_gather_rows<int32_t><<<grid_for(n * k), GT, 0, st>>>(src, (const int32_t *)idx, n, k, dst);
    else k_gather_rows<int64_t><<<grid_for(n * k), GT, 0, st>>>(src, (const int64_t *)idx, n, k, dst);
    LS_LAUNCH_CHECK();
    return LS_OK;
}

extern "C" int ls_gather_rows_bwd_f32(const float *gdst, const int32_t *ptr, const int32_t *items, int64_t V, int k, float *gsrc,
                                      void *stream) {
    LS_REQUIRE(V >= 0 && k >= 1, "bad size");
    if (V == 0) return LS_OK;
    LS_REQUIRE(gdst && ptr && items && gsrc, "NULL pointer");
    k_gather_rows_bwd<<<grid_for(V * k), GT, 0, (cudaStream_t)stream>>>(gdst, ptr, items, V, k, gsrc);
    LS_LAUNCH_CHECK();
    return LS_OK;
}

#define LS_DISPATCH_IDX(KERNEL, GRID, ...)                                                        \
    do {                                                                                          \
        if (idx_bytes == 4) KERNEL<int32_t><<<GRID, GT, 0, st>>>(verts, (const int32_t *)faces, __VA_ARGS__); \
        else KERNEL<int64_t><<<GRID, GT, 0, st>>>(verts, (const int64_t *)faces, __VA_ARGS__);     \
        LS_LAUNCH_CHECK();                                                                        \
    } while (0)

extern "C" int ls_face_normals_f32(const float *verts, const void *faces, int idx_bytes, int64_t F, float *n, void *stream) {
    LS_REQUIRE(idx_bytes == 4 || idx_bytes == 8, "idx_bytes must be 4 or 8");
    LS_REQUIRE(F >= 0, "bad size");
    if (F == 0) return LS_OK;
    LS_REQUIRE(verts && faces && n, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    LS_DISPATCH_IDX(k_face_normals, grid_for(F), F, n);
    return LS_OK;
}

extern "C" int ls_face_normals_bwd_f32(const float *verts, const void *faces, int idx_bytes, int64_t F, int64_t V,
                                       const int32_t *inc_ptr, const int32_t *inc, const float *gn, float *gverts, void *stream) {
    LS_REQUIRE(idx_bytes == 4 || idx_bytes == 8, "idx_bytes must be 4 or 8");
    LS_REQUIRE(F >= 0 && V >= 0, "bad size");
    if (V == 0) return LS_OK;
    LS_REQUIRE(verts && (faces || F == 0) && inc_ptr && inc && gn && gverts, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    LS_DISPATCH_IDX(k_face_normals_bwd, grid_for(V), F, V, inc_ptr, inc, gn, gverts);
    return LS_OK;
}

// The launches of one vertex-normals call, after the entry point's checks: B packed meshes on the reduction grid `red`, or
// one mesh (B = 1, null device offsets, red_grid(F) blocks), with the scratch layout of ls_vertex_normals_batch_scratch_bytes(B).
static int vertex_normals_launch(const float *verts, const void *faces, int idx_bytes, int64_t F, int64_t V, int B, dim3 red,
                                 const int64_t *vert_offsets, const int64_t *face_offsets, const int32_t *inc_ptr,
                                 const int32_t *inc, const float *face_normals, float *out, float *raw_len, float *edge_norms,
                                 void *scratch, cudaStream_t st) {
    double *partials = (double *)scratch;
    unsigned int *tickets = (unsigned int *)((char *)scratch + batch_partials_bytes(B));
    LS_CUDA_TRY(cudaMemsetAsync(tickets, 0, batch_ticket_bytes(B), st));
    LS_DISPATCH_IDX(k_edge_norms_batch, red, F, face_offsets, partials, tickets, edge_norms);
    if (V == 0) return LS_OK;
    LS_DISPATCH_IDX(k_vertex_normals_batch, grid_for(V), F, V, B, vert_offsets, inc_ptr, inc, face_normals, edge_norms, out, raw_len);
    return LS_OK;
}

static int vertex_normals_bwd_launch(const float *verts, const void *faces, int idx_bytes, int64_t F, int64_t V, int B, dim3 red,
                                     const int64_t *vert_offsets, const int64_t *face_offsets, const int32_t *inc_ptr,
                                     const int32_t *inc, const float *face_normals, const float *out, const float *raw_len,
                                     const float *edge_norms, const float *gout, float *gverts, float *gface_normals,
                                     void *scratch, cudaStream_t st) {
    double *partials = (double *)scratch;
    unsigned int *tickets = (unsigned int *)((char *)scratch + batch_partials_bytes(B));
    float *T = (float *)((char *)scratch + batch_partials_bytes(B) + batch_ticket_bytes(B));
    LS_CUDA_TRY(cudaMemsetAsync(tickets, 0, batch_ticket_bytes(B), st));
    LS_DISPATCH_IDX(k_vertex_normals_batch_bwd1, red, F, face_offsets, face_normals, edge_norms, out, gout, raw_len, gface_normals,
                    partials, tickets, T);
    if (V == 0) return LS_OK;
    LS_DISPATCH_IDX(k_vertex_normals_batch_bwd2, grid_for(V), F, V, B, vert_offsets, inc_ptr, inc, face_normals, edge_norms, out,
                    gout, raw_len, T, gverts);
    return LS_OK;
}

extern "C" int ls_vertex_normals_f32(const float *verts, const void *faces, int idx_bytes, int64_t F, int64_t V,
                                     const int32_t *inc_ptr, const int32_t *inc, const float *face_normals, float *out,
                                     float *raw_len, float *edge_norms, void *scratch, void *stream) {
    LS_REQUIRE(idx_bytes == 4 || idx_bytes == 8, "idx_bytes must be 4 or 8");
    LS_REQUIRE(F >= 0 && V >= 0, "bad size");
    if (V == 0) return LS_OK;
    LS_REQUIRE(verts && (faces || F == 0) && inc_ptr && inc && face_normals && out && raw_len && edge_norms && scratch, "NULL pointer");
    return vertex_normals_launch(verts, faces, idx_bytes, F, V, 1, dim3(red_grid(F)), nullptr, nullptr, inc_ptr, inc, face_normals,
                                 out, raw_len, edge_norms, scratch, (cudaStream_t)stream);
}

extern "C" int ls_vertex_normals_bwd_f32(const float *verts, const void *faces, int idx_bytes, int64_t F, int64_t V,
                                         const int32_t *inc_ptr, const int32_t *inc, const float *face_normals, const float *out,
                                         const float *raw_len, const float *edge_norms, const float *gout, float *gverts,
                                         float *gface_normals, void *scratch, void *stream) {
    LS_REQUIRE(idx_bytes == 4 || idx_bytes == 8, "idx_bytes must be 4 or 8");
    LS_REQUIRE(F >= 0 && V >= 0, "bad size");
    if (V == 0) return LS_OK;
    LS_REQUIRE(verts && (faces || F == 0) && inc_ptr && inc && face_normals && out && raw_len && edge_norms && gout && gverts &&
                   gface_normals && scratch, "NULL pointer");
    return vertex_normals_bwd_launch(verts, faces, idx_bytes, F, V, 1, dim3(red_grid(F)), nullptr, nullptr, inc_ptr, inc,
                                     face_normals, out, raw_len, edge_norms, gout, gverts, gface_normals, scratch,
                                     (cudaStream_t)stream);
}

extern "C" int ls_vertex_normals_batch_scratch_bytes(int B, size_t *bytes_out) {
    LS_REQUIRE(bytes_out != nullptr, "bytes_out is NULL");
    LS_REQUIRE(B >= 1 && B <= 65535, "B must be in [1, 65535]");
    *bytes_out = batch_partials_bytes(B) + batch_ticket_bytes(B) + (size_t)B * 3 * 4;
    return LS_OK;
}

// host checks of the packed layout; returns the reduction grid (max_i red_grid(F_i), B)
static int check_batch(int64_t F, int64_t V, int B, const int64_t *vo, const int64_t *fo, size_t scratch_bytes, dim3 *red) {
    size_t need = 0;
    int rc = ls_vertex_normals_batch_scratch_bytes(B, &need);
    if (rc) return rc;
    LS_REQUIRE(scratch_bytes >= need, "scratch smaller than ls_vertex_normals_batch_scratch_bytes(B)");
    LS_REQUIRE(vo && fo, "NULL host offsets");
    LS_REQUIRE(vo[0] == 0 && fo[0] == 0, "offsets must start at 0");
    unsigned nb = 1;
    for (int i = 0; i < B; ++i) {
        LS_REQUIRE(vo[i + 1] >= vo[i] && fo[i + 1] >= fo[i], "offsets must be non-decreasing");
        const unsigned g = red_grid(fo[i + 1] - fo[i]);
        nb = g > nb ? g : nb;
    }
    LS_REQUIRE(vo[B] == V && fo[B] == F, "offsets must end at V and F");
    *red = dim3(nb, (unsigned)B);
    return LS_OK;
}

extern "C" int ls_vertex_normals_batch_f32(const float *verts, const void *faces, int idx_bytes, int64_t F, int64_t V, int B,
                                           const int64_t *vert_offsets, const int64_t *face_offsets,
                                           const int64_t *vert_offsets_host, const int64_t *face_offsets_host,
                                           const int32_t *inc_ptr, const int32_t *inc, const float *face_normals, float *out,
                                           float *raw_len, float *edge_norms, void *scratch, size_t scratch_bytes, void *stream) {
    LS_REQUIRE(idx_bytes == 4 || idx_bytes == 8, "idx_bytes must be 4 or 8");
    LS_REQUIRE(F >= 0 && V >= 0, "bad size");
    dim3 red;
    int rc = check_batch(F, V, B, vert_offsets_host, face_offsets_host, scratch_bytes, &red);
    if (rc) return rc;
    LS_REQUIRE(verts && (faces || F == 0) && vert_offsets && face_offsets && inc_ptr && inc && face_normals && out && raw_len &&
                   edge_norms && scratch, "NULL pointer");
    return vertex_normals_launch(verts, faces, idx_bytes, F, V, B, red, vert_offsets, face_offsets, inc_ptr, inc, face_normals, out,
                                 raw_len, edge_norms, scratch, (cudaStream_t)stream);
}

extern "C" int ls_vertex_normals_batch_bwd_f32(const float *verts, const void *faces, int idx_bytes, int64_t F, int64_t V, int B,
                                               const int64_t *vert_offsets, const int64_t *face_offsets,
                                               const int64_t *vert_offsets_host, const int64_t *face_offsets_host,
                                               const int32_t *inc_ptr, const int32_t *inc, const float *face_normals,
                                               const float *out, const float *raw_len, const float *edge_norms, const float *gout,
                                               float *gverts, float *gface_normals, void *scratch, size_t scratch_bytes,
                                               void *stream) {
    LS_REQUIRE(idx_bytes == 4 || idx_bytes == 8, "idx_bytes must be 4 or 8");
    LS_REQUIRE(F >= 0 && V >= 0, "bad size");
    dim3 red;
    int rc = check_batch(F, V, B, vert_offsets_host, face_offsets_host, scratch_bytes, &red);
    if (rc) return rc;
    LS_REQUIRE(verts && (faces || F == 0) && vert_offsets && face_offsets && inc_ptr && inc && face_normals && out && raw_len &&
                   edge_norms && gout && gverts && gface_normals && scratch, "NULL pointer");
    return vertex_normals_bwd_launch(verts, faces, idx_bytes, F, V, B, red, vert_offsets, face_offsets, inc_ptr, inc, face_normals,
                                     out, raw_len, edge_norms, gout, gverts, gface_normals, scratch, (cudaStream_t)stream);
}

extern "C" int ls_massmatrix_voronoi_f32(const float *verts, const void *faces, int idx_bytes, int64_t F, int64_t V,
                                         const int32_t *inc_ptr, const int32_t *inc, float *out, void *stream) {
    LS_REQUIRE(idx_bytes == 4 || idx_bytes == 8, "idx_bytes must be 4 or 8");
    LS_REQUIRE(F >= 0 && V >= 0, "bad size");
    if (V == 0) return LS_OK;
    LS_REQUIRE(verts && (faces || F == 0) && inc_ptr && inc && out, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    LS_DISPATCH_IDX(k_massmatrix_voronoi, grid_for(V), V, inc_ptr, inc, out);
    return LS_OK;
}

extern "C" int ls_massmatrix_voronoi_bwd_f32(const float *verts, const void *faces, int idx_bytes, int64_t F, int64_t V,
                                             const int32_t *inc_ptr, const int32_t *inc, const float *gout, float *gverts,
                                             void *stream) {
    LS_REQUIRE(idx_bytes == 4 || idx_bytes == 8, "idx_bytes must be 4 or 8");
    LS_REQUIRE(F >= 0 && V >= 0, "bad size");
    if (V == 0) return LS_OK;
    LS_REQUIRE(verts && (faces || F == 0) && inc_ptr && inc && gout && gverts, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    LS_DISPATCH_IDX(k_massmatrix_voronoi_bwd, grid_for(V), V, inc_ptr, inc, gout, gverts);
    return LS_OK;
}
