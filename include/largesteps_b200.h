/*
 * largesteps_b200.h -- C ABI of the CUDA-native (H100, sm_90a) large-steps hot path (libls_b200.so).
 *
 * Every entry point replaces a piece of the reference's Python hot path; the reference interface each one
 * stands in for is cited as (file:line) relative to rgl-epfl/large-steps-pytorch.  The reference has no FFI
 * of its own for this path (its device arithmetic lives in torch sparse ops and in the third-party wheel
 * `cholespy`), so this header is the boundary a maintainer would bind with ctypes -- see INTEGRATION.md.
 *
 * Conventions
 *   - plain C types only; device pointers are raw `void*`/typed pointers into CUDA global memory of the
 *     CURRENT device; `stream` is a `cudaStream_t` passed as `void*` (NULL = legacy default stream).
 *   - every function returns an `ls_status` (0 = LS_OK).  `ls_last_error()` gives a thread-local message.
 *   - all work is stream-ordered and asynchronous unless a HOST out-pointer is documented as synchronising.
 *   - arrays named rowptr/col/val must be 16-byte aligned and readable up to the next 16-byte boundary
 *     past their last element (true for any cudaMalloc / torch allocation): the SpMM streams them with
 *     1-D TMA bulk copies (cp.async.bulk), which move whole 16-byte granules.
 *   - a handle is not thread-safe; distinct handles are independent.
 */
#ifndef LARGESTEPS_B200_H
#define LARGESTEPS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    LS_OK = 0,
    LS_ERR_BAD_ARG = 1,        /* null pointer, bad size, misaligned array, k out of range            */
    LS_ERR_CUDA = 2,           /* a CUDA runtime call failed (message in ls_last_error)                */
    LS_ERR_BREAKDOWN = 3,      /* CG breakdown: p.Ap <= 0 or NaN (matrix not SPD / NaN input)          */
    LS_ERR_NOT_CONVERGED = 4,  /* maxit reached before the relative residual target                    */
    LS_ERR_UNSUPPORTED = 5,    /* configuration not supported by this build                            */
    LS_ERR_INDEX_RANGE = 6,    /* face / COO index outside [0, V)                                      */
    LS_ERR_WORKSPACE = 7       /* workspace too small                                                  */
} ls_status;

/* ---- library ------------------------------------------------------------------------------------- */
int         ls_version(void);                 /* 10000*major + 100*minor + patch                        */
const char *ls_last_error(void);              /* thread-local, never NULL                               */
const char *ls_status_string(int status);
/* number of kernels this library has launched since load (bench.py's `gpu_launches` evidence)          */
uint64_t    ls_launch_count(void);
/* persisting kernels in a graph count once per graph launch * nodes; see DESIGN.md                      */

/* ---- system-matrix assembly  (replaces largesteps/geometry.py:3-133: laplacian_cot, laplacian_uniform,
 *      compute_matrix -- torch.unique / coalesce / sparse add on the device) ------------------------------
 * Two-phase because nnz(M) = V + 2E is only known after the directed edges have been de-duplicated.
 *   faces      (F,3) int32 (idx_bytes=4) or int64 (idx_bytes=8), row-major, device
 *   workspace  ls_assemble_workspace_bytes(F, V) bytes, device, 16-byte aligned; must be kept untouched
 *              between _count and _fill
 *   nnz_out    HOST pointer; _count synchronises the stream to write it                               */
int ls_assemble_workspace_bytes(int64_t F, int64_t V, size_t *bytes_out);
int ls_assemble_count(const void *faces, int idx_bytes, int64_t F, int64_t V,
                      void *workspace, size_t workspace_bytes, int64_t *nnz_out, void *stream);
/*   verts      (V,3) float32 device (only read when cotan != 0; geometry.py:20-41)
 *   diag_shift 1.0f for M = I + lambda L, float(1-alpha) for M = (1-alpha) I + alpha L  (geometry.py:127-132)
 *   scale      lambda or alpha
 *   outputs (any group may be NULL):
 *     coo_row, coo_col (nnz) int64 + coo_val (nnz) float32 : the coalesced, row-major sorted COO triplets
 *                         torch.sparse_coo_tensor(...).coalesce() would hold (geometry.py:133)
 *     csr_rowptr (V+1) int32, csr_col (nnz) int32, csr_val (nnz) float32 : the CSR the solver streams    */
int ls_assemble_fill(const void *faces, int idx_bytes, const float *verts, int64_t F, int64_t V,
                     int cotan, float diag_shift, float scale,
                     void *workspace, size_t workspace_bytes, int64_t nnz,
                     int64_t *coo_row, int64_t *coo_col, float *coo_val,
                     int32_t *csr_rowptr, int32_t *csr_col, float *csr_val, void *stream);
/* ---- backward of the cotangent assembly  (completes laplacian_cot / compute_matrix(cotan=True), geometry.py:3-63,96-133:
 *      the reference builds M's values from differentiable torch ops of the vertex positions) ------------------------------
 *   gverts (V,3) float32 out = d(sum_e gval[e] M.values[e]) / d verts for M = diag_shift I + scale L as ls_assemble_fill built
 *   it (diag_shift does not enter the gradient).
 *     verts, faces, F, V, scale: as given to ls_assemble_fill.  rowptr, col: its CSR of M.  gval (nnz): the gradient of M's
 *     values in their row-major order.  inc_ptr / inc: ls_face_incidence of the same faces.
 *     scratch: ls_laplacian_cot_bwd_scratch_bytes(F) bytes, device, 16-byte aligned.
 *   Per face, each cotangent weight w on edge (i, j) receives scale (gval_ii + gval_jj - gval_ij - gval_ji), 0 on a self-edge;
 *   per vertex, the chain of geometry.py:20-41 is followed back as torch's autograd runs it (the area clamp passes the gradient
 *   where the product is >= 1e-12, a zero-length edge's direction counts as 0), summed in face order.  No atomics:
 *   bit-reproducible.                                                                                                          */
int ls_laplacian_cot_bwd_scratch_bytes(int64_t F, size_t *bytes_out);
int ls_laplacian_cot_bwd_f32(const float *verts, const void *faces, int idx_bytes, int64_t F, int64_t V, float scale,
                             const int32_t *rowptr, const int32_t *col, const float *gval,
                             const int32_t *inc_ptr, const int32_t *inc, void *scratch, size_t scratch_bytes,
                             float *gverts, void *stream);
/* ---- matrix-free product with the cotangent Laplacian  (laplacian_cot(verts, faces) @ x of geometry.py:3-63 without the
 *      matrix: the per-step regulariser of scripts/main.py:192-195 on a cotangent L recomputed from the current shape) ---------
 *   ls_cot_laplacian_product_f32:  y (V,k) = L x with L = diag(colsum W) - W, i.e. y_i = sum over the edges (i, j) of the faces
 *     at i of w (x_i - x_j), w the face's cotangent weight as ls_assemble_fill computes it (scale 1).  A self-edge adds nothing,
 *     a duplicated face adds twice, an unused vertex gets 0.  Also writes w_out (3F floats, face f's weights on edges (v1, v2),
 *     (v2, v0), (v0, v1) at 3f..3f+2), which the backward reads.  Sums run over the incidence list in its order: no atomics,
 *     bit-reproducible.  Two kernels, no synchronisation, no scratch.
 *   ls_cot_laplacian_product_bwd_f32:  for the gradient gy (V,k) of y,
 *     gx (V,k) = L gy (L is symmetric: the forward's gather with the same w), and
 *     gverts (V,3) = the gradient through the weights: w_e gets sum_q (gy_i,q - gy_j,q)(x_i,q - x_j,q) on edge e = (i, j)
 *       (0 on a self-edge), then the chain of geometry.py:20-41 as ls_laplacian_cot_bwd_f32 follows it.
 *     Either output may be NULL; only the kernels of the requested ones run (gx: one, gverts: two).  w is only read for gx, x
 *     and scratch only for gverts.  scratch: ls_cot_laplacian_product_scratch_bytes(F) bytes, device, 16-byte aligned.
 *   Both:  verts (V,3), x, y, gy, gx: float32 row-major contiguous, k >= 1; faces and F, V as for ls_face_incidence, every
 *     index in [0, V) (not checked here: ls_face_incidence checks it); inc_ptr / inc: ls_face_incidence of the same faces.   */
int ls_cot_laplacian_product_scratch_bytes(int64_t F, size_t *bytes_out);
int ls_cot_laplacian_product_f32(const float *verts, const void *faces, int idx_bytes, int64_t F, int64_t V,
                                 const int32_t *inc_ptr, const int32_t *inc, const float *x, int k,
                                 float *y, float *w_out, void *stream);
int ls_cot_laplacian_product_bwd_f32(const float *verts, const void *faces, int idx_bytes, int64_t F, int64_t V,
                                     const int32_t *inc_ptr, const int32_t *inc, const float *w, const float *x, int k,
                                     const float *gy, float *gx /* nullable */, float *gverts /* nullable */,
                                     void *scratch, size_t scratch_bytes, void *stream);

/* ---- locality order of the vertices (no reference counterpart: the reference hands the native numbering to
 *      CHOLMOD, which re-orders internally with AMD; here the solver's matrix copy is re-ordered along a Morton curve
 *      of the vertex positions so that consecutive rows are a compact patch of the surface) ------------------------
 *   verts (V,3) float32 device; perm_new2old (V) int32 device out; deterministic.                               */
int ls_order_workspace_bytes(int64_t V, size_t *bytes_out);
int ls_order_morton(const float *verts, int64_t V, int32_t *perm_new2old,
                    void *workspace, size_t workspace_bytes, void *stream);

/* ---- COO -> CSR  (what CholeskySolver.__init__ hands to cholespy: solvers.py:33-34, M.indices(), M.values())
 *   coo_row/coo_col: coalesced, row-major sorted int64 (nnz).  Writes rowptr (V+1) and col (nnz) int32.
 *   Unsorted rows or out-of-range indices -> LS_ERR_INDEX_RANGE (synchronises to report it).            */
int ls_coo_to_csr(const int64_t *coo_row, const int64_t *coo_col, int64_t nnz, int64_t V,
                  int32_t *csr_rowptr, int32_t *csr_col, void *stream);

/* ---- y = A x  (replaces torch sparse `M @ v`: parameterize.py:30 to_differential; scripts/main.py:192-195)
 *   CSR float32 / int32;  x, y: (V,k) float32 row-major with leading dimensions ldx, ldy (>= k), k >= 1.
 *   rowptr, col and val must be 16-byte aligned (they are streamed with bulk copies), else LS_ERR_BAD_ARG.  */
int ls_spmm_csr_f32(int64_t V, const int32_t *rowptr, const int32_t *col, const float *val,
                    const float *x, int64_t ldx, float *y, int64_t ldy, int k, void *stream);
/* ---- gradient of y = A x with respect to A's values  (completes `L @ v` of parameterize.py:30 and scripts/main.py:192-195,
 *      which torch differentiates in both arguments)
 *   gval[e] = sum_{q=0..k-1} gy[row_e, q] x[col_e, q] over A's CSR pattern, q summed in order.  x, gy: (V,k) float32
 *   row-major with leading dimensions ldx, ldgy (>= k), k >= 1; gval (nnz) float32 out.  No atomics: bit-reproducible.      */
int ls_spmm_csr_grad_val_f32(int64_t V, const int32_t *rowptr, const int32_t *col, const float *x, int64_t ldx,
                             const float *gy, int64_t ldgy, int k, float *gval, void *stream);

/* ---- preconditioned conjugate gradients  (replaces solvers.py:26-39 CholeskySolver.solve via cholespy and
 *      solvers.py:41-126 ConjugateGradientSolver: solve M X = B for all k columns in one pass) ------------
 *   ls_pcg_workspace_bytes: bytes of device workspace a handle for (V, nnz, k_max) needs.
 *   ls_pcg_create: copies the CSR into the (caller-owned, 256-byte aligned) workspace in the solver's padded
 *       streaming layout (re-ordered by perm_new2old when given; b/x/x0 of ls_pcg_solve stay in the caller's
 *       numbering), extracts the Jacobi diagonal, balances the row partition, plans the SpMM blocks.
 *       The caller keeps `workspace` alive until ls_pcg_destroy.  Synchronises `stream`.
 *       precond: 0 = none, 1 = Jacobi, 2 = Chebyshev polynomial of degree 3 in D^-1 M on top of Jacobi (spectrum bounds from a
 *       Gershgorin row scan; ~3x fewer CG iterations and reductions for ~1.3x the SpMVs), 3 = auto: 2 where it is measured
 *       faster (meshes whose solver vectors fit in shared memory on the cooperative grid, ~1K..430K vertices), else 1.
 *       k_max in [1,4].
 *       The workspace size depends on (V, nnz, k_max) only -- never on the environment.
 *   ls_pcg_solve:  b, x: (V,k) float32 row-major contiguous (ld = k); x0 = NULL for a cold start (x0 may alias x).
 *       rtol: stop when ||r_j||_2 <= rtol * ||b_j||_2 for every column j (columns freeze independently, which
 *       is what the reference's per-axis solves do, solvers.py:115-118).  maxit > 0.
 *       info_dev (optional, device, 8 floats): [iterations, status, relres_0..relres_3, 0, 0] written
 *       stream-ordered; info_host (optional, HOST, same 8 floats): if non-NULL the call synchronises and
 *       returns LS_ERR_NOT_CONVERGED / LS_ERR_BREAKDOWN as status; if NULL the call stays asynchronous.   */
int ls_pcg_workspace_bytes(int64_t V, int64_t nnz, int k_max, size_t *bytes_out);
int ls_pcg_create(void **handle_out, int64_t V, int64_t nnz,
                  const int32_t *rowptr, const int32_t *col, const float *val,
                  const int32_t *perm_new2old /* optional locality order from ls_order_morton, or NULL */,
                  int precond, int k_max, void *workspace, size_t workspace_bytes, void *stream);
int ls_pcg_solve(void *handle, const float *b, float *x, const float *x0, int k,
                 float rtol, int maxit, float *info_dev, float *info_host, void *stream);
int ls_pcg_destroy(void *handle);
/* Accuracy guard of the fused solver (csrc/ls_pcg_fused.cuh).  When the iteration has converged on its recursive residual
 * the kernel evaluates the TRUE residual b - M x with fp64 accumulation; if, for some column, it exceeds both rtol ||b|| and
 * theta * 2^-24 * || |M| |x| || (theta times the floor that storing x in fp32 imposes), the iteration restarts from that
 * residual, at most max_restarts times per solve.  Defaults: max_restarts = 1, theta = 3.  max_restarts = 0 switches the
 * check off.  (The reference's direct solve has no such knob: solvers.py:36-39.)                                            */
int ls_pcg_set_refinement(void *handle, int max_restarts, float theta);
/* ---- batched solve: n independent meshes per call, one thread-block cluster of 1..16 CTAs per mesh ----------------------
 * For many small and mid-size meshes with DIFFERENT matrices (meshes sharing one matrix are already one ls_pcg_solve with
 * 3n columns).  Each mesh iterates, checks its true residual and stops on its own; results and iteration counts of a mesh do
 * not depend on the other meshes of the batch.
 *   ls_pcg_batch_create: plans the batch over existing handles from ls_pcg_create (the handles must outlive the batch
 *       and may not appear twice) and uploads its argument table (cudaMalloc'd, freed by ls_pcg_batch_destroy).  Each
 *       handle's own preconditioner is used: Jacobi, or for a handle whose preconditioner is Chebyshev (precond 2) the same
 *       polynomial as ls_pcg_solve, always at RES 2.  Each mesh gets the smallest cluster of 1, 2, 4, 8 or 16 CTAs whose
 *       shared memory holds its solver vectors; meshes with the same preconditioner, cluster size and kernel form one launch.
 *       A mesh larger than one cluster of 16 (Jacobi: 71,680 rows with the pattern-only matrix copy, 68,096 with the general
 *       one; Chebyshev: 48,128 / 46,592; at 227 KB of shared memory per CTA) returns LS_ERR_BAD_ARG: solve it with
 *       ls_pcg_solve.  Synchronises `stream`.
 *   ls_pcg_batch_solve: b, x (and the optional warm start x0) are packed (sum V_i, k) float32 row-major: mesh i's rows
 *       follow mesh i-1's, in the order of `handles`.  k in [1,3].  info_dev (optional, device, 8 n floats): mesh i's
 *       record [iterations, status, relres_0..relres_3, restarts, 0] at info_dev + 8 i.  info_host (optional, HOST, 8 n
 *       floats): as ls_pcg_solve, the call then synchronises and returns LS_ERR_BREAKDOWN / LS_ERR_NOT_CONVERGED for the
 *       first mesh that failed (named in ls_last_error); if NULL the call stays asynchronous.  One launch per plan group,
 *       no host-to-device copy.                                                                                                  */
int ls_pcg_batch_create(void **batch_out, void *const *handles, int n, void *stream);
int ls_pcg_batch_solve(void *batch, const float *b, float *x, const float *x0, int k, float rtol, int maxit,
                       float *info_dev /* 8 n */, float *info_host, void *stream);
int ls_pcg_batch_destroy(void *batch);
/* introspection.  Fused solver (default): out8 = [matrix copy (2 pattern-only SELL-32 / 1 general SELL-32), padded SELL
 *   entries, CTAs, cluster size (0 = cooperative grid), 10 + residency level (0 vectors in global memory, 1 r/s/D^-1 in
 *   shared memory, 2 also x and p, 3 also the gathered vector), preconditioner in use (0 / 1 / 2), threads per CTA, re-ordered].
 *   Graph-mode solver (LS_PCG_MODE=graph, or when the fused kernel cannot run): out8 = [engine (1 SELL-32, 0 = TMA-staged
 *   CSR), padded SELL entries, SpMM grid, vector-kernel grid, 0, 0, block plan valid, re-ordered].  (Values 1 and 2 of
 *   out8[4] are retired and not produced.)                                                                           */
int ls_pcg_describe(void *handle, int64_t *out8);
/* algorithmic bytes of one in-solver SpMM launch: 8 nnz + 4 (V+1) + 8 k V  (SURVEY.md section 8 d)      */
int64_t ls_pcg_spmm_bytes(void *handle, int k);

/* ---- per-step glue either side of the solve  (replaces scripts/geometry.py:91-147 compute_face_normals /
 *      compute_vertex_normals and the `v_unique[duplicate_idx]` gathers of scripts/main.py:176-180; csrc/ls_glue.cu) ---------
 * All differentiable: the *_bwd entry points are the adjoints the Python autograd wrappers call.  Scatter-adds are gathers
 * over a list built once per connectivity, so the per-step kernels use no atomics and are bit-reproducible.
 *   faces (F,3) / idx (n): int32 (idx_bytes = 4) or int64 (8), device.  verts (V,3) float32.
 *   ls_face_incidence: inc_ptr (V+1), inc (3F) int32: for vertex v the sorted codes 4*face + corner of its face corners.
 *   ls_index_buckets:  ptr (V+1), items (n): positions i with idx[i] == v, sorted (the adjoint of a row gather).
 *     both: workspace of ls_bucket_workspace_bytes(V) bytes; synchronise the stream; LS_ERR_INDEX_RANGE on a bad index.
 *   ls_gather_rows_f32:      dst[i,:] = src[idx[i],:]               (n,k) <- (V,k), row-major contiguous
 *   ls_gather_rows_bwd_f32:  gsrc[v,:] = sum_{i in bucket v} gdst[i,:]
 *   ls_face_normals_f32:     n (3,F) = normalised cross(v1 - v0, v2 - v0), the reference's layout (geometry.py:104-110)
 *   ls_vertex_normals_f32:   out (V,3) = normalised sum over incident corners of face_normal * acos(<d0,d1>), d0/d1 the corner's
 *                            edge vectors divided by the Frobenius norm of the WHOLE edge field as in geometry.py:137-140;
 *                            also writes raw_len (V) and edge_norms (3) for the backward.  scratch: ls_glue_scratch_bytes().  */
int ls_glue_scratch_bytes(size_t *bytes_out);
int ls_bucket_workspace_bytes(int64_t n_keys, size_t *bytes_out);
int ls_face_incidence(const void *faces, int idx_bytes, int64_t F, int64_t V, int32_t *inc_ptr, int32_t *inc,
                      void *workspace, size_t workspace_bytes, void *stream);
int ls_index_buckets(const void *idx, int idx_bytes, int64_t n, int64_t V, int32_t *ptr, int32_t *items,
                     void *workspace, size_t workspace_bytes, void *stream);
int ls_gather_rows_f32(const float *src, const void *idx, int idx_bytes, int64_t n, int k, float *dst, void *stream);
int ls_gather_rows_bwd_f32(const float *gdst, const int32_t *ptr, const int32_t *items, int64_t V, int k, float *gsrc, void *stream);
int ls_face_normals_f32(const float *verts, const void *faces, int idx_bytes, int64_t F, float *n, void *stream);
int ls_face_normals_bwd_f32(const float *verts, const void *faces, int idx_bytes, int64_t F, int64_t V,
                            const int32_t *inc_ptr, const int32_t *inc, const float *gn, float *gverts, void *stream);
int ls_vertex_normals_f32(const float *verts, const void *faces, int idx_bytes, int64_t F, int64_t V,
                          const int32_t *inc_ptr, const int32_t *inc, const float *face_normals, float *out,
                          float *raw_len, float *edge_norms, void *scratch, void *stream);
int ls_vertex_normals_bwd_f32(const float *verts, const void *faces, int idx_bytes, int64_t F, int64_t V,
                              const int32_t *inc_ptr, const int32_t *inc, const float *face_normals, const float *out,
                              const float *raw_len, const float *edge_norms, const float *gout, float *gverts,
                              float *gface_normals, void *scratch, void *stream);
/*   Per-mesh vertex normals of B meshes packed into one mesh: verts (sum V_i, 3), faces (sum F_i, 3) with mesh i's indices
 *   shifted by its first vertex, face_normals (3, sum F_i).  The edge-field norms (and the backward's T_i) are taken per mesh,
 *   with mesh i's faces split over the same blocks as the single-mesh call, so every output is bitwise what
 *   ls_vertex_normals_f32 / _bwd_f32 give mesh i on its own.  One memset and two kernels per direction, whatever B is.
 *     vert_offsets, face_offsets:  (B + 1) int64, device: mesh i owns vertices [vert_offsets[i], vert_offsets[i+1]) and faces
 *                                  [face_offsets[i], face_offsets[i+1]); the *_host arrays hold the same values in host
 *                                  memory (checked there: monotone, starting at 0, ending at V and F; else LS_ERR_BAD_ARG).
 *                                  Faces must index their own mesh's vertices (not checked here).
 *     edge_norms (3 B): mesh i's three norms at 3 i.   inc_ptr / inc: ls_face_incidence of the packed faces.
 *     scratch: ls_vertex_normals_batch_scratch_bytes(B) bytes, device, 16-byte aligned.  B in [1, 65535].              */
int ls_vertex_normals_batch_scratch_bytes(int B, size_t *bytes_out);
int ls_vertex_normals_batch_f32(const float *verts, const void *faces, int idx_bytes, int64_t F, int64_t V, int B,
                                const int64_t *vert_offsets, const int64_t *face_offsets,
                                const int64_t *vert_offsets_host, const int64_t *face_offsets_host,
                                const int32_t *inc_ptr, const int32_t *inc, const float *face_normals, float *out,
                                float *raw_len, float *edge_norms, void *scratch, size_t scratch_bytes, void *stream);
int ls_vertex_normals_batch_bwd_f32(const float *verts, const void *faces, int idx_bytes, int64_t F, int64_t V, int B,
                                    const int64_t *vert_offsets, const int64_t *face_offsets,
                                    const int64_t *vert_offsets_host, const int64_t *face_offsets_host,
                                    const int32_t *inc_ptr, const int32_t *inc, const float *face_normals, const float *out,
                                    const float *raw_len, const float *edge_norms, const float *gout, float *gverts,
                                    float *gface_normals, void *scratch, size_t scratch_bytes, void *stream);
/*   ls_massmatrix_voronoi_f32:  out (V) = mixed Voronoi area of each vertex, massmatrix_voronoi of scripts/geometry.py:35-89:
 *     per face the law-of-cosines barycentric cells, Heron's area with no clamp, the obtuse override (0.5 area at the obtuse
 *     corner, 0.25 at the others), summed per vertex in the reference's float32 order.  A face with a zero-length edge gives
 *     NaN at its vertices, as in the reference; an unused vertex gets 0.  inc_ptr / inc: ls_face_incidence of the same faces.
 *   ls_massmatrix_voronoi_bwd_f32:  gverts (V,3) = d(sum_v gout[v] out[v]) / d verts, through the branch the override took.
 *     Both: no scratch, no atomics, bit-reproducible.                                                                       */
int ls_massmatrix_voronoi_f32(const float *verts, const void *faces, int idx_bytes, int64_t F, int64_t V,
                              const int32_t *inc_ptr, const int32_t *inc, float *out, void *stream);
int ls_massmatrix_voronoi_bwd_f32(const float *verts, const void *faces, int idx_bytes, int64_t F, int64_t V,
                                  const int32_t *inc_ptr, const int32_t *inc, const float *gout, float *gverts, void *stream);

/* ---- point-to-mesh distances  (igl.point_mesh_squared_distance and igl.hausdorff, which the figure scripts score their runs
 *      with: figures/comparison/generate_data.py:78-88; csrc/ls_distance.cu) ------------------------------------------------
 *   ls_distance_bvh_bytes:  bytes of the BVH of F faces (F in [1, 2^30]): 256 + 48 F + 64 (F - 1), or the build scratch if
 *     that is larger.
 *   ls_distance_bvh_build:  builds the BVH of the mesh (verts (V,3) float32, faces (F,3) int32 / int64 as idx_bytes says,
 *     every index in [0, V): not checked here) into `bvh` (256-byte aligned; the caller keeps it while it queries).
 *     Asynchronous.  The BVH does not refer to verts or faces afterwards.
 *   ls_distance_query_workspace_bytes:  bytes of the workspace of a query of n points.
 *   ls_distance_query:  for each point q of points (n,3) float32: sqrD[q] (float64) the least squared distance to a face,
 *     face[q] (int64) the lowest face index at that distance, closest (n,3) float64 the closest point on that face, all in
 *     the caller's order (each output may be NULL).  The closest point on a face is computed in float64 from the float32
 *     corners.  A point with a non-finite coordinate, or any point when a face has a non-finite corner, gets NaN, -1 and
 *     NaN.  max_mode: 0 = no maximum; 1 = the workspace's record holds the maximum of this query's sqrD; 2 = folds it into
 *     the record of an earlier query on the same workspace (NaN-propagating).  Asynchronous; bitwise reproducible.
 *   ls_distance_result:  synchronises `stream`, writes the record's maximum to *max_host (if non-NULL) and returns
 *     LS_ERR_UNSUPPORTED if a query folded into it overflowed its traversal stack (the tree's depth bound rules it out).
 *   workspace: 256-byte aligned; a query may not overlap another on the same workspace.
 *   ls_distance_grad_workspace_bytes:  bytes of the workspace of a gradient w.r.t. the vertices of n queries on a mesh of F
 *     faces and V vertices (n in [0, 2^31 - 16), F in [1, 0x1ffffff0 / 3), V in [1, 2^31 - 16)).
 *   ls_distance_grad_f32:  the backward of sqrD from a query's face (n) and closest (n,3) outputs and the upstream
 *     grad_sqrD (n) float64: with C = closest[q] and beta the weights of C on the corners (a, b, c) of face[q] in face order
 *     (recomputed in float64 from points[q] and the corners by the query's Voronoi regions),
 *       grad_points[q] = 2 g[q] (p_q - C)                        (n,3) float32, NULL to skip
 *       grad_verts[k] += -2 g[q] beta_k (p_q - C) per corner k   (V,3) float32, NULL to skip; overwritten, not accumulated
 *     A face that repeats a vertex adds once per corner; an unreferenced vertex gets 0.  A row with face -1 (a non-finite
 *     point or corner) gets NaN in grad_points and adds nothing to grad_verts.  Sums run in float64 in a fixed order and
 *     are rounded once: no atomics, bitwise reproducible for either index type and on any stream.  verts, faces and
 *     workspace (256-byte aligned, ls_distance_grad_workspace_bytes) are needed only with grad_verts.  Asynchronous.  */
int ls_distance_bvh_bytes(int64_t F, size_t *bytes_out);
int ls_distance_bvh_build(const float *verts, int64_t V, const void *faces, int idx_bytes, int64_t F, void *bvh,
                          size_t bvh_bytes, void *stream);
int ls_distance_query_workspace_bytes(int64_t n, size_t *bytes_out);
int ls_distance_query(const void *bvh, int64_t F, const float *points, int64_t n, double *sqrD, int64_t *face, double *closest,
                      int max_mode, void *workspace, size_t workspace_bytes, void *stream);
int ls_distance_result(const void *workspace, double *max_host, void *stream);
int ls_distance_grad_workspace_bytes(int64_t n, int64_t F, int64_t V, size_t *bytes_out);
int ls_distance_grad_f32(const float *points, int64_t n, const float *verts, int64_t V, const void *faces, int idx_bytes,
                         int64_t F, const int64_t *face, const double *closest, const double *grad_sqrD, float *grad_points,
                         float *grad_verts, void *workspace, size_t workspace_bytes, void *stream);

/* ---- point-to-mesh distances over a packed batch of B meshes  (csrc/ls_distance.cu) -------------------------------------
 *   The meshes are packed as by batch.pack_meshes: faces (F,3) with mesh b's rows [face_offsets[b], face_offsets[b+1]) indexing
 *   vertices of mesh b only (not checked here), each mesh with at least one face.  Their BVHs are one forest, built in the
 *   same launches for any B; the single-mesh entry points above are the case B = 1.
 *   ls_distance_bvh_batch_bytes:  bytes of the forest of B meshes and F faces in all (1 <= B <= min(F, 2^24)):
 *     align256(16 B + 8) + 48 F + 64 (F - B), or the build scratch if that is larger.
 *   ls_distance_bvh_batch_build:  ls_distance_bvh_build of every mesh, with face_offsets (B + 1) int64 on the device (copied
 *     into the BVH).  Each mesh has its own non-finite flag and prune slack.  Asynchronous.
 *   ls_distance_query_batch_workspace_bytes:  bytes of the workspace of a query of n points in S segments.
 *   ls_distance_query_batch:  the rows [point_offsets[s], point_offsets[s+1]) of points (point_offsets (S + 1) int64 on the
 *     device, from 0 to n, non-decreasing: not checked here) are answered by mesh s, or by the only mesh when B == 1 (then S
 *     is any count >= 1; otherwise S == B).  sqrD, face (packed face index) and closest as ls_distance_query, each bitwise
 *     what ls_distance_query on a BVH of that mesh alone gives, up to the face offset.  max_out (S) float64 on the device,
 *     NULL exactly when max_mode is 0: max_mode 1 sets max_out[s] to the NaN-propagating maximum of segment s's sqrD, 2 folds
 *     it into max_out (0 for an empty segment).  The workspace's record counts stack overflows for ls_distance_result.
 *     Asynchronous; bitwise reproducible.
 *   ls_distance_segment_sum_f64:  out[s] = the sum of x[offsets[s] .. offsets[s+1]) in float64 (offsets (S + 1) on the
 *     device), in a fixed order without atomics: bitwise reproducible.  The per-mesh chamfer means.  Asynchronous.  */
int ls_distance_bvh_batch_bytes(int64_t F, int64_t B, size_t *bytes_out);
int ls_distance_bvh_batch_build(const float *verts, int64_t V, const void *faces, int idx_bytes, int64_t F, int64_t B,
                                const int64_t *face_offsets, void *bvh, size_t bvh_bytes, void *stream);
int ls_distance_query_batch_workspace_bytes(int64_t n, int64_t S, size_t *bytes_out);
int ls_distance_query_batch(const void *bvh, int64_t F, int64_t B, const float *points, int64_t n, int64_t S,
                            const int64_t *point_offsets, double *sqrD, int64_t *face, double *closest, double *max_out,
                            int max_mode, void *workspace, size_t workspace_bytes, void *stream);
int ls_distance_segment_sum_f64(const double *x, int64_t n, int64_t S, const int64_t *offsets, double *out, void *stream);

/* ---- isotropic remeshing  (the reference loop's remesh_botsch: scripts/main.py:149; csrc/ls_remesh.cu) ---------------------
 *   For closed, edge-manifold, consistently oriented meshes: verts (V,3) float32 and faces (F,3) int32, both device buffers the
 *   stages rewrite in place.  Each stage runs on `workspace` (device, 256-byte aligned, ls_remesh_workspace_bytes of the
 *   buffers' capacity V_cap, F_cap) and synchronises `stream` once to read back its counts.  With F == 0, split, collapse,
 *   flip and compact launch nothing and report 0 (compact: no vertex is referenced); faces with V == 0 are LS_ERR_BAD_ARG,
 *   or LS_ERR_INDEX_RANGE in ls_remesh_check.
 *   ls_remesh_workspace_bytes:  bytes of the workspace for meshes of up to V vertices and F faces.
 *   ls_remesh_check:  *flags_out = the defects found, OR of 1 (an edge with one face), 2 (an edge with more than two faces),
 *     4 (a directed edge held by two faces), 8 (a face repeating a vertex), 16 (an index outside [0, V): LS_ERR_INDEX_RANGE).
 *   ls_remesh_split:  splits every edge longer than `high` at its midpoint, all at once (new vertices V.., new faces F..);
 *     needs V_cap >= V + 3F/2 and F_cap >= 4F; *n_split = edges split (V += n, F += 2n).
 *   ls_remesh_collapse_round:  one round of midpoint collapses of edges shorter than `low` (an independent set of local
 *     minima of the edge length; an edge whose ends both have valence 3 never collapses); a collapsed vertex is left
 *     unreferenced and its two faces become rows of -1.
 *     V_live: the live vertices (no collapse when <= 4).  *n_collapsed = collapses applied.
 *   ls_remesh_compact:  drops the rows of -1 and the unreferenced vertices, keeping the order; *V_out, *F_out the new sizes.
 *   ls_remesh_flip_round:  one round of valence-improving edge flips; *n_flipped = flips applied.
 *   ls_remesh_relax:  tangential relaxation towards the neighbours' mean, then projection onto the mesh of the BVH `bvh`
 *     (F0 faces, ls_distance_bvh_build).
 *   The _v entry points are the same stages for the reference's adaptive remesh_botsch(V, F, target, iters, feature,
 *   project).  They take three per-vertex device buffers with the vertices' capacity: vhigh = 1.4 t and vlow = 0.7 t
 *   (float64, t the target edge length) and feature (uint8, nonzero for a feature vertex).  Either all three are NULL, and the
 *   call equals the entry point without _v (scalar bounds, no features), or all three are set, and the scalar high and low
 *   are not read; one or two set is LS_ERR_BAD_ARG.  With the attributes set:
 *     split:  edge (a, b) splits iff neither end is a feature and |ab|^2 > ((vhigh[a] + vhigh[b]) / 2)^2; its midpoint gets
 *       vhigh = (vhigh[a] + vhigh[b]) / 2, vlow = (vlow[a] + vlow[b]) / 2 and feature = 0.  Writes the new vertices' attributes.
 *     collapse:  edge (a, b) is eligible iff neither end is a feature, |ab|^2 < ((vlow[a] + vlow[b]) / 2)^2, every neighbour
 *       of a (b) other than b (a) is within vhigh[a] (vhigh[b]) of the midpoint, and the scalar call's other checks pass.  The
 *       survivor a (the lower index) keeps its own attributes.  Reads the attributes.
 *     flip:  no flip of edge (a, b) whose a, b or opposite vertices c, d is a feature.  Reads feature.
 *     compact:  moves the attributes with the vertices; an unreferenced vertex's attributes are dropped.
 *     relax:  a feature vertex is neither relaxed nor projected: it keeps its position bit for bit.  Reads feature.
 *   A constant target equal to h with no feature gives the scalar call's result (high = 1.4 h, low = 0.7 h) bit for bit.      */
int ls_remesh_workspace_bytes(int64_t V, int64_t F, size_t *bytes_out);
int ls_remesh_check(const int32_t *faces, int64_t F, int64_t V, void *workspace, size_t workspace_bytes, uint32_t *flags_out,
                    void *stream);
int ls_remesh_split(float *verts, int32_t *faces, int64_t V, int64_t F, int64_t V_cap, int64_t F_cap, double high, void *workspace,
                    size_t workspace_bytes, int64_t *n_split, void *stream);
int ls_remesh_collapse_round(float *verts, int32_t *faces, int64_t V, int64_t F, int64_t V_live, double low, double high,
                             void *workspace, size_t workspace_bytes, int64_t *n_collapsed, void *stream);
int ls_remesh_compact(float *verts, int32_t *faces, int64_t V, int64_t F, void *workspace, size_t workspace_bytes, int64_t *V_out,
                      int64_t *F_out, void *stream);
int ls_remesh_flip_round(const float *verts, int32_t *faces, int64_t V, int64_t F, void *workspace, size_t workspace_bytes,
                         int64_t *n_flipped, void *stream);
int ls_remesh_relax(float *verts, const int32_t *faces, int64_t V, int64_t F, const void *bvh, int64_t F0, void *workspace,
                    size_t workspace_bytes, void *stream);
int ls_remesh_split_v(float *verts, int32_t *faces, int64_t V, int64_t F, int64_t V_cap, int64_t F_cap, double high, double *vhigh,
                      double *vlow, uint8_t *feature, void *workspace, size_t workspace_bytes, int64_t *n_split, void *stream);
int ls_remesh_collapse_round_v(float *verts, int32_t *faces, int64_t V, int64_t F, int64_t V_live, double low, double high,
                               double *vhigh, double *vlow, uint8_t *feature, void *workspace, size_t workspace_bytes,
                               int64_t *n_collapsed, void *stream);
int ls_remesh_compact_v(float *verts, int32_t *faces, int64_t V, int64_t F, double *vhigh, double *vlow, uint8_t *feature,
                        void *workspace, size_t workspace_bytes, int64_t *V_out, int64_t *F_out, void *stream);
int ls_remesh_flip_round_v(const float *verts, int32_t *faces, int64_t V, int64_t F, double *vhigh, double *vlow, uint8_t *feature,
                           void *workspace, size_t workspace_bytes, int64_t *n_flipped, void *stream);
int ls_remesh_relax_v(float *verts, const int32_t *faces, int64_t V, int64_t F, const void *bvh, int64_t F0, double *vhigh,
                      double *vlow, uint8_t *feature, void *workspace, size_t workspace_bytes, void *stream);

/* ---- fused AdamUniform step  (replaces largesteps/optimize.py:17-41) ----------------------------------
 *   n elements float32; one_minus_beta{1,2} = 1 - beta and c1 = 1 - beta1^t, c2 = 1 - beta2^t are computed by
 *   the caller in double (as the reference's Python does) and rounded once to float.
 *   scratch: device, >= 16 bytes, zero-initialised by the callee.                                        */
int ls_adam_uniform_step(float *param, const float *grad, float *g1, float *g2, int64_t n,
                         float lr, float beta1, float beta2, float one_minus_beta1, float one_minus_beta2,
                         float c1, float c2, void *scratch, void *stream);
/* ---- the same step for n tensors at once: each tensor gets its own normaliser (the max of its own g2, NaN if its moments
 *   hold a NaN), so every tensor comes out bitwise as ls_adam_uniform_step would leave it.  Two kernels per
 *   LS_ADAM_MULTI_MAX tensors (the table travels as a kernel parameter: no allocation, no copy, no synchronisation).
 *   tensors: HOST array of n entries (n >= 0; entries with n == 0 are skipped); lr / betas / c1 / c2 per tensor, so
 *   tensors of different parameter groups and step counts share a call.
 *   scratch: device, >= 8 n bytes (scratch_bytes), zero-initialised by the callee.                                     */
#define LS_ADAM_MULTI_MAX 256
typedef struct {
    float *param;
    const float *grad;
    float *g1;
    float *g2;
    int64_t n;
    float lr, beta1, beta2, one_minus_beta1, one_minus_beta2, c1, c2;
} ls_adam_tensor;
int ls_adam_uniform_step_multi(const ls_adam_tensor *tensors, int n, void *scratch, size_t scratch_bytes, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* LARGESTEPS_B200_H */
