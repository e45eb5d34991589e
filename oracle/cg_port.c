/*
 * cg_port.c -- TEST INFRASTRUCTURE / CPU BASELINE ONLY (see oracle/__init__.py).
 *
 * Plain-C restatement of the reference's ConjugateGradientSolver (largesteps/solvers.py:41-126), the one solve path
 * of the reference that runs without the cholespy wheel.  Same algorithm, same arithmetic type (fp32), same absolute
 * tolerance, one axis at a time; the reference gets its host parallelism from torch's intra-op threads, here every
 * vector operation and the CSR matvec are OpenMP loops, so it can use all the host cores it is given
 * (`bench.py --impl reference`, `cpu_baseline`).  Never linked into the product library.
 *
 *   solve_axis  solvers.py:58-84     r = A x - b; p = -r; while ||r|| > 1e-5: ...
 *   solve       solvers.py:86-126    per-axis loop with separate forward / backward warm starts (the caller keeps them)
 *
 * It also holds lsref_sell_spmv_f32, the exact model of the solver's SELL-32 SpMV that tests/test_gpu_sell_spmv.py
 * compares the device with bit for bit.
 *
 * Build: gcc -O3 -fopenmp -shared -fPIC oracle/cg_port.c -o oracle/_build/libcg_port.so   (oracle/cport.py does it)
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#ifdef _OPENMP
#include <omp.h>
#endif

int lsref_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

void lsref_set_num_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

/* y = A x, CSR, fp32 (torch: `self.M @ p`, solvers.py:70,74) */
static void spmv(int64_t n, const int32_t *rowptr, const int32_t *col, const float *val, const float *x, float *y) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        float s = 0.f;
        for (int32_t j = rowptr[i]; j < rowptr[i + 1]; ++j) s += val[j] * x[col[j]];
        y[i] = s;
    }
}

static float dot(int64_t n, const float *a, const float *b) {
    double s = 0.0; /* torch reduces fp32 with wider partial sums per chunk; double keeps the port thread-count independent */
#pragma omp parallel for reduction(+ : s) schedule(static)
    for (int64_t i = 0; i < n; ++i) s += (double)a[i] * (double)b[i];
    return (float)s;
}

/* solvers.py:58-84.  x holds x0 on entry, the solution on exit.  work: 3 n floats.  Returns the iteration count. */
int lsref_cg_axis(int64_t n, const int32_t *rowptr, const int32_t *col, const float *val, const float *b, float *x,
                  float tol, int maxit, float *work) {
    float *r = work, *p = work + n, *Ap = work + 2 * n;
    spmv(n, rowptr, col, val, x, r);                       /* r = M x - b        (solvers.py:70) */
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        r[i] -= b[i];
        p[i] = -r[i];                                      /* p = -r             (solvers.py:71) */
    }
    float r_norm = sqrtf(dot(n, r, r));                    /* r.norm()           (solvers.py:72) */
    int it = 0;
    while (r_norm > tol && it < maxit) {                   /* absolute tolerance (solvers.py:73); maxit is a safety net */
        spmv(n, rowptr, col, val, p, Ap);                  /* Ap = M p           (solvers.py:74) */
        const float r2 = r_norm * r_norm;                  /*                    (solvers.py:75) */
        const float alpha = r2 / dot(n, p, Ap);            /*                    (solvers.py:76) */
#pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < n; ++i) {
            x[i] += alpha * p[i];                          /*                    (solvers.py:77) */
            r[i] += alpha * Ap[i];                         /*                    (solvers.py:80) */
        }
        r_norm = sqrtf(dot(n, r, r));                      /*                    (solvers.py:81) */
        const float beta = r_norm * r_norm / r2;           /*                    (solvers.py:82) */
#pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < n; ++i) p[i] = -r[i] + beta * p[i];   /*        (solvers.py:83) */
        ++it;
    }
    return it;
}

/* y = A x, (V, K) row-major, exactly as the solver's SELL-32 SpMM kernels compute it (csrc/ls_sell_kernel.cuh): every
 * row is padded to the widest row of its slice of 32 rows with entries {own row, 0.0f}, and its entries, the CSR ones in
 * order and then the padding, are accumulated one fmaf(val, x[col], acc) after the other from acc = 0.  fmaf() rounds once
 * per step whatever the compiler's contraction setting, so the result is the device's bit for bit. */
void lsref_sell_spmv_f32(int64_t V, int K, const int32_t *rowptr, const int32_t *col, const float *val, const float *x,
                         float *y) {
#pragma omp parallel for schedule(static)
    for (int64_t s = 0; s < (V + 31) / 32; ++s) {
        const int64_t r0 = 32 * s, r1 = r0 + 32 < V ? r0 + 32 : V;
        int32_t w = 0;
        for (int64_t i = r0; i < r1; ++i)
            if (rowptr[i + 1] - rowptr[i] > w) w = rowptr[i + 1] - rowptr[i];
        for (int64_t i = r0; i < r1; ++i)
            for (int k = 0; k < K; ++k) {
                float acc = 0.f;
                for (int32_t j = 0; j < w; ++j) {
                    const int32_t e = rowptr[i] + j;
                    acc = (e < rowptr[i + 1]) ? fmaf(val[e], x[(int64_t)col[e] * K + k], acc) : fmaf(0.f, x[i * K + k], acc);
                }
                y[i * K + k] = acc;
            }
    }
}

/* solvers.py:115-118: one CG per axis of a (n,k) row-major right-hand side; x0 / x are (n,k) row-major too.
 * iters_out[k] receives the iteration counts. */
int lsref_cg_solve(int64_t n, int k, const int32_t *rowptr, const int32_t *col, const float *val, const float *b,
                   const float *x0, float *x, float tol, int maxit, int *iters_out) {
    float *bb = (float *)malloc(sizeof(float) * (size_t)n * 5);
    if (!bb) return -1;
    float *xx = bb + n, *work = bb + 2 * n;
    for (int a = 0; a < k; ++a) {
#pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < n; ++i) {
            bb[i] = b[i * k + a];
            xx[i] = x0 ? x0[i * k + a] : 0.f;
        }
        const int it = lsref_cg_axis(n, rowptr, col, val, bb, xx, tol, maxit, work);
        if (iters_out) iters_out[a] = it;
#pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < n; ++i) x[i * k + a] = xx[i];
    }
    free(bb);
    return 0;
}
