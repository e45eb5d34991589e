// ls_pcg_handle.h -- the solver's handle and the host functions its translation units call in one another (internal: nothing
// here is exported from libls_b200.so).  The solver's host code is split by concern:
//   ls_pcg.cu         the workspace carve, the C entry points create / solve / destroy, the fused solver's device checks and launch
//   ls_pcg_copies.cu  the matrix copies: CSR (optionally re-ordered), dinv, SELL-32, pattern-only, the Chebyshev coefficients
//   ls_pcg_graph.cu   the graph-mode fallback solver and every launch of the stand-alone SpMV kernels (and their diagnostics)
//   ls_pcg_plan.cu    the launch plans of the fused and the batched solve: host only, no CUDA call
//   ls_pcg_batch.cu   the batched solve
// A kernel is referenced from exactly one translation unit: a template kernel named in two is compiled and registered twice
// (tests/test_kernel_inventory.py).  So the stand-alone SpMV kernels, their occupancy query included, stay in ls_pcg_graph.cu,
// the copy kernels in ls_pcg_copies.cu, and the fused kernel is reached only through the ls_fused_fn_* tables.
#pragma once
#include "ls_spmm_host.h"
#include "ls_pcg_fused.cuh"

#pragma GCC visibility push(hidden)
namespace lspcg {

constexpr int KMAX = 4;
// upper bound on the graph-mode kernels' grids (workspace sizing of their partials and SpMM descriptors; 132 SMs on H100 SXM).
// The fused solver's grid is at most 255 CTAs: its partials are carved for 256.
constexpr int GRID_CAP = 132 * 8 * 2;

struct PcgCtrl {
    double rz[KMAX], pAp[KMAX], rr[KMAX], bb[KMAX];
    float beta[KMAX];
    float rtol2;
    int maxit;
    int it;
    int done;        // 0 running, 1 converged, 2 maxit reached, 3 breakdown
    int conv[KMAX];  // column frozen
    int k;
    int restart;     // warm start was worse than a cold start for some column: redo the initialisation from x = 0
};

// How the fused solver runs a mesh for one K (plan_fused).  on = 0: it does not, the graph-mode solver runs.
struct FusedPlan {
    int on, grid, cluster, res, nw, sync, nsl_max;   // nw warps per CTA; sync 1: one CTA or one cluster (cluster = grid), 0: grid
    size_t smem;
};

// The environment switches of the fused solver's launch plan (DESIGN 4.6), read once per ls_pcg_create / ls_pcg_plan.
struct PlanEnv {
    int graph;       // LS_PCG_MODE=graph: no fused solver
    int cluster;     // LS_PCG_CLUSTER: -1 auto, 0 never one CTA or cluster, N a cluster of N CTAs
    int res;         // LS_PCG_RES: cap on the residency level, -1 none
    int onecta;      // LS_PCG_ONECTA: largest mesh (slices) on one CTA
    int clres;       // LS_PCG_CLRES: largest mesh (slices) on one cluster of CLRES_CS CTAs at RES 4
    int small_cta;   // 256-thread CTAs where they apply (LS_PCG_SMALLCTA=0: never)
};

// The environment switches of the matrix copies and the handle's defaults (DESIGN 4.6), read once per ls_pcg_create.
struct CreateEnv {
    int force_reorder;   // LS_FORCE_REORDER set: use the caller's permutation without comparing gather locality
    int pattern;         // pattern-only copy where every off-diagonal value is equal (LS_PCG_PATTERN=0: never)
    int patshare;        // ... with identical slices stored once (LS_PCG_PATSHARE=0: one copy per slice)
    int csr;             // LS_SPMM_ENGINE=csr: the TMA-staged CSR engine even when the SELL-32 copy fits
    int cheb_m;          // LS_PCG_CHEB_M: Chebyshev steps, 2..8
    int refine;          // LS_PCG_REFINE: restarts from the true residual per solve
    int sell_tma;        // LS_SELL_TMA: stand-alone SpMM variant (3: 32 warps x 2 slots of 2 KB)
    int sell_pf;         // LS_SELL_PF: halo (rows) of its L2 prefetch
};

struct PcgHandle {
    int64_t V, nnz, Vp;
    int k_max, precond;
    int device;
    int sm_count;
    // workspace carve-out (device)
    int *rowptr, *col;
    float *val, *dinv;
    float *x, *r, *p, *Ap;
    PcgCtrl *ctrl;
    double *part_spmm, *part_vec;
    unsigned int *tickets;   // [0] spmm, [1] vec
    float *info;
    int *flags;
    int *perm;       // new -> old row (NULL-equivalent when has_perm == 0)
    int *inv;        // old -> new
    int *scan;
    int has_perm;
    // SELL-32 engine (fast path)
    int *soff;
    int2 *ent;
    long long sell_cap;      // capacity of `ent` in entries
    long long sell_entries;  // padded entry count
    int nslices;
    int sell_on;
    // pattern-only copy for matrices with one common off-diagonal value (ls_sell_kernel.cuh "PAT"; LS_PCG_PATTERN=0 switches it off)
    int *poff;
    unsigned int *pcol;
    unsigned char *pcls;     // diagonal class per row
    unsigned long long *pcls_tab;   // [PAT_CLASSES] classes, then an int: more classes than the table holds
    unsigned int *patmm;     // [min, max] of the off-diagonal value bits
    long long pat_cap;       // capacity of `pcol` in words
    float offc;
    int pat_on;
    int pat_shared;          // identical compact slices share one stored copy (LS_PCG_PATSHARE=0 keeps one copy per slice)
    int pat_stored;          // slices stored (distinct, plus the ones never shared)
    int pat_words;           // words of `pcol` in use
    // fused two-synchronisation solver (ls_pcg_fused.cuh): the default; one configuration for K = 3 (k = 1..3) and one for K = 4
    lsf::GridBar *gbar;      // grid barrier counter
    double *partials;        // fenced all-reduce partials, [2][NVMAX][grid]
    long long *dbg;          // LS_PCG_PROFILE cycle counters
    unsigned long long *ring;   // fast all-reduce slots
    int ring_slots;
    float *pv;               // owner copy of p, k_max planes
    float *z2, *cy, *cd;     // Chebyshev preconditioner: second published row buffer, iterate and direction planes
    int cheb_m;              // 0 / 1: Jacobi only; m >= 2: polynomial of degree m - 1 (precond = 2)
    float cheb_c0, cheb_c1[8], cheb_c2[8];
    float *gersh;            // [1] max_i sum_j |a_ij| / a_ii
    struct FusedCfg : FusedPlan {
        int pat;
        const void *fn, *fn_prof;
    } fused[2];
    int max_smem_optin;
    int refine;              // max restarts from the true residual per solve
    float theta;
    // the graph-mode solver and the stand-alone SpMV launches (ls_pcg_graph.cu)
    struct Graph {
        lsk::SpmmCfg cfg;    // CSR engine
        int spmm_grid;
        int vec_grid;
        int sell_grid;       // spmm_sell_kernel
        int4 *desc;          // CSR engine's block plan (workspace)
        int *desc_cnt;
        int *part;           // ... and its row partition
        int planned;         // the block plan fits
        int sell_tma;        // stand-alone SpMM: TMA-staged variant (0 = register-prefetch kernel)
        int sell_pf;         // ... halo (rows) of its bulk L2 prefetch of the gathered vector, 0 = off
        cudaGraphExec_t exec[KMAX + 1];   // one per K
        cudaStream_t cap_stream;
        int *pinned_done;    // 2 ints, host pinned
        cudaEvent_t ev[2];
    } graph;
    size_t ws_bytes;
    struct Span {
        char *at;
        size_t bytes;
    } zeroed[2];             // workspace regions ls_pcg_create zeroes (carve_handle)
};

// ---- ls_pcg_plan.cu --------------------------------------------------------------------------------------------------
PlanEnv plan_env();
CreateEnv create_env();
// precond = 3 (auto) -> 1 (Jacobi) or 2 (Chebyshev)
int auto_precond(int nslices, int sm_count, int max_smem, const PlanEnv &env);
FusedPlan plan_fused(int nslices, int K, int pat, int cheb, int sm_count, int max_smem, int coop, const PlanEnv &env);
// the fused kernel for (K, RES, NW, PAT, SYNC, PROF, CHEB), or NULL when that combination is not built
const void *fused_fn(int K, int res, int nw, int pat, int sync, int prof, int cheb = 0);

// ---- ls_pcg_copies.cu: the stages of ls_pcg_create that build the matrix copies, in the order it runs them --------------
int copy_matrix(PcgHandle *h, const int *rowptr, const int *col, const float *val, const int *perm, int force_reorder,
                cudaStream_t stream);
int sell_copy(PcgHandle *h, cudaStream_t stream);
// What create needs from the device, brought back in one round trip
struct Readback {
    int flags[2];          // the CSR checks' bits (k_dinv, the permuted copy); the block plan's overflow
    unsigned int mm[2];    // [min, max] of the off-diagonal value bits (equal: a pattern-only matrix)
    float gersh;           // Gershgorin bound of lambda_max(D^-1 A) (precond 2 only)
};
int read_back(PcgHandle *h, const CreateEnv &ce, Readback &rb, cudaStream_t stream);
int build_pattern_copy(PcgHandle *h, unsigned int offc_bits, int share, cudaStream_t stream);
void chebyshev_coefficients(float gersh, int m, float &c0, float (&c1)[8], float (&c2)[8]);
int flag_error(int flags);

// ---- ls_pcg_graph.cu ---------------------------------------------------------------------------------------------------
int graph_geometry(PcgHandle *h, cudaStream_t stream);
// writes x and the 8-float status record to info
int solve_graph(PcgHandle *h, int k, const float *b, float *x, const float *x0, float rtol, int maxit, float *info,
                cudaStream_t stream);
void graph_destroy(PcgHandle::Graph &g);

// ---- ls_pcg.cu -------------------------------------------------------------------------------------------------------
cudaLaunchConfig_t cluster_launch(int grid, int cluster, int threads, size_t smem, cudaStream_t stream, cudaLaunchAttribute *at);
bool cluster_fits(const void *fn, int cluster, int threads, size_t smem, const LsDevInfo &di);
void fused_handle_args(const PcgHandle *h, int nsl_max, lsf::FusedArgs &a);
int finish_info(const float *info, float *info_host, int n, bool batch, float rtol, int maxit, cudaStream_t stream);

}  // namespace lspcg
#pragma GCC visibility pop
