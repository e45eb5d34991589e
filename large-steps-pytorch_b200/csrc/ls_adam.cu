// ls_adam.cu -- fused AdamUniform step (sm_90a).  Replaces largesteps/optimize.py:17-41 (8 eager torch kernels
// + a max reduction per parameter): two streaming passes over (param, grad, g1, g2).
//   pass 1: g1 = b1 g1 + (1-b1) g ; g2 = b2 g2 + (1-b2) g^2 ; gmax = max(g2)        (optimize.py:35-36)
//   pass 2: p -= lr * (g1/c1) / (1e-8 + sqrt(gmax/c2))                                 (optimize.py:37-41)
// max(sqrt(g2/c2)) == sqrt(max(g2)/c2) in fp32 (both maps are monotone), so the scalar normaliser of optimize.py:40 is
// reproduced to the last bit or one ulp (torch divides by a Python scalar as multiply-by-reciprocal; here it is a division);
// the max itself is order independent (deterministic).  A NaN in the moments makes the normaliser NaN, as torch's max() does:
// divergence poisons every parameter and is visible, instead of being dropped by fmaxf.
// ls_adam_uniform_step_multi runs the same two passes for many tensors per launch, each with its own normaliser.
#include "ls_common.cuh"

namespace {
constexpr int AT = 256;

// ---- one launch per pass for a table of tensors (ls_adam_uniform_step is a table of one) ---------------------------------
// Block b works on tensor t with blk[t] <= b < blk[t+1], chunk b - blk[t] of blk[t+1] - blk[t] (a grid-stride loop over that
// tensor alone, at most sm_count * 8 blocks), so small and large tensors share one grid.  Each tensor keeps its own [max g2
// bits, NaN flag] pair in scratch, and a max does not depend on the partition, so every tensor's result is bitwise that of
// a call on it alone.  The table is a kernel parameter, and the launch cost grows with it (20 KB at CAP 256): a call with few
// tensors uses the small table (CAP 16, 1.3 KB), and ls_adam_uniform_step a table of one.
template <int CAP>
struct AdamTable {
    int blk[CAP + 1];                  // prefix of per-tensor block counts
    ls_adam_tensor t[CAP];
};
constexpr int ADAM_SMALL_TABLE = 16;
static_assert(sizeof(AdamTable<LS_ADAM_MULTI_MAX>) + 16 <= 32764, "kernel parameter space of sm_90 (CUDA >= 12.1)");

template <int CAP>
__device__ __forceinline__ int table_slot(const AdamTable<CAP> &tab, int n, int b) {
    int lo = 0, hi = n - 1;                      // the last slot with blk[slot] <= b
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (tab.blk[mid] <= b) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// The kernels copy their tensor's size out of the table before the loop, and read grad through __ldg: nvcc cannot tell that
// the loop's stores leave the table alone, nor that grad is read-only, and without these the two passes took 8 % longer.
template <int CAP>
__global__ void __launch_bounds__(AT) k_adam_moments_multi(const __grid_constant__ AdamTable<CAP> tab, int n,
                                                           unsigned int *__restrict__ gmax_bits) {
    const int s = table_slot(tab, n, blockIdx.x);
    const ls_adam_tensor &e = tab.t[s];
    const int64_t nb = tab.blk[s + 1] - tab.blk[s], b0 = (int64_t)blockIdx.x - tab.blk[s], ne = e.n;
    const float *__restrict__ grad = e.grad;
    float *__restrict__ g1 = e.g1;
    float *__restrict__ g2 = e.g2;
    const float b1 = e.beta1, b2 = e.beta2, omb1 = e.one_minus_beta1, omb2 = e.one_minus_beta2;
    float m = 0.f;
    bool nan_seen = false;
    for (int64_t i = b0 * blockDim.x + threadIdx.x; i < ne; i += nb * blockDim.x) {
        const float g = __ldg(grad + i);
        // g1.mul_(b1).add_(grad, alpha=1-b1): the in-place mul rounds, torch's CUDA add(alpha) contracts to an fma
        const float a = fmaf(omb1, g, __fmul_rn(g1[i], b1));
        const float b = fmaf(omb2, __fmul_rn(g, g), __fmul_rn(g2[i], b2));
        g1[i] = a;
        g2[i] = b;
        m = fmaxf(m, b);
        nan_seen |= (b != b);
    }
    unsigned int *slot = gmax_bits + 2 * s;
    if (__any_sync(0xffffffffu, nan_seen) && (threadIdx.x & 31) == 0) atomicOr(slot + 1, 1u);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    __shared__ float wm[AT / 32];
    if ((threadIdx.x & 31) == 0) wm[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x < 32) {
        float v = threadIdx.x < AT / 32 ? wm[threadIdx.x] : 0.f;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
        if (threadIdx.x == 0) atomicMax(slot, __float_as_uint(v));   // g2 >= 0: uint order == float order
    }
}

template <int CAP>
__global__ void __launch_bounds__(AT) k_adam_apply_multi(const __grid_constant__ AdamTable<CAP> tab, int n,
                                                         const unsigned int *__restrict__ gmax_bits) {
    const int s = table_slot(tab, n, blockIdx.x);
    const ls_adam_tensor &e = tab.t[s];
    const int64_t nb = tab.blk[s + 1] - tab.blk[s], b0 = (int64_t)blockIdx.x - tab.blk[s], ne = e.n;
    const unsigned int *slot = gmax_bits + 2 * s;
    const float gmax = slot[1] ? __int_as_float(0x7fc00000) : __uint_as_float(*slot);
    const float denom = __fadd_rn(1e-8f, __fsqrt_rn(__fdiv_rn(gmax, e.c2)));   // 1e-8 + m2.sqrt().max()
    float *__restrict__ param = e.param;
    const float *__restrict__ g1 = e.g1;
    const float lr = e.lr, c1 = e.c1;
    for (int64_t i = b0 * blockDim.x + threadIdx.x; i < ne; i += nb * blockDim.x) {
        const float m1 = __fdiv_rn(g1[i], c1);
        const float gr = __fdiv_rn(m1, denom);
        param[i] = fmaf(-lr, gr, param[i]);                                  // p.data.sub_(gr, alpha=lr)
    }
}

// tensors [0, m) of one table (m <= CAP): both passes
template <int CAP>
int adam_multi_launch(const ls_adam_tensor *tensors, int m, int64_t cap, unsigned int *bits, cudaStream_t stream) {
    AdamTable<CAP> tab;
    int64_t blocks = 0;
    for (int i = 0; i < m; ++i) {
        tab.t[i] = tensors[i];
        int64_t g = (tab.t[i].n + AT - 1) / AT;
        if (g > cap) g = cap;
        tab.blk[i] = (int)blocks;
        blocks += g;
    }
    tab.blk[m] = (int)blocks;
    if (blocks == 0) return LS_OK;                         // only empty tensors in this part of the table
    k_adam_moments_multi<CAP><<<(unsigned)blocks, AT, 0, stream>>>(tab, m, bits);
    LS_LAUNCH_CHECK();
    k_adam_apply_multi<CAP><<<(unsigned)blocks, AT, 0, stream>>>(tab, m, bits);
    LS_LAUNCH_CHECK();
    return LS_OK;
}
}  // namespace

extern "C" int ls_adam_uniform_step(float *param, const float *grad, float *g1, float *g2, int64_t n, float lr,
                                    float beta1, float beta2, float one_minus_beta1, float one_minus_beta2, float c1,
                                    float c2, void *scratch, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    LS_REQUIRE(n >= 0, "negative size");
    if (n == 0) return LS_OK;
    LS_REQUIRE(param && grad && g1 && g2 && scratch, "NULL pointer");
    LsDevInfo di;
    int rc = ls_dev_info(&di);
    if (rc) return rc;
    const ls_adam_tensor t = {param, grad, g1, g2, n, lr, beta1, beta2, one_minus_beta1, one_minus_beta2, c1, c2};
    LS_CUDA_TRY(cudaMemsetAsync(scratch, 0, 16, stream));
    return adam_multi_launch<1>(&t, 1, (int64_t)di.sm_count * 8, (unsigned int *)scratch, stream);
}

extern "C" int ls_adam_uniform_step_multi(const ls_adam_tensor *tensors, int n, void *scratch, size_t scratch_bytes,
                                          void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    LS_REQUIRE(n >= 0, "negative tensor count");
    if (n == 0) return LS_OK;
    LS_REQUIRE(tensors && scratch, "NULL pointer");
    LS_REQUIRE(scratch_bytes >= (size_t)8 * n, "scratch smaller than 8 n bytes");
    for (int i = 0; i < n; ++i) {
        const ls_adam_tensor &e = tensors[i];
        LS_REQUIRE(e.n >= 0, "negative size");
        LS_REQUIRE(e.n == 0 || (e.param && e.grad && e.g1 && e.g2), "NULL tensor pointer");
    }
    LsDevInfo di;
    int rc = ls_dev_info(&di);
    if (rc) return rc;
    const int64_t cap = (int64_t)di.sm_count * 8;          // grid cap per tensor
    LS_CUDA_TRY(cudaMemsetAsync(scratch, 0, (size_t)8 * n, stream));
    for (int base = 0; base < n; base += LS_ADAM_MULTI_MAX) {
        const int m = n - base < LS_ADAM_MULTI_MAX ? n - base : LS_ADAM_MULTI_MAX;
        unsigned int *bits = (unsigned int *)scratch + 2 * base;
        rc = m <= ADAM_SMALL_TABLE ? adam_multi_launch<ADAM_SMALL_TABLE>(tensors + base, m, cap, bits, stream)
                                   : adam_multi_launch<LS_ADAM_MULTI_MAX>(tensors + base, m, cap, bits, stream);
        if (rc) return rc;
    }
    return LS_OK;
}
