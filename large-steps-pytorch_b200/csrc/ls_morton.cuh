// ls_morton.cuh -- the Morton cell code of a point set's bounding-box grid, and the segment of an item in a packed batch
// (device helpers; ls_order.cu, ls_distance.cu).
#pragma once
#include "ls_common.cuh"

__device__ __forceinline__ unsigned int f2ord(float f) {   // order-preserving float -> uint
    unsigned int u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned int u) {
    return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

__device__ __forceinline__ unsigned int spread3(unsigned int x) {   // 10 bits -> every third bit
    x &= 0x3ffu;
    x = (x | (x << 16)) & 0x030000ffu;
    x = (x | (x << 8)) & 0x0300f00fu;
    x = (x | (x << 4)) & 0x030c30c3u;
    x = (x | (x << 2)) & 0x09249249u;
    return x;
}

// the cell of point i in the grid of 2^bits cells per axis over the box [lo, hi] (three f2ord-encoded coordinates each)
__device__ __forceinline__ unsigned int cell_code(const float *__restrict__ verts, int64_t i, const unsigned int *__restrict__ mlo,
                                                  const unsigned int *__restrict__ mhi, int bits) {
    float lo[3], ext = 0.f;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        lo[d] = ord2f(mlo[d]);
        ext = fmaxf(ext, ord2f(mhi[d]) - lo[d]);
    }
    const float scale = (ext > 0.f) ? (float)(1 << bits) / ext : 0.f;
    unsigned int q[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        float x = verts[3 * i + d];
        float t = (x == x) ? (x - lo[d]) * scale : 0.f;
        int c = (int)t;
        c = max(0, min((1 << bits) - 1, c));
        q[d] = (unsigned int)c;
    }
    return spread3(q[0]) | (spread3(q[1]) << 1) | (spread3(q[2]) << 2);
}

// The segment of item x in a packed batch of B segments: the largest b < B with off[b] - b * shift <= x (shift 1 for the
// internal nodes of a BVH forest, whose mesh b holds off[b + 1] - off[b] - 1 of them).  B == 1 reads nothing.
__device__ __forceinline__ int ls_segment_of(const int64_t *__restrict__ off, int B, int64_t x, int shift) {
    int lo = 0, hi = B;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (off[mid] - (int64_t)mid * shift <= x) lo = mid;
        else hi = mid;
    }
    return lo;
}
