// The Gram triangle of a short list of item rows in shared memory, shared by the intra-list diversity of offline_eval.cu
// (DESIGN.md 4.14) and the MMR re-ranking of rerank.cu (DESIGN.md 4.15), so that ild@K and the reranker measure the
// same cosine.  Everything is in an unnamed namespace: each translation unit compiles its own copy.
#pragma once
#include <cstdint>

namespace {

constexpr int GRAM_TD = 32;            // Gram tile: columns of d per pass
constexpr int GRAM_TDS = GRAM_TD + 4;  // its row stride in floats: rows stay 16-byte aligned, thread b's reads of row b
                                       // spread over 8 banks

// G[b * (b + 1) / 2 + a] (a <= b < kmax) = the fp32 dot product of the first d columns of rows item[a] and item[b] of
// `items` (pitch ld); an entry item[x] < 0 reads as a zero row.  The CTA has at least kmax threads.  item[], tile
// ([kmax][GRAM_TDS] floats, 16-byte aligned) and G (kmax (kmax + 1) / 2 floats) are shared memory; item[] may be
// written just before the call, the first barrier publishes it.  Thread b owns column b of the triangle: every tile
// adds its GRAM_TD products to G[a, b] for a = 0..b in that order, so each dot product has one fixed order.  Returns
// after a barrier, with G complete.
__device__ __forceinline__ void gram_triangle(const int32_t* item, int kmax, const float* __restrict__ items, int ld,
                                              int d, float* tile, float* G) {
    const int tid = threadIdx.x, nt = blockDim.x;
    for (int p = tid; p < kmax * (kmax + 1) / 2; p += nt) G[p] = 0.f;
    __syncthreads();
    const int b = tid;
    const size_t gb = (size_t)b * (b + 1) / 2;
    for (int d0 = 0; d0 < d; d0 += GRAM_TD) {
        for (int e = tid; e < kmax * GRAM_TD; e += nt) {
            const int a = e / GRAM_TD, t = e - a * GRAM_TD;
            const int32_t it = item[a];
            tile[a * GRAM_TDS + t] = it >= 0 && d0 + t < d ? items[(int64_t)it * ld + d0 + t] : 0.f;
        }
        __syncthreads();
        if (b < kmax) {
            float xb[GRAM_TD];
#pragma unroll
            for (int t = 0; t < GRAM_TD; ++t) xb[t] = tile[b * GRAM_TDS + t];
            for (int a = 0; a <= b; ++a) {
                const float4* xa = reinterpret_cast<const float4*>(tile + a * GRAM_TDS);
                float acc = 0.f;
#pragma unroll
                for (int t = 0; t < GRAM_TD / 4; ++t) {
                    const float4 v = xa[t];
                    acc = fmaf(v.x, xb[4 * t], acc);
                    acc = fmaf(v.y, xb[4 * t + 1], acc);
                    acc = fmaf(v.z, xb[4 * t + 2], acc);
                    acc = fmaf(v.w, xb[4 * t + 3], acc);
                }
                G[gb + a] += acc;
            }
        }
        __syncthreads();
    }
}

// cos(a, b) of two entries of the triangle in fp64 (either order): 0 when either row has zero norm
__device__ __forceinline__ double gram_cos(const float* G, int a, int b) {
    const int lo = a < b ? a : b, hi = a < b ? b : a;
    const double na = (double)G[(size_t)lo * (lo + 1) / 2 + lo], nb = (double)G[(size_t)hi * (hi + 1) / 2 + hi];
    return na > 0.0 && nb > 0.0 ? (double)G[(size_t)hi * (hi + 1) / 2 + lo] / sqrt(na * nb) : 0.0;
}

__host__ __device__ constexpr size_t gram_tile_floats(int kmax) { return (size_t)kmax * GRAM_TDS; }
__host__ __device__ constexpr size_t gram_triangle_floats(int kmax) { return (size_t)kmax * (kmax + 1) / 2; }

}  // namespace
