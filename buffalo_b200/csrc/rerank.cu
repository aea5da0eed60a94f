// Maximal Marginal Relevance re-ranking of candidate lists (DESIGN.md 4.15): the device path of ParALS / ParBPRMF
// topk_recommendation(diversify=w) and buffalo_b200.parallel.rerank_mmr.  Per row, from its m candidates c_j with
// scores s_j (-1 pads), k of them are picked greedily: at step t the unpicked valid candidate of the largest
//   obj_j = (1 - w) rel_j - w maxsim_j      (the maxsim term left out at t = 0)
// with rel_j = (s_j - s_min) / (s_max - s_min) over the row's valid candidates (1 when they are all equal) and maxsim_j
// the largest cosine of item c_j to the items picked so far, ties to the smaller position.  Every cosine is the one of
// oe_ild_kernel (the same Gram triangle builder, gram_common.cuh), so ild@K and the reranker measure the same thing.
//   mmr_rerank_kernel: one CTA per row, thread j owns candidate j (m <= 256).  The Gram triangle of the row's item rows
//                      is built in shared memory; each step is a block argmax over (obj, position): a warp butterfly,
//                      then the per-warp winners through shared memory (double-buffered, one barrier per step).
// A row's output depends on that row alone.  No atomics, no global scratch.
#include <algorithm>

#include "gram_common.cuh"
#include "serve_common.cuh"

using namespace bfl;

namespace {

constexpr int MMR_MMAX = 256;
constexpr int MMR_WARPS = MMR_MMAX / 32;

// (obj, pos) beats (o2, p2): larger objective, ties to the smaller position
__device__ __forceinline__ void mmr_better(double& obj, int& pos, double o2, int p2) {
    if (o2 > obj || (o2 == obj && p2 < pos)) {
        obj = o2;
        pos = p2;
    }
}

// Shared memory: the Gram tile [m][GRAM_TDS] (first: its rows are read as float4), per-warp reduction slots (the score
// range, then two buffers of step winners), the row's items and the Gram triangle.
__global__ void __launch_bounds__(MMR_MMAX) mmr_rerank_kernel(const int32_t* __restrict__ cand_idx,
                                                              const float* __restrict__ cand_val, int m, int k, double w,
                                                              const float* __restrict__ items, int ld, int d,
                                                              int32_t* __restrict__ out_idx,
                                                              float* __restrict__ out_val) {
    extern __shared__ __align__(16) unsigned char mmr_smem[];
    float* tile = reinterpret_cast<float*>(mmr_smem);                              // [m][GRAM_TDS]
    double* red_lo = reinterpret_cast<double*>(tile + gram_tile_floats(m));        // [MMR_WARPS]
    double* red_hi = red_lo + MMR_WARPS;                                           // [MMR_WARPS]
    double* red_obj = red_hi + MMR_WARPS;                                          // [2][MMR_WARPS]
    int* red_pos = reinterpret_cast<int*>(red_obj + 2 * MMR_WARPS);                // [2][MMR_WARPS]
    int32_t* item = red_pos + 2 * MMR_WARPS;                                       // [m]
    float* G = reinterpret_cast<float*>(item + m);                                 // [m (m + 1) / 2]
    const int j = threadIdx.x, lane = j & 31, warp = j >> 5, nw = blockDim.x >> 5;
    const int64_t r = blockIdx.x;
    const int32_t c = j < m ? cand_idx[r * m + j] : -1;
    const float s = c >= 0 ? cand_val[r * m + j] : 0.f;
    if (j < m) item[j] = c;
    // the row's score range (min / max are exact, so any order gives the same pair)
    double lo = c >= 0 ? (double)s : INFINITY, hi = c >= 0 ? (double)s : -INFINITY;
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        lo = fmin(lo, __shfl_xor_sync(FULL, lo, o));
        hi = fmax(hi, __shfl_xor_sync(FULL, hi, o));
    }
    if (lane == 0) {
        red_lo[warp] = lo;
        red_hi[warp] = hi;
    }
    gram_triangle(item, m, items, ld, d, tile, G);   // its barriers publish item[] and the score range too
    for (int i = 0; i < nw; ++i) {
        lo = fmin(lo, red_lo[i]);
        hi = fmax(hi, red_hi[i]);
    }
    const double rel = hi > lo ? ((double)s - lo) / (hi - lo) : 1.0;
    const double a = 1.0 - w;
    double maxsim = -INFINITY;
    bool live = c >= 0;
    int32_t* oi = out_idx + r * k;
    float* ov = out_val + r * k;
    for (int t = 0; t < k; ++t) {
        // a live candidate's objective is finite, so -inf marks "nothing left"
        double obj = live ? (t == 0 ? a * rel : a * rel - w * maxsim) : -INFINITY;
        int pos = j;
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            const double o2 = __shfl_xor_sync(FULL, obj, o);
            const int p2 = __shfl_xor_sync(FULL, pos, o);
            mmr_better(obj, pos, o2, p2);
        }
        double* ro = red_obj + (t & 1) * MMR_WARPS;
        int* rp = red_pos + (t & 1) * MMR_WARPS;
        if (lane == 0) {
            ro[warp] = obj;
            rp[warp] = pos;
        }
        __syncthreads();   // the other buffer was last read before this barrier's previous use
        obj = ro[0];
        pos = rp[0];
        for (int i = 1; i < nw; ++i) mmr_better(obj, pos, ro[i], rp[i]);
        if (obj == -INFINITY) {   // the same decision in every thread
            for (int u = t + j; u < k; u += blockDim.x) {
                oi[u] = -1;
                ov[u] = 0.f;
            }
            return;
        }
        if (j == pos) {
            oi[t] = c;
            ov[t] = s;
            live = false;
        }
        if (live) maxsim = fmax(maxsim, gram_cos(G, pos, j));
    }
}

size_t mmr_smem_bytes(int m) {
    static_assert((sizeof(float) * GRAM_TDS) % 16 == 0, "tile rows must keep float4 alignment");
    return sizeof(float) * gram_tile_floats(m) + sizeof(double) * 4 * MMR_WARPS + sizeof(int) * 2 * MMR_WARPS +
           sizeof(int32_t) * m + sizeof(float) * gram_triangle_floats(m);
}

}  // namespace

namespace bfl {

int mmr_rerank(const float* items, int ld, int d, const int32_t* cand_idx, const float* cand_val, int64_t n, int m,
               int k, float diversify, int32_t* out_idx, float* out_val, cudaStream_t st) {
    if (n == 0) return BFL_OK;
    const size_t smem = mmr_smem_bytes(m);
    BFL_CUDA(cudaFuncSetAttribute(mmr_rerank_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int threads = std::max(32, (m + 31) / 32 * 32);
    mmr_rerank_kernel<<<(unsigned)n, threads, smem, st>>>(cand_idx, cand_val, m, k, (double)diversify, items, ld, d,
                                                         out_idx, out_val);
    BFL_LAUNCHED();
    return BFL_OK;
}

}  // namespace bfl
