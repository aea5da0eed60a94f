// Pieces shared by the top-k kernels of topk.cu and the masked validation top-k of evaluate.cu: the order-preserving
// float key and the per-slice scoring loop.  Both kernels score through topk_score_slice, so a score depends only on
// (query row, item row, bias, d, ldq, ldi) and is bitwise the same in either kernel, whatever number of queries a CTA
// blocks together.
#pragma once
#include "bfl_common.cuh"

namespace bfl {

constexpr int TK_THREADS = 256;
constexpr int TK_SLICE = 4096;
constexpr int TK_KMAX = 4096;

__device__ __forceinline__ uint32_t ord_of(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);   // larger float <=> larger unsigned
}

// Loads QB query rows (zero-padded to dpad = ceil4(d)) into qv, then scores[qi * TK_SLICE + it] = q_qi . item(i0 + it)
// (+ bias) for it < ni.  One warp per item row: every lane sums its columns with fmaf, then a butterfly warp sum.
// All threads of the CTA call it; it ends with __syncthreads().
template <int QB>
__device__ __forceinline__ void topk_score_slice(const float* __restrict__ Qr, int64_t q0, int nqb, int ldq,
                                                 const float* __restrict__ It, int64_t i0, int ni, int ldi,
                                                 const float* __restrict__ bias, int d, float* qv, float* scores) {
    const int dpad = (d + 3) & ~3;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    for (int e = tid; e < QB * dpad; e += TK_THREADS) {
        const int qi = e / dpad, c = e - qi * dpad;
        qv[e] = (qi < nqb && c < d) ? Qr[(q0 + qi) * ldq + c] : 0.f;
    }
    __syncthreads();
    const bool vec = (ldi & 3) == 0 && (d & 3) == 0;
    for (int it = w; it < ni; it += TK_THREADS / 32) {
        const float* row = It + (i0 + it) * ldi;
        float acc[QB];
#pragma unroll
        for (int qi = 0; qi < QB; ++qi) acc[qi] = 0.f;
        if (vec) {
            for (int c = lane * 4; c < d; c += 128) {
                const float4 v = __ldg(reinterpret_cast<const float4*>(row + c));
#pragma unroll
                for (int qi = 0; qi < QB; ++qi) {
                    const float4 x = *reinterpret_cast<const float4*>(qv + qi * dpad + c);
                    acc[qi] = fmaf(v.x, x.x, fmaf(v.y, x.y, fmaf(v.z, x.z, fmaf(v.w, x.w, acc[qi]))));
                }
            }
        } else {
            for (int c = lane; c < d; c += 32) {
                const float v = __ldg(row + c);
#pragma unroll
                for (int qi = 0; qi < QB; ++qi) acc[qi] = fmaf(v, qv[qi * dpad + c], acc[qi]);
            }
        }
#pragma unroll
        for (int qi = 0; qi < QB; ++qi) acc[qi] = warp_sum(acc[qi]);
        if (lane == 0) {
            const float b = bias ? bias[i0 + it] : 0.f;
#pragma unroll
            for (int qi = 0; qi < QB; ++qi) scores[qi * TK_SLICE + it] = acc[qi] + b;
        }
    }
    __syncthreads();
}

// topk.cu: per query, the k best of its ncand candidates (score, index; index -1 = empty) ordered best first, ties to
// the smaller index, into out_idx / out_val [nq x k] (-1 / -inf where fewer than k candidates exist).  Stream-ordered.
int topk_merge(const float* cand_v, const int32_t* cand_i, int64_t nq, int ncand, int k, int32_t* out_idx, float* out_val,
               cudaStream_t st);

}  // namespace bfl
