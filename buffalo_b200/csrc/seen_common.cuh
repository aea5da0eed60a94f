// Top-k that leaves out each query's seen items: the pieces shared by the validation top-k of evaluate.cu and the
// seen-aware serving paths of serve.cu.  A "seen" CSR has END offsets (int64) and int32 keys, every row non-decreasing
// (duplicates allowed); seen_row[q] names the row of query q (no seen_row: row q).  Ranking is on one 64-bit key per
// candidate, (~ord(score)) << 32 | position: smaller key = better candidate, so the order is score descending, then
// position ascending, distinct positions have distinct keys, and no score value ever marks a seen item.
#pragma once
#include <cuda_runtime.h>

#include "topk_common.cuh"

namespace bfl {

constexpr unsigned long long SEEN_EMPTY = ~0ull;   // never a rank key: the position half of a key is below 2^31

__device__ __forceinline__ unsigned long long rank_key(float s, int64_t pos) {
    return ((unsigned long long)(~ord_of(s)) << 32) | (unsigned long long)(uint32_t)pos;
}

// the score a rank key was made from, bit for bit
__device__ __forceinline__ float rank_key_score(unsigned long long key) {
    const uint32_t o = ~(uint32_t)(key >> 32);
    return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o);
}

__device__ __forceinline__ int64_t seen_row_begin(const int64_t* __restrict__ indptr, int64_t r) {
    return r > 0 ? indptr[r - 1] : 0;
}

// First position in [lo, hi) of the non-decreasing a[] holding a value >= x.  All 32 lanes of a warp call it.
__device__ inline int64_t warp_lower_bound(const int32_t* __restrict__ a, int64_t lo, int64_t hi, int32_t x, int lane) {
    while (hi - lo > 32) {
        const int64_t step = (hi - lo + 31) / 32;
        const int64_t p = lo + lane * step;
        const int c = __popc(__ballot_sync(FULL, p < hi && a[p] < x));   // probes 0..c-1 are below x
        const int64_t nlo = c == 0 ? lo : lo + (int64_t)(c - 1) * step + 1;
        hi = min(hi, lo + (int64_t)c * step);
        lo = nlo;
    }
    return lo + __popc(__ballot_sync(FULL, lo + lane < hi && a[lo + lane] < x));
}

// Marks in bits[] (bit p = candidate i0 + p) the keys a[lo..hi) of a sorted row, all inside [i0, i0 + slice): one
// thread per key from `first` with stride `stride`; duplicates set the same bit.
__device__ __forceinline__ void mark_seen_range(const int32_t* __restrict__ a, int64_t lo, int64_t hi, int64_t i0,
                                                uint32_t* bits, int first, int stride) {
    for (int64_t e = lo + first; e < hi; e += stride) {
        const int p = a[e] - (int)i0;
        atomicOr(&bits[p >> 5], 1u << (p & 31));
    }
}

// Whether the sorted a[lo..hi) holds x: one thread's binary search (candidates in an arbitrary order, as a pool's).
__device__ __forceinline__ bool row_contains(const int32_t* __restrict__ a, int64_t lo, int64_t hi, int32_t x) {
    const int64_t end = hi;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (a[mid] < x) lo = mid + 1;
        else hi = mid;
    }
    return lo < end && a[lo] == x;
}

struct KeySel {
    unsigned int hist[256];
    unsigned long long prefix;
    unsigned int kk, cnt;
    int stop;
};

// The k smallest of the keys get(0..n) that are not SEEN_EMPTY (n_valid of them, all distinct) -> out[0..min(k, n_valid))
// in no particular order; returns that count.  MSB-first radix select over 8-bit digits, stopping as soon as the
// remaining bin is taken whole.  All threads of the CTA (TK_THREADS) call it.
template <class Get>
__device__ int select_smallest(Get get, int64_t n, int64_t n_valid, int k, unsigned long long* out, KeySel& sc) {
    const int tid = threadIdx.x, lane = tid & 31;
    unsigned long long prefix = 0, mask = 0;
    if (n_valid > k) {
        if (tid == 0) sc.kk = (unsigned)k;
        for (int shift = 56; shift >= 0; shift -= 8) {
            sc.hist[tid] = 0;
            __syncthreads();
            for (int64_t i = tid; i < n; i += TK_THREADS) {
                const unsigned long long key = get(i);
                if (key != SEEN_EMPTY && (key & mask) == prefix) atomicAdd(&sc.hist[(unsigned)(key >> shift) & 255u], 1u);
            }
            __syncthreads();
            if (tid == 0) {
                const unsigned kk = sc.kk;
                unsigned cum = 0;
                int b = 0;
                for (; b < 255; ++b) {
                    if (cum + sc.hist[b] >= kk) break;
                    cum += sc.hist[b];
                }
                sc.kk = kk - cum;
                sc.stop = sc.hist[b] == kk - cum;
                sc.prefix = prefix | ((unsigned long long)b << shift);
            }
            __syncthreads();
            prefix = sc.prefix;
            mask |= 255ull << shift;
            if (sc.stop) break;
        }
    }
    // every key whose digits so far are at most the selected ones: exactly min(k, n_valid) keys
    if (tid == 0) sc.cnt = 0;
    __syncthreads();
    for (int64_t i0 = 0; i0 < n; i0 += TK_THREADS) {
        const int64_t i = i0 + tid;
        const unsigned long long key = i < n ? get(i) : SEEN_EMPTY;
        const bool take = key != SEEN_EMPTY && (key & mask) <= prefix;
        const unsigned bal = __ballot_sync(FULL, take);
        unsigned base = 0;
        if (lane == 0 && bal) base = atomicAdd(&sc.cnt, (unsigned)__popc(bal));
        base = __shfl_sync(FULL, base, 0);
        if (take) out[base + __popc(bal & ((1u << lane) - 1u))] = key;
    }
    __syncthreads();
    return n_valid > k ? k : (int)n_valid;
}

// Stream-ordered, implemented in evaluate.cu.
// masked_topk: per query q, the k best of the n_items candidate rows (scores of bfl_topk_device for the same
// arguments) outside seen row seen_row[q]; candidate c is item pool[c] when a pool is given (the rows of `items` are
// then the pool's rows, gathered), else item c.  out_idx [nq x k] candidate positions best first, -1 pads;
// out_val [nq x k] (nullable) their scores, 0 on the padding.
int masked_topk(const float* queries, int64_t nq, int ldq, const float* items, int64_t n_items, int ldi,
                const float* item_bias, int d, int k, const int64_t* seen_indptr, const int32_t* seen_keys,
                const int32_t* seen_row, const int32_t* pool, int32_t* out_idx, float* out_val, cudaStream_t st);
// seen_merge: per query, the k best of its nslices lists of rank keys (list s holds cand_cnt[q * nslices + s] keys
// at cand + (q * nslices + s) * k) -> out_idx / out_val as masked_topk.
int seen_merge(const unsigned long long* cand, const int32_t* cand_cnt, int64_t nq, int nslices, int k,
               int32_t* out_idx, float* out_val, cudaStream_t st);

}  // namespace bfl
