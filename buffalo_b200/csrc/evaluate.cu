// Validation metrics on the device (DESIGN.md 4.8): the path behind Evaluable.get_validation_results for dot-product
// models (buffalo/evaluate/base.py:44-148 in the reference).
//   eval_slice_kernel      : a CTA scores EV_QB users against a slice of TK_SLICE items with topk.cu's scoring loop,
//                            drops the items of each user's sorted training row that fall in the slice (found by a
//                            warp binary search, marked in a shared bitmask), and keeps the k best of the rest;
//   eval_merge_kernel      : per user, the k best of the slices' candidates, ordered;
//   eval_rank_terms_kernel : per user, hits against the held-out row, DCG, AP, accuracy and AUC in fp64;
//   eval_score_terms_kernel: per held-out triple, the model's score with NumPy's float32 arithmetic and its error;
//   eval_sum_*_kernel      : column sums of per-row terms in a fixed order (bitwise repeatable).
// Ranking is on the 64-bit rank keys of seen_common.cuh, so selection needs no tie rule and no score is ever used as a
// marker.  masked_topk (a pool, scores out) and seen_merge also serve the seen-aware calls of serve.cu.
#include "seen_common.cuh"

using namespace bfl;

namespace {

constexpr int EV_QB = 4;
constexpr unsigned long long EV_EMPTY = SEEN_EMPTY;
constexpr int EV_SUM_BLOCKS = 128;
constexpr int EV_SUM_WIDTH = 8;

__global__ void __launch_bounds__(TK_THREADS) eval_slice_kernel(
    const float* __restrict__ Qr, int64_t nq, int ldq, const float* __restrict__ It, int64_t n_items, int ldi,
    const float* __restrict__ bias, int d, int k, int nslices, const int64_t* __restrict__ seen_indptr,
    const int32_t* __restrict__ seen_keys, const int32_t* __restrict__ seen_row, const int32_t* __restrict__ pool,
    unsigned long long* __restrict__ cand, int32_t* __restrict__ cand_cnt) {
    extern __shared__ __align__(16) unsigned char ev_smem[];
    unsigned long long* keys = reinterpret_cast<unsigned long long*>(ev_smem);   // [TK_SLICE]
    float* scores = reinterpret_cast<float*>(keys + TK_SLICE);                    // [EV_QB][TK_SLICE]
    float* qv = scores + EV_QB * TK_SLICE;                                         // [EV_QB][dpad]
    __shared__ uint32_t seen_bits[TK_SLICE / 32];
    __shared__ int64_t seen_lo[EV_QB], seen_hi[EV_QB];
    __shared__ KeySel sc;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int64_t q0 = (int64_t)blockIdx.x * EV_QB;
    const int nqb = (int)min((long long)EV_QB, (long long)(nq - q0));
    const int slice = blockIdx.y;
    const int64_t i0 = (int64_t)slice * TK_SLICE;
    const int ni = (int)min((long long)TK_SLICE, (long long)(n_items - i0));
    if (w < nqb) {   // the user's seen items inside [i0, i0 + ni); with a pool, the whole row
        const int64_t r = seen_row ? seen_row[q0 + w] : q0 + w;
        const int64_t b = seen_row_begin(seen_indptr, r), e = seen_indptr[r];
        const int64_t lo = pool ? b : warp_lower_bound(seen_keys, b, e, (int32_t)i0, lane);
        const int64_t hi = pool ? e : warp_lower_bound(seen_keys, lo, e, (int32_t)(i0 + ni), lane);
        if (lane == 0) {
            seen_lo[w] = lo;
            seen_hi[w] = hi;
        }
    }
    topk_score_slice<EV_QB>(Qr, q0, nqb, ldq, It, i0, ni, ldi, bias, d, qv, scores);   // ends with __syncthreads
    for (int qi = 0; qi < nqb; ++qi) {
        for (int j = tid; j < TK_SLICE / 32; j += TK_THREADS) seen_bits[j] = 0;
        if (tid == 0) sc.cnt = 0;
        __syncthreads();
        if (!pool) {
            mark_seen_range(seen_keys, seen_lo[qi], seen_hi[qi], i0, seen_bits, tid, TK_THREADS);
        } else if (seen_hi[qi] > seen_lo[qi]) {   // candidate it is item pool[i0 + it], pool order is arbitrary
            for (int it = tid; it < ni; it += TK_THREADS)
                if (row_contains(seen_keys, seen_lo[qi], seen_hi[qi], pool[i0 + it]))
                    atomicOr(&seen_bits[it >> 5], 1u << (it & 31));
        }
        __syncthreads();
        for (int it0 = 0; it0 < ni; it0 += TK_THREADS) {
            const int it = it0 + tid;
            const bool keep = it < ni && !((seen_bits[it >> 5] >> (it & 31)) & 1u);
            const unsigned bal = __ballot_sync(FULL, keep);
            unsigned base = 0;
            if (lane == 0 && bal) base = atomicAdd(&sc.cnt, (unsigned)__popc(bal));
            base = __shfl_sync(FULL, base, 0);
            if (keep) keys[base + __popc(bal & ((1u << lane) - 1u))] = rank_key(scores[qi * TK_SLICE + it], i0 + it);
        }
        __syncthreads();
        const int n_unseen = (int)sc.cnt;
        __syncthreads();
        const size_t o = (size_t)(q0 + qi) * nslices + slice;
        const int got = select_smallest([&](int64_t i) { return keys[i]; }, n_unseen, n_unseen, k, cand + o * k, sc);
        if (tid == 0) cand_cnt[o] = got;
    }
}

__global__ void __launch_bounds__(TK_THREADS) eval_merge_kernel(const unsigned long long* __restrict__ cand,
                                                                const int32_t* __restrict__ cand_cnt, int nslices,
                                                                int k, int kpad, int32_t* __restrict__ out_idx,
                                                                float* __restrict__ out_val) {
    extern __shared__ __align__(16) unsigned long long ev_sorted[];   // [kpad]
    __shared__ KeySel sc;
    __shared__ long long part[TK_THREADS / 32];
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const size_t q = blockIdx.x;
    const unsigned long long* cq = cand + q * (size_t)nslices * k;
    const int32_t* cnt = cand_cnt + q * nslices;
    long long nv = 0;
    for (int s = tid; s < nslices; s += TK_THREADS) nv += cnt[s];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nv += __shfl_xor_sync(FULL, nv, o);
    if (lane == 0) part[w] = nv;
    __syncthreads();
    long long n_valid = 0;
#pragma unroll
    for (int i = 0; i < TK_THREADS / 32; ++i) n_valid += part[i];
    const int got = select_smallest(
        [&](int64_t i) {
            const int64_t s = i / k;
            return (i - s * k) < cnt[s] ? cq[i] : EV_EMPTY;
        },
        (int64_t)nslices * k, n_valid, k, ev_sorted, sc);
    for (int i = got + tid; i < kpad; i += TK_THREADS) ev_sorted[i] = EV_EMPTY;
    __syncthreads();
    for (int size = 2; size <= kpad; size <<= 1) {
        for (int strd = size >> 1; strd > 0; strd >>= 1) {
            for (int i = tid; i < kpad / 2; i += TK_THREADS) {
                const int lo = 2 * i - (i & (strd - 1)), hi = lo + strd;
                const bool up = (lo & size) == 0;
                const unsigned long long a = ev_sorted[lo], b = ev_sorted[hi];
                if ((a > b) == up) {
                    ev_sorted[lo] = b;
                    ev_sorted[hi] = a;
                }
            }
            __syncthreads();
        }
    }
    for (int i = tid; i < k; i += TK_THREADS) {
        out_idx[q * k + i] = i < got ? (int32_t)(uint32_t)(ev_sorted[i] & 0xffffffffull) : -1;
        if (out_val) out_val[q * k + i] = i < got ? rank_key_score(ev_sorted[i]) : 0.f;
    }
}

__global__ void eval_unsorted_rows_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ keys,
                                          int64_t rows, unsigned long long* __restrict__ count) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < rows; r += warps) {
        const int64_t b = r > 0 ? indptr[r - 1] : 0, e = indptr[r];
        bool bad = false;
        for (int64_t i = b + 1 + lane; i < e; i += 32) bad |= keys[i] < keys[i - 1];
        if (__any_sync(FULL, bad) && lane == 0) atomicAdd(count, 1ull);
    }
}

// One thread per evaluated row: the per-row terms of buffalo_b200/evaluate/base.py's host loop.
// terms[r] = (ndcg, ap / min(n_pos, topk), accuracy, auc, 1 if the row counts, 1 if it has no negative item).
__global__ void eval_rank_terms_kernel(const int32_t* __restrict__ ranked, int64_t nq, int k,
                                       const int32_t* __restrict__ users, const int64_t* __restrict__ seen_indptr,
                                       const int32_t* __restrict__ seen_row, const int64_t* __restrict__ gt_indptr,
                                       const int32_t* __restrict__ gt_keys, const double* __restrict__ gains,
                                       const double* __restrict__ ideal, int64_t num_items, double* __restrict__ terms) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nq) return;
    double* t = terms + r * 6;
    const int64_t sr = seen_row[r];
    if (seen_indptr[sr] == (sr > 0 ? seen_indptr[sr - 1] : 0)) {   // no training items: skipped, like the host
        for (int c = 0; c < 6; ++c) t[c] = 0.0;
        return;
    }
    const int64_t u = users[r];
    const int64_t g0 = u > 0 ? gt_indptr[u - 1] : 0, g1 = gt_indptr[u];
    int64_t n_pos = 0;   // distinct held-out items (the host's set)
    for (int64_t e = g0; e < g1; ++e) n_pos += (e == g0 || gt_keys[e] != gt_keys[e - 1]) ? 1 : 0;
    double cum = 0.0, dcg = 0.0, ap = 0.0, auc_sum = 0.0, miss = 0.0;
    int len = 0;
    const int32_t* rk = ranked + r * k;
    for (int j = 0; j < k; ++j) {
        const int32_t item = rk[j];
        if (item < 0) break;
        int64_t lo = g0, hi = g1;
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (gt_keys[mid] < item) lo = mid + 1;
            else hi = mid;
        }
        const double h = (lo < g1 && gt_keys[lo] == item) ? 1.0 : 0.0;
        cum += h;
        dcg += h * gains[j];
        ap += h * cum / (double)(j + 1);
        auc_sum += (1.0 - h) * cum;
        miss += 1.0 - h;
        ++len;
    }
    const int64_t n_neg = num_items - n_pos;
    const double auc = auc_sum + ((len ? cum : 0.0) + (double)n_pos) / 2.0 * ((double)n_neg - miss);
    const int64_t m = n_pos < k ? n_pos : k;
    t[0] = dcg / ideal[m - 1];
    t[1] = ap / (double)m;
    t[2] = cum / (double)n_pos;
    t[3] = n_neg != 0 ? auc / (double)(n_pos * n_neg) : 0.0;
    t[4] = 1.0;
    t[5] = n_neg == 0 ? 1.0 : 0.0;
}

// NumPy's float32 add.reduce over a contiguous run (numpy/_core/src/umath/loops_utils.h.src, pairwise_sum with
// PW_BLOCKSIZE 128): fewer than 8 values summed in order, else 8 interleaved accumulators, else split in halves
// rounded down to a multiple of 8.  Intrinsics keep the compiler from contracting or reassociating.
template <class F>
__device__ float np_pairwise_block(F a, int off, int n) {
    if (n < 8) {
        float res = 0.f;
        for (int i = 0; i < n; ++i) res = __fadd_rn(res, a(off + i));
        return res;
    }
    float r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = a(off + j);
    int i = 8;
    for (; i < n - (n % 8); i += 8) {
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = __fadd_rn(r[j], a(off + i + j));
    }
    float res = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])),
                          __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
    for (; i < n; ++i) res = __fadd_rn(res, a(off + i));
    return res;
}

template <int DEPTH, class F>
__device__ float np_pairwise(F a, int off, int n) {
    if constexpr (DEPTH == 0) {
        return np_pairwise_block(a, off, n);
    } else {
        if (n <= 128) return np_pairwise_block(a, off, n);
        int n2 = n / 2;
        n2 -= n2 % 8;
        return __fadd_rn(np_pairwise<DEPTH - 1>(a, off, n2), np_pairwise<DEPTH - 1>(a, off + n2, n - n2));
    }
}

// mode 0: (P[r] * Q[c]).sum(1); 1: the same + Qb[c]; 2: 1 - ((P[r] - Q[c]) ** 2).sum(-1) -- all float32 like the host's
// _get_scores -- then err = float64(score) - float64(val): terms[i] = (err^2, |err|).
__global__ void eval_score_terms_kernel(const float* __restrict__ P, const float* __restrict__ Q,
                                        const float* __restrict__ Qb, int width, int mode,
                                        const int32_t* __restrict__ rows, const int32_t* __restrict__ cols,
                                        const float* __restrict__ vals, int64_t n, double* __restrict__ terms) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* p = P + (int64_t)rows[i] * width;
    const float* q = Q + (int64_t)cols[i] * width;
    float s;
    if (mode == 2) {
        s = np_pairwise<3>([&](int c) { const float x = __fsub_rn(p[c], q[c]); return __fmul_rn(x, x); }, 0, width);
        s = __fsub_rn(1.0f, __fadd_rn(0.f, s));
    } else {
        s = __fadd_rn(0.f, np_pairwise<3>([&](int c) { return __fmul_rn(p[c], q[c]); }, 0, width));
        if (mode == 1) s = __fadd_rn(s, Qb[cols[i]]);
    }
    const double err = (double)s - (double)vals[i];
    terms[2 * i] = err * err;
    terms[2 * i + 1] = fabs(err);
}

// Fixed-order column sums: thread g of the EV_SUM_BLOCKS x TK_THREADS grid adds rows g, g + grid, ... in order, then
// a shared-memory tree per block and one more over the blocks.
__global__ void __launch_bounds__(TK_THREADS) eval_sum_partial_kernel(const double* __restrict__ terms, int64_t n,
                                                                      int width, double* __restrict__ partial) {
    __shared__ double red[EV_SUM_WIDTH][TK_THREADS];
    const int tid = threadIdx.x;
    double acc[EV_SUM_WIDTH];
#pragma unroll
    for (int c = 0; c < EV_SUM_WIDTH; ++c) acc[c] = 0.0;
    for (int64_t r = (int64_t)blockIdx.x * TK_THREADS + tid; r < n; r += (int64_t)EV_SUM_BLOCKS * TK_THREADS) {
#pragma unroll
        for (int c = 0; c < EV_SUM_WIDTH; ++c)
            if (c < width) acc[c] += terms[r * width + c];
    }
#pragma unroll
    for (int c = 0; c < EV_SUM_WIDTH; ++c) red[c][tid] = acc[c];
    __syncthreads();
    for (int s = TK_THREADS / 2; s > 0; s >>= 1) {
        if (tid < s) {
#pragma unroll
            for (int c = 0; c < EV_SUM_WIDTH; ++c) red[c][tid] += red[c][tid + s];
        }
        __syncthreads();
    }
    if (tid < width) partial[blockIdx.x * EV_SUM_WIDTH + tid] = red[tid][0];
}

__global__ void __launch_bounds__(EV_SUM_BLOCKS) eval_sum_final_kernel(const double* __restrict__ partial, int width,
                                                                       double* __restrict__ out) {
    __shared__ double red[EV_SUM_WIDTH][EV_SUM_BLOCKS];
    const int tid = threadIdx.x;
    for (int c = 0; c < width; ++c) red[c][tid] = partial[tid * EV_SUM_WIDTH + c];
    __syncthreads();
    for (int s = EV_SUM_BLOCKS / 2; s > 0; s >>= 1) {
        if (tid < s)
            for (int c = 0; c < width; ++c) red[c][tid] += red[c][tid + s];
        __syncthreads();
    }
    if (tid < width) out[tid] = red[tid][0];
}

}  // namespace

int bfl::masked_topk(const float* queries, int64_t nq, int ldq, const float* items, int64_t n_items, int ldi,
                     const float* item_bias, int d, int k, const int64_t* seen_indptr, const int32_t* seen_keys,
                     const int32_t* seen_row, const int32_t* pool, int32_t* out_idx, float* out_val, cudaStream_t st) {
    const int64_t nslices = (n_items + TK_SLICE - 1) / TK_SLICE;
    if (n_items > INT32_MAX || nslices > 65535) BFL_FAIL(BFL_ERR_ARG, "masked top-k: too many items");
    unsigned long long* cand = nullptr;
    int32_t* cand_cnt = nullptr;
    BFL_CUDA(cudaMallocAsync(&cand, sizeof(unsigned long long) * (size_t)nq * nslices * k, st));
    BFL_CUDA(cudaMallocAsync(&cand_cnt, sizeof(int32_t) * (size_t)nq * nslices, st));
    const int dpad = (d + 3) & ~3;
    const size_t smem1 = sizeof(unsigned long long) * TK_SLICE + sizeof(float) * ((size_t)EV_QB * TK_SLICE + (size_t)EV_QB * dpad);
    BFL_CUDA(cudaFuncSetAttribute(eval_slice_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem1));
    dim3 grid((unsigned)((nq + EV_QB - 1) / EV_QB), (unsigned)nslices);
    eval_slice_kernel<<<grid, TK_THREADS, smem1, st>>>(queries, nq, ldq, items, n_items, ldi, item_bias, d, k,
                                                       (int)nslices, seen_indptr, seen_keys, seen_row, pool, cand,
                                                       cand_cnt);
    BFL_LAUNCHED();
    const int rc = seen_merge(cand, cand_cnt, nq, (int)nslices, k, out_idx, out_val, st);
    BFL_CUDA(cudaFreeAsync(cand, st));
    BFL_CUDA(cudaFreeAsync(cand_cnt, st));
    return rc;
}

int bfl::seen_merge(const unsigned long long* cand, const int32_t* cand_cnt, int64_t nq, int nslices, int k,
                    int32_t* out_idx, float* out_val, cudaStream_t st) {
    int kpad = 2;
    while (kpad < k) kpad <<= 1;
    eval_merge_kernel<<<(unsigned)nq, TK_THREADS, kpad * sizeof(unsigned long long), st>>>(cand, cand_cnt, nslices, k,
                                                                                          kpad, out_idx, out_val);
    BFL_LAUNCHED();
    return BFL_OK;
}

extern "C" {

int bfl_eval_unsorted_rows_device(const int64_t* d_indptr, const int32_t* d_keys, int64_t rows,
                                  unsigned long long* d_count, void* stream) {
    if (BFL_OK != require_device()) return BFL_ERR_CUDA;
    if (!d_indptr || !d_keys || !d_count || rows < 0) BFL_FAIL(BFL_ERR_ARG, "bad unsorted-rows arguments");
    cudaStream_t st = (cudaStream_t)stream;
    BFL_CUDA(cudaMemsetAsync(d_count, 0, sizeof(unsigned long long), st));
    if (rows == 0) return BFL_OK;
    const unsigned g = (unsigned)std::min<int64_t>((rows + 7) / 8, 4096);
    eval_unsorted_rows_kernel<<<g, 256, 0, st>>>(d_indptr, d_keys, rows, d_count);
    BFL_LAUNCHED();
    return BFL_OK;
}

int bfl_eval_topk_masked_device(const float* d_queries, int64_t nq, int ldq, const float* d_items, int64_t n_items,
                                int ldi, const float* d_item_bias, int d, int k, const int64_t* d_seen_indptr,
                                const int32_t* d_seen_keys, const int32_t* d_seen_row, int32_t* d_out_idx,
                                void* stream) {
    if (BFL_OK != require_device()) return BFL_ERR_CUDA;
    if (!d_queries || !d_items || !d_seen_indptr || !d_seen_keys || !d_seen_row || !d_out_idx || nq <= 0 ||
        n_items <= 0 || d <= 0 || ldq < d || ldi < d)
        BFL_FAIL(BFL_ERR_ARG, "bad masked top-k arguments");
    if (k <= 0 || k > TK_KMAX) BFL_FAIL(BFL_ERR_ARG, "masked top-k: k must be in [1, 4096]");
    return masked_topk(d_queries, nq, ldq, d_items, n_items, ldi, d_item_bias, d, k, d_seen_indptr, d_seen_keys,
                       d_seen_row, nullptr, d_out_idx, nullptr, (cudaStream_t)stream);
}

int bfl_eval_ranking_terms_device(const int32_t* d_ranked, int64_t nq, int k, const int32_t* d_users,
                                  const int64_t* d_seen_indptr, const int32_t* d_seen_row, const int64_t* d_gt_indptr,
                                  const int32_t* d_gt_keys, const double* d_gains, const double* d_ideal,
                                  int64_t num_items, double* d_terms, void* stream) {
    if (BFL_OK != require_device()) return BFL_ERR_CUDA;
    if (!d_ranked || !d_users || !d_seen_indptr || !d_seen_row || !d_gt_indptr || !d_gt_keys || !d_gains || !d_ideal ||
        !d_terms || nq < 0 || k <= 0 || num_items <= 0)
        BFL_FAIL(BFL_ERR_ARG, "bad ranking-terms arguments");
    if (nq == 0) return BFL_OK;
    cudaStream_t st = (cudaStream_t)stream;
    eval_rank_terms_kernel<<<(unsigned)((nq + 127) / 128), 128, 0, st>>>(d_ranked, nq, k, d_users, d_seen_indptr,
                                                                        d_seen_row, d_gt_indptr, d_gt_keys, d_gains,
                                                                        d_ideal, num_items, d_terms);
    BFL_LAUNCHED();
    return BFL_OK;
}

int bfl_eval_score_terms_device(const float* d_P, const float* d_Q, const float* d_Qb, int width, int mode,
                                const int32_t* d_rows, const int32_t* d_cols, const float* d_vals, int64_t n,
                                double* d_terms, void* stream) {
    if (BFL_OK != require_device()) return BFL_ERR_CUDA;
    if (!d_P || !d_Q || !d_rows || !d_cols || !d_vals || !d_terms || n < 0 || width <= 0 || width > 1024 ||
        mode < 0 || mode > 2 || (mode == 1 && !d_Qb))
        BFL_FAIL(BFL_ERR_ARG, "bad score-terms arguments");
    if (n == 0) return BFL_OK;
    cudaStream_t st = (cudaStream_t)stream;
    eval_score_terms_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(d_P, d_Q, d_Qb, width, mode, d_rows, d_cols,
                                                                         d_vals, n, d_terms);
    BFL_LAUNCHED();
    return BFL_OK;
}

int bfl_eval_sum_device(const double* d_terms, int64_t n, int width, double* d_out, void* stream) {
    if (BFL_OK != require_device()) return BFL_ERR_CUDA;
    if ((!d_terms && n > 0) || !d_out || n < 0 || width <= 0 || width > EV_SUM_WIDTH)
        BFL_FAIL(BFL_ERR_ARG, "bad sum arguments");
    cudaStream_t st = (cudaStream_t)stream;
    double* partial = nullptr;
    BFL_CUDA(cudaMallocAsync(&partial, sizeof(double) * EV_SUM_BLOCKS * EV_SUM_WIDTH, st));
    eval_sum_partial_kernel<<<EV_SUM_BLOCKS, TK_THREADS, 0, st>>>(d_terms, n, width, partial);
    BFL_LAUNCHED();
    eval_sum_final_kernel<<<1, EV_SUM_BLOCKS, 0, st>>>(partial, width, d_out);
    BFL_LAUNCHED();
    BFL_CUDA(cudaFreeAsync(partial, st));
    return BFL_OK;
}

}  // extern "C"
