// Evaluation top-k on the device (SURVEY.md 8(f-2)): scores = P[rows] . Q^T (+ item bias) and the k best items per
// query row, replacing the reference's host quickselect (buffalo/parallel/_core.hpp:69-142, used by
// buffalo/evaluate/base.py:31-128 and Algo.topk_recommendation).  Two kernels, no library calls:
//   topk_slice_kernel : a CTA scores QB queries against a slice of SLICE items (item rows read once per QB queries),
//                       keeps the scores in shared memory and radix-selects the slice's k best per query;
//   topk_merge_kernel : per query, radix-selects the k best of the slices' candidates and orders them with a
//                       shared-memory bitonic sort on (score descending, item index ascending) -- deterministic ties.
#include "topk_common.cuh"

using namespace bfl;

namespace {

constexpr int TK_QB = 4;

struct SelScratch {
    unsigned int hist[256];
    unsigned int warp_tot[TK_THREADS / 32];
    unsigned int prefix, kk, cnt, base;
};

// k largest of vals[0..n) -> (out_v, out_i)[0..k) unordered; idxs == nullptr: index = idx0 + position.  n > 0, k > 0.
// Ties at the k-th value are resolved towards the smaller position (deterministic).  All threads of the CTA call it.
__device__ void block_select(const float* vals, const int32_t* idxs, int idx0, int n, int k, float* out_v,
                             int32_t* out_i, SelScratch& sc) {
    const int tid = threadIdx.x;
    if (n <= k) {
        for (int i = tid; i < k; i += TK_THREADS) {
            out_v[i] = i < n ? vals[i] : -INFINITY;
            out_i[i] = i < n ? (idxs ? idxs[i] : idx0 + i) : -1;
        }
        __syncthreads();
        return;
    }
    if (tid == 0) { sc.prefix = 0; sc.kk = (unsigned)k; }
    uint32_t mask = 0;
    for (int shift = 24; shift >= 0; shift -= 8) {
        sc.hist[tid] = 0;   // TK_THREADS == 256
        __syncthreads();
        const uint32_t prefix = sc.prefix;
        for (int i = tid; i < n; i += TK_THREADS) {
            const uint32_t u = ord_of(vals[i]);
            if ((u & mask) == prefix) atomicAdd(&sc.hist[(u >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (tid == 0) {
            unsigned cum = 0, kk = sc.kk;
            int b = 255;
            for (; b > 0; --b) {
                if (cum + sc.hist[b] >= kk) break;
                cum += sc.hist[b];
            }
            sc.kk = kk - cum;                       // still needed inside bin b
            sc.prefix = prefix | ((uint32_t)b << shift);
        }
        mask |= 255u << shift;
        __syncthreads();
    }
    const uint32_t T = sc.prefix;
    const unsigned kk = sc.kk;                       // ties to take; k - kk elements are strictly larger
    if (tid == 0) { sc.cnt = 0; sc.base = 0; }
    __syncthreads();
    for (int i = tid; i < n; i += TK_THREADS) {
        const float v = vals[i];
        if (ord_of(v) > T) {
            const unsigned pos = atomicAdd(&sc.cnt, 1u);
            out_v[pos] = v;
            out_i[pos] = idxs ? idxs[i] : idx0 + i;
        }
    }
    const int lane = tid & 31, w = tid >> 5;
    for (int i0 = 0; i0 < n; i0 += TK_THREADS) {
        __syncthreads();
        const unsigned base = sc.base;
        if (base >= kk) break;
        const int i = i0 + tid;
        const float v = i < n ? vals[i] : 0.f;
        const bool tie = i < n && ord_of(v) == T;
        const unsigned bal = __ballot_sync(FULL, tie);
        if (lane == 0) sc.warp_tot[w] = __popc(bal);
        __syncthreads();
        unsigned before = 0, total = 0;
#pragma unroll
        for (int ww = 0; ww < TK_THREADS / 32; ++ww) {
            const unsigned t = sc.warp_tot[ww];
            before += ww < w ? t : 0u;
            total += t;
        }
        const unsigned r = base + before + __popc(bal & ((1u << lane) - 1u));
        if (tie && r < kk) {
            out_v[(k - kk) + r] = v;
            out_i[(k - kk) + r] = idxs ? idxs[i] : idx0 + i;
        }
        __syncthreads();
        if (tid == 0) sc.base = base + total;
    }
    __syncthreads();
}

__global__ void __launch_bounds__(TK_THREADS) topk_slice_kernel(const float* __restrict__ Qr, int64_t nq, int ldq,
                                                                const float* __restrict__ It, int64_t n_items, int ldi,
                                                                const float* __restrict__ bias, int d, int k, int nslices,
                                                                float* __restrict__ cand_v, int32_t* __restrict__ cand_i) {
    extern __shared__ __align__(16) float tk_smem[];
    float* scores = tk_smem;                       // [TK_QB][TK_SLICE]
    float* qv = scores + TK_QB * TK_SLICE;         // [TK_QB][dpad]
    __shared__ SelScratch sc;
    const int slice = blockIdx.x;
    const int64_t q0 = (int64_t)blockIdx.y * TK_QB;
    const int nqb = (int)min((long long)TK_QB, (long long)(nq - q0));
    const int64_t i0 = (int64_t)slice * TK_SLICE;
    const int ni = (int)min((long long)TK_SLICE, (long long)(n_items - i0));
    topk_score_slice<TK_QB>(Qr, q0, nqb, ldq, It, i0, ni, ldi, bias, d, qv, scores);
    for (int qi = 0; qi < nqb; ++qi) {
        const size_t o = ((size_t)(q0 + qi) * nslices + slice) * k;
        block_select(scores + qi * TK_SLICE, nullptr, (int)i0, ni, k, cand_v + o, cand_i + o, sc);
    }
}

__global__ void __launch_bounds__(TK_THREADS) topk_merge_kernel(const float* __restrict__ cand_v,
                                                                const int32_t* __restrict__ cand_i, int ncand, int k,
                                                                int kpad, float* __restrict__ sel_v,
                                                                int32_t* __restrict__ sel_i, int32_t* __restrict__ out_i,
                                                                float* __restrict__ out_v) {
    extern __shared__ __align__(16) unsigned long long tk_keys[];   // [kpad]
    __shared__ SelScratch sc;
    const int tid = threadIdx.x;
    const size_t q = blockIdx.x;
    float* sv = sel_v + q * k;
    int32_t* si = sel_i + q * k;
    block_select(cand_v + q * ncand, cand_i + q * ncand, 0, ncand, k, sv, si, sc);
    __threadfence_block();
    __syncthreads();
    // sort ascending on (~ord(score), index): best score first, smaller index first among equal scores; empty slots last
    for (int i = tid; i < kpad; i += TK_THREADS) {
        unsigned long long key = ~0ull;
        if (i < k && si[i] >= 0) key = ((unsigned long long)(~ord_of(sv[i])) << 32) | (unsigned int)si[i];
        tk_keys[i] = key;
    }
    __syncthreads();
    for (int size = 2; size <= kpad; size <<= 1) {
        for (int strd = size >> 1; strd > 0; strd >>= 1) {
            for (int i = tid; i < kpad / 2; i += TK_THREADS) {
                const int lo = 2 * i - (i & (strd - 1)), hi = lo + strd;
                const bool up = (lo & size) == 0;
                const unsigned long long a = tk_keys[lo], b = tk_keys[hi];
                if ((a > b) == up) { tk_keys[lo] = b; tk_keys[hi] = a; }
            }
            __syncthreads();
        }
    }
    for (int i = tid; i < k; i += TK_THREADS) {
        const unsigned long long key = tk_keys[i];
        if (key == ~0ull) {
            out_i[q * k + i] = -1;
            out_v[q * k + i] = -INFINITY;
        } else {
            const uint32_t o = ~(uint32_t)(key >> 32);
            const uint32_t u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
            out_i[q * k + i] = (int32_t)(uint32_t)(key & 0xffffffffu);
            out_v[q * k + i] = __uint_as_float(u);
        }
    }
}

}  // namespace

int bfl::topk_merge(const float* cand_v, const int32_t* cand_i, int64_t nq, int ncand, int k, int32_t* out_idx,
                    float* out_val, cudaStream_t st) {
    float* sel_v = nullptr;
    int32_t* sel_i = nullptr;
    const size_t ns = (size_t)nq * k;
    BFL_CUDA(cudaMallocAsync(&sel_v, ns * sizeof(float), st));
    BFL_CUDA(cudaMallocAsync(&sel_i, ns * sizeof(int32_t), st));
    int kpad = 2;
    while (kpad < k) kpad <<= 1;
    topk_merge_kernel<<<(unsigned)nq, TK_THREADS, kpad * sizeof(unsigned long long), st>>>(cand_v, cand_i, ncand, k, kpad,
                                                                                          sel_v, sel_i, out_idx, out_val);
    BFL_LAUNCHED();
    BFL_CUDA(cudaFreeAsync(sel_v, st));
    BFL_CUDA(cudaFreeAsync(sel_i, st));
    return BFL_OK;
}

extern "C" {

// all pointers are device pointers; out_idx [nq x k] (best first, -1 = fewer than k items), out_val [nq x k]
int bfl_topk_device(const float* queries, int64_t nq, int ldq, const float* items, int64_t n_items, int ldi,
                    const float* item_bias, int d, int k, int32_t* out_idx, float* out_val, void* stream) {
    if (BFL_OK != require_device()) return BFL_ERR_CUDA;
    if (!queries || !items || !out_idx || !out_val || nq <= 0 || n_items <= 0 || d <= 0 || ldq < d || ldi < d)
        BFL_FAIL(BFL_ERR_ARG, "bad top-k arguments");
    if (k <= 0 || k > TK_KMAX) BFL_FAIL(BFL_ERR_ARG, "top-k: k must be in [1, 4096]");
    cudaStream_t st = (cudaStream_t)stream;
    const int nslices = (int)((n_items + TK_SLICE - 1) / TK_SLICE);
    const int ncand = nslices * k;
    float* cand_v = nullptr;
    int32_t* cand_i = nullptr;
    const size_t nc = (size_t)nq * ncand;
    BFL_CUDA(cudaMallocAsync(&cand_v, nc * sizeof(float), st));
    BFL_CUDA(cudaMallocAsync(&cand_i, nc * sizeof(int32_t), st));
    const int dpad = (d + 3) & ~3;
    const size_t smem1 = sizeof(float) * ((size_t)TK_QB * TK_SLICE + (size_t)TK_QB * dpad);
    BFL_CUDA(cudaFuncSetAttribute(topk_slice_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem1));
    dim3 grid(nslices, (unsigned)((nq + TK_QB - 1) / TK_QB));
    topk_slice_kernel<<<grid, TK_THREADS, smem1, st>>>(queries, nq, ldq, items, n_items, ldi, item_bias, d, k, nslices,
                                                       cand_v, cand_i);
    BFL_LAUNCHED();
    const int rc = topk_merge(cand_v, cand_i, nq, ncand, k, out_idx, out_val, st);
    BFL_CUDA(cudaFreeAsync(cand_v, st));
    BFL_CUDA(cudaFreeAsync(cand_i, st));
    return rc;
}

// host pointers: copies queries / items / bias to the device, runs bfl_topk_device, copies the result back
int bfl_topk_host(const float* queries, int64_t nq, int ldq, const float* items, int64_t n_items, int ldi,
                  const float* item_bias, int d, int k, int32_t* out_idx, float* out_val) {
    if (BFL_OK != require_device()) return BFL_ERR_CUDA;
    if (!queries || !items || !out_idx || nq <= 0 || n_items <= 0) BFL_FAIL(BFL_ERR_ARG, "bad top-k arguments");
    DevBuf<float> dq, di, db, dv;
    DevBuf<int32_t> dix;
    if (BFL_OK != dq.reserve((size_t)nq * ldq) || BFL_OK != di.reserve((size_t)n_items * ldi) ||
        BFL_OK != dv.reserve((size_t)nq * k) || BFL_OK != dix.reserve((size_t)nq * k))
        return BFL_ERR_CUDA;
    if (item_bias && BFL_OK != db.reserve((size_t)n_items)) return BFL_ERR_CUDA;
    BFL_CUDA(cudaMemcpy(dq.p, queries, sizeof(float) * (size_t)nq * ldq, cudaMemcpyHostToDevice));
    BFL_CUDA(cudaMemcpy(di.p, items, sizeof(float) * (size_t)n_items * ldi, cudaMemcpyHostToDevice));
    if (item_bias) BFL_CUDA(cudaMemcpy(db.p, item_bias, sizeof(float) * (size_t)n_items, cudaMemcpyHostToDevice));
    const int rc = bfl_topk_device(dq.p, nq, ldq, di.p, n_items, ldi, item_bias ? db.p : nullptr, d, k, dix.p, dv.p, nullptr);
    if (rc != BFL_OK) return rc;
    BFL_CUDA(cudaDeviceSynchronize());
    BFL_CUDA(cudaMemcpy(out_idx, dix.p, sizeof(int32_t) * (size_t)nq * k, cudaMemcpyDeviceToHost));
    if (out_val) BFL_CUDA(cudaMemcpy(out_val, dv.p, sizeof(float) * (size_t)nq * k, cudaMemcpyDeviceToHost));
    return BFL_OK;
}

}  // extern "C"
