// Per-query candidate lists for batch serving (DESIGN.md 4.13): query q of a batch ranks only the items of its own
// list, row cand.row[q] (or cand.base + q) of a CSR of item ids in any order, duplicates allowed.  Row q of the answer
// is bitwise what bfl_serve_topk (bfl_seen_topk with seen rows) returns for that query with its list as the pool:
// the same fp32 score bits, the same rank keys (~ord(score)) << 32 | list position, so ties go to the earlier position.
//   cand_units_kernel : per query, the units of its list (ceil(len / 1024), one per slice of 1024 positions) and the
//                       rank-key slots they fill (min(k, slice length) each); two int64 scans make them a work list, so
//                       a long row costs its own units and short rows are not padded to it.
//   cand_slice_kernel : one warp per unit: the query row staged once in shared memory, each candidate row read straight
//                       from the resident items with 16-byte loads (plain loads for unaligned rows), every pair scored
//                       in topk_score_slice's order (lane partials, warp_sum's butterfly, then the bias), seen items
//                       marked by a binary search in the query's sorted seen row, then warp_select<true> -> rank keys
//                       and a count per unit.
//   cand_merge_kernel : per query, the segmented merge of its units' rank keys (select_smallest, a bitonic sort);
//                       positions map to item ids through the query's list; -1 / 0.0f pad.
// No atomics outside a warp's own shared scratch, so the result does not depend on batch cuts, grid or SM count.
#include <algorithm>
#include <climits>

#include "serve_common.cuh"

using namespace bfl;

namespace {

constexpr int CD_PAIRS = 4;                         // candidate rows a warp has in flight
constexpr int CD_SMEM_MAX = 227 * 1024;             // dynamic shared memory per CTA on sm_90

__device__ __forceinline__ int64_t row_of(const CandRows& c, int64_t q) { return c.row ? c.row[q] : c.base + q; }

__device__ __forceinline__ int64_t row_begin(const int64_t* __restrict__ indptr, int64_t r) {
    return r > 0 ? indptr[r - 1] : 0;
}

// floats of one warp's shared scratch: the query row, the unit's scores, the select histogram and the seen bitmask
__host__ __device__ inline int warp_floats(int d) { return ((d + 3) & ~3) + SV_SLICE + sel_words(true); }

__global__ void cand_units_kernel(CandRows cand, int64_t nb, int k, long long* __restrict__ unit_end,
                                  long long* __restrict__ key_end) {
    const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nb) return;
    const int64_t r = row_of(cand, q);
    const int64_t len = cand.indptr[r] - row_begin(cand.indptr, r);
    const int64_t full = len / SV_SLICE, rest = len - full * SV_SLICE;
    unit_end[q] = full + (rest > 0);
    key_end[q] = full * min(k, SV_SLICE) + min((int64_t)k, rest);
}

__global__ void __launch_bounds__(SV_THREADS)
    cand_slice_kernel(const float* __restrict__ Qm, int64_t n_qrows, int ldq, const int32_t* __restrict__ qidx,
                      int64_t nb, const float* __restrict__ It, int ldi, const float* __restrict__ bias, int d, int k,
                      CandRows cand, CandRows seen, const long long* __restrict__ unit_end,
                      const long long* __restrict__ key_end, long long n_units, unsigned long long* __restrict__ cand_key,
                      int32_t* __restrict__ cand_cnt) {
    extern __shared__ __align__(16) float cd_smem[];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const long long u = (long long)blockIdx.x * (blockDim.x >> 5) + w;
    if (u >= n_units) return;                       // the warp's work is a unit or nothing: no block barrier below
    const int dpad = (d + 3) & ~3;
    float* qs = cd_smem + (size_t)w * warp_floats(d);   // [dpad]
    float* scores = qs + dpad;                          // [SV_SLICE]
    unsigned* hist = reinterpret_cast<unsigned*>(scores + SV_SLICE);
    uint32_t* bits = hist + 256;

    // the unit: query q (the first with unit_end[q] > u), slice j of its list
    int64_t lo = 0, hi = nb - 1;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (unit_end[mid] > u) hi = mid;
        else lo = mid + 1;
    }
    const int64_t q = lo;
    const long long j = u - (q > 0 ? unit_end[q - 1] : 0);
    const int64_t r = row_of(cand, q);
    const int32_t* list = cand.keys + row_begin(cand.indptr, r);
    const int64_t i0 = j * SV_SLICE;
    const int ni = (int)min((int64_t)SV_SLICE, cand.indptr[r] - row_begin(cand.indptr, r) - i0);
    const size_t slot = (size_t)(q > 0 ? key_end[q - 1] : 0) + (size_t)j * min(k, SV_SLICE);

    const int64_t qr = qidx[q];
    for (int c = lane; c < dpad; c += 32) qs[c] = (c < d && qr >= 0 && qr < n_qrows) ? Qm[qr * ldq + c] : 0.f;
    __syncwarp();

    const bool vec = (ldi & 3) == 0 && (d & 3) == 0;
    for (int i = 0; i < ni; i += CD_PAIRS) {
        int32_t item[CD_PAIRS];
        float acc[CD_PAIRS];
#pragma unroll
        for (int p = 0; p < CD_PAIRS; ++p) {
            item[p] = list[i0 + min(i + p, ni - 1)];    // past the unit's end: its last row again, scored and dropped
            acc[p] = 0.f;
        }
        if (vec) {
            for (int c = lane * 4; c < d; c += 128) {
                const float4 x = *reinterpret_cast<const float4*>(qs + c);
                float4 v[CD_PAIRS];
#pragma unroll
                for (int p = 0; p < CD_PAIRS; ++p) v[p] = __ldg(reinterpret_cast<const float4*>(It + (int64_t)item[p] * ldi + c));
#pragma unroll
                for (int p = 0; p < CD_PAIRS; ++p)
                    acc[p] = fmaf(v[p].x, x.x, fmaf(v[p].y, x.y, fmaf(v[p].z, x.z, fmaf(v[p].w, x.w, acc[p]))));
            }
        } else {
            for (int c = lane; c < d; c += 32) {
                const float x = qs[c];
                float v[CD_PAIRS];
#pragma unroll
                for (int p = 0; p < CD_PAIRS; ++p) v[p] = __ldg(It + (int64_t)item[p] * ldi + c);
#pragma unroll
                for (int p = 0; p < CD_PAIRS; ++p) acc[p] = fmaf(v[p], x, acc[p]);
            }
        }
        // every lane ends warp_sum with lane 0's sum (each butterfly step adds the same two values)
#pragma unroll
        for (int p = 0; p < CD_PAIRS; ++p) acc[p] = warp_sum(acc[p]);
#pragma unroll
        for (int p = 0; p < CD_PAIRS; ++p)
            if (lane == p && i + p < ni) scores[i + p] = acc[p] + (bias ? bias[item[p]] : 0.f);
    }

    bits[lane] = 0;
    __syncwarp();
    if (seen.indptr) {   // list order is arbitrary: each candidate is looked up in the sorted seen row
        const int64_t sr = row_of(seen, q);
        const int64_t sb = row_begin(seen.indptr, sr), se = seen.indptr[sr];
        if (se > sb)
            for (int c0 = 0; c0 < ni; c0 += 32) {
                const int c = c0 + lane;
                const unsigned m = __ballot_sync(FULL, c < ni && row_contains(seen.keys, sb, se, list[i0 + c]));
                if (lane == 0) bits[c0 >> 5] = m;
            }
    }
    __syncwarp();
    warp_select<true>(scores, (int)i0, ni, k, nullptr, nullptr, hist, bits, cand_key + slot, cand_cnt + u);
}

// The segmented merge of one query's units: unit s holds cnt[s] keys at cand + s * stride (n keys of storage in all, the
// last unit may be shorter).  The k best of them go to sorted[0..kpad) ascending (best first), SEEN_EMPTY after the
// first `got`; returns got.  part: TK_THREADS / 32 words of shared scratch.  All TK_THREADS threads of the CTA call it.
__device__ __forceinline__ int merge_rank_lists(const unsigned long long* __restrict__ cand,
                                                const int32_t* __restrict__ cnt, int nunits, int stride, int64_t n,
                                                int k, int kpad, unsigned long long* sorted, KeySel& sc,
                                                long long* part) {
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    long long nv = 0;
    for (int s = tid; s < nunits; s += TK_THREADS) nv += cnt[s];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nv += __shfl_xor_sync(FULL, nv, o);
    if (lane == 0) part[w] = nv;
    __syncthreads();
    long long n_valid = 0;
#pragma unroll
    for (int i = 0; i < TK_THREADS / 32; ++i) n_valid += part[i];
    const int got = select_smallest(
        [&](int64_t i) {
            const int64_t s = i / stride;
            return (i - s * stride) < cnt[s] ? cand[i] : SEEN_EMPTY;
        },
        n, n_valid, k, sorted, sc);
    for (int i = got + tid; i < kpad; i += TK_THREADS) sorted[i] = SEEN_EMPTY;
    __syncthreads();
    for (int size = 2; size <= kpad; size <<= 1) {
        for (int strd = size >> 1; strd > 0; strd >>= 1) {
            for (int i = tid; i < kpad / 2; i += TK_THREADS) {
                const int lo = 2 * i - (i & (strd - 1)), hi = lo + strd;
                const bool up = (lo & size) == 0;
                const unsigned long long a = sorted[lo], b = sorted[hi];
                if ((a > b) == up) {
                    sorted[lo] = b;
                    sorted[hi] = a;
                }
            }
            __syncthreads();
        }
    }
    return got;
}

__global__ void __launch_bounds__(TK_THREADS)
    cand_merge_kernel(CandRows cand, const long long* __restrict__ unit_end, const long long* __restrict__ key_end,
                      const unsigned long long* __restrict__ cand_key, const int32_t* __restrict__ cand_cnt, int k,
                      int kpad, int32_t* __restrict__ out_idx, float* __restrict__ out_val) {
    extern __shared__ __align__(16) unsigned long long cd_sorted[];   // [kpad]
    __shared__ KeySel sc;
    __shared__ long long part[TK_THREADS / 32];
    const int64_t q = blockIdx.x;
    const long long u0 = q > 0 ? unit_end[q - 1] : 0, kb = q > 0 ? key_end[q - 1] : 0;
    const int got = merge_rank_lists(cand_key + kb, cand_cnt + u0, (int)(unit_end[q] - u0), min(k, SV_SLICE),
                                     key_end[q] - kb, k, kpad, cd_sorted, sc, part);
    const int32_t* list = cand.keys + row_begin(cand.indptr, row_of(cand, q));
    for (int i = threadIdx.x; i < k; i += TK_THREADS) {
        const unsigned long long key = cd_sorted[i];
        out_idx[q * k + i] = i < got ? list[(uint32_t)key] : -1;
        if (out_val) out_val[q * k + i] = i < got ? rank_key_score(key) : 0.f;
    }
}

}  // namespace

int bfl::cand_plan(CandRows cand, int64_t nb, int k, long long* unit_end, long long* key_end, cudaStream_t st) {
    cand_units_kernel<<<(unsigned)((nb + 255) / 256), 256, 0, st>>>(cand, nb, k, unit_end, key_end);
    BFL_LAUNCHED();
    if (int rc = inclusive_scan_i64(unit_end, unit_end, nb, st)) return rc;
    return inclusive_scan_i64(key_end, key_end, nb, st);
}

int bfl::cand_batch(const float* queries, int64_t n_q, int ldq, const int32_t* qidx, int64_t nb, const float* items,
                    int ldi, const float* bias, int d, int k, CandRows cand, CandRows seen, const long long* unit_end,
                    const long long* key_end, long long n_units, unsigned long long* cand_key, int32_t* cand_cnt,
                    int32_t* out_idx, float* out_val, cudaStream_t st) {
    const int per_warp = (int)sizeof(float) * warp_floats(d);
    const int warps = std::min(SV_THREADS / 32, CD_SMEM_MAX / per_warp);
    if (warps < 1) BFL_FAIL(BFL_ERR_ARG, "candidates: item rows too wide for one warp's shared memory");
    if (n_units > 0) {
        const long long blocks = (n_units + warps - 1) / warps;
        if (blocks > INT_MAX) BFL_FAIL(BFL_ERR_ARG, "candidates: too many candidates for one batch");
        const int smem = warps * per_warp;
        BFL_CUDA(cudaFuncSetAttribute(cand_slice_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        cand_slice_kernel<<<(unsigned)blocks, warps * 32, smem, st>>>(queries, n_q, ldq, qidx, nb, items, ldi, bias, d,
                                                                      k, cand, seen, unit_end, key_end, n_units,
                                                                      cand_key, cand_cnt);
        BFL_LAUNCHED();
    }
    int kpad = 2;
    while (kpad < k) kpad <<= 1;
    cand_merge_kernel<<<(unsigned)nb, TK_THREADS, kpad * sizeof(unsigned long long), st>>>(
        cand, unit_end, key_end, cand_key, cand_cnt, k, kpad, out_idx, out_val);
    BFL_LAUNCHED();
    return BFL_OK;
}
