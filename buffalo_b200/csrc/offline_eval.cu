// Offline evaluation on held-out interactions (DESIGN.md 4.14): the device path of Evaluable.evaluate and
// buffalo_b200.evaluate.evaluate_lists.  Ranked lists come in as int32 [n x k] (-1 pads), the held-out items as a truth
// CSR whose rows are sorted and free of duplicates.  Every per-row value is a function of that row alone, so it does not
// depend on the batch split or the launch configuration; the means are left to bfl_eval_sum_device (fixed order).
//   oe_cutoff_terms_kernel  : one warp per row; lane i of a 32-entry chunk binary-searches entry i in the truth row, a
//                             ballot and a warp scan give the hit count, the DCG and the AP sum up to each entry, and the
//                             values at every cutoff inside the chunk are written to that cutoff's [n x 8] slab;
//   oe_ild_kernel           : one CTA per row; the Gram matrix of the row's first kmax item rows (kmax <= 256) is built
//                             in shared memory (gram_common.cuh), then 1 - cos per pair summed per cutoff;
//   oe_coverage_mark_kernel : first[item] = min over every list entry of the cutoff index the entry's position falls in;
//   oe_coverage_count_kernel: the number of items per first cutoff index (integers, so any order gives the same count).
#include <algorithm>

#include "gram_common.cuh"
#include "seen_common.cuh"

using namespace bfl;

namespace {

constexpr int OE_WIDTH = 8;          // hit, recall, precision, ndcg, ap, rr, ild, ild counted
constexpr int OE_TERMS_THREADS = 256;
constexpr int OE_ILD_KMAX = 256;
constexpr int OE_COUNT_THREADS = 256;

// terms[c * slab + r * OE_WIDTH + j]: slab c is the [n x 8] block of cutoff c.
__global__ void __launch_bounds__(OE_TERMS_THREADS) oe_cutoff_terms_kernel(
    const int32_t* __restrict__ ranked, int64_t n, int k, const int64_t* __restrict__ truth_indptr,
    const int32_t* __restrict__ truth_keys, const int32_t* __restrict__ truth_row, const int32_t* __restrict__ cutoffs,
    int n_cut, const double* __restrict__ gains, const double* __restrict__ ideal, double* __restrict__ terms,
    int64_t slab) {
    const int lane = threadIdx.x & 31;
    const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (r >= n) return;   // the whole warp leaves together
    const int64_t tr = truth_row ? truth_row[r] : r;
    const int64_t g0 = seen_row_begin(truth_indptr, tr), g1 = truth_indptr[tr];
    const int64_t n_pos = g1 - g0;
    const int32_t* rk = ranked + r * (int64_t)k;
    const int kmax = cutoffs[n_cut - 1];
    int cum = 0, first = 0, c = 0;   // hits before the chunk, 1-based position of the first hit (0: none), next cutoff
    double dcg = 0.0, ap = 0.0;      // sums over the entries before the chunk
    for (int base = 0; base < kmax; base += 32) {
        const int i = base + lane;
        bool h = false;
        if (i < kmax && i < k) {   // entries past the list's width count as padding
            const int32_t e = rk[i];
            h = e >= 0 && row_contains(truth_keys, g0, g1, e);
        }
        const unsigned bal = __ballot_sync(FULL, h);
        const int ci = cum + __popc(bal & (0xffffffffu >> (31 - lane)));   // hits among entries 0..i
        double td = h ? gains[i] : 0.0, ta = h ? (double)ci / (double)(i + 1) : 0.0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const double x = __shfl_up_sync(FULL, td, o), y = __shfl_up_sync(FULL, ta, o);
            if (lane >= o) {
                td += x;
                ta += y;
            }
        }
        td += dcg;
        ta += ap;
        if (!first && bal) first = base + __ffs(bal);
        for (; c < n_cut && cutoffs[c] <= base + 32; ++c) {
            const int kc = cutoffs[c], src = kc - 1 - base;
            const double D = __shfl_sync(FULL, td, src), A = __shfl_sync(FULL, ta, src);
            const int C = __shfl_sync(FULL, ci, src);
            if (lane == 0) {
                double* t = terms + c * slab + r * OE_WIDTH;
                const int64_t m = n_pos < kc ? n_pos : kc;
                const bool any = n_pos > 0;
                t[0] = C > 0 ? 1.0 : 0.0;
                t[1] = any ? (double)C / (double)n_pos : 0.0;
                t[2] = (double)C / (double)kc;
                t[3] = any ? D / ideal[m - 1] : 0.0;
                t[4] = any ? A / (double)m : 0.0;
                t[5] = first && first <= kc ? 1.0 / (double)first : 0.0;
                t[6] = 0.0;
                t[7] = 0.0;
            }
        }
        dcg = __shfl_sync(FULL, td, 31);
        ap = __shfl_sync(FULL, ta, 31);
        cum += __popc(bal);
    }
}

// Shared memory: one tile [kmax][GRAM_TDS] of item rows, per position b the fp64 sum over valid a < b of 1 - cos(a, b),
// the row's items, and the Gram triangle of gram_triangle (gram_common.cuh).
__global__ void __launch_bounds__(OE_ILD_KMAX) oe_ild_kernel(const int32_t* __restrict__ ranked, int k, int kmax,
                                                             const float* __restrict__ items, int ld, int d,
                                                             const int32_t* __restrict__ cutoffs, int n_cut,
                                                             double* __restrict__ terms, int64_t slab) {
    extern __shared__ __align__(16) unsigned char oe_smem[];
    // tile first: its rows are read as float4, so it must start on 16 bytes (its size, 144 kmax, keeps pair_sum on 8)
    float* tile = reinterpret_cast<float*>(oe_smem);                        // [kmax][GRAM_TDS]
    double* pair_sum = reinterpret_cast<double*>(tile + gram_tile_floats(kmax));   // [kmax]
    int32_t* item = reinterpret_cast<int32_t*>(pair_sum + kmax);            // [kmax]
    float* G = reinterpret_cast<float*>(item + kmax);                       // [kmax * (kmax + 1) / 2]
    const int tid = threadIdx.x, nt = blockDim.x;
    const int64_t r = blockIdx.x;
    const int32_t* rk = ranked + r * (int64_t)k;
    for (int b = tid; b < kmax; b += nt) item[b] = rk[b];
    gram_triangle(item, kmax, items, ld, d, tile, G);
    const int b = tid;
    const size_t gb = (size_t)b * (b + 1) / 2;
    if (b < kmax) {
        double s = 0.0;
        if (item[b] >= 0) {
            const double nb = (double)G[gb + b];
            for (int a = 0; a < b; ++a) {
                if (item[a] < 0) continue;
                const double na = (double)G[(size_t)a * (a + 1) / 2 + a];
                const double cosv = na > 0.0 && nb > 0.0 ? (double)G[gb + a] / sqrt(na * nb) : 0.0;
                s += 1.0 - cosv;
            }
        }
        pair_sum[b] = s;
    }
    __syncthreads();
    for (int c = tid; c < n_cut; c += nt) {
        const int kc = min(cutoffs[c], kmax);
        double s = 0.0;
        long long m = 0;
        for (int p = 0; p < kc; ++p) {
            s += pair_sum[p];
            m += item[p] >= 0;
        }
        double* t = terms + c * slab + r * OE_WIDTH;
        t[6] = m >= 2 ? s / (0.5 * (double)m * (double)(m - 1)) : 0.0;
        t[7] = m >= 2 ? 1.0 : 0.0;
    }
}

__global__ void oe_coverage_mark_kernel(const int32_t* __restrict__ ranked, int64_t n, int k, int kmax,
                                        const int32_t* __restrict__ bucket, int32_t* __restrict__ first) {
    const int64_t total = n * kmax;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = e / kmax;
        const int p = (int)(e - r * kmax);
        const int32_t it = ranked[r * k + p];
        if (it >= 0) atomicMin(first + it, bucket[p]);
    }
}

__global__ void __launch_bounds__(OE_COUNT_THREADS) oe_coverage_count_kernel(const int32_t* __restrict__ first,
                                                                              int64_t n_items, int n_cut,
                                                                              unsigned long long* __restrict__ count) {
    extern __shared__ unsigned int oe_hist[];   // [n_cut]
    for (int c = threadIdx.x; c < n_cut; c += blockDim.x) oe_hist[c] = 0;
    __syncthreads();
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_items; i += (int64_t)gridDim.x * blockDim.x) {
        const int f = first[i];
        if (f < n_cut) atomicAdd(&oe_hist[f], 1u);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < n_cut; c += blockDim.x)
        if (oe_hist[c]) atomicAdd(count + c, (unsigned long long)oe_hist[c]);
}

size_t ild_smem_bytes(int kmax) {
    static_assert((sizeof(float) * GRAM_TDS) % 16 == 0, "tile rows must keep float4 alignment");
    return sizeof(float) * gram_tile_floats(kmax) + sizeof(double) * kmax + sizeof(int32_t) * kmax +
           sizeof(float) * gram_triangle_floats(kmax);
}

}  // namespace

extern "C" {

int bfl_eval_cutoff_terms_device(const int32_t* d_ranked, int64_t n, int k, const int64_t* d_truth_indptr,
                                 const int32_t* d_truth_keys, const int32_t* d_truth_row, const int32_t* d_cutoffs,
                                 int n_cut, const double* d_gains, const double* d_ideal, double* d_terms,
                                 int64_t slab_stride, void* stream) {
    if (BFL_OK != require_device()) return BFL_ERR_CUDA;
    if (!d_ranked || !d_truth_indptr || !d_truth_keys || !d_cutoffs || !d_gains || !d_ideal || !d_terms || n < 0 ||
        k <= 0 || k > TK_KMAX || n_cut <= 0 || slab_stride < n * OE_WIDTH)
        BFL_FAIL(BFL_ERR_ARG, "bad cutoff-terms arguments");
    if (n == 0) return BFL_OK;
    const int64_t warps_per_block = OE_TERMS_THREADS / 32;
    oe_cutoff_terms_kernel<<<(unsigned)((n + warps_per_block - 1) / warps_per_block), OE_TERMS_THREADS, 0,
                             (cudaStream_t)stream>>>(d_ranked, n, k, d_truth_indptr, d_truth_keys, d_truth_row,
                                                     d_cutoffs, n_cut, d_gains, d_ideal, d_terms, slab_stride);
    BFL_LAUNCHED();
    return BFL_OK;
}

int bfl_eval_ild_device(const int32_t* d_ranked, int64_t n, int k, int kmax, const float* d_items, int ld, int d,
                        const int32_t* d_cutoffs, int n_cut, double* d_terms, int64_t slab_stride, void* stream) {
    if (BFL_OK != require_device()) return BFL_ERR_CUDA;
    if (!d_ranked || !d_items || !d_cutoffs || !d_terms || n < 0 || k <= 0 || d <= 0 || ld < d || n_cut <= 0 ||
        slab_stride < n * OE_WIDTH)
        BFL_FAIL(BFL_ERR_ARG, "bad ild arguments");
    if (kmax < 1 || kmax > OE_ILD_KMAX || kmax > k) BFL_FAIL(BFL_ERR_ARG, "ild: cutoffs must be in [1, min(k, 256)]");
    if (n == 0) return BFL_OK;
    if (n > INT32_MAX) BFL_FAIL(BFL_ERR_ARG, "ild: too many rows in one call");
    const size_t smem = ild_smem_bytes(kmax);
    BFL_CUDA(cudaFuncSetAttribute(oe_ild_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int threads = std::max(32, (kmax + 31) / 32 * 32);
    oe_ild_kernel<<<(unsigned)n, threads, smem, (cudaStream_t)stream>>>(d_ranked, k, kmax, d_items, ld, d, d_cutoffs,
                                                                        n_cut, d_terms, slab_stride);
    BFL_LAUNCHED();
    return BFL_OK;
}

int bfl_eval_coverage_mark_device(const int32_t* d_ranked, int64_t n, int k, const int32_t* d_bucket, int kmax,
                                  int32_t* d_first, void* stream) {
    if (BFL_OK != require_device()) return BFL_ERR_CUDA;
    if (!d_ranked || !d_bucket || !d_first || n < 0 || k <= 0 || kmax <= 0 || kmax > k)
        BFL_FAIL(BFL_ERR_ARG, "bad coverage-mark arguments");
    if (n == 0) return BFL_OK;
    const int64_t total = n * kmax;
    const unsigned g = (unsigned)std::min<int64_t>((total + 255) / 256, 132 * 64);
    oe_coverage_mark_kernel<<<g, 256, 0, (cudaStream_t)stream>>>(d_ranked, n, k, kmax, d_bucket, d_first);
    BFL_LAUNCHED();
    return BFL_OK;
}

int bfl_eval_coverage_count_device(const int32_t* d_first, int64_t n_items, int n_cut, unsigned long long* d_count,
                                   void* stream) {
    if (BFL_OK != require_device()) return BFL_ERR_CUDA;
    if (!d_first || !d_count || n_items <= 0 || n_cut <= 0 || n_cut > TK_KMAX)
        BFL_FAIL(BFL_ERR_ARG, "bad coverage-count arguments");
    cudaStream_t st = (cudaStream_t)stream;
    BFL_CUDA(cudaMemsetAsync(d_count, 0, sizeof(unsigned long long) * n_cut, st));
    const unsigned g = (unsigned)std::min<int64_t>((n_items + OE_COUNT_THREADS - 1) / OE_COUNT_THREADS, 264);
    oe_coverage_count_kernel<<<g, OE_COUNT_THREADS, sizeof(unsigned int) * n_cut, st>>>(d_first, n_items, n_cut,
                                                                                       d_count);
    BFL_LAUNCHED();
    return BFL_OK;
}

}  // extern "C"
