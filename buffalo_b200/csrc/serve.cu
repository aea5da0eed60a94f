// Batch serving top-k on the device (DESIGN.md 4.9): the device path of buffalo.parallel's ParALS / ParBPRMF
// (dot_topn, buffalo/parallel/_core.hpp:88-142).  A bfl_serve_t keeps the item and query factors resident and answers
// "k best items for these n query rows" for any n, cut into batches.  Scores are bitwise those of topk_score_slice
// (topk_common.cuh), so Algo, validation and Par* share one ranking.
//   serve_slice_kernel : a CTA scores 32 gathered query rows against a slice of 1024 candidates.  Candidate rows (pool
//                        indirection resolved here) are staged in shared memory in tiles through cp.async.bulk on two
//                        mbarriers; a thread holds a 4 query x IR item register tile; each warp then radix-selects the
//                        slice's k best for its own 4 queries without block barriers.
//   topk_merge         : the merge of topk.cu, unchanged.
// The scoring tree, the warp select and the slice's shared-memory budget are in serve_common.cuh (the IVF search of
// ivf.cu runs them too).
//   serve_finish_kernel: candidate positions -> item ids through the pool, 0.0f scores on the -1 padding.
// The seen-aware calls (bfl_seen_topk*) leave each query's seen items out: serve_slice_seen_kernel marks them in a
// per-warp bitmask before its warp_select, which then never counts them and hands the merge rank keys and a count per
// slice (seen_merge); calls that go to the 4-query kernels run masked_topk on the gathered rows.  Both in
// seen_common.cuh / evaluate.cu.
#include <algorithm>
#include <climits>
#include <new>

#include "sm90_ptx.cuh"
#include "serve_common.cuh"

using namespace bfl;

namespace {

constexpr int64_t SV_SEEN_KEYS = (int64_t)1 << 24;  // seen keys per internal batch aimed at (a longer row is a batch)
constexpr int64_t SV_CAND_LIST = (int64_t)1 << 24;  // list entries per internal batch of bfl_cand_topk (likewise)

// A seen CSR on the device (END offsets, every row non-decreasing); query q of a batch reads row row[q], or row q.
struct SeenRows {
    const int64_t* indptr;
    const int32_t* keys;
    const int32_t* row;
};

// Qm rows are gathered through qidx (an index outside [0, n_qrows) reads as a zero row); candidate c of the slice is
// item row pool[c] (or c).  cand_i holds candidate POSITIONS (so ties resolve as on a gathered item matrix).
// SEEN: query q leaves out the items of row seen.row[q] (or q) of the sorted seen CSR; the slice's candidates go to
// cand_key / cand_cnt (rank keys and their number) instead of cand_v / cand_i.  The body of serve_slice_kernel and
// serve_slice_seen_kernel.
template <int IR, bool SEEN>
__device__ __forceinline__ void serve_slice(const float* __restrict__ Qm, int64_t n_qrows, int ldq,
                                            const int32_t* __restrict__ qidx, int nq, const float* __restrict__ It,
                                            int ldi, int64_t n_cand, const int32_t* __restrict__ pool,
                                            const float* __restrict__ bias, int d, int k, int nslices, int bulk,
                                            int tile_floats, float* __restrict__ cand_v, int32_t* __restrict__ cand_i,
                                            SeenRows seen, unsigned long long* __restrict__ cand_key,
                                            int32_t* __restrict__ cand_cnt) {
    constexpr int IT = 32 * IR;
    extern __shared__ __align__(128) float sv_smem[];
    __shared__ __align__(8) uint64_t bar[2];
    const int dpad = (d + 3) & ~3, pitch = tile_pitch(dpad);
    float* scores = sv_smem;                        // [SV_QT][SV_SLICE]
    float* qs = scores + SV_QT * SV_SLICE;          // [SV_QT][dpad]
    float* tiles = qs + SV_QT * dpad;               // [2][tile_floats]; the select histograms afterwards
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int slice = blockIdx.x;
    const int q0 = blockIdx.y * SV_QT;
    const int64_t i0 = (int64_t)slice * SV_SLICE;
    const int ni = (int)min((long long)SV_SLICE, (long long)(n_cand - i0));
    const int ntiles = (ni + IT - 1) / IT;

    if (tid == 0) {
        sm90::mbar_init(&bar[0], 1);
        sm90::mbar_init(&bar[1], 1);
        sm90::mbar_init_fence();
    }
    for (int e = tid; e < SV_QT * dpad; e += SV_THREADS) {
        const int qi = e / dpad, c = e - qi * dpad;
        float v = 0.f;
        if (q0 + qi < nq && c < d) {
            const int64_t r = qidx[q0 + qi];
            if (r >= 0 && r < n_qrows) v = Qm[r * ldq + c];
        }
        qs[e] = v;
    }
    __syncthreads();

    // warp 0 stages tile t with one bulk copy per row, all completing on bar[t & 1]
    auto stage_bulk = [&](int t) {
        const int nt = min(IT, ni - t * IT);
        float* dst = tiles + (t & 1) * tile_floats;
        if (lane == 0) sm90::mbar_arrive_expect_tx(&bar[t & 1], (uint32_t)nt * d * 4u);
        __syncwarp();
        for (int j = lane; j < nt; j += 32) {
            const int64_t c = i0 + t * IT + j;
            const int64_t row = pool ? pool[c] : c;
            sm90::cp_async_bulk_g2s(dst + j * pitch, It + row * ldi, (uint32_t)d * 4u, &bar[t & 1]);
        }
    };
    if (bulk && w == 0) stage_bulk(0);

    ScoreCtx s;
    s.q = qs + w * SV_QR * dpad;
    s.dpad = dpad;
    s.pitch = pitch;
    s.d = d;
    s.vec = (ldi & 3) == 0 && (d & 3) == 0;
    for (int t = 0; t < ntiles; ++t) {
        float* tile = tiles + (t & 1) * tile_floats;
        if (bulk) {
            if (w == 0 && t + 1 < ntiles) stage_bulk(t + 1);   // its buffer was released by the barrier ending tile t - 1
            sm90::mbar_wait(&bar[t & 1], (t >> 1) & 1);
        } else {
            const int nt = min(IT, ni - t * IT);
            for (int e = tid; e < nt * d; e += SV_THREADS) {
                const int j = e / d, c = e - j * d;
                const int64_t cp = i0 + t * IT + j;
                const int64_t row = pool ? pool[cp] : cp;
                tile[j * pitch + c] = It[row * ldi + c];
            }
            __syncthreads();
        }
        s.t = tile + lane * pitch;
        float acc[SV_QR][IR];
        tree<0, 0, IR>(s, acc);
#pragma unroll
        for (int b = 0; b < IR; ++b) {
            const int it = t * IT + b * 32 + lane;
            if (it < ni) {
                float bv = 0.f;
                if (bias) bv = bias[pool ? (int64_t)pool[i0 + it] : i0 + it];
#pragma unroll
                for (int a = 0; a < SV_QR; ++a) scores[(w * SV_QR + a) * SV_SLICE + it] = acc[a][b] + bv;
            }
        }
        __syncthreads();
    }
    unsigned* hist = reinterpret_cast<unsigned*>(tiles) + w * sel_words(SEEN);
    for (int a = 0; a < SV_QR; ++a) {
        const int q = q0 + w * SV_QR + a;
        if (q >= nq) break;
        const size_t o = ((size_t)q * nslices + slice) * k;
        if constexpr (SEEN) {
            // bit c of `bits`: candidate i0 + c is one of the query's seen items
            uint32_t* bits = hist + 256;
            const int64_t r = seen.row ? seen.row[q] : q;
            const int64_t b = seen_row_begin(seen.indptr, r), e = seen.indptr[r];
            bits[lane] = 0;
            __syncwarp();
            if (e > b && pool) {   // pool order is arbitrary: each candidate is looked up in the row
                for (int c0 = 0; c0 < ni; c0 += 32) {
                    const int c = c0 + lane;
                    const unsigned m = __ballot_sync(FULL, c < ni && row_contains(seen.keys, b, e, pool[i0 + c]));
                    if (lane == 0) bits[c0 >> 5] = m;
                }
            } else if (e > b) {    // the slice's seen items are one run of the sorted row
                const int64_t lo = warp_lower_bound(seen.keys, b, e, (int32_t)i0, lane);
                const int64_t hi = warp_lower_bound(seen.keys, lo, e, (int32_t)(i0 + ni), lane);
                mark_seen_range(seen.keys, lo, hi, i0, bits, lane, 32);
            }
            __syncwarp();
            warp_select<true>(scores + (w * SV_QR + a) * SV_SLICE, (int)i0, ni, k, nullptr, nullptr, hist, bits,
                              cand_key + o, cand_cnt + (size_t)q * nslices + slice);
        } else {
            warp_select<false>(scores + (w * SV_QR + a) * SV_SLICE, (int)i0, ni, k, cand_v + o, cand_i + o, hist);
        }
        __syncwarp();
    }
}

template <int IR>
__global__ void __launch_bounds__(SV_THREADS)
    serve_slice_kernel(const float* __restrict__ Qm, int64_t n_qrows, int ldq, const int32_t* __restrict__ qidx, int nq,
                       const float* __restrict__ It, int ldi, int64_t n_cand, const int32_t* __restrict__ pool,
                       const float* __restrict__ bias, int d, int k, int nslices, int bulk, int tile_floats,
                       float* __restrict__ cand_v, int32_t* __restrict__ cand_i) {
    serve_slice<IR, false>(Qm, n_qrows, ldq, qidx, nq, It, ldi, n_cand, pool, bias, d, k, nslices, bulk, tile_floats,
                           cand_v, cand_i, SeenRows{nullptr, nullptr, nullptr}, nullptr, nullptr);
}

template <int IR>
__global__ void __launch_bounds__(SV_THREADS)
    serve_slice_seen_kernel(const float* __restrict__ Qm, int64_t n_qrows, int ldq, const int32_t* __restrict__ qidx,
                            int nq, const float* __restrict__ It, int ldi, int64_t n_cand,
                            const int32_t* __restrict__ pool, const float* __restrict__ bias, int d, int k, int nslices,
                            int bulk, int tile_floats, SeenRows seen, unsigned long long* __restrict__ cand_key,
                            int32_t* __restrict__ cand_cnt) {
    serve_slice<IR, true>(Qm, n_qrows, ldq, qidx, nq, It, ldi, n_cand, pool, bias, d, k, nslices, bulk, tile_floats,
                          nullptr, nullptr, seen, cand_key, cand_cnt);
}

__global__ void serve_finish_kernel(int32_t* __restrict__ idx, float* __restrict__ val, size_t n,
                                    const int32_t* __restrict__ pool) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t c = idx[i];
    if (c < 0) {
        val[i] = 0.f;
    } else if (pool) {
        idx[i] = pool[c];
    }
}

// dst[r] = src[idx[r]] for rows of d floats (pitch ld on both sides, padding columns zero)
__global__ void serve_gather_rows_kernel(const float* __restrict__ src, int64_t n_src, int ld, const int32_t* __restrict__ idx,
                                         int64_t n, int d, float* __restrict__ dst) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n * ld) return;
    const int64_t r = e / ld;
    const int c = (int)(e - r * ld);
    const int64_t s = idx[r];
    dst[e] = (c < d && s >= 0 && s < n_src) ? src[s * ld + c] : 0.f;
}

// writes r to major[indptr[r - 1] .. indptr[r]) for every row r: the row ids the device radix sort orders by
__global__ void seen_row_ids_kernel(const int64_t* __restrict__ indptr, int64_t rows, int32_t* __restrict__ major) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < rows; r += warps)
        for (int64_t e = seen_row_begin(indptr, r) + lane; e < indptr[r]; e += 32) major[e] = (int32_t)r;
}

}  // namespace

struct bfl_serve {
    // items / queries: owned uploads of host arrays, or borrowed device memory
    DevBuf<float> own_items, own_bias, own_queries;
    const float *items = nullptr, *bias = nullptr, *queries = nullptr;
    const float* host_items = nullptr;              // the host array own_items mirrors (alias check of set_queries)
    int64_t n_items = 0, n_q = 0;
    int ldi = 0, ldq = 0, d = 0;
    DevBuf<int32_t> pool;
    int64_t n_pool = -1;                            // -1: no pool

    int num_sms = 0;
    cudaStream_t compute = nullptr, copy = nullptr;
    cudaEvent_t scored[2] = {nullptr, nullptr}, copied[2] = {nullptr, nullptr};
    DevBuf<float> cand_v;
    DevBuf<int32_t> cand_i;
    DevBuf<int32_t> qidx;
    DevBuf<int32_t> out_i[2];
    DevBuf<float> out_v[2];
    DevBuf<float> gq, gi, gb;                       // gathered rows for the widths the batch kernel does not take
    int32_t* pin_i[2] = {nullptr, nullptr};
    float* pin_v[2] = {nullptr, nullptr};
    size_t pin_cap = 0;
    // seen-aware calls: candidate rank keys and counts of the batch kernel; the batch's seen rows as uploaded (sp / sk,
    // staged through two pinned slots) and, for rows given unsorted, the device radix sort's scratch and output
    DevBuf<unsigned long long> cand_k;
    DevBuf<int32_t> cand_cnt;
    DevBuf<int64_t> sp, sorted_sp;
    DevBuf<int32_t> sk, sorted_sk, sort_major;
    DevBuf<float> sort_vals;
    cudaEvent_t staged[2] = {nullptr, nullptr};
    int64_t* pin_sp[2] = {nullptr, nullptr};
    int32_t* pin_sk[2] = {nullptr, nullptr};
    size_t pin_sp_cap = 0, pin_sk_cap = 0;
    // candidate-list calls (candidates.cu): the batch's lists as uploaded (cp / ck, staged through their own two pinned
    // slots), the work list (unit_end / key_end); the rank keys and counts go to cand_k / cand_cnt
    DevBuf<int64_t> cp;
    DevBuf<int32_t> ck;
    DevBuf<long long> unit_end, key_end;
    cudaEvent_t cstaged[2] = {nullptr, nullptr};
    int64_t* pin_cp[2] = {nullptr, nullptr};
    int32_t* pin_ck[2] = {nullptr, nullptr};
    size_t pin_cp_cap = 0, pin_ck_cap = 0;
    int64_t cand_budget = 0;                        // list entries per batch; 0: SV_CAND_LIST

    int attach() {
        if (compute) return BFL_OK;
        if (BFL_OK != require_device()) return BFL_ERR_CUDA;
        int dev = 0;
        BFL_CUDA(cudaGetDevice(&dev));
        BFL_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
        BFL_CUDA(cudaStreamCreateWithFlags(&compute, cudaStreamNonBlocking));
        BFL_CUDA(cudaStreamCreateWithFlags(&copy, cudaStreamNonBlocking));
        for (int s = 0; s < 2; ++s) {
            BFL_CUDA(cudaEventCreateWithFlags(&scored[s], cudaEventDisableTiming));
            BFL_CUDA(cudaEventCreateWithFlags(&copied[s], cudaEventDisableTiming));
            BFL_CUDA(cudaEventCreateWithFlags(&staged[s], cudaEventDisableTiming));
            BFL_CUDA(cudaEventCreateWithFlags(&cstaged[s], cudaEventDisableTiming));
        }
        return BFL_OK;
    }
    int reserve_pinned(size_t n) {
        if (n <= pin_cap) return BFL_OK;
        release_pinned();
        for (int s = 0; s < 2; ++s) {
            BFL_CUDA(cudaMallocHost(&pin_i[s], n * sizeof(int32_t)));
            BFL_CUDA(cudaMallocHost(&pin_v[s], n * sizeof(float)));
        }
        pin_cap = n;
        return BFL_OK;
    }
    void release_pinned() {
        for (int s = 0; s < 2; ++s) {
            if (pin_i[s]) cudaFreeHost(pin_i[s]);
            if (pin_v[s]) cudaFreeHost(pin_v[s]);
            pin_i[s] = nullptr;
            pin_v[s] = nullptr;
        }
        pin_cap = 0;
    }
    // the two pinned slots the seen rows of a batch are staged in: rows END offsets and n_keys keys each
    int reserve_seen_pinned(size_t rows, size_t n_keys) {
        return reserve_rows_pinned(rows, n_keys, pin_sp, pin_sk, pin_sp_cap, pin_sk_cap);
    }
    void release_seen_pinned() { release_rows_pinned(pin_sp, pin_sk, pin_sp_cap, pin_sk_cap); }
    static int reserve_rows_pinned(size_t rows, size_t n_keys, int64_t** pp, int32_t** pk, size_t& cap_p, size_t& cap_k) {
        if (rows <= cap_p && n_keys <= cap_k) return BFL_OK;
        release_rows_pinned(pp, pk, cap_p, cap_k);
        for (int s = 0; s < 2; ++s) {
            BFL_CUDA(cudaMallocHost(&pp[s], rows * sizeof(int64_t)));
            BFL_CUDA(cudaMallocHost(&pk[s], n_keys * sizeof(int32_t)));
        }
        cap_p = rows;
        cap_k = n_keys;
        return BFL_OK;
    }
    static void release_rows_pinned(int64_t** pp, int32_t** pk, size_t& cap_p, size_t& cap_k) {
        for (int s = 0; s < 2; ++s) {
            if (pp[s]) cudaFreeHost(pp[s]);
            if (pk[s]) cudaFreeHost(pk[s]);
            pp[s] = nullptr;
            pk[s] = nullptr;
        }
        cap_p = cap_k = 0;
    }
    ~bfl_serve() {
        if (compute) cudaStreamSynchronize(compute);
        if (copy) cudaStreamSynchronize(copy);
        release_pinned();
        release_seen_pinned();
        release_rows_pinned(pin_cp, pin_ck, pin_cp_cap, pin_ck_cap);
        for (int s = 0; s < 2; ++s) {
            if (scored[s]) cudaEventDestroy(scored[s]);
            if (copied[s]) cudaEventDestroy(copied[s]);
            if (staged[s]) cudaEventDestroy(staged[s]);
            if (cstaged[s]) cudaEventDestroy(cstaged[s]);
        }
        if (compute) cudaStreamDestroy(compute);
        if (copy) cudaStreamDestroy(copy);
    }

    // new items invalidate what was set relative to the old ones: the pool and the queries (which may alias the old
    // item buffer or be narrower than the new d)
    void items_changed() {
        n_pool = -1;
        own_queries.release();
        queries = nullptr;
        n_q = 0;
        ldq = 0;
    }
    int64_t n_cand() const { return n_pool >= 0 ? n_pool : n_items; }
    // The one place that picks the kernels for a batch of nb queries.  The batch kernel takes every width its
    // shared-memory tiles hold, except a call of fewer queries than one CTA's tile over more slices than the card has
    // SMs: such a call runs whole waves of mostly empty 32-query CTAs, and the 4-query kernels of topk.cu on gathered
    // rows answer it sooner (benchmarks/serve_bench.py --small, DESIGN.md 4.9).  Wider rows always go there.
    bool batch_kernel(int64_t nb) const {
        return d <= SV_DMAX && (nb >= SV_QT || (n_cand() + SV_SLICE - 1) / SV_SLICE <= num_sms);
    }
    int slice_len() const { return d <= SV_DMAX ? SV_SLICE : TK_SLICE; }
    // queries per internal batch for this k: the candidate scratch stays near SV_CAND_BYTES
    int64_t batch_rows(int k) const {
        const int64_t nsl = (n_cand() + slice_len() - 1) / slice_len();
        int64_t b = (int64_t)(SV_CAND_BYTES / ((size_t)nsl * k * 8));
        b = b / SV_QT * SV_QT;
        return b < SV_QT ? SV_QT : (b > SV_BATCH_MAX ? SV_BATCH_MAX : b);
    }
    int check_ready(int64_t n, int k, const void* a, const void* b) {
        if (!items || !queries) BFL_FAIL(BFL_ERR_STATE, "serve: set the items and the queries before topk");
        if (!a || !b || n <= 0) BFL_FAIL(BFL_ERR_ARG, "bad serve top-k arguments");
        if (k <= 0 || k > TK_KMAX) BFL_FAIL(BFL_ERR_ARG, "top-k: k must be in [1, 4096]");
        const int64_t nsl = (n_cand() + slice_len() - 1) / slice_len();
        if (nsl * k > INT_MAX) BFL_FAIL(BFL_ERR_ARG, "serve: too many candidates for this k");
        return BFL_OK;
    }
    // one batch, stream-ordered: d_qidx[0..nb) -> d_out_i / d_out_v [nb x k]; with seen rows, query q of the batch
    // leaves out the items of its row
    int run_batch(const int32_t* d_qidx, int64_t nb, int k, int32_t* d_out_i, float* d_out_v, cudaStream_t st,
                  const SeenRows* seen = nullptr);
    // one batch of candidate-list queries, stream-ordered: query q of the batch ranks its list (row q of `cand`) ->
    // d_out_i / d_out_v [nb x k]; n_units / n_keys: the batch's work-list totals, or -1 to read them back (synchronises)
    int run_cand_batch(const int32_t* d_qidx, int64_t nb, int k, const CandRows& cand, const CandRows* seen,
                       long long n_units, long long n_keys, int32_t* d_out_i, float* d_out_v, cudaStream_t st);
    // the host-array call of bfl_serve_topk, bfl_seen_topk (seen_indptr == nullptr: no seen rows) and bfl_cand_topk
    // (cand_indptr != nullptr: row i of the host CSR is query i's candidate list)
    int topk_host(const int32_t* query_idx, int64_t n, int k, int32_t* out_idx, float* out_val,
                  const int64_t* seen_indptr, const int32_t* seen_keys, const int64_t* cand_indptr = nullptr,
                  const int32_t* cand_keys = nullptr);
    // uploads the rows [r0, r0 + nb) of a host CSR through pinned slot s (pin_p / pin_k, released by event ev) into
    // dp / dk, offsets from 0, on `compute`
    int upload_rows(const int64_t* indptr, const int32_t* keys, int64_t r0, int64_t nb, int64_t* pin_p, int32_t* pin_k,
                    cudaEvent_t ev, DevBuf<int64_t>& dp, DevBuf<int32_t>& dk);
    // uploads the seen rows [r0, r0 + nb) of a host CSR through pinned slot s; sorts them on the device when unsorted
    int stage_seen(const int64_t* indptr, const int32_t* keys, int64_t r0, int64_t nb, bool unsorted, int s,
                   SeenRows* out);
};

int bfl::serve_gather_rows(const float* src, int64_t n_src, int ld, const int32_t* idx, int64_t n, int d, float* dst,
                           cudaStream_t st) {
    serve_gather_rows_kernel<<<(unsigned)((n * ld + 255) / 256), 256, 0, st>>>(src, n_src, ld, idx, n, d, dst);
    BFL_LAUNCHED();
    return BFL_OK;
}

int bfl_serve::run_batch(const int32_t* d_qidx, int64_t nb, int k, int32_t* d_out_i, float* d_out_v, cudaStream_t st,
                         const SeenRows* seen) {
    const int64_t nc = n_cand();
    const int32_t* dpool = n_pool >= 0 ? pool.p : nullptr;
    if (!batch_kernel(nb)) {
        const int ew = 256;
        if (BFL_OK != gq.reserve((size_t)nb * ldq)) return BFL_ERR_CUDA;
        serve_gather_rows_kernel<<<(unsigned)((nb * ldq + ew - 1) / ew), ew, 0, st>>>(queries, n_q, ldq, d_qidx, nb, d, gq.p);
        BFL_LAUNCHED();
        const float *it = items, *bs = bias;
        if (dpool) {
            if (BFL_OK != gi.reserve((size_t)nc * ldi)) return BFL_ERR_CUDA;
            serve_gather_rows_kernel<<<(unsigned)((nc * ldi + ew - 1) / ew), ew, 0, st>>>(items, n_items, ldi, dpool, nc, d, gi.p);
            BFL_LAUNCHED();
            it = gi.p;
            if (bias) {
                if (BFL_OK != gb.reserve((size_t)nc)) return BFL_ERR_CUDA;
                serve_gather_rows_kernel<<<(unsigned)((nc + ew - 1) / ew), ew, 0, st>>>(bias, n_items, 1, dpool, nc, 1, gb.p);
                BFL_LAUNCHED();
                bs = gb.p;
            }
        }
        const int rc = seen ? masked_topk(gq.p, nb, ldq, it, nc, ldi, bs, d, k, seen->indptr, seen->keys, seen->row,
                                          dpool, d_out_i, d_out_v, st)
                            : bfl_topk_device(gq.p, nb, ldq, it, nc, ldi, bs, d, k, d_out_i, d_out_v, st);
        if (rc != BFL_OK) return rc;
    } else {
        const int nslices = (int)((nc + SV_SLICE - 1) / SV_SLICE);
        const int ncand = nslices * k;
        if (seen ? (BFL_OK != cand_k.reserve((size_t)nb * ncand) || BFL_OK != cand_cnt.reserve((size_t)nb * nslices))
                 : (BFL_OK != cand_v.reserve((size_t)nb * ncand) || BFL_OK != cand_i.reserve((size_t)nb * ncand)))
            return BFL_ERR_CUDA;
        const int IR = d <= 128 ? 2 : 1;
        int tile_floats = 0;
        const size_t smem = slice_smem_bytes(d, IR, seen != nullptr, &tile_floats);
        // bulk copies need 16-byte aligned rows of a multiple of 16 bytes (bind_items_device checks the base address);
        // other row shapes are staged with plain loads
        const int bulk = (ldi & 3) == 0 && (d & 3) == 0;
        dim3 grid(nslices, (unsigned)((nb + SV_QT - 1) / SV_QT));
        if (seen) {
            auto kern = IR == 2 ? serve_slice_seen_kernel<2> : serve_slice_seen_kernel<1>;
            BFL_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            kern<<<grid, SV_THREADS, smem, st>>>(queries, n_q, ldq, d_qidx, (int)nb, items, ldi, nc, dpool, bias, d, k,
                                                 nslices, bulk, tile_floats, *seen, cand_k.p, cand_cnt.p);
        } else {
            auto kern = IR == 2 ? serve_slice_kernel<2> : serve_slice_kernel<1>;
            BFL_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            kern<<<grid, SV_THREADS, smem, st>>>(queries, n_q, ldq, d_qidx, (int)nb, items, ldi, nc, dpool, bias, d, k,
                                                 nslices, bulk, tile_floats, cand_v.p, cand_i.p);
        }
        BFL_LAUNCHED();
        const int rc = seen ? seen_merge(cand_k.p, cand_cnt.p, nb, nslices, k, d_out_i, d_out_v, st)
                            : topk_merge(cand_v.p, cand_i.p, nb, ncand, k, d_out_i, d_out_v, st);
        if (rc != BFL_OK) return rc;
    }
    const size_t n = (size_t)nb * k;
    serve_finish_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_out_i, d_out_v, n, dpool);
    BFL_LAUNCHED();
    return BFL_OK;
}

int bfl_serve::run_cand_batch(const int32_t* d_qidx, int64_t nb, int k, const CandRows& cand, const CandRows* seen,
                              long long n_units, long long n_keys, int32_t* d_out_i, float* d_out_v, cudaStream_t st) {
    if (BFL_OK != unit_end.reserve((size_t)nb) || BFL_OK != key_end.reserve((size_t)nb)) return BFL_ERR_CUDA;
    if (int rc = cand_plan(cand, nb, k, unit_end.p, key_end.p, st)) return rc;
    if (n_units < 0) {
        BFL_CUDA(cudaMemcpyAsync(&n_units, unit_end.p + nb - 1, sizeof(long long), cudaMemcpyDeviceToHost, st));
        BFL_CUDA(cudaMemcpyAsync(&n_keys, key_end.p + nb - 1, sizeof(long long), cudaMemcpyDeviceToHost, st));
        BFL_CUDA(cudaStreamSynchronize(st));
    }
    if (BFL_OK != cand_k.reserve((size_t)std::max(n_keys, 1ll)) || BFL_OK != cand_cnt.reserve((size_t)std::max(n_units, 1ll)))
        return BFL_ERR_CUDA;
    return cand_batch(queries, n_q, ldq, d_qidx, nb, items, ldi, bias, d, k, cand,
                      seen ? *seen : CandRows{nullptr, nullptr, nullptr, 0}, unit_end.p, key_end.p, n_units, cand_k.p,
                      cand_cnt.p, d_out_i, d_out_v, st);
}

int bfl_serve::upload_rows(const int64_t* indptr, const int32_t* keys, int64_t r0, int64_t nb, int64_t* pin_p,
                           int32_t* pin_k, cudaEvent_t ev, DevBuf<int64_t>& dp, DevBuf<int32_t>& dk) {
    const int64_t kb = r0 > 0 ? indptr[r0 - 1] : 0, nk = indptr[r0 + nb - 1] - kb;
    // the slot was last read by the upload of the batch before the previous one
    BFL_CUDA(cudaEventSynchronize(ev));
    memcpy(pin_k, keys + kb, sizeof(int32_t) * (size_t)nk);
    for (int64_t i = 0; i < nb; ++i) pin_p[i] = indptr[r0 + i] - kb;
    if (BFL_OK != dp.reserve((size_t)nb) || BFL_OK != dk.reserve((size_t)(nk > 0 ? nk : 1))) return BFL_ERR_CUDA;
    BFL_CUDA(cudaMemcpyAsync(dp.p, pin_p, sizeof(int64_t) * (size_t)nb, cudaMemcpyHostToDevice, compute));
    BFL_CUDA(cudaMemcpyAsync(dk.p, pin_k, sizeof(int32_t) * (size_t)nk, cudaMemcpyHostToDevice, compute));
    BFL_CUDA(cudaEventRecord(ev, compute));
    return BFL_OK;
}

int bfl_serve::stage_seen(const int64_t* indptr, const int32_t* keys, int64_t r0, int64_t nb, bool unsorted, int s,
                          SeenRows* out) {
    if (int rc = upload_rows(indptr, keys, r0, nb, pin_sp[s], pin_sk[s], staged[s], sp, sk)) return rc;
    const int64_t nk = indptr[r0 + nb - 1] - (r0 > 0 ? indptr[r0 - 1] : 0);
    *out = SeenRows{sp.p, sk.p, nullptr};
    if (!unsorted) return BFL_OK;
    // rows in session order (or with duplicates out of place): the device radix sort of the ingest path, by (row, key)
    if (BFL_OK != sorted_sp.reserve((size_t)nb) || BFL_OK != sorted_sk.reserve((size_t)nk) ||
        BFL_OK != sort_major.reserve((size_t)nk) || BFL_OK != sort_vals.reserve((size_t)nk))
        return BFL_ERR_CUDA;
    const unsigned g = (unsigned)std::min<int64_t>((nb + 7) / 8, 4096);
    seen_row_ids_kernel<<<g, 256, 0, compute>>>(sp.p, nb, sort_major.p);
    BFL_LAUNCHED();
    // the values ride along and are dropped: only the order of the keys is wanted
    const int rc = bfl_csr_from_triples_device(sort_major.p, sk.p, sort_vals.p, nk, (int32_t)nb, (int32_t)n_items, 1,
                                               sorted_sp.p, sorted_sk.p, sort_vals.p, compute);
    if (rc != BFL_OK) return rc;
    *out = SeenRows{sorted_sp.p, sorted_sk.p, nullptr};
    return BFL_OK;
}

int bfl_serve::topk_host(const int32_t* query_idx, int64_t n, int k, int32_t* out_idx, float* out_val,
                         const int64_t* seen_indptr, const int32_t* seen_keys, const int64_t* cand_indptr,
                         const int32_t* cand_keys) {
    int rc = BFL_OK;
    // batches of at most batch_rows(k) queries; with seen rows also of at most SV_SEEN_KEYS seen keys, with candidate
    // lists of at most cand_budget list entries, unless a single row holds more (it is then a batch of its own)
    const int64_t B = batch_rows(k) < n ? batch_rows(k) : n;
    const int64_t list_budget = cand_budget > 0 ? cand_budget : SV_CAND_LIST;
    std::vector<int64_t> start{0};
    int64_t max_keys = 1, max_list = 1;
    while (start.back() < n) {
        const int64_t b0 = start.back();
        int64_t e = n - b0 < B ? n : b0 + B;
        if (seen_indptr) {
            const int64_t kb = b0 > 0 ? seen_indptr[b0 - 1] : 0;
            e = std::max<int64_t>(b0 + 1, std::upper_bound(seen_indptr + b0, seen_indptr + e, kb + SV_SEEN_KEYS) - seen_indptr);
            max_keys = std::max<int64_t>(max_keys, seen_indptr[e - 1] - kb);
        }
        if (cand_indptr) {
            const int64_t cb = b0 > 0 ? cand_indptr[b0 - 1] : 0;
            e = std::max<int64_t>(b0 + 1, std::upper_bound(cand_indptr + b0, cand_indptr + e, cb + list_budget) - cand_indptr);
            max_list = std::max<int64_t>(max_list, cand_indptr[e - 1] - cb);
        }
        start.push_back(e);
    }
    const int64_t nbatch = (int64_t)start.size() - 1;
    // the work-list totals of each batch of candidate lists (as cand_units_kernel counts them)
    std::vector<long long> n_units(cand_indptr ? nbatch : 0, 0), n_keys(cand_indptr ? nbatch : 0, 0);
    long long max_units = 1, max_rank_keys = 1;
    for (int64_t b = 0; b < (int64_t)n_units.size(); ++b) {
        for (int64_t r = start[b]; r < start[b + 1]; ++r) {
            const int64_t len = cand_indptr[r] - (r > 0 ? cand_indptr[r - 1] : 0);
            const int64_t full = len / SV_SLICE, rest = len - full * SV_SLICE;
            n_units[b] += full + (rest > 0);
            n_keys[b] += full * std::min(k, SV_SLICE) + std::min<int64_t>(k, rest);
        }
        max_units = std::max(max_units, n_units[b]);
        max_rank_keys = std::max(max_rank_keys, n_keys[b]);
    }
    // batches holding a row that is not non-decreasing are sorted on the device
    std::vector<char> unsorted(seen_indptr ? nbatch : 0, 0);
    bool any_unsorted = false;
    for (int64_t b = 0; b < (int64_t)unsorted.size(); ++b) {
        for (int64_t r = start[b]; r < start[b + 1] && !unsorted[b]; ++r)
            for (int64_t e = (r > 0 ? seen_indptr[r - 1] : 0) + 1; e < seen_indptr[r]; ++e)
                if (seen_keys[e] < seen_keys[e - 1]) {
                    unsorted[b] = 1;
                    break;
                }
        any_unsorted |= unsorted[b] != 0;
    }
    const size_t per = (size_t)B * k;
    if (BFL_OK != qidx.reserve((size_t)n) || BFL_OK != reserve_pinned(per)) return BFL_ERR_CUDA;
    for (int s = 0; s < 2; ++s)
        if (BFL_OK != out_i[s].reserve(per) || BFL_OK != out_v[s].reserve(per)) return BFL_ERR_CUDA;
    // the seen buffers at their largest before the first batch: a reserve that grows frees a buffer kernels may read
    if (seen_indptr && (BFL_OK != reserve_seen_pinned((size_t)B, (size_t)max_keys) || BFL_OK != sp.reserve((size_t)B) ||
                        BFL_OK != sk.reserve((size_t)max_keys)))
        return BFL_ERR_CUDA;
    if (any_unsorted && (BFL_OK != sorted_sp.reserve((size_t)B) || BFL_OK != sorted_sk.reserve((size_t)max_keys) ||
                         BFL_OK != sort_major.reserve((size_t)max_keys) || BFL_OK != sort_vals.reserve((size_t)max_keys)))
        return BFL_ERR_CUDA;
    if (cand_indptr && (BFL_OK != reserve_rows_pinned((size_t)B, (size_t)max_list, pin_cp, pin_ck, pin_cp_cap, pin_ck_cap) ||
                        BFL_OK != cp.reserve((size_t)B) || BFL_OK != ck.reserve((size_t)max_list) ||
                        BFL_OK != unit_end.reserve((size_t)B) || BFL_OK != key_end.reserve((size_t)B) ||
                        BFL_OK != cand_k.reserve((size_t)max_rank_keys) || BFL_OK != cand_cnt.reserve((size_t)max_units)))
        return BFL_ERR_CUDA;
    BFL_CUDA(cudaMemcpyAsync(qidx.p, query_idx, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, compute));
    // batch b is scored on `compute` into slot b & 1 and copied to that slot's pinned buffers on `copy`; the host
    // drains batch b - 1 into the caller's arrays (and stages the seen rows of batch b + 1) while batch b runs
    auto drain = [&](int64_t b) -> int {
        const int s = (int)(b & 1);
        const int64_t b0 = start[b], nb = start[b + 1] - b0;
        BFL_CUDA(cudaEventSynchronize(copied[s]));
        memcpy(out_idx + b0 * k, pin_i[s], sizeof(int32_t) * (size_t)nb * k);
        if (out_val) memcpy(out_val + b0 * k, pin_v[s], sizeof(float) * (size_t)nb * k);
        return BFL_OK;
    };
    for (int64_t b = 0; b < nbatch; ++b) {
        const int s = (int)(b & 1);
        const int64_t b0 = start[b], nb = start[b + 1] - b0;
        SeenRows seen{};
        if (seen_indptr) rc = stage_seen(seen_indptr, seen_keys, b0, nb, unsorted[b] != 0, s, &seen);
        if (rc == BFL_OK && cand_indptr) {
            rc = upload_rows(cand_indptr, cand_keys, b0, nb, pin_cp[s], pin_ck[s], cstaged[s], cp, ck);
            const CandRows cand{cp.p, ck.p, nullptr, 0}, cseen{seen.indptr, seen.keys, nullptr, 0};
            if (rc == BFL_OK)
                rc = run_cand_batch(qidx.p + b0, nb, k, cand, seen_indptr ? &cseen : nullptr, n_units[b], n_keys[b],
                                    out_i[s].p, out_v[s].p, compute);
        } else if (rc == BFL_OK) {
            rc = run_batch(qidx.p + b0, nb, k, out_i[s].p, out_v[s].p, compute, seen_indptr ? &seen : nullptr);
        }
        if (rc == BFL_OK) {
            BFL_CUDA(cudaEventRecord(scored[s], compute));
            BFL_CUDA(cudaStreamWaitEvent(copy, scored[s], 0));
            BFL_CUDA(cudaMemcpyAsync(pin_i[s], out_i[s].p, sizeof(int32_t) * (size_t)nb * k, cudaMemcpyDeviceToHost,
                                     copy));
            BFL_CUDA(cudaMemcpyAsync(pin_v[s], out_v[s].p, sizeof(float) * (size_t)nb * k, cudaMemcpyDeviceToHost,
                                     copy));
            BFL_CUDA(cudaEventRecord(copied[s], copy));
            if (b > 0) rc = drain(b - 1);
        }
        if (rc != BFL_OK) {   // leave nothing in flight behind a failed call
            cudaStreamSynchronize(compute);
            cudaStreamSynchronize(copy);
            return rc;
        }
    }
    rc = drain(nbatch - 1);
    BFL_CUDA(cudaStreamSynchronize(compute));
    return rc;
}

extern "C" {

bfl_serve_t* bfl_serve_create(void) { return new (std::nothrow) bfl_serve(); }

void bfl_serve_destroy(bfl_serve_t* h) { delete h; }

static int check_matrix(const void* p, int64_t rows, int ld, int d) {
    if (!p || rows <= 0 || d <= 0 || ld < d) BFL_FAIL(BFL_ERR_ARG, "serve: bad matrix arguments");
    if (rows > INT_MAX) BFL_FAIL(BFL_ERR_ARG, "serve: the row count must be below 2^31");
    return BFL_OK;
}

int bfl_serve_bind_items_device(bfl_serve_t* h, const float* d_items, int64_t n_items, int ld, int d,
                                const float* d_item_bias) {
    if (!h) BFL_FAIL(BFL_ERR_ARG, "serve: null handle");
    if (BFL_OK != check_matrix(d_items, n_items, ld, d)) return BFL_ERR_ARG;
    // aligned-shaped rows are read 16 bytes at a time (float4 loads, bulk copies), as topk_score_slice reads them
    if ((ld & 3) == 0 && (d & 3) == 0 && ((uintptr_t)d_items & 15) != 0)
        BFL_FAIL(BFL_ERR_ARG, "serve: device item rows of a multiple of 4 floats must be 16-byte aligned");
    if (BFL_OK != h->attach()) return BFL_ERR_CUDA;
    h->items_changed();
    h->items = nullptr;
    h->own_items.release();
    h->own_bias.release();
    h->host_items = nullptr;
    h->items = d_items;
    h->bias = d_item_bias;
    h->n_items = n_items;
    h->ldi = ld;
    h->d = d;
    return BFL_OK;
}

int bfl_serve_set_items(bfl_serve_t* h, const float* items, int64_t n_items, int ld, int d, const float* item_bias) {
    if (!h) BFL_FAIL(BFL_ERR_ARG, "serve: null handle");
    if (BFL_OK != check_matrix(items, n_items, ld, d)) return BFL_ERR_ARG;
    if (BFL_OK != h->attach()) return BFL_ERR_CUDA;
    h->items_changed();
    h->items = nullptr;                             // stays unset if the upload below fails
    if (BFL_OK != h->own_items.reserve((size_t)n_items * ld)) return BFL_ERR_CUDA;
    BFL_CUDA(cudaMemcpy(h->own_items.p, items, sizeof(float) * (size_t)n_items * ld, cudaMemcpyHostToDevice));
    if (item_bias) {
        if (BFL_OK != h->own_bias.reserve((size_t)n_items)) return BFL_ERR_CUDA;
        BFL_CUDA(cudaMemcpy(h->own_bias.p, item_bias, sizeof(float) * (size_t)n_items, cudaMemcpyHostToDevice));
    }
    h->host_items = items;
    h->items = h->own_items.p;
    h->bias = item_bias ? h->own_bias.p : nullptr;
    h->n_items = n_items;
    h->ldi = ld;
    h->d = d;
    return BFL_OK;
}

int bfl_serve_bind_queries_device(bfl_serve_t* h, const float* d_queries, int64_t n_q, int ld) {
    if (!h) BFL_FAIL(BFL_ERR_ARG, "serve: null handle");
    if (!h->items) BFL_FAIL(BFL_ERR_STATE, "serve: set the items before the queries");
    if (BFL_OK != check_matrix(d_queries, n_q, ld, h->d)) return BFL_ERR_ARG;
    h->own_queries.release();
    h->queries = d_queries;
    h->n_q = n_q;
    h->ldq = ld;
    return BFL_OK;
}

int bfl_serve_set_queries(bfl_serve_t* h, const float* queries, int64_t n_q, int ld) {
    if (!h) BFL_FAIL(BFL_ERR_ARG, "serve: null handle");
    if (!h->items) BFL_FAIL(BFL_ERR_STATE, "serve: set the items before the queries");
    if (BFL_OK != check_matrix(queries, n_q, ld, h->d)) return BFL_ERR_ARG;
    if (queries == h->host_items && n_q == h->n_items && ld == h->ldi) {   // most_similar: one resident copy
        h->own_queries.release();
        h->queries = h->items;
    } else {
        if (BFL_OK != h->own_queries.reserve((size_t)n_q * ld)) return BFL_ERR_CUDA;
        BFL_CUDA(cudaMemcpy(h->own_queries.p, queries, sizeof(float) * (size_t)n_q * ld, cudaMemcpyHostToDevice));
        h->queries = h->own_queries.p;
    }
    h->n_q = n_q;
    h->ldq = ld;
    return BFL_OK;
}

int bfl_serve_set_pool(bfl_serve_t* h, const int32_t* pool_idx, int64_t n_pool) {
    if (!h) BFL_FAIL(BFL_ERR_ARG, "serve: null handle");
    if (!h->items) BFL_FAIL(BFL_ERR_STATE, "serve: set the items before the pool");
    if (!pool_idx) {
        h->n_pool = -1;
        return BFL_OK;
    }
    if (n_pool <= 0) BFL_FAIL(BFL_ERR_ARG, "serve: pool is empty");
    if (n_pool > INT_MAX) BFL_FAIL(BFL_ERR_ARG, "serve: the pool must hold fewer than 2^31 indices");
    for (int64_t i = 0; i < n_pool; ++i)
        if (pool_idx[i] < 0 || pool_idx[i] >= h->n_items) BFL_FAIL(BFL_ERR_ARG, "serve: pool index out of range");
    if (BFL_OK != h->pool.reserve((size_t)n_pool)) return BFL_ERR_CUDA;
    BFL_CUDA(cudaMemcpy(h->pool.p, pool_idx, sizeof(int32_t) * (size_t)n_pool, cudaMemcpyHostToDevice));
    h->n_pool = n_pool;
    return BFL_OK;
}

int bfl_serve_topk_device(bfl_serve_t* h, const int32_t* d_query_idx, int64_t n, int k, int32_t* d_out_idx,
                          float* d_out_val, void* stream) {
    if (!h) BFL_FAIL(BFL_ERR_ARG, "serve: null handle");
    int rc = h->check_ready(n, k, d_query_idx, d_out_idx);
    if (rc != BFL_OK) return rc;
    if (!d_out_val) BFL_FAIL(BFL_ERR_ARG, "serve: the device variant needs d_out_val");
    const int64_t B = h->batch_rows(k);
    for (int64_t b0 = 0; b0 < n; b0 += B) {
        const int64_t nb = n - b0 < B ? n - b0 : B;
        rc = h->run_batch(d_query_idx + b0, nb, k, d_out_idx + b0 * k, d_out_val + b0 * k, (cudaStream_t)stream);
        if (rc != BFL_OK) return rc;
    }
    return BFL_OK;
}

int bfl_serve_topk(bfl_serve_t* h, const int32_t* query_idx, int64_t n, int k, int32_t* out_idx, float* out_val) {
    if (!h) BFL_FAIL(BFL_ERR_ARG, "serve: null handle");
    int rc = h->check_ready(n, k, query_idx, out_idx);
    if (rc != BFL_OK) return rc;
    for (int64_t i = 0; i < n; ++i)
        if (query_idx[i] < 0 || query_idx[i] >= h->n_q) BFL_FAIL(BFL_ERR_ARG, "serve: query index out of range");
    return h->topk_host(query_idx, n, k, out_idx, out_val, nullptr, nullptr);
}

// n rows of a host CSR of item ids ("seen" or "candidate" rows): END offsets non-decreasing from 0, keys in the items
static int check_rows(const bfl_serve_t* h, const int64_t* indptr, const int32_t* keys, int64_t n, const char* what) {
    const std::string w(what);
    if (!indptr) BFL_FAIL(BFL_ERR_ARG, "serve: the " + w + " rows need their END offsets");
    int64_t prev = 0;
    for (int64_t i = 0; i < n; ++i) {
        if (indptr[i] < prev) BFL_FAIL(BFL_ERR_ARG, "serve: " + w + " END offsets must be non-decreasing from 0");
        prev = indptr[i];
    }
    if (prev > 0 && !keys) BFL_FAIL(BFL_ERR_ARG, "serve: " + w + " keys missing");
    for (int64_t e = 0; e < prev; ++e)
        if (keys[e] < 0 || keys[e] >= h->n_items) BFL_FAIL(BFL_ERR_ARG, "serve: " + w + " key out of range");
    return BFL_OK;
}

static int check_query_idx(const bfl_serve_t* h, const int32_t* query_idx, int64_t n) {
    for (int64_t i = 0; i < n; ++i)
        if (query_idx[i] < 0 || query_idx[i] >= h->n_q) BFL_FAIL(BFL_ERR_ARG, "serve: query index out of range");
    return BFL_OK;
}

int bfl_seen_topk(bfl_serve_t* h, const int32_t* query_idx, int64_t n, int k, const int64_t* seen_indptr,
                  const int32_t* seen_keys, int32_t* out_idx, float* out_val) {
    if (!h) BFL_FAIL(BFL_ERR_ARG, "serve: null handle");
    int rc = h->check_ready(n, k, query_idx, out_idx);
    if (rc != BFL_OK) return rc;
    if (!seen_indptr) BFL_FAIL(BFL_ERR_ARG, "serve: the seen rows need their END offsets");
    if (BFL_OK != check_query_idx(h, query_idx, n) || BFL_OK != check_rows(h, seen_indptr, seen_keys, n, "seen"))
        return BFL_ERR_ARG;
    return h->topk_host(query_idx, n, k, out_idx, out_val, seen_indptr, seen_keys);
}

int bfl_seen_topk_device(bfl_serve_t* h, const int32_t* d_query_idx, int64_t n, int k, const int64_t* d_seen_indptr,
                         const int32_t* d_seen_keys, const int32_t* d_seen_row, int32_t* d_out_idx, float* d_out_val,
                         void* stream) {
    if (!h) BFL_FAIL(BFL_ERR_ARG, "serve: null handle");
    int rc = h->check_ready(n, k, d_query_idx, d_out_idx);
    if (rc != BFL_OK) return rc;
    if (!d_out_val) BFL_FAIL(BFL_ERR_ARG, "serve: the device variant needs d_out_val");
    if (!d_seen_indptr || !d_seen_keys || !d_seen_row) BFL_FAIL(BFL_ERR_ARG, "serve: bad seen rows");
    const int64_t B = h->batch_rows(k);
    for (int64_t b0 = 0; b0 < n; b0 += B) {
        const int64_t nb = n - b0 < B ? n - b0 : B;
        const SeenRows seen{d_seen_indptr, d_seen_keys, d_seen_row + b0};
        rc = h->run_batch(d_query_idx + b0, nb, k, d_out_idx + b0 * k, d_out_val + b0 * k, (cudaStream_t)stream, &seen);
        if (rc != BFL_OK) return rc;
    }
    return BFL_OK;
}

int bfl_cand_topk(bfl_serve_t* h, const int32_t* query_idx, int64_t n, int k, const int64_t* cand_indptr,
                  const int32_t* cand_keys, const int64_t* seen_indptr, const int32_t* seen_keys, int32_t* out_idx,
                  float* out_val) {
    if (!h) BFL_FAIL(BFL_ERR_ARG, "serve: null handle");
    int rc = h->check_ready(n, k, query_idx, out_idx);
    if (rc != BFL_OK) return rc;
    if (BFL_OK != check_query_idx(h, query_idx, n) || BFL_OK != check_rows(h, cand_indptr, cand_keys, n, "candidate") ||
        (seen_indptr && BFL_OK != check_rows(h, seen_indptr, seen_keys, n, "seen")))
        return BFL_ERR_ARG;
    return h->topk_host(query_idx, n, k, out_idx, out_val, seen_indptr, seen_keys, cand_indptr, cand_keys);
}

int bfl_cand_topk_device(bfl_serve_t* h, const int32_t* d_query_idx, int64_t n, int k, const int64_t* d_cand_indptr,
                         const int32_t* d_cand_keys, const int32_t* d_cand_row, const int64_t* d_seen_indptr,
                         const int32_t* d_seen_keys, const int32_t* d_seen_row, int32_t* d_out_idx, float* d_out_val,
                         void* stream) {
    if (!h) BFL_FAIL(BFL_ERR_ARG, "serve: null handle");
    int rc = h->check_ready(n, k, d_query_idx, d_out_idx);
    if (rc != BFL_OK) return rc;
    if (!d_cand_indptr || !d_cand_keys) BFL_FAIL(BFL_ERR_ARG, "serve: bad candidate rows");
    if (d_seen_indptr && !d_seen_keys) BFL_FAIL(BFL_ERR_ARG, "serve: bad seen rows");
    const int64_t B = h->batch_rows(k);
    for (int64_t b0 = 0; b0 < n; b0 += B) {
        const int64_t nb = n - b0 < B ? n - b0 : B;
        const CandRows cand{d_cand_indptr, d_cand_keys, d_cand_row ? d_cand_row + b0 : nullptr, b0};
        const CandRows seen{d_seen_indptr, d_seen_keys, d_seen_row ? d_seen_row + b0 : nullptr, b0};
        rc = h->run_cand_batch(d_query_idx + b0, nb, k, cand, d_seen_indptr ? &seen : nullptr, -1, -1,
                               d_out_idx + b0 * k, d_out_val ? d_out_val + b0 * k : nullptr, (cudaStream_t)stream);
        if (rc != BFL_OK) return rc;
    }
    return BFL_OK;
}

int bfl_mmr_rerank_device(bfl_serve_t* h, const int32_t* d_cand_idx, const float* d_cand_val, int64_t n, int m,
                          int k, float diversify, int32_t* d_out_idx, float* d_out_val, void* stream) {
    if (!h) BFL_FAIL(BFL_ERR_ARG, "serve: null handle");
    if (!d_cand_idx || !d_cand_val || !d_out_idx || !d_out_val || n < 0)
        BFL_FAIL(BFL_ERR_ARG, "mmr: bad arguments");
    if (m < 1 || m > 256 || k < 1 || k > m) BFL_FAIL(BFL_ERR_ARG, "mmr: need 1 <= k <= m <= 256");
    if (!(diversify >= 0.f && diversify <= 1.f)) BFL_FAIL(BFL_ERR_ARG, "mmr: diversify must be in [0, 1]");
    if (n > INT_MAX) BFL_FAIL(BFL_ERR_ARG, "mmr: too many rows in one call");
    if (!h->items) BFL_FAIL(BFL_ERR_STATE, "mmr: set the items first");
    return mmr_rerank(h->items, h->ldi, h->d, d_cand_idx, d_cand_val, n, m, k, diversify, d_out_idx, d_out_val,
                      (cudaStream_t)stream);
}

int bfl_cand_set_budget(bfl_serve_t* h, int64_t list_entries) {
    if (!h || list_entries < 0) BFL_FAIL(BFL_ERR_ARG, "serve: bad candidate budget");
    h->cand_budget = list_entries;
    return BFL_OK;
}

}  // extern "C"
