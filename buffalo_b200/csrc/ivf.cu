// Inverted-file (IVF-Flat) index for batch serving (DESIGN.md 4.12): the rows are clustered by spherical k-means into
// nlist lists, and a query scores only the rows of the nprobe lists whose centroids it scores best.  Every scored pair
// gets the exact path's fp32 score bits and every candidate the exact path's 64-bit rank key, so nprobe = nlist returns
// bfl_serve_topk's answer bit for bit.
//   Build:  ivf_inv_norm_kernel (1 / |row|), ivf_seed_kernel (the drawn unit rows), then per iteration the assignment
//           (a bfl_serve top-1 of the rows against the centroids), the members grouped by list with the device radix
//           sort and ivf_update_kernel (ordered sums, no atomics).  A last assignment makes the lists; the rows, ids and
//           bias are gathered list-major (serve_gather_rows).
//   Search: coarse (a bfl_serve top-nprobe of the queries against the centroids), the (query, list) pairs sorted by
//           list, ivf_fine_kernel (a CTA scores up to 32 queries probing one list against one 1024-row chunk of it,
//           serve_slice's scoring and warp select), seen_merge over each query's chunk slots.
#include <algorithm>
#include <climits>
#include <functional>
#include <new>

#include "sm90_ptx.cuh"
#include "serve_common.cuh"

using namespace bfl;

namespace {

constexpr int IVF_MAX_LISTS = 65536;

// inv[r] = 1 / |row r| (0 for a zero row): one warp per row, lane-strided squares summed by warp_sum
__global__ void ivf_inv_norm_kernel(const float* __restrict__ X, int64_t n, int ld, int d, float* __restrict__ inv) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n; r += warps) {
        float s = 0.f;
        for (int c = lane; c < d; c += 32) s = fmaf(X[r * ld + c], X[r * ld + c], s);
        s = warp_sum(s);
        if (lane == 0) inv[r] = s > 0.f ? 1.f / sqrtf(s) : 0.f;
    }
}

// centroid l = unit row pick[l]; padding columns zero
__global__ void ivf_seed_kernel(const float* __restrict__ X, int ld, int d, const float* __restrict__ inv,
                                const int32_t* __restrict__ pick, int nlist, float* __restrict__ cent) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (int64_t)nlist * ld) return;
    const int l = (int)(e / ld), c = (int)(e - (int64_t)l * ld);
    const int64_t r = pick[l];
    cent[e] = c < d ? X[r * ld + c] * inv[r] : 0.f;
}

__global__ void ivf_iota_kernel(int32_t* __restrict__ a, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) a[i] = (int32_t)i;
}

// One CTA per list: the sum of the member unit rows in ascending row order (thread c owns column c), then divided by
// its norm (a fixed shared-memory tree).  An empty list, or one whose sum is zero, keeps its previous centroid.
__global__ void __launch_bounds__(SV_DMAX) ivf_update_kernel(const float* __restrict__ X, int ld, int d,
                                                              const float* __restrict__ inv,
                                                              const int64_t* __restrict__ indptr,
                                                              const int32_t* __restrict__ members,
                                                              float* __restrict__ cent) {
    __shared__ float red[SV_DMAX];
    const int l = blockIdx.x, c = threadIdx.x;
    const int64_t b = l > 0 ? indptr[l - 1] : 0, e = indptr[l];
    float s = 0.f;
    if (c < d)
        for (int64_t m = b; m < e; ++m) {
            const int64_t r = members[m];
            s += X[r * ld + c] * inv[r];
        }
    red[c] = s * s;
    __syncthreads();
    for (int o = SV_DMAX / 2; o > 0; o >>= 1) {
        if (c < o) red[c] += red[c + o];
        __syncthreads();
    }
    const float nrm = sqrtf(red[0]);
    if (e > b && nrm > 0.f && c < d) cent[(int64_t)l * ld + c] = s / nrm;
}

// probe j of every query is list j (nprobe = nlist)
__global__ void ivf_all_lists_kernel(int32_t* __restrict__ probes, int64_t nb, int nlist) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nb * nlist) probes[i] = (int32_t)(i % nlist);
}

// slot[q * nprobe + j] = the first candidate slot of query q's j-th probe: its lists' chunk counts summed in probe order
__global__ void ivf_slots_kernel(const int32_t* __restrict__ probes, int64_t nb, int nprobe,
                                 const int32_t* __restrict__ chunks, int32_t* __restrict__ slot) {
    const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nb) return;
    int32_t s = 0;
    for (int j = 0; j < nprobe; ++j) {
        slot[q * nprobe + j] = s;
        s += chunks[probes[q * nprobe + j]];
    }
}

// work[l] = CTAs of list l: ceil(pairs / SV_QT) query groups times its chunk count
__global__ void ivf_work_kernel(const int64_t* __restrict__ pind, const int32_t* __restrict__ chunks, int nlist,
                                long long* __restrict__ work) {
    const int l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= nlist) return;
    const int64_t np = pind[l] - (l > 0 ? pind[l - 1] : 0);
    work[l] = (long long)((np + SV_QT - 1) / SV_QT) * chunks[l];
}

// One CTA per (list l, group of up to SV_QT of the queries probing it, chunk of SV_SLICE of its rows).  Rows are the
// list-major copy L (pitch ld); query q of the batch is row q of Qm.  Scores are serve_slice's (tree / leaf); each
// query's chunk goes through warp_select as rank keys of list-major positions, which are then rewritten to the row ids
// (ascending within a list, so the order of the keys does not change) and stored in the query's slot for the chunk.
template <int IR>
__global__ void __launch_bounds__(SV_THREADS)
    ivf_fine_kernel(const float* __restrict__ Qm, int ldq, const float* __restrict__ L, int ld,
                    const float* __restrict__ lbias, const int32_t* __restrict__ lids,
                    const int64_t* __restrict__ loff, const int32_t* __restrict__ chunks,
                    const int64_t* __restrict__ pind, const int32_t* __restrict__ pairs,
                    const int32_t* __restrict__ slot, int nprobe, const long long* __restrict__ work, int nlist, int d,
                    int k, int nslots, int bulk, int tile_floats, unsigned long long* __restrict__ cand_key,
                    int32_t* __restrict__ cand_cnt) {
    constexpr int IT = 32 * IR;
    extern __shared__ __align__(128) float sv_smem[];
    __shared__ __align__(8) uint64_t bar[2];
    const int dpad = (d + 3) & ~3, pitch = tile_pitch(dpad);
    float* scores = sv_smem;                        // [SV_QT][SV_SLICE]
    float* qs = scores + SV_QT * SV_SLICE;          // [SV_QT][dpad]
    float* tiles = qs + SV_QT * dpad;               // [2][tile_floats]; the select scratch afterwards
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;

    // the work item: list l holds CTAs [work[l - 1], work[l])
    const long long wi = blockIdx.x;
    int lo = 0, hi = nlist - 1;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (work[mid] > wi) hi = mid;
        else lo = mid + 1;
    }
    const int l = lo;
    const long long r = wi - (l > 0 ? work[l - 1] : 0);
    const int nch = chunks[l];
    const int g = (int)(r / nch), ch = (int)(r - (long long)g * nch);
    const int64_t p0 = (l > 0 ? pind[l - 1] : 0) + (int64_t)g * SV_QT;
    const int nq = (int)min((int64_t)SV_QT, pind[l] - p0);
    const int64_t i0 = (l > 0 ? loff[l - 1] : 0) + (int64_t)ch * SV_SLICE;
    const int ni = (int)min((int64_t)SV_SLICE, loff[l] - i0);
    const int ntiles = (ni + IT - 1) / IT;

    if (tid == 0) {
        sm90::mbar_init(&bar[0], 1);
        sm90::mbar_init(&bar[1], 1);
        sm90::mbar_init_fence();
    }
    for (int e = tid; e < SV_QT * dpad; e += SV_THREADS) {
        const int qi = e / dpad, c = e - qi * dpad;
        float v = 0.f;
        if (qi < nq && c < d) v = Qm[(int64_t)(pairs[p0 + qi] / nprobe) * ldq + c];
        qs[e] = v;
    }
    __syncthreads();

    auto stage_bulk = [&](int t) {
        const int nt = min(IT, ni - t * IT);
        float* dst = tiles + (t & 1) * tile_floats;
        if (lane == 0) sm90::mbar_arrive_expect_tx(&bar[t & 1], (uint32_t)nt * d * 4u);
        __syncwarp();
        for (int j = lane; j < nt; j += 32)
            sm90::cp_async_bulk_g2s(dst + j * pitch, L + (i0 + t * IT + j) * ld, (uint32_t)d * 4u, &bar[t & 1]);
    };
    if (bulk && w == 0) stage_bulk(0);

    ScoreCtx s;
    s.q = qs + w * SV_QR * dpad;
    s.dpad = dpad;
    s.pitch = pitch;
    s.d = d;
    s.vec = (ld & 3) == 0 && (d & 3) == 0;
    for (int t = 0; t < ntiles; ++t) {
        float* tile = tiles + (t & 1) * tile_floats;
        if (bulk) {
            if (w == 0 && t + 1 < ntiles) stage_bulk(t + 1);
            sm90::mbar_wait(&bar[t & 1], (t >> 1) & 1);
        } else {
            const int nt = min(IT, ni - t * IT);
            for (int e = tid; e < nt * d; e += SV_THREADS) {
                const int j = e / d, c = e - j * d;
                tile[j * pitch + c] = L[(i0 + t * IT + j) * ld + c];
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
                const float bv = lbias ? lbias[i0 + it] : 0.f;
#pragma unroll
                for (int a = 0; a < SV_QR; ++a) scores[(w * SV_QR + a) * SV_SLICE + it] = acc[a][b] + bv;
            }
        }
        __syncthreads();
    }
    unsigned* hist = reinterpret_cast<unsigned*>(tiles) + w * sel_words(true);
    uint32_t* bits = hist + 256;                    // no candidate is left out
    bits[lane] = 0;
    __syncwarp();
    for (int a = 0; a < SV_QR; ++a) {
        const int qi = w * SV_QR + a;
        if (qi >= nq) break;
        const int32_t pr = pairs[p0 + qi];
        const size_t o = (size_t)(pr / nprobe) * nslots + slot[pr] + ch;
        warp_select<true>(scores + qi * SV_SLICE, (int)i0, ni, k, nullptr, nullptr, hist, bits, cand_key + o * k,
                          cand_cnt + o);
        __syncwarp();
        const int cnt = min(ni, k);
        for (int i = lane; i < cnt; i += 32) {
            const unsigned long long key = cand_key[o * k + i];
            cand_key[o * k + i] = (key & 0xffffffff00000000ull) | (uint32_t)lids[(uint32_t)key];
        }
        __syncwarp();
    }
}

uint64_t splitmix64(uint64_t& x) {
    uint64_t z = (x += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

unsigned blocks_for(int64_t n, int t = 256) { return (unsigned)((n + t - 1) / t); }

}  // namespace

struct bfl_ivf {
    int64_t n = 0;
    int ld = 0, d = 0, nlist = 0;
    bool built = false;
    DevBuf<float> cent;                             // [nlist][ld] unit centroids
    DevBuf<int64_t> offs;                           // [nlist] END offsets of the lists
    DevBuf<int32_t> ids;                            // [n] row ids, list-major, ascending within a list
    DevBuf<float> rows;                             // [n][ld] the original rows, list-major
    DevBuf<float> bias;                             // [n] list-major bias (has_bias)
    bool has_bias = false;
    DevBuf<int32_t> chunks;                         // [nlist] SV_SLICE-row chunks per list
    std::vector<int64_t> h_offs;
    std::vector<int64_t> top_slots;                 // [nlist + 1]: chunk slots the nprobe longest lists need
    bfl_serve_t* coarse = nullptr;                  // top-k over the centroids
    int num_sms = 0;
    int64_t batch_cap = 0;                          // 0: automatic
    cudaStream_t st = nullptr;
    // search scratch
    DevBuf<int32_t> probes, slot, iota, pairs;
    DevBuf<float> pval, dummy;
    DevBuf<int64_t> pind;
    DevBuf<long long> work;
    DevBuf<unsigned long long> cand_k;
    DevBuf<int32_t> cand_cnt;

    int attach() {
        if (st) return BFL_OK;
        if (BFL_OK != require_device()) return BFL_ERR_CUDA;
        int dev = 0;
        BFL_CUDA(cudaGetDevice(&dev));
        BFL_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
        BFL_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
        if (!coarse) coarse = bfl_serve_create();
        if (!coarse) BFL_FAIL(BFL_ERR_CUDA, "ivf: out of host memory");
        return BFL_OK;
    }
    ~bfl_ivf() {
        if (st) cudaStreamSynchronize(st);
        bfl_serve_destroy(coarse);
        if (st) cudaStreamDestroy(st);
    }
    // list id of every row against the current centroids (top-1, ties to the smaller list) -> assign[0..n)
    int assign_rows(const float* X, int32_t* assign) {
        if (BFL_OK != bfl_serve_bind_items_device(coarse, cent.p, nlist, ld, d, nullptr)) return BFL_ERR_CUDA;
        if (BFL_OK != bfl_serve_bind_queries_device(coarse, X, n, ld)) return BFL_ERR_CUDA;
        return bfl_serve_topk_device(coarse, iota.p, n, 1, assign, pval.p, st);
    }
    int build(const float* X, int64_t n_rows, int ld_, int d_, const float* b, int nlist_, int iters, uint64_t seed);
    int search(const float* Q, int64_t nq, int ldq, int nprobe, int k, bool use_bias, int32_t* out_i, float* out_v,
               cudaStream_t caller);
};

int bfl_ivf::build(const float* X, int64_t n_rows, int ld_, int d_, const float* b, int nlist_, int iters,
                   uint64_t seed) {
    built = false;
    n = n_rows;
    ld = ld_;
    d = d_;
    nlist = nlist_;
    // the caller's rows may have been written on any stream
    BFL_CUDA(cudaDeviceSynchronize());
    DevBuf<float> inv;
    DevBuf<int32_t> assign, members, pick;
    if (BFL_OK != inv.reserve(n) || BFL_OK != assign.reserve(n) || BFL_OK != members.reserve(n) ||
        BFL_OK != pick.reserve(nlist) || BFL_OK != iota.reserve(n) || BFL_OK != pval.reserve(n) ||
        BFL_OK != dummy.reserve(n) || BFL_OK != cent.reserve((size_t)nlist * ld) || BFL_OK != offs.reserve(nlist) ||
        BFL_OK != ids.reserve(n) || BFL_OK != rows.reserve((size_t)n * ld) || BFL_OK != chunks.reserve(nlist))
        return BFL_ERR_CUDA;
    has_bias = b != nullptr;
    if (has_bias && BFL_OK != bias.reserve(n)) return BFL_ERR_CUDA;
    // nlist distinct rows: the first nlist draws of a partial Fisher-Yates shuffle seeded with `seed`
    std::vector<int32_t> perm(n);
    for (int64_t i = 0; i < n; ++i) perm[i] = (int32_t)i;
    uint64_t state = seed;
    for (int i = 0; i < nlist; ++i) std::swap(perm[i], perm[i + (int64_t)(splitmix64(state) % (uint64_t)(n - i))]);
    BFL_CUDA(cudaMemcpyAsync(pick.p, perm.data(), sizeof(int32_t) * nlist, cudaMemcpyHostToDevice, st));
    ivf_inv_norm_kernel<<<blocks_for(n * 32), 256, 0, st>>>(X, n, ld, d, inv.p);
    BFL_LAUNCHED();
    ivf_seed_kernel<<<blocks_for((int64_t)nlist * ld), 256, 0, st>>>(X, ld, d, inv.p, pick.p, nlist, cent.p);
    BFL_LAUNCHED();
    ivf_iota_kernel<<<blocks_for(n), 256, 0, st>>>(iota.p, n);
    BFL_LAUNCHED();
    BFL_CUDA(cudaMemsetAsync(dummy.p, 0, sizeof(float) * n, st));
    // members of each list in ascending row order: a stable sort by list of the rows in row order
    auto group = [&]() -> int {
        if (int rc = assign_rows(X, assign.p)) return rc;
        return bfl_csr_from_triples_device(assign.p, iota.p, dummy.p, n, nlist, (int32_t)n, 0, offs.p, members.p,
                                           pval.p, st);
    };
    for (int it = 0; it < iters; ++it) {
        if (int rc = group()) return rc;
        ivf_update_kernel<<<nlist, SV_DMAX, 0, st>>>(X, ld, d, inv.p, offs.p, members.p, cent.p);
        BFL_LAUNCHED();
    }
    if (int rc = group()) return rc;
    BFL_CUDA(cudaMemcpyAsync(ids.p, members.p, sizeof(int32_t) * n, cudaMemcpyDeviceToDevice, st));
    if (int rc = serve_gather_rows(X, n, ld, ids.p, n, d, rows.p, st)) return rc;
    if (has_bias)
        if (int rc = serve_gather_rows(b, n, 1, ids.p, n, 1, bias.p, st)) return rc;
    h_offs.resize(nlist);
    BFL_CUDA(cudaMemcpyAsync(h_offs.data(), offs.p, sizeof(int64_t) * nlist, cudaMemcpyDeviceToHost, st));
    BFL_CUDA(cudaStreamSynchronize(st));
    std::vector<int32_t> nch(nlist);
    for (int l = 0; l < nlist; ++l) {
        const int64_t len = h_offs[l] - (l > 0 ? h_offs[l - 1] : 0);
        nch[l] = (int32_t)((len + SV_SLICE - 1) / SV_SLICE);
    }
    BFL_CUDA(cudaMemcpy(chunks.p, nch.data(), sizeof(int32_t) * nlist, cudaMemcpyHostToDevice));
    std::sort(nch.begin(), nch.end(), std::greater<int32_t>());
    top_slots.assign(nlist + 1, 0);
    for (int l = 0; l < nlist; ++l) top_slots[l + 1] = top_slots[l] + nch[l];
    built = true;
    return BFL_OK;
}

int bfl_ivf::search(const float* Q, int64_t nq, int ldq, int nprobe, int k, bool use_bias, int32_t* out_i,
                    float* out_v, cudaStream_t caller) {
    // the caller's queries may have been written on `caller`
    BFL_CUDA(cudaStreamSynchronize(caller));
    const int nslots = (int)std::max<int64_t>(top_slots[nprobe], 1);
    // queries per batch: candidate keys and counts, and the pair arrays with the radix sort's scratch
    const size_t per = (size_t)nslots * k * 8 + (size_t)nslots * 4 + (size_t)nprobe * 48;
    int64_t B = (int64_t)(SV_CAND_BYTES / per);
    B = std::max<int64_t>(1, std::min<int64_t>(B, SV_BATCH_MAX));
    if (batch_cap > 0) B = std::min(B, batch_cap);
    B = std::min(B, nq);
    const int64_t npair = B * nprobe;
    if (npair > INT_MAX) BFL_FAIL(BFL_ERR_ARG, "ivf: too many probes for one query batch");
    if (BFL_OK != probes.reserve(npair) || BFL_OK != slot.reserve(npair) || BFL_OK != pairs.reserve(npair) ||
        BFL_OK != dummy.reserve(npair) || BFL_OK != pval.reserve(std::max<int64_t>(npair, n)) ||
        BFL_OK != iota.reserve(std::max<int64_t>(std::max(npair, nq), n)) || BFL_OK != pind.reserve(nlist) ||
        BFL_OK != work.reserve(nlist) || BFL_OK != cand_k.reserve((size_t)B * nslots * k) ||
        BFL_OK != cand_cnt.reserve((size_t)B * nslots))
        return BFL_ERR_CUDA;
    ivf_iota_kernel<<<blocks_for(iota.cap), 256, 0, st>>>(iota.p, (int64_t)iota.cap);
    BFL_LAUNCHED();
    if (nprobe < nlist) {
        if (BFL_OK != bfl_serve_bind_items_device(coarse, cent.p, nlist, ld, d, nullptr)) return BFL_ERR_CUDA;
        if (BFL_OK != bfl_serve_bind_queries_device(coarse, Q, nq, ldq)) return BFL_ERR_CUDA;
    }
    const int IR = d <= 128 ? 2 : 1;
    int tile_floats = 0;
    const size_t smem = slice_smem_bytes(d, IR, true, &tile_floats);
    auto kern = IR == 2 ? ivf_fine_kernel<2> : ivf_fine_kernel<1>;
    BFL_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int bulk = (ld & 3) == 0 && (d & 3) == 0;
    for (int64_t b0 = 0; b0 < nq; b0 += B) {
        const int64_t nb = std::min(B, nq - b0), np = nb * nprobe;
        if (nprobe < nlist) {
            if (int rc = bfl_serve_topk_device(coarse, iota.p + b0, nb, nprobe, probes.p, pval.p, st)) return rc;
        } else {
            ivf_all_lists_kernel<<<blocks_for(np), 256, 0, st>>>(probes.p, nb, nlist);
            BFL_LAUNCHED();
        }
        ivf_slots_kernel<<<blocks_for(nb), 256, 0, st>>>(probes.p, nb, nprobe, chunks.p, slot.p);
        BFL_LAUNCHED();
        // the pairs of each list in query order
        if (int rc = bfl_csr_from_triples_device(probes.p, iota.p, pval.p, np, nlist, (int32_t)np, 0, pind.p, pairs.p,
                                                 dummy.p, st))
            return rc;
        ivf_work_kernel<<<blocks_for(nlist), 256, 0, st>>>(pind.p, chunks.p, nlist, work.p);
        BFL_LAUNCHED();
        if (int rc = inclusive_scan_i64(work.p, work.p, nlist, st)) return rc;
        BFL_CUDA(cudaMemsetAsync(cand_cnt.p, 0, sizeof(int32_t) * (size_t)nb * nslots, st));
        long long total = 0;
        BFL_CUDA(cudaMemcpyAsync(&total, work.p + nlist - 1, sizeof(long long), cudaMemcpyDeviceToHost, st));
        BFL_CUDA(cudaStreamSynchronize(st));
        if (total > INT_MAX) BFL_FAIL(BFL_ERR_ARG, "ivf: too much work for one query batch");
        if (total > 0) {
            kern<<<(unsigned)total, SV_THREADS, smem, st>>>(Q + b0 * ldq, ldq, rows.p, ld, use_bias ? bias.p : nullptr,
                                                            ids.p, offs.p, chunks.p, pind.p, pairs.p, slot.p, nprobe,
                                                            work.p, nlist, d, k, nslots, bulk, tile_floats, cand_k.p,
                                                            cand_cnt.p);
            BFL_LAUNCHED();
        }
        if (int rc = seen_merge(cand_k.p, cand_cnt.p, nb, nslots, k, out_i + b0 * k, out_v + b0 * k, st)) return rc;
    }
    BFL_CUDA(cudaStreamSynchronize(st));
    return BFL_OK;
}

extern "C" {

bfl_ivf_t* bfl_ivf_create(void) { return new (std::nothrow) bfl_ivf(); }

void bfl_ivf_destroy(bfl_ivf_t* h) { delete h; }

int bfl_ivf_attach(bfl_ivf_t* h) {
    if (!h) BFL_FAIL(BFL_ERR_ARG, "ivf: null handle");
    return h->attach();
}

int bfl_ivf_build_device(bfl_ivf_t* h, const float* d_rows, int64_t n, int ld, int d, const float* d_bias, int nlist,
                         int iters, uint64_t seed) {
    if (!h) BFL_FAIL(BFL_ERR_ARG, "ivf: null handle");
    if (!d_rows || n <= 0 || n > INT_MAX || d <= 0 || ld < d) BFL_FAIL(BFL_ERR_ARG, "ivf: bad row arguments");
    if (d > SV_DMAX) BFL_FAIL(BFL_ERR_ARG, "ivf: rows of at most 256 floats");
    if (nlist < 1 || nlist > std::min<int64_t>(n, IVF_MAX_LISTS)) BFL_FAIL(BFL_ERR_ARG, "ivf: nlist must be in [1, min(rows, 65536)]");
    if (iters < 1) BFL_FAIL(BFL_ERR_ARG, "ivf: iters must be at least 1");
    if ((ld & 3) == 0 && (d & 3) == 0 && ((uintptr_t)d_rows & 15) != 0)
        BFL_FAIL(BFL_ERR_ARG, "ivf: device rows of a multiple of 4 floats must be 16-byte aligned");
    if (BFL_OK != h->attach()) return BFL_ERR_CUDA;
    const int rc = h->build(d_rows, n, ld, d, d_bias, nlist, iters, seed);
    if (rc != BFL_OK) cudaStreamSynchronize(h->st);
    return rc;
}

int bfl_ivf_search_device(bfl_ivf_t* h, const float* d_queries, int64_t n, int ldq, int nprobe, int k, int use_bias,
                          int32_t* d_out_idx, float* d_out_val, void* stream) {
    if (!h) BFL_FAIL(BFL_ERR_ARG, "ivf: null handle");
    if (!h->built) BFL_FAIL(BFL_ERR_STATE, "ivf: build the index before searching it");
    if (!d_queries || n <= 0 || n > INT_MAX || ldq < h->d || !d_out_idx || !d_out_val)
        BFL_FAIL(BFL_ERR_ARG, "ivf: bad search arguments");
    if (nprobe < 1 || nprobe > h->nlist) BFL_FAIL(BFL_ERR_ARG, "ivf: nprobe must be in [1, nlist]");
    if (nprobe > TK_KMAX && nprobe != h->nlist) BFL_FAIL(BFL_ERR_ARG, "ivf: nprobe above 4096 must be nlist");
    if (k < 1 || k > TK_KMAX) BFL_FAIL(BFL_ERR_ARG, "ivf: k must be in [1, 4096]");
    if (use_bias && !h->has_bias) BFL_FAIL(BFL_ERR_ARG, "ivf: the index holds no bias");
    const int rc = h->search(d_queries, n, ldq, nprobe, k, use_bias != 0, d_out_idx, d_out_val, (cudaStream_t)stream);
    if (rc != BFL_OK) cudaStreamSynchronize(h->st);
    return rc;
}

int bfl_ivf_set_batch_rows(bfl_ivf_t* h, int64_t rows) {
    if (!h || rows < 0) BFL_FAIL(BFL_ERR_ARG, "ivf: bad batch rows");
    h->batch_cap = rows;
    return BFL_OK;
}

int bfl_ivf_info(bfl_ivf_t* h, int64_t* n, int* nlist, int* ld, int* d) {
    if (!h || !n || !nlist || !ld || !d) BFL_FAIL(BFL_ERR_ARG, "ivf: bad info arguments");
    if (!h->built) BFL_FAIL(BFL_ERR_STATE, "ivf: no index built");
    *n = h->n;
    *nlist = h->nlist;
    *ld = h->ld;
    *d = h->d;
    return BFL_OK;
}

int bfl_ivf_read(bfl_ivf_t* h, float* centroids, int64_t* offsets, int32_t* ids) {
    if (!h) BFL_FAIL(BFL_ERR_ARG, "ivf: null handle");
    if (!h->built) BFL_FAIL(BFL_ERR_STATE, "ivf: no index built");
    if (centroids)
        BFL_CUDA(cudaMemcpy(centroids, h->cent.p, sizeof(float) * (size_t)h->nlist * h->ld, cudaMemcpyDeviceToHost));
    if (offsets) memcpy(offsets, h->h_offs.data(), sizeof(int64_t) * (size_t)h->nlist);
    if (ids) BFL_CUDA(cudaMemcpy(ids, h->ids.p, sizeof(int32_t) * (size_t)h->n, cudaMemcpyDeviceToHost));
    return BFL_OK;
}

}  // extern "C"
