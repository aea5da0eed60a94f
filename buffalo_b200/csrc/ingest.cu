// Device-side ingest helpers (SURVEY.md 8(f-1), 8(f-4)), hand-written, no library sort:
//   * CSR build from (row, col, val) triples: a stable LSD radix sort (8-bit digits) of the combined (major, minor) key
//     + histogram/scan of the major index -> `indptr` (exclusive END offsets), `key`, `val` in the reference's layout
//     (buffalo/data/base.py:187-192; ordering of fileio.hpp:330-341: by (row, col) resp. (col, row), duplicates kept).
//     Replaces the text -> temp files -> parallel sort pipeline's sort/compress stage (fileio.hpp:263-419, mm.py:236-279).
//   * cumulative popularity table of BPRMF.prepare_sampling (buffalo/algo/bpr.py:99-111): histogram of the item keys,
//     integer power, inclusive scan.
//   * the core the two device text parsers share (text_ingest.cuh): handle setup, staging, the stage clock and the
//     CSR build into host arrays.
// Sort pass = per-warp digit histograms over contiguous sub-tiles, one exclusive scan of the digit-major counter
// matrix, and a stable scatter in which every warp walks its sub-tile in order and ranks equal digits with
// __match_any_sync -- no atomics on the data path, so the result is deterministic.
#include <algorithm>
#include <vector>

#include "bfl_common.cuh"
#include "text_ingest.cuh"

using namespace bfl;

namespace {

constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 8;                      // per thread
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

// ---- int64 inclusive scan (three kernels) ------------------------------------------------------
__device__ __forceinline__ long long block_exclusive_scan(long long v, long long* total, long long* warp_buf) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    long long inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const long long t = __shfl_up_sync(FULL, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) warp_buf[w] = inc;
    __syncthreads();
    long long before = 0, tot = 0;
#pragma unroll
    for (int i = 0; i < SCAN_THREADS / 32; ++i) {
        const long long t = warp_buf[i];
        before += i < w ? t : 0;
        tot += t;
    }
    __syncthreads();
    *total = tot;
    return before + inc - v;
}

__global__ void __launch_bounds__(SCAN_THREADS) scan_tiles_kernel(const long long* __restrict__ in, long long* __restrict__ out,
                                                                  long long n, long long* __restrict__ tile_sums) {
    __shared__ long long wb[SCAN_THREADS / 32];
    const long long base = (long long)blockIdx.x * SCAN_TILE + (long long)threadIdx.x * SCAN_ITEMS;
    long long v[SCAN_ITEMS], s = 0;
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i) {
        v[i] = base + i < n ? in[base + i] : 0;
        s += v[i];
    }
    long long tot;
    long long run = block_exclusive_scan(s, &tot, wb);
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i) {
        run += v[i];
        if (base + i < n) out[base + i] = run;     // inclusive within the tile
    }
    if (threadIdx.x == 0) tile_sums[blockIdx.x] = tot;
}
__global__ void __launch_bounds__(SCAN_THREADS) scan_add_kernel(long long* __restrict__ out, long long n,
                                                                const long long* __restrict__ tile_prefix) {
    const long long add = blockIdx.x == 0 ? 0 : tile_prefix[blockIdx.x - 1];
    const long long base = (long long)blockIdx.x * SCAN_TILE + (long long)threadIdx.x * SCAN_ITEMS;
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i)
        if (base + i < n) out[base + i] += add;
}

}  // namespace

namespace bfl {

// out[i] = in[0] + ... + in[i]; in == out allowed; recursion over the tile sums
int inclusive_scan_i64(const long long* in, long long* out, long long n, cudaStream_t st) {
    if (n <= 0) return BFL_OK;
    const long long tiles = (n + SCAN_TILE - 1) / SCAN_TILE;
    long long* sums = nullptr;
    BFL_CUDA(cudaMallocAsync(&sums, sizeof(long long) * tiles, st));
    scan_tiles_kernel<<<(unsigned)tiles, SCAN_THREADS, 0, st>>>(in, out, n, sums);
    BFL_LAUNCHED();
    if (tiles > 1) {
        const int rc = inclusive_scan_i64(sums, sums, tiles, st);
        if (rc != BFL_OK) return rc;
        scan_add_kernel<<<(unsigned)tiles, SCAN_THREADS, 0, st>>>(out, n, sums);
        BFL_LAUNCHED();
    }
    BFL_CUDA(cudaFreeAsync(sums, st));
    return BFL_OK;
}

}  // namespace bfl

namespace {

// ---- histograms ----------------------------------------------------------------------------------
__global__ void hist_i32_kernel(const int32_t* __restrict__ idx, long long n, long long* __restrict__ counts, int32_t nbins) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int32_t k = idx[i];
        if (k >= 0 && k < nbins) atomicAdd(reinterpret_cast<unsigned long long*>(counts + k), 1ull);
    }
}
__global__ void ipow_kernel(long long* __restrict__ t, long long n, int power) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long b = t[i];
        long long r = 1;
        for (int p = 0; p < power; ++p) r *= b;    // table **= int(power) (bpr.py:108); power 0 -> all ones
        t[i] = r;
    }
}

// ---- stable LSD radix sort of 64-bit keys with a float payload ---------------------------------------
constexpr int RS_THREADS = 256;                     // 8 warps per CTA
constexpr int RS_WARP_ITEMS = 8192;                 // contiguous sub-tile of one warp

__global__ void make_keys_kernel(const int32_t* __restrict__ major, const int32_t* __restrict__ minor, long long n,
                                 unsigned long long* __restrict__ keys) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        keys[i] = ((unsigned long long)(uint32_t)major[i] << 32) | (uint32_t)minor[i];
}

// counts[digit * nwarps + warp] = number of keys of the warp's sub-tile with that digit
__global__ void __launch_bounds__(RS_THREADS) rs_hist_kernel(const unsigned long long* __restrict__ keys, long long n, int shift,
                                                             long long nwarps, long long* __restrict__ counts) {
    __shared__ unsigned int h[RS_THREADS / 32][256];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const long long gw = (long long)blockIdx.x * (RS_THREADS / 32) + w;
    for (int i = lane; i < 256; i += 32) h[w][i] = 0;
    __syncwarp();
    if (gw < nwarps) {
        const long long b = gw * RS_WARP_ITEMS, e = min(n, b + RS_WARP_ITEMS);
        for (long long i = b + lane; i < e; i += 32) atomicAdd(&h[w][(unsigned)(keys[i] >> shift) & 255u], 1u);
        __syncwarp();
        for (int i = lane; i < 256; i += 32) counts[(long long)i * nwarps + gw] = h[w][i];
    }
}
// offsets = exclusive scan of counts (digit-major): position of the first key of (digit, warp)
__global__ void __launch_bounds__(RS_THREADS) rs_scatter_kernel(const unsigned long long* __restrict__ keys,
                                                                const float* __restrict__ vals, long long n, int shift,
                                                                long long nwarps, const long long* __restrict__ incl,
                                                                unsigned long long* __restrict__ keys_out,
                                                                float* __restrict__ vals_out) {
    __shared__ long long pos[RS_THREADS / 32][256];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const long long gw = (long long)blockIdx.x * (RS_THREADS / 32) + w;
    if (gw >= nwarps) return;
    for (int i = lane; i < 256; i += 32) {
        const long long flat = (long long)i * nwarps + gw;
        pos[w][i] = flat == 0 ? 0 : incl[flat - 1];          // exclusive prefix
    }
    __syncwarp();
    const long long b = gw * RS_WARP_ITEMS, e = min(n, b + RS_WARP_ITEMS);
    for (long long i0 = b; i0 < e; i0 += 32) {
        const long long i = i0 + lane;
        const bool ok = i < e;
        const unsigned long long k = ok ? keys[i] : 0ull;
        const unsigned dgt = ok ? ((unsigned)(k >> shift) & 255u) : 256u + lane;   // inactive lanes match nobody
        const unsigned same = __match_any_sync(FULL, dgt);
        const int rank = __popc(same & ((1u << lane) - 1u));
        long long p = 0;
        if (ok) p = pos[w][dgt] + rank;
        __syncwarp();
        if (ok && rank == 0) pos[w][dgt] += __popc(same);    // one leader per digit advances the cursor
        __syncwarp();
        if (ok) {
            keys_out[p] = k;
            vals_out[p] = vals[i];
        }
    }
}

__global__ void split_keys_kernel(const unsigned long long* __restrict__ keys, long long n, int32_t* __restrict__ minor_out) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        minor_out[i] = (int32_t)(uint32_t)(keys[i] & 0xffffffffull);
}

int bits_for(long long v) {
    int b = 0;
    while ((1ll << b) < v && b < 32) ++b;
    return std::max(b, 1);
}

}  // namespace

extern "C" {

// Cumulative popularity table on the device: cum[i] = sum_{j <= i} count(j)^power (int64), bpr.py:99-111.
int bfl_popularity_table_device(const int32_t* d_keys, int64_t nnz, int32_t n_items, int power, int64_t* d_cum, void* stream) {
    if (BFL_OK != require_device()) return BFL_ERR_CUDA;
    if (!d_cum || n_items <= 0 || nnz < 0 || (nnz > 0 && !d_keys) || power < 0) BFL_FAIL(BFL_ERR_ARG, "bad popularity-table arguments");
    cudaStream_t st = (cudaStream_t)stream;
    BFL_CUDA(cudaMemsetAsync(d_cum, 0, sizeof(int64_t) * n_items, st));
    if (nnz > 0) {
        hist_i32_kernel<<<grid_for(nnz), 256, 0, st>>>(d_keys, nnz, reinterpret_cast<long long*>(d_cum), n_items);
        BFL_LAUNCHED();
    }
    if (power != 1) {
        ipow_kernel<<<grid_for(n_items), 256, 0, st>>>(reinterpret_cast<long long*>(d_cum), n_items, power);
        BFL_LAUNCHED();
    }
    return inclusive_scan_i64(reinterpret_cast<long long*>(d_cum), reinterpret_cast<long long*>(d_cum), n_items, st);
}

int bfl_popularity_table_host(const int32_t* keys, int64_t nnz, int32_t n_items, int power, int64_t* cum) {
    if (BFL_OK != require_device()) return BFL_ERR_CUDA;
    if (!cum || n_items <= 0 || nnz < 0 || (nnz > 0 && !keys)) BFL_FAIL(BFL_ERR_ARG, "bad popularity-table arguments");
    DevBuf<int32_t> dk;
    DevBuf<int64_t> dc;
    if (BFL_OK != dk.reserve((size_t)std::max<int64_t>(nnz, 1)) || BFL_OK != dc.reserve((size_t)n_items)) return BFL_ERR_CUDA;
    if (nnz > 0) BFL_CUDA(cudaMemcpy(dk.p, keys, sizeof(int32_t) * (size_t)nnz, cudaMemcpyHostToDevice));
    const int rc = bfl_popularity_table_device(dk.p, nnz, n_items, power, dc.p, nullptr);
    if (rc != BFL_OK) return rc;
    BFL_CUDA(cudaDeviceSynchronize());
    BFL_CUDA(cudaMemcpy(cum, dc.p, sizeof(int64_t) * (size_t)n_items, cudaMemcpyDeviceToHost));
    return BFL_OK;
}

// CSR of one orientation from device triples: entries sorted by (major, minor) with a stable sort (equal pairs keep their
// input order), d_indptr[num_major] = exclusive end offsets, d_key_out = minor index, d_val_out = value.
// sort_minor == 0: stable sort by the major index only (Stream's internal_data_type="stream" keeps the token order).
int bfl_csr_from_triples_device(const int32_t* d_major, const int32_t* d_minor, const float* d_vals, int64_t nnz,
                                int32_t num_major, int32_t num_minor, int sort_minor, int64_t* d_indptr,
                                int32_t* d_key_out, float* d_val_out, void* stream) {
    if (BFL_OK != require_device()) return BFL_ERR_CUDA;
    if (!d_indptr || num_major <= 0 || num_minor <= 0 || nnz < 0) BFL_FAIL(BFL_ERR_ARG, "bad CSR-build arguments");
    if (nnz > 0 && (!d_major || !d_minor || !d_vals || !d_key_out || !d_val_out)) BFL_FAIL(BFL_ERR_ARG, "bad CSR-build arguments");
    cudaStream_t st = (cudaStream_t)stream;
    // indptr: histogram of the major index + inclusive scan
    BFL_CUDA(cudaMemsetAsync(d_indptr, 0, sizeof(int64_t) * num_major, st));
    if (nnz == 0) return BFL_OK;
    const int g = grid_for(nnz);
    hist_i32_kernel<<<g, 256, 0, st>>>(d_major, nnz, reinterpret_cast<long long*>(d_indptr), num_major);
    BFL_LAUNCHED();
    int rc = inclusive_scan_i64(reinterpret_cast<long long*>(d_indptr), reinterpret_cast<long long*>(d_indptr), num_major, st);
    if (rc != BFL_OK) return rc;
    // radix sort of (major << 32 | minor) carrying the value
    unsigned long long *k0 = nullptr, *k1 = nullptr;
    float* v1 = nullptr;
    long long* counts = nullptr;
    const long long nwarps = (nnz + RS_WARP_ITEMS - 1) / RS_WARP_ITEMS;
    BFL_CUDA(cudaMallocAsync(&k0, sizeof(unsigned long long) * nnz, st));
    BFL_CUDA(cudaMallocAsync(&k1, sizeof(unsigned long long) * nnz, st));
    BFL_CUDA(cudaMallocAsync(&v1, sizeof(float) * nnz, st));
    BFL_CUDA(cudaMallocAsync(&counts, sizeof(long long) * 256 * nwarps, st));
    make_keys_kernel<<<g, 256, 0, st>>>(d_major, d_minor, nnz, k0);
    BFL_LAUNCHED();
    BFL_CUDA(cudaMemcpyAsync(d_val_out, d_vals, sizeof(float) * nnz, cudaMemcpyDeviceToDevice, st));
    std::vector<int> shifts;
    if (sort_minor)
        for (int s = 0; s < bits_for(num_minor); s += 8) shifts.push_back(s);
    for (int s = 0; s < bits_for(num_major); s += 8) shifts.push_back(32 + s);
    unsigned long long *src = k0, *dst = k1;
    float *vsrc = d_val_out, *vdst = v1;
    const unsigned gb = (unsigned)((nwarps + RS_THREADS / 32 - 1) / (RS_THREADS / 32));
    for (int shift : shifts) {
        rs_hist_kernel<<<gb, RS_THREADS, 0, st>>>(src, nnz, shift, nwarps, counts);
        BFL_LAUNCHED();
        rc = inclusive_scan_i64(counts, counts, 256 * nwarps, st);
        if (rc != BFL_OK) return rc;
        rs_scatter_kernel<<<gb, RS_THREADS, 0, st>>>(src, vsrc, nnz, shift, nwarps, counts, dst, vdst);
        BFL_LAUNCHED();
        std::swap(src, dst);
        std::swap(vsrc, vdst);
    }
    split_keys_kernel<<<g, 256, 0, st>>>(src, nnz, d_key_out);
    BFL_LAUNCHED();
    if (vsrc != d_val_out) BFL_CUDA(cudaMemcpyAsync(d_val_out, vsrc, sizeof(float) * nnz, cudaMemcpyDeviceToDevice, st));
    BFL_CUDA(cudaFreeAsync(k0, st));
    BFL_CUDA(cudaFreeAsync(k1, st));
    BFL_CUDA(cudaFreeAsync(v1, st));
    BFL_CUDA(cudaFreeAsync(counts, st));
    return BFL_OK;
}

// host triples in, host CSR out (copies around bfl_csr_from_triples_device)
int bfl_csr_from_triples_host(const int32_t* major, const int32_t* minor, const float* vals, int64_t nnz, int32_t num_major,
                              int32_t num_minor, int sort_minor, int64_t* indptr, int32_t* key_out, float* val_out) {
    if (BFL_OK != require_device()) return BFL_ERR_CUDA;
    if (!indptr || num_major <= 0 || nnz < 0) BFL_FAIL(BFL_ERR_ARG, "bad CSR-build arguments");
    DevBuf<int32_t> dmj, dmn, dk;
    DevBuf<float> dv, dvo;
    DevBuf<int64_t> dind;
    const size_t n1 = (size_t)std::max<int64_t>(nnz, 1);
    if (BFL_OK != dmj.reserve(n1) || BFL_OK != dmn.reserve(n1) || BFL_OK != dk.reserve(n1) || BFL_OK != dv.reserve(n1) ||
        BFL_OK != dvo.reserve(n1) || BFL_OK != dind.reserve((size_t)num_major))
        return BFL_ERR_CUDA;
    if (nnz > 0) {
        BFL_CUDA(cudaMemcpy(dmj.p, major, sizeof(int32_t) * nnz, cudaMemcpyHostToDevice));
        BFL_CUDA(cudaMemcpy(dmn.p, minor, sizeof(int32_t) * nnz, cudaMemcpyHostToDevice));
        BFL_CUDA(cudaMemcpy(dv.p, vals, sizeof(float) * nnz, cudaMemcpyHostToDevice));
    }
    const int rc = bfl_csr_from_triples_device(dmj.p, dmn.p, dv.p, nnz, num_major, num_minor, sort_minor, dind.p, dk.p, dvo.p, nullptr);
    if (rc != BFL_OK) return rc;
    BFL_CUDA(cudaDeviceSynchronize());
    BFL_CUDA(cudaMemcpy(indptr, dind.p, sizeof(int64_t) * num_major, cudaMemcpyDeviceToHost));
    if (nnz > 0) {
        BFL_CUDA(cudaMemcpy(key_out, dk.p, sizeof(int32_t) * nnz, cudaMemcpyDeviceToHost));
        BFL_CUDA(cudaMemcpy(val_out, dvo.p, sizeof(float) * nnz, cudaMemcpyDeviceToHost));
    }
    return BFL_OK;
}

}  // extern "C"

// ---- core of the device text parsers (text_ingest.cuh) ------------------------------------------
namespace bfl {

int grid_for(long long n) {
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
        sms <= 0)
        sms = 1;
    return (int)std::max<long long>(1, std::min<long long>((n + 255) / 256, (long long)sms * 16));
}

TextIngest::~TextIngest() {
    if (comp) cudaStreamSynchronize(comp);
    for (int i = 0; i < 2; ++i) {
        if (host[i]) cudaFreeHost(host[i]);
        if (copied[i]) cudaEventDestroy(copied[i]);
    }
    for (auto& v : marks)
        for (cudaEvent_t e : v) cudaEventDestroy(e);
    if (comp) cudaStreamDestroy(comp);
}

bool setup(TextIngest* h, long long block_bytes, int stages) {
    h->block_bytes = block_bytes;
    h->marks.resize((size_t)stages);
    int dev = 0;
    uint64_t zero = 0;
    bool ok = cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetDefaultMemPool(&h->mem_pool, dev) == cudaSuccess &&
              cudaMemPoolSetAttribute(h->mem_pool, cudaMemPoolAttrUsedMemHigh, &zero) == cudaSuccess &&
              cudaStreamCreateWithFlags(&h->comp, cudaStreamNonBlocking) == cudaSuccess;
    for (int i = 0; ok && i < 2; ++i)
        ok = cudaHostAlloc(&h->host[i], (size_t)block_bytes, cudaHostAllocDefault) == cudaSuccess &&
             cudaEventCreateWithFlags(&h->copied[i], cudaEventDisableTiming) == cudaSuccess;
    return ok;
}

int mark(TextIngest* h, int stage, cudaStream_t st) {
    cudaEvent_t e;
    BFL_CUDA(cudaEventCreate(&e));
    h->marks[stage].push_back(e);
    BFL_CUDA(cudaEventRecord(e, st));
    return BFL_OK;
}

int staging(TextIngest* h, int slot, void** host_ptr) {
    if (!h || slot < 0 || slot > 1 || !host_ptr) BFL_FAIL(BFL_ERR_ARG, "bad staging arguments");
    if (h->copy_pending[slot]) BFL_CUDA(cudaEventSynchronize(h->copied[slot]));
    h->copy_pending[slot] = false;
    *host_ptr = h->host[slot];
    return BFL_OK;
}

int check_feed(TextIngest* h, int slot, long long n, int is_last) {
    if (!h || slot < 0 || slot > 1 || n < 0 || n > h->block_bytes) BFL_FAIL(BFL_ERR_ARG, "bad feed arguments");
    if (h->last_fed) BFL_FAIL(BFL_ERR_STATE, "feed after the last block");
    if (!is_last && (n == 0 || h->host[slot][n - 1] != '\n')) BFL_FAIL(BFL_ERR_ARG, "a block that is not the last must end with '\\n'");
    h->last_fed = is_last != 0;
    return BFL_OK;
}

int build_to_host(TextIngest* h, int orientation, const int32_t* row, const int32_t* col, const float* val, long long nnz,
                  int32_t num_rows, int32_t num_cols, int sort_minor, int csr_stage, int d2h_stage, int64_t* indptr,
                  int32_t* key, float* out_val) {
    const int32_t nmaj = orientation ? num_cols : num_rows, nmin = orientation ? num_rows : num_cols;
    int64_t* d_ind = nullptr;
    int32_t* d_key = nullptr;
    float* d_val = nullptr;
    const size_t m = (size_t)std::max<long long>(nnz, 1);
    BFL_CUDA(cudaMallocAsync(&d_ind, sizeof(int64_t) * nmaj, h->comp));
    BFL_CUDA(cudaMallocAsync(&d_key, sizeof(int32_t) * m, h->comp));
    BFL_CUDA(cudaMallocAsync(&d_val, sizeof(float) * m, h->comp));
    if (int rc = mark(h, csr_stage, h->comp)) return rc;
    int rc = bfl_csr_from_triples_device(orientation ? col : row, orientation ? row : col, val, nnz, nmaj, std::max(nmin, 1),
                                         sort_minor, d_ind, d_key, d_val, h->comp);
    if (rc != BFL_OK) return rc;
    if ((rc = mark(h, csr_stage, h->comp))) return rc;
    h->built[orientation] = true;
    if ((rc = mark(h, d2h_stage, h->comp))) return rc;
    BFL_CUDA(cudaMemcpyAsync(indptr, d_ind, sizeof(int64_t) * nmaj, cudaMemcpyDeviceToHost, h->comp));
    if (nnz) {
        BFL_CUDA(cudaMemcpyAsync(key, d_key, sizeof(int32_t) * nnz, cudaMemcpyDeviceToHost, h->comp));
        BFL_CUDA(cudaMemcpyAsync(out_val, d_val, sizeof(float) * nnz, cudaMemcpyDeviceToHost, h->comp));
    }
    if ((rc = mark(h, d2h_stage, h->comp))) return rc;
    BFL_CUDA(cudaFreeAsync(d_ind, h->comp));
    BFL_CUDA(cudaFreeAsync(d_key, h->comp));
    BFL_CUDA(cudaFreeAsync(d_val, h->comp));
    BFL_CUDA(cudaStreamSynchronize(h->comp));
    return BFL_OK;
}

int stats(TextIngest* h, double* stage_ms, int64_t* peak_bytes) {
    if (!h || !stage_ms || !peak_bytes) BFL_FAIL(BFL_ERR_ARG, "bad stats arguments");
    BFL_CUDA(cudaStreamSynchronize(h->comp));
    for (size_t s = 0; s < h->marks.size(); ++s) {
        double tot = 0.0;
        for (size_t i = 0; i + 1 < h->marks[s].size(); i += 2) {
            float ms = 0.f;
            BFL_CUDA(cudaEventElapsedTime(&ms, h->marks[s][i], h->marks[s][i + 1]));
            tot += ms;
        }
        stage_ms[s] = tot;
    }
    uint64_t hi = 0;
    BFL_CUDA(cudaMemPoolGetAttribute(h->mem_pool, cudaMemPoolAttrUsedMemHigh, &hi));
    *peak_bytes = (int64_t)hi;
    return BFL_OK;
}

}  // namespace bfl
