// Shared host/device helpers for the buffalo_b200 CUDA backend (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/buffalo_b200.h"

namespace bfl {

// ---------------------------------------------------------------------------------------
// error plumbing (replaces CHECK_CUDA's throw, include/buffalo/cuda/utils.cuh:24-31)
// ---------------------------------------------------------------------------------------
void set_error(const std::string& msg);
extern std::atomic<long long> g_launches;

#define BFL_CUDA(expr)                                                                       \
    do {                                                                                     \
        cudaError_t _e = (expr);                                                             \
        if (_e != cudaSuccess) {                                                             \
            bfl::set_error(std::string(#expr) + ": " + cudaGetErrorString(_e) + " (" +       \
                           __FILE__ + ":" + std::to_string(__LINE__) + ")");                 \
            return BFL_ERR_CUDA;                                                             \
        }                                                                                    \
    } while (0)

#define BFL_LAUNCHED()                                                                       \
    do {                                                                                     \
        bfl::g_launches.fetch_add(1, std::memory_order_relaxed);                             \
        BFL_CUDA(cudaGetLastError());                                                        \
    } while (0)

#define BFL_FAIL(code, msg)                                                                  \
    do {                                                                                     \
        bfl::set_error(msg);                                                                 \
        return (code);                                                                       \
    } while (0)

int require_device();  // BFL_OK iff a CUDA device of compute capability 9.0 is current

// out[i] = in[0] + ... + in[i] on `st` (in == out allowed); ingest.cu
int inclusive_scan_i64(const long long* in, long long* out, long long n, cudaStream_t st);

// ---------------------------------------------------------------------------------------
// minimal JSON reader for the option file (the reference uses json11, lib/algo.cc:19-37).
// Flat access to top-level scalars; nested objects/arrays are skipped.
// ---------------------------------------------------------------------------------------
struct JsonOpt {
    std::map<std::string, double> num;
    std::map<std::string, bool> boolean;
    std::map<std::string, std::string> str;
    bool parse(const std::string& text, std::string* err);
    bool load(const char* path, std::string* err);
    double number(const char* k, double dflt) const {
        auto it = num.find(k);
        if (it != num.end()) return it->second;
        auto ib = boolean.find(k);
        if (ib != boolean.end()) return ib->second ? 1.0 : 0.0;
        return dflt;
    }
    int integer(const char* k, int dflt) const { return (int)number(k, (double)dflt); }
    bool flag(const char* k, bool dflt) const {
        auto ib = boolean.find(k);
        if (ib != boolean.end()) return ib->second;
        auto it = num.find(k);
        if (it != num.end()) return it->second != 0.0;
        return dflt;
    }
    std::string string(const char* k, const char* dflt) const {
        auto it = str.find(k);
        return it != str.end() ? it->second : std::string(dflt);
    }
};

// device buffer with explicit ownership
template <typename T>
struct DevBuf {
    T* p = nullptr;
    size_t cap = 0;
    int reserve(size_t n) {
        if (n <= cap) return BFL_OK;
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
        BFL_CUDA(cudaMalloc(&p, n * sizeof(T)));
        cap = n;
        return BFL_OK;
    }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    ~DevBuf() { release(); }
};

#ifdef __CUDACC__
// ---------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------
constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
    return v;
}
// Warp-uniform broadcasts: all lanes already hold the same value, but routing it through lane 0 tells the
// compiler so; branches on the result are then uniform and shuffles under them stay plain SHFL instead of
// WARPSYNC.COLLECTIVE calls.
__device__ __forceinline__ int uni(int v) { return __shfl_sync(FULL, v, 0); }
__device__ __forceinline__ float uni(float v) { return __shfl_sync(FULL, v, 0); }
__device__ __forceinline__ bool uni(bool v) { return __shfl_sync(FULL, (int)v, 0) != 0; }
__device__ __forceinline__ long long uni(long long v) {
    const int lo = __shfl_sync(FULL, (int)(v & 0xffffffffll), 0), hi = __shfl_sync(FULL, (int)(v >> 32), 0);
    return ((long long)hi << 32) | (unsigned int)lo;
}
__device__ __forceinline__ int warp_id_uniform() { return __shfl_sync(FULL, (int)(threadIdx.x >> 5), 0); }

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
    return v;
}

// Philox4x32-10, identical to oracle/buffalo_oracle.c::philox4x32_10
__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                              uint32_t k0, uint32_t k1, uint32_t out[4]) {
#pragma unroll
    for (int i = 0; i < 10; ++i) {
        uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        uint32_t n0 = hi1 ^ c1 ^ k0;
        uint32_t n2 = hi0 ^ c3 ^ k1;
        c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}
__device__ __forceinline__ uint32_t draw_u32(uint32_t seed, uint32_t epoch, uint64_t idx, uint32_t t) {
    uint32_t o[4];
    philox4x32_10((uint32_t)idx, (uint32_t)(idx >> 32), t >> 2, epoch, seed, 0x5EEDu, o);
    return o[t & 3];
}
__device__ __forceinline__ int32_t draw_range(uint32_t seed, uint32_t epoch, uint64_t idx, uint32_t t,
                                              uint32_t range) {
    return (int32_t)__umulhi(draw_u32(seed, epoch, idx, t), range);
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}

// ---------------------------------------------------------------------------------------
// Deterministic loss: per-row terms (NV doubles per row, interleaved) summed by a fixed two-stage tree whose shape
// depends on the row count only.  Stage 1: fixed ranges of kLossRows rows, one CTA of 256 threads each.
// ---------------------------------------------------------------------------------------
constexpr int kLossRows = 4096;

template <int NV>
__global__ void __launch_bounds__(256) loss_tree_partial_kernel(const double* row_loss, int64_t n, double* part) {
    __shared__ double s[NV][256];
    const int64_t lo = (int64_t)blockIdx.x * kLossRows, hi = min(n, lo + kLossRows);
    double t[NV];
#pragma unroll
    for (int v = 0; v < NV; ++v) t[v] = 0.0;
    for (int64_t i = lo + threadIdx.x; i < hi; i += 256)
#pragma unroll
        for (int v = 0; v < NV; ++v) t[v] += row_loss[i * NV + v];
#pragma unroll
    for (int v = 0; v < NV; ++v) s[v][threadIdx.x] = t[v];
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o)
#pragma unroll
            for (int v = 0; v < NV; ++v) s[v][threadIdx.x] += s[v][threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x < NV) part[(int64_t)blockIdx.x * NV + threadIdx.x] = s[threadIdx.x][0];
}

// Stage 2 (one CTA of 256 threads): the partials by the same tree, added into loss[0 .. NV).
template <int NV>
__global__ void __launch_bounds__(256) loss_tree_final_kernel(const double* part, int64_t nblk, double* loss) {
    __shared__ double s[NV][256];
    double t[NV];
#pragma unroll
    for (int v = 0; v < NV; ++v) t[v] = 0.0;
    for (int64_t i = threadIdx.x; i < nblk; i += 256)
#pragma unroll
        for (int v = 0; v < NV; ++v) t[v] += part[i * NV + v];
#pragma unroll
    for (int v = 0; v < NV; ++v) s[v][threadIdx.x] = t[v];
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o)
#pragma unroll
            for (int v = 0; v < NV; ++v) s[v][threadIdx.x] += s[v][threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x < NV) loss[threadIdx.x] += s[threadIdx.x][0];
}
#endif  // __CUDACC__

// ---------------------------------------------------------------------------------------
// holder core shared by the ALS, SGD and pLSI handles: options state, device attach and the P/Q factor pointers
// ---------------------------------------------------------------------------------------
struct Holder {
    bool opt_set = false;
    int d = 0, vdim = 0;
    int num_sms = 0;
    cudaStream_t stream = nullptr;

    // factors: either owned device mirrors of retained host pointers, or borrowed device memory
    float *hostP = nullptr, *hostQ = nullptr;
    DevBuf<float> ownP, ownQ;
    float *dP = nullptr, *dQ = nullptr;
    int64_t P_rows = 0, Q_rows = 0;
    bool factors_ready = false;

    virtual ~Holder();
    // parses the handle's options; option errors (BFL_ERR_OPTION) come before attach_device()
    virtual int apply_options(const JsonOpt& j) = 0;
    // require_device(), the SM count and the non-blocking stream (created once)
    int attach_device();
    // caller-owned device factors of 16-byte aligned rows; releases the owned mirrors
    int borrow_factors(float* P, int64_t P_rows, float* Q, int64_t Q_rows);
    // retains the caller's host factors and points dP/dQ at owned mirrors of rows * vdim floats (not yet copied)
    int mirror_factors(float* P, int64_t P_rows, float* Q, int64_t Q_rows);
};

// bfl_*_init (src is a file path) and bfl_*_init_json (src is the JSON text)
int init_holder(Holder* h, const char* src, bool is_path);

// a device CSR of END offsets: borrowed through bind_csr_device, or a holder's own upload of the caller's indptr
struct CsrBinding {
    const int64_t* indptr = nullptr;
    const int32_t* keys = nullptr;
    const float* vals = nullptr;
    int64_t rows = 0, nnz = 0;
    // borrows a device CSR; with_vals: the holder reads values as well as keys
    int bind(const int64_t* d_indptr, const int32_t* d_keys, const float* d_vals, int64_t n_rows, int64_t n_nnz,
             bool with_vals);
    int check_range(int64_t row_begin, int64_t row_end) const;
};

// begin/end entry offsets of rows [row_begin, row_end) read from a device `indptr` of END offsets; synchronises `st`
int read_row_span(const int64_t* indptr, int64_t row_begin, int64_t row_end, cudaStream_t st, int64_t* begin,
                  int64_t* end);

}  // namespace bfl
