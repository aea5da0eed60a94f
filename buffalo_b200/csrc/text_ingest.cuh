// Core shared by the device text parsers (mm_ingest.cu, stream_ingest.cu; DESIGN.md 4.6, 4.7): the compute stream,
// two pinned staging buffers, the feed state, the per-stage device clock and the CSR build into host arrays.
// Implemented in ingest.cu.  Each parser derives its handle from TextIngest and keeps its own device buffers, kernels
// and stage enum.
#pragma once
#include <vector>

#include "bfl_common.cuh"

namespace bfl {

// grid of the grid-stride helper kernels of 256 threads: one CTA per 256 items, at most 16 CTAs per SM of the device
int grid_for(long long n);

struct TextIngest {
    long long block_bytes = 0;
    cudaStream_t comp = nullptr;                           // compute stream
    unsigned char* host[2] = {nullptr, nullptr};           // pinned staging buffers of block_bytes
    cudaEvent_t copied[2] = {nullptr, nullptr};            // recorded by a parser whose upload of a slot is asynchronous
    bool copy_pending[2] = {false, false};
    long long fed = 0;                                     // bytes fed so far
    bool last_fed = false, built[2] = {false, false};
    std::vector<std::vector<cudaEvent_t>> marks;           // (begin, end) event pairs per stage
    cudaMemPool_t mem_pool = nullptr;                      // the device's default pool, high-water mark reset at setup

    virtual ~TextIngest();
};

// Resets the pool's high-water mark, creates the compute stream, the staging buffers and their copy events; false
// when a call fails (the CUDA error is left for setup_done).
bool setup(TextIngest* h, long long block_bytes, int stages);

// h, or nullptr after reporting "<what> ingest setup failed" and deleting h when !ok
template <class H>
H* setup_done(H* h, bool ok, const char* what) {
    if (ok) return h;
    set_error(std::string(what) + " ingest setup failed: " + cudaGetErrorString(cudaGetLastError()));
    delete h;
    return nullptr;
}

// records the next begin or end event of `stage` on st
int mark(TextIngest* h, int stage, cudaStream_t st);

// host_ptr = staging buffer `slot` once its pending upload (if any) has finished
int staging(TextIngest* h, int slot, void** host_ptr);

// argument and state checks of a feed of n bytes from `slot`; every block but the last ends with '\n'.  Records
// whether this is the last block.
int check_feed(TextIngest* h, int slot, long long n, int is_last);

// CSR of one orientation (0: by row, 1: by column) of the nnz device triples, built on the compute stream into host
// arrays of num_major END offsets and nnz entries; the build is timed as csr_stage, the copy as d2h_stage.  Marks the
// orientation built and synchronises.
int build_to_host(TextIngest* h, int orientation, const int32_t* row, const int32_t* col, const float* val, long long nnz,
                  int32_t num_rows, int32_t num_cols, int sort_minor, int csr_stage, int d2h_stage, int64_t* indptr,
                  int32_t* key, float* out_val);

// stage_ms[s] = summed device time of the (begin, end) pairs of stage s; *peak_bytes = the pool's high-water mark
int stats(TextIngest* h, double* stage_ms, int64_t* peak_bytes);

}  // namespace bfl
