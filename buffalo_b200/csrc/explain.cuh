// ALS explanations and posterior draws (explain.cu, DESIGN.md 4.11, 4.17): the launchers behind bfl_als_explain_device
// and bfl_als_posterior_sample_device, and the row-system build and Cholesky factorisation both kernels run.
#pragma once
#include "bfl_common.cuh"

namespace bfl {

constexpr int EXPLAIN_DMAX = 256;      // the packed lower triangle of A_r fits in shared memory up to here
constexpr int EXPLAIN_KMAX = 4096;     // targets per history row (the serve handle's largest k)
constexpr int EXPLAIN_TOPM_MAX = 64;   // contributions kept per (row, target)

struct ExplainArgs {
    const float* G;          // d x d Gram Q'Q (row-major)
    const float* Q;          // [Q_rows, ld] item factors
    int64_t Q_rows;
    int D, ld;
    float alpha, reg;        // alpha and reg_u of the user half-epoch
    bool adaptive_reg;       // reg * (entries of the row)
    const int64_t* indptr;   // [n] END offsets of the history rows
    const int32_t* keys;     // items in [0, Q_rows), ascending within a row (duplicates adjacent)
    const float* vals;
    int64_t n;
    const int32_t* targets;  // [n, k] item indexes, -1 (or anything outside [0, Q_rows)) for no target
    int k, topm;
    float* scores;           // [n, k]
    int32_t* out_keys;       // [n, k, topm]
    float* out_contrib;      // [n, k, topm]
};

// a.n rows on `st`; arguments are checked by the caller (k, topm and D within the limits above)
int explain_launch(const ExplainArgs& a, int num_sms, cudaStream_t st);

// Philox epoch word of the posterior draws (draw_u32(seed, POSTERIOR_TAG, draw key, t)): "TS" + 0x0417, a domain no
// training or fold-in stream uses
constexpr uint32_t POSTERIOR_TAG = 0x54530417u;

struct PosteriorArgs {
    const float* G;          // d x d Gram Q'Q (row-major)
    const float* Q;          // [Q_rows, ldq] item factors
    int D, ldq;
    float alpha, reg;        // alpha and reg_u of the user half-epoch
    bool adaptive_reg;
    const int64_t* indptr;   // [n] END offsets of the history rows
    const int32_t* keys;     // items in [0, Q_rows), ascending within a row (duplicates adjacent)
    const float* vals;
    int64_t n;
    int ld;                  // row pitch of mean and out (>= D), independent of Q's
    const float* mean;       // [n, ld]
    const int64_t* draw_keys;   // [n] Philox counter of each row's normal draws
    uint32_t seed;
    float scale;             // sigma; 0 copies the mean
    float* out;              // [n, ld], may alias mean
    int64_t* failed;         // += rows whose A_r met a non-positive or NaN pivot (written as their mean)
};

// a.n rows on `st`; arguments are checked by the caller (D <= EXPLAIN_DMAX)
int posterior_sample_launch(const PosteriorArgs& a, int num_sms, cudaStream_t st);

// ---- the row system and its factorisation, shared by explain_kernel and posterior_sample_kernel ------------------
constexpr int EX_THREADS = 256, EX_WARPS = EX_THREADS / 32;
constexpr int EX_NB = 16;   // history entries per gathered chunk

__device__ __forceinline__ int tri(int i) { return i * (i + 1) / 2; }   // start of row i of the packed lower triangle

// the chunk's item rows into Qc (warp per entry, coalesced, rows S floats apart), its keys into ck and w(v) into cw
template <typename W>
__device__ __forceinline__ void gather_chunk(const float* Q, int ld, int D, const int32_t* keys, const float* vals,
                                             int64_t b0, int nb, int S, float* Qc, float* cw, int* ck, W w) {
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    for (int b = wid; b < nb; b += EX_WARPS) {
        const float* q = Q + (int64_t)__ldg(keys + b0 + b) * ld;
        for (int c = lane; c < D; c += 32) Qc[b * S + c] = __ldg(q + c);
    }
    if (tid < nb) {
        ck[tid] = __ldg(keys + b0 + tid);
        cw[tid] = w(__ldg(vals + b0 + tid));
    }
}

// A_r = G + regk*I + sum alpha v q q' (packed lower triangle L) and, with WITH_B, b_r = sum (1 + alpha v) q into bv,
// over entries [beg, end) in entry order.  Qc [EX_NB][S], cw, ck [EX_NB] are scratch.  Ends with a __syncthreads.
template <bool WITH_B>
__device__ __forceinline__ void build_row_system(const float* G, const float* Q, int ld, int D, int S, float alpha,
                                                 float regk, const int32_t* keys, const float* vals, int64_t beg,
                                                 int64_t end, float* L, float* bv, float* Qc, float* cw, int* ck) {
    const int tid = threadIdx.x, lane = tid & 31, wid = warp_id_uniform();
    for (int i = wid; i < D; i += EX_WARPS)
        for (int j = lane; j <= i; j += 32) L[tri(i) + j] = G[i * D + j] + (i == j ? regk : 0.f);
    if (WITH_B)
        for (int i = tid; i < D; i += EX_THREADS) bv[i] = 0.f;
    for (int64_t b0 = beg; b0 < end; b0 += EX_NB) {
        const int nb = (int)min((int64_t)EX_NB, end - b0);
        __syncthreads();
        gather_chunk(Q, ld, D, keys, vals, b0, nb, S, Qc, cw, ck, [](float v) { return v; });
        __syncthreads();
        for (int i = wid; i < D; i += EX_WARPS)
            for (int j = lane; j <= i; j += 32) {
                float acc = 0.f;
                for (int b = 0; b < nb; ++b) acc += (alpha * cw[b] * Qc[b * S + i]) * Qc[b * S + j];
                L[tri(i) + j] += acc;
            }
        if (WITH_B)
            for (int i = tid; i < D; i += EX_THREADS) {
                float acc = 0.f;
                for (int b = 0; b < nb; ++b) acc += (1.0f + alpha * cw[b]) * Qc[b * S + i];
                bv[i] += acc;
            }
    }
    __syncthreads();
}

// Cholesky A = L L' of the packed lower triangle, right-looking, in place: the strictly lower part of L in L, its
// diagonal in diag; colv [D] is scratch.  Every thread reads the same pivot, so a non-positive (or NaN) one stops all
// of them at the same column and they all return false.  Ends with a __syncthreads when it returns true.
__device__ __forceinline__ bool cholesky_packed(float* L, float* diag, float* colv, int D) {
    const int tid = threadIdx.x, lane = tid & 31, wid = warp_id_uniform();
    for (int j = 0; j < D; ++j) {
        const float p = L[tri(j) + j];
        if (!(p > 0.f)) return false;
        const float ljj = sqrtf(p);
        for (int i = j + 1 + tid; i < D; i += EX_THREADS) {
            const float lij = L[tri(i) + j] / ljj;
            L[tri(i) + j] = lij;
            colv[i] = lij;
        }
        if (tid == 0) diag[j] = ljj;
        __syncthreads();
        for (int i = j + 1 + wid; i < D; i += EX_WARPS) {
            const float lij = colv[i];
            float* row = L + tri(i);
            for (int c = j + 1 + lane; c <= i; c += 32) row[c] -= lij * colv[c];
        }
        __syncthreads();
    }
    return true;
}

}  // namespace bfl
