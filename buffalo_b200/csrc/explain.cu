// ALS explanations (DESIGN.md 4.11): for a history row r and a target item i, the score q_i' x_r of the exact row solve
// x_r = A_r^-1 b_r of the user half-epoch, and its split into one term per history item,
//   contribution_rij = (q_i' A_r^-1 q_j) * (1 + alpha v_j),
// with the top-m terms per (row, target).  One CTA owns one row at a time; no atomics, so a row's outputs depend only on
// the row, its targets, Q, the Gram and the options.
#include "explain.cuh"

namespace bfl {
namespace {

constexpr int EX_THREADS = 256, EX_WARPS = EX_THREADS / 32;
constexpr int EX_T = 16;    // targets per tile
constexpr int EX_NB = 16;   // history entries per gathered chunk (EX_T * EX_NB == EX_THREADS: one dot per thread)
static_assert(EX_T * EX_NB == EX_THREADS, "one (target, entry) pair per thread");

__device__ __forceinline__ int tri(int i) { return i * (i + 1) / 2; }   // start of row i of the packed lower triangle

// floats of dynamic shared memory: the packed lower triangle, pivots, one column, b, the target tile, the gathered
// chunk, its contributions, weights and keys, and the top-m lists.  Rows of the tiles are S = D | 1 floats apart, an
// odd stride, so the 16 chunk rows a warp reads in the dot products sit in 16 different banks.
size_t explain_smem_floats(int D, int topm) {
    const size_t S = (size_t)(D | 1);
    return (size_t)D * (D + 1) / 2 + 3 * (size_t)D + (EX_T + EX_NB) * S + EX_T * EX_NB + 2 * EX_NB + 2 * (size_t)EX_T * topm;
}

// the chunk's item rows into Qc (warp per entry, coalesced), its keys into ck and w(v) into cw
template <typename W>
__device__ __forceinline__ void gather_chunk(const ExplainArgs& a, int64_t b0, int nb, int S, float* Qc, float* cw, int* ck,
                                             W w) {
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    for (int b = wid; b < nb; b += EX_WARPS) {
        const float* q = a.Q + (int64_t)__ldg(a.keys + b0 + b) * a.ld;
        for (int c = lane; c < a.D; c += 32) Qc[b * S + c] = __ldg(q + c);
    }
    if (tid < nb) {
        ck[tid] = __ldg(a.keys + b0 + tid);
        cw[tid] = w(__ldg(a.vals + b0 + tid));
    }
}

// one item's total into a descending list of cnt <= topm entries.  Keys arrive in ascending order, so on a tie the
// kept (smaller) item wins: a new item enters only when its total is strictly larger.
__device__ __forceinline__ void topm_push(float* v, int* keys, int topm, int& cnt, int key, float val) {
    if (cnt == topm && !(val > v[topm - 1])) return;
    int p = cnt < topm ? cnt++ : topm - 1;
    while (p > 0 && val > v[p - 1]) {
        v[p] = v[p - 1];
        keys[p] = keys[p - 1];
        --p;
    }
    v[p] = val;
    keys[p] = key;
}

__global__ void __launch_bounds__(EX_THREADS) explain_kernel(ExplainArgs a) {
    extern __shared__ float sm[];
    const int D = a.D, S = D | 1, topm = a.topm, k = a.k;
    float* L = sm;                        // packed lower triangle: A_r, then its Cholesky factor (strictly lower part)
    float* diag = L + tri(D);             // [D] pivots L[j][j]
    float* colv = diag + D;               // [D] column j of L while step j updates the trailing matrix
    float* bv = colv + D;                 // [D] b_r
    float* U = bv + D;                    // [EX_T][S] target rows q_i, solved in place to A_r^-1 q_i
    float* Qc = U + EX_T * S;             // [EX_NB][S] gathered history rows
    float* Cc = Qc + EX_NB * S;           // [EX_T][EX_NB] the chunk's contributions
    float* cw = Cc + EX_T * EX_NB;        // [EX_NB] v (building A_r) or 1 + alpha v (contributions)
    int* ck = (int*)(cw + EX_NB);         // [EX_NB] the chunk's keys
    float* tv = (float*)(ck + EX_NB);     // [EX_T][topm] kept contributions, descending
    int* tk = (int*)(tv + EX_T * topm);   // [EX_T][topm] their items
    __shared__ int s_fail;                // the row's factorisation met a non-positive pivot
    const int tid = threadIdx.x, lane = tid & 31, wid = warp_id_uniform();
    const float alpha = a.alpha;

    for (int64_t r = blockIdx.x; r < a.n; r += gridDim.x) {
        const int64_t beg = r == 0 ? 0 : a.indptr[r - 1], end = a.indptr[r];
        const int32_t* tg = a.targets + r * k;
        float* score = a.scores + r * k;
        int32_t* okeys = a.out_keys + r * k * topm;
        float* ocon = a.out_contrib + r * k * topm;
        if (end <= beg) {   // no history: nothing to explain
            for (int t = tid; t < k; t += EX_THREADS) score[t] = 0.f;
            for (int64_t e = tid; e < (int64_t)k * topm; e += EX_THREADS) {
                okeys[e] = -1;
                ocon[e] = 0.f;
            }
            continue;
        }
        __syncthreads();   // the previous row is done with the shared arrays
        if (tid == 0) s_fail = 0;

        // 1. A_r = G + reg*kappa*I + sum alpha v q q' (lower part), b_r = sum (1 + alpha v) q, in entry order
        const float regk = a.reg * (a.adaptive_reg ? (float)(end - beg) : 1.0f);
        for (int i = wid; i < D; i += EX_WARPS)
            for (int j = lane; j <= i; j += 32) L[tri(i) + j] = a.G[i * D + j] + (i == j ? regk : 0.f);
        for (int i = tid; i < D; i += EX_THREADS) bv[i] = 0.f;
        for (int64_t b0 = beg; b0 < end; b0 += EX_NB) {
            const int nb = (int)min((int64_t)EX_NB, end - b0);
            __syncthreads();
            gather_chunk(a, b0, nb, S, Qc, cw, ck, [](float v) { return v; });
            __syncthreads();
            for (int i = wid; i < D; i += EX_WARPS)
                for (int j = lane; j <= i; j += 32) {
                    float acc = 0.f;
                    for (int b = 0; b < nb; ++b) acc += (alpha * cw[b] * Qc[b * S + i]) * Qc[b * S + j];
                    L[tri(i) + j] += acc;
                }
            for (int i = tid; i < D; i += EX_THREADS) {
                float acc = 0.f;
                for (int b = 0; b < nb; ++b) acc += (1.0f + alpha * cw[b]) * Qc[b * S + i];
                bv[i] += acc;
            }
        }
        __syncthreads();

        // 2. Cholesky A_r = L L', right-looking, in place.  Every thread reads the same pivot, so a non-positive (or
        // NaN) one stops all of them at the same column.
        for (int j = 0; j < D; ++j) {
            const float p = L[tri(j) + j];
            if (!(p > 0.f)) {
                if (tid == 0) s_fail = 1;
                break;
            }
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

        // 3.-6. per tile of EX_T targets
        for (int t0 = 0; t0 < k; t0 += EX_T) {
            const int nt = min(EX_T, k - t0);
            __syncthreads();   // the previous tile is done with U and the top-m lists (and s_fail is set)
            const bool fail = s_fail != 0;
            // 3. u_i = A_r^-1 q_i: warp w solves targets w and w + 8 (forward L y = q, then backward L' u = y)
            bool any = false;
            for (int t = wid; t < nt; t += EX_WARPS) {
                const int key = tg[t0 + t];
                if (key < 0 || key >= a.Q_rows) {
                    if (lane == 0) score[t0 + t] = 0.f;
                    continue;
                }
                if (fail) {
                    if (lane == 0) score[t0 + t] = __int_as_float(0x7fc00000);   // NaN
                    continue;
                }
                any = true;
                float* u = U + t * S;
                const float* q = a.Q + (int64_t)key * a.ld;
                for (int c = lane; c < D; c += 32) u[c] = __ldg(q + c);
                __syncwarp();
                for (int j = 0; j < D; ++j) {
                    const float uj = u[j] / diag[j];
                    __syncwarp();
                    if (lane == 0) u[j] = uj;
                    for (int i = j + 1 + lane; i < D; i += 32) u[i] -= L[tri(i) + j] * uj;
                    __syncwarp();
                }
                for (int j = D - 1; j >= 0; --j) {
                    const float uj = u[j] / diag[j];
                    __syncwarp();
                    if (lane == 0) u[j] = uj;
                    const float* row = L + tri(j);
                    for (int i = lane; i < j; i += 32) u[i] -= row[i] * uj;
                    __syncwarp();
                }
                // 4. score = u_i' b_r
                float s = 0.f;
                for (int c = lane; c < D; c += 32) s += u[c] * bv[c];
                s = warp_sum(s);
                if (lane == 0) score[t0 + t] = s;
            }
            any = __syncthreads_or(any);

            // 5. one more pass over the row: (1 + alpha v_j) * (u_i . q_j) for every (target, entry) pair of a chunk,
            // then 6. thread t folds target t's terms in entry order: equal adjacent keys (duplicates) are summed, and
            // each item's total goes through the top-m list
            const int my_key = tid < nt ? tg[t0 + tid] : -1;
            const bool mine = tid < nt && my_key >= 0 && my_key < a.Q_rows && !fail;
            int cnt = 0, pend_key = -1;
            float pend = 0.f;
            float* myv = tv + tid * topm;
            int* myk = tk + tid * topm;
            if (any) {
                const int pt = tid / EX_NB, pb = tid % EX_NB;
                for (int64_t b0 = beg; b0 < end; b0 += EX_NB) {
                    const int nb = (int)min((int64_t)EX_NB, end - b0);
                    __syncthreads();
                    gather_chunk(a, b0, nb, S, Qc, cw, ck, [alpha](float v) { return 1.0f + alpha * v; });
                    __syncthreads();
                    if (pt < nt && pb < nb) {
                        const float* u = U + pt * S;
                        const float* q = Qc + pb * S;
                        float acc = 0.f;
                        for (int c = 0; c < D; ++c) acc += u[c] * q[c];
                        Cc[pt * EX_NB + pb] = cw[pb] * acc;
                    }
                    __syncthreads();
                    if (mine) {
                        for (int b = 0; b < nb; ++b) {
                            const int key = ck[b];
                            const float c = Cc[tid * EX_NB + b];
                            if (key == pend_key) {
                                pend += c;
                            } else {
                                if (pend_key >= 0) topm_push(myv, myk, topm, cnt, pend_key, pend);
                                pend_key = key;
                                pend = c;
                            }
                        }
                    }
                }
            }
            if (tid < nt) {
                if (mine && pend_key >= 0) topm_push(myv, myk, topm, cnt, pend_key, pend);
                int32_t* ok = okeys + (int64_t)(t0 + tid) * topm;
                float* oc = ocon + (int64_t)(t0 + tid) * topm;
                for (int p = 0; p < topm; ++p) {
                    ok[p] = p < cnt ? myk[p] : -1;
                    oc[p] = p < cnt ? myv[p] : 0.f;
                }
            }
        }
    }
}

}  // namespace

int explain_launch(const ExplainArgs& a, int num_sms, cudaStream_t st) {
    if (a.n <= 0) return BFL_OK;
    const size_t smem = explain_smem_floats(a.D, a.topm) * sizeof(float);
    BFL_CUDA(cudaFuncSetAttribute(explain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    BFL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, explain_kernel, EX_THREADS, smem));
    if (per_sm < 1) BFL_FAIL(BFL_ERR_CUDA, "explain_kernel does not fit on an SM with " + std::to_string(smem) + " B of shared memory");
    const int grid = (int)std::min<int64_t>(a.n, (int64_t)num_sms * per_sm);
    explain_kernel<<<grid, EX_THREADS, smem, st>>>(a);
    BFL_LAUNCHED();
    return BFL_OK;
}

}  // namespace bfl
