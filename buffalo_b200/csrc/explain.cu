// ALS explanations (DESIGN.md 4.11): for a history row r and a target item i, the score q_i' x_r of the exact row solve
// x_r = A_r^-1 b_r of the user half-epoch, and its split into one term per history item,
//   contribution_rij = (q_i' A_r^-1 q_j) * (1 + alpha v_j),
// with the top-m terms per (row, target).  One CTA owns one row at a time; no atomics, so a row's outputs depend only on
// the row, its targets, Q, the Gram and the options.
//
// Posterior draws (DESIGN.md 4.17): for the same A_r, x~ = mean + scale * L^-T z with A_r = L L' and z ~ N(0, I) from
// Philox, i.e. a draw from N(mean, scale^2 A_r^-1), the posterior of the row under the Gaussian reading of the user
// half-epoch.  One CTA per row at a time, no atomics: a row's draw depends only on the seed, its draw key, its history,
// its mean, Q, the Gram and the options.
#include "explain.cuh"

namespace bfl {
namespace {

constexpr int EX_T = 16;    // targets per tile (EX_T * EX_NB == EX_THREADS: one dot per thread)
static_assert(EX_T * EX_NB == EX_THREADS, "one (target, entry) pair per thread");

// floats of dynamic shared memory: the packed lower triangle, pivots, one column, b, the target tile, the gathered
// chunk, its contributions, weights and keys, and the top-m lists.  Rows of the tiles are S = D | 1 floats apart, an
// odd stride, so the 16 chunk rows a warp reads in the dot products sit in 16 different banks.
size_t explain_smem_floats(int D, int topm) {
    const size_t S = (size_t)(D | 1);
    return (size_t)D * (D + 1) / 2 + 3 * (size_t)D + (EX_T + EX_NB) * S + EX_T * EX_NB + 2 * EX_NB + 2 * (size_t)EX_T * topm;
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
        build_row_system<true>(a.G, a.Q, a.ld, D, S, alpha, regk, a.keys, a.vals, beg, end, L, bv, Qc, cw, ck);

        // 2. Cholesky A_r = L L', right-looking, in place
        if (!cholesky_packed(L, diag, colv, D) && tid == 0) s_fail = 1;

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
                    gather_chunk(a.Q, a.ld, D, a.keys, a.vals, b0, nb, S, Qc, cw, ck, [alpha](float v) { return 1.0f + alpha * v; });
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

// floats of dynamic shared memory: the packed lower triangle, pivots, z (also the factorisation's column), y, the
// gathered chunk (rows S = D | 1 floats apart), its weights and keys
size_t posterior_smem_floats(int D) {
    const size_t S = (size_t)(D | 1);
    return (size_t)D * (D + 1) / 2 + 3 * (size_t)D + EX_NB * S + 2 * EX_NB;
}

// z_c for c < D of one row: quad q of the draw key's Philox stream gives words w[0..3] = draw_u32(seed, POSTERIOR_TAG,
// key, 4q + i), and pair k = 2q + h the Box-Muller normals of u1 = (w[2h] + 1) 2^-32, u2 = w[2h + 1] 2^-32:
// sqrt(-2 ln u1) cos(2 pi u2), sqrt(-2 ln u1) sin(2 pi u2) (u1 and u2 rounded to fp32; precise logf / sincospif)
__device__ __forceinline__ void normal_draws(uint32_t seed, uint64_t key, int D, float* z) {
    for (int q = threadIdx.x; 4 * q < D; q += EX_THREADS) {
        uint32_t w[4];
        philox4x32_10((uint32_t)key, (uint32_t)(key >> 32), (uint32_t)q, POSTERIOR_TAG, seed, 0x5EEDu, w);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int c = 4 * q + 2 * h;
            if (c < D) {
                const float u1 = (float)((uint64_t)w[2 * h] + 1u) * 0x1p-32f, u2 = (float)w[2 * h + 1] * 0x1p-32f;
                const float rad = sqrtf(-2.0f * logf(u1));
                float sn, cs;
                sincospif(2.0f * u2, &sn, &cs);
                z[c] = rad * cs;
                if (c + 1 < D) z[c + 1] = rad * sn;
            }
        }
    }
}

__global__ void __launch_bounds__(EX_THREADS) posterior_sample_kernel(PosteriorArgs a, int64_t* failed_part) {
    extern __shared__ float sm[];
    const int D = a.D, S = D | 1;
    float* L = sm;                        // packed lower triangle: A_r, then its Cholesky factor (strictly lower part)
    float* diag = L + tri(D);             // [D] pivots L[j][j]
    float* zv = diag + D;                 // [D] the factorisation's column j, then z, solved in place
    float* yv = zv + D;                   // [D] y = L'^-1 z
    float* Qc = yv + D;                   // [EX_NB][S] gathered history rows
    float* cw = Qc + EX_NB * S;           // [EX_NB] v
    int* ck = (int*)(cw + EX_NB);         // [EX_NB] the chunk's keys
    const int tid = threadIdx.x, lane = tid & 31;
    int64_t nfail = 0;                    // rows of this CTA left at their mean (thread 0's count)

    for (int64_t r = blockIdx.x; r < a.n; r += gridDim.x) {
        const float* mean = a.mean + r * a.ld;
        float* out = a.out + r * a.ld;
        if (a.scale == 0.f) {             // no exploration: the mean itself, whatever its bits
            for (int c = tid; c < D; c += EX_THREADS) out[c] = mean[c];
            continue;
        }
        const int64_t beg = r == 0 ? 0 : a.indptr[r - 1], end = a.indptr[r];
        __syncthreads();   // the previous row is done with the shared arrays

        // 1.-2. A_r = G + reg*kappa*I + sum alpha v q q' in entry order, then A_r = L L'
        const float regk = a.reg * (a.adaptive_reg ? (float)(end - beg) : 1.0f);
        build_row_system<false>(a.G, a.Q, a.ldq, D, S, a.alpha, regk, a.keys, a.vals, beg, end, L, nullptr, Qc, cw, ck);
        if (!cholesky_packed(L, diag, zv, D)) {
            for (int c = tid; c < D; c += EX_THREADS) out[c] = mean[c];
            if (tid == 0) ++nfail;
            continue;
        }

        // 3. z ~ N(0, I)
        normal_draws(a.seed, (uint64_t)a.draw_keys[r], D, zv);
        __syncthreads();

        // 4. L' y = z by back substitution, one warp: column j from D - 1 down, y_j = z_j / L_jj, then
        // z_i -= L_ji y_j for i < j (row j of the packed triangle, contiguous)
        if (tid < 32) {
            for (int j = D - 1; j >= 0; --j) {
                const float yj = zv[j] / diag[j];
                if (lane == 0) yv[j] = yj;
                const float* row = L + tri(j);
                for (int i = lane; i < j; i += 32) zv[i] -= row[i] * yj;
                __syncwarp();
            }
        }
        __syncthreads();

        // 5. out = mean + scale y (out may be mean: each element is read before it is written, by the same thread)
        for (int c = tid; c < D; c += EX_THREADS) out[c] = mean[c] + a.scale * yv[c];
    }
    if (tid == 0) failed_part[blockIdx.x] = nfail;
}

// *failed += the per-CTA counts, one CTA
__global__ void __launch_bounds__(256) failed_sum_kernel(const int64_t* part, int n, int64_t* failed) {
    __shared__ int64_t s[256];
    int64_t t = 0;
    for (int i = threadIdx.x; i < n; i += 256) t += part[i];
    s[threadIdx.x] = t;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
        if (threadIdx.x < w) s[threadIdx.x] += s[threadIdx.x + w];
        __syncthreads();
    }
    if (threadIdx.x == 0) *failed += s[0];
}

}  // namespace

int posterior_sample_launch(const PosteriorArgs& a, int num_sms, cudaStream_t st) {
    if (a.n <= 0) return BFL_OK;
    const size_t smem = posterior_smem_floats(a.D) * sizeof(float);
    BFL_CUDA(cudaFuncSetAttribute(posterior_sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    BFL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, posterior_sample_kernel, EX_THREADS, smem));
    if (per_sm < 1)
        BFL_FAIL(BFL_ERR_CUDA, "posterior_sample_kernel does not fit on an SM with " + std::to_string(smem) + " B of shared memory");
    const int grid = (int)std::min<int64_t>(a.n, (int64_t)num_sms * per_sm);
    int64_t* part = nullptr;
    BFL_CUDA(cudaMallocAsync(&part, sizeof(int64_t) * (size_t)grid, st));
    posterior_sample_kernel<<<grid, EX_THREADS, smem, st>>>(a, part);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) {
        g_launches.fetch_add(1, std::memory_order_relaxed);
        failed_sum_kernel<<<1, 256, 0, st>>>(part, grid, a.failed);
        e = cudaGetLastError();
    }
    cudaFreeAsync(part, st);
    BFL_CUDA(e);
    BFL_LAUNCHED();
    return BFL_OK;
}

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
