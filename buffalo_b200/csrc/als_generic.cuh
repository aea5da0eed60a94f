// Generic ALS row-solve kernels: one warp per row, lane-strided columns.  They accept every
// (d <= 512, block_size, optimizer) combination the option file can express and define the
// baseline the tuned kernels in als_fast.cuh are tested against.
//
// Maths follows the reference CPU path (lib/algo_impl/als/als.cc:107-358, lib/algo.cc:39-82);
// the normal-equation matrix of the manual_cg path is applied as an operator
// (G + a*sum v q q^T + reg*kappa*I) instead of being materialised (als.cc:194-202), which is the
// same arithmetic the reference's own CUDA kernel uses (lib/cuda/als/als.cu:44-107).
#pragma once
#include "bfl_common.cuh"

namespace bfl {

struct AlsArgs {
    float* X;             // matrix being updated [rows x ld]
    const float* Y;       // opposite factors     [Y_rows x ld]
    const float* G;       // Y^T Y                [D x D] dense
    const int64_t* indptr;  // global exclusive end offsets (device), indexed by absolute row
    const int32_t* keys;  // chunk buffers, element (it - shift)
    const float* vals;
    float* yui;           // scratch [chunk nnz] (generic ialspp only)
    double* loss;         // [0] numerator, [1] denominator (may be null).  Kernels instantiated with DET = true take it
                          // as per-row terms instead: row r's pair is stored (not added) at loss[2 r], loss[2 r + 1]
    const int32_t* row_list;  // optional explicit row list (absolute row ids), else null
    int64_t shift;        // global offset of keys[0]
    int64_t row_begin, row_end;  // absolute rows [begin, end) (or range into row_list)
    int64_t Y_rows;
    int D, ld;
    int block_size;
    int max_iters;
    int adaptive_reg, compute_loss, axis;
    float alpha, reg, eps, tol;
    int n_peer;           // fused multi-GPU exchange: every solved row is also stored to these replicas of X
    float* peerX[15];
    const float* tc_scales;  // tensor-core path: [0] operand scale 2^e, [1] 2^-2e (device; null when that path is off)
};
constexpr int BFL_MAX_PEERS = 15;

constexpr int GEN_WARPS = 8;

// ---------------------------------------------------------------------------------------
// manual_cg  (lib/algo.cc:58-82 on the system of als.cc:180-202)
// ---------------------------------------------------------------------------------------
template <int NC, bool DET = false>
__global__ void __launch_bounds__(GEN_WARPS * 32) als_cg_warp_kernel(AlsArgs a) {
    __shared__ float ps_all[GEN_WARPS][NC * 32];
    const int lane = threadIdx.x & 31, wib = warp_id_uniform();
    float* ps = ps_all[wib];
    const int64_t warp0 = (int64_t)blockIdx.x * GEN_WARPS + wib;
    const int64_t nwarps = (int64_t)gridDim.x * GEN_WARPS;
    const int D = a.D, ld = a.ld;
    double l_nume = 0.0, l_deno = 0.0;
    for (int64_t ri = a.row_begin + warp0; ri < a.row_end; ri += nwarps) {
        const int64_t row = uni((long long)(a.row_list ? a.row_list[ri] : ri));
        const int64_t beg = uni((long long)(row == 0 ? 0 : a.indptr[row - 1]));
        const int64_t end = uni((long long)a.indptr[row]);
        const int64_t n = end - beg;
        if (n == 0) continue;  // als.cc:159-162: skipped, not zeroed
        float x[NC], y[NC], t[NC], r[NC], p[NC], Ap[NC];
        float* xrow = a.X + row * ld;
#pragma unroll
        for (int k = 0; k < NC; ++k) {
            const int c = lane + 32 * k;
            x[k] = c < D ? xrow[c] : 0.f;
            y[k] = 0.f;
            t[k] = 0.f;
        }
        const float regk = a.reg * (a.adaptive_reg ? (float)n : 1.0f);
        // xG
#pragma unroll
        for (int k = 0; k < NC; ++k) ps[lane + 32 * k] = x[k];
        __syncwarp();
        float xg[NC];
#pragma unroll
        for (int k = 0; k < NC; ++k) xg[k] = 0.f;
        for (int j = 0; j < D; ++j) {
            const float xj = ps[j];
#pragma unroll
            for (int k = 0; k < NC; ++k) {
                const int c = lane + 32 * k;
                if (c < D) xg[k] += xj * __ldg(a.G + (int64_t)j * D + c);
            }
        }
        if (a.compute_loss) {
            float s = 0.f, xx = 0.f;
#pragma unroll
            for (int k = 0; k < NC; ++k) {
                s += x[k] * xg[k];
                xx += x[k] * x[k];
            }
            s = warp_sum(s);
            xx = warp_sum(xx);
            if (a.axis == 1) {
                l_nume += s;                 // als.cc:175-178
                l_deno += (double)a.Y_rows;
            }
            l_nume += (double)(regk * xx);   // als.cc:198-200
        }
        for (int64_t it = beg; it < end; ++it) {
            const int key = a.keys[it - a.shift];
            const float v = a.vals[it - a.shift];
            const float* qrow = a.Y + (int64_t)key * ld;
            float q[NC], part = 0.f;
#pragma unroll
            for (int k = 0; k < NC; ++k) {
                const int c = lane + 32 * k;
                q[k] = c < D ? __ldg(qrow + c) : 0.f;
                part += x[k] * q[k];
            }
            const float dot = warp_sum(part);
            const float av = a.alpha * v;
            const float coef = 1.0f + av;     // als.cc:185
            const float tc = av * dot;
#pragma unroll
            for (int k = 0; k < NC; ++k) {
                y[k] += coef * q[k];
                t[k] += tc * q[k];
            }
            if (a.compute_loss && a.axis == 1) {  // als.cc:187-192
                l_nume -= (double)(dot * dot);
                l_nume += (double)((dot - 1.f) * (dot - 1.f)) * (1.0 + (double)av);
                l_deno += (double)av;
            }
        }
        float yy = 0.f, rr = 0.f;
#pragma unroll
        for (int k = 0; k < NC; ++k) {
            r[k] = y[k] - t[k] - xg[k] - regk * x[k];  // r = y - xA (algo.cc:62)
            yy += y[k] * y[k];
            rr += r[k] * r[k];
        }
        yy = uni(warp_sum(yy));
        rr = uni(warp_sum(rr));
        if (yy < rr) {  // algo.cc:64-67
#pragma unroll
            for (int k = 0; k < NC; ++k) {
                x[k] = 0.f;
                r[k] = y[k];
            }
            rr = yy;
        }
#pragma unroll
        for (int k = 0; k < NC; ++k) p[k] = r[k];
        float rs_old = rr;
        for (int iter = 0; iter < a.max_iters; ++iter) {
            __syncwarp();
#pragma unroll
            for (int k = 0; k < NC; ++k) ps[lane + 32 * k] = p[k];
            __syncwarp();
#pragma unroll
            for (int k = 0; k < NC; ++k) Ap[k] = regk * p[k];
            for (int j = 0; j < D; ++j) {
                const float pj = ps[j];
#pragma unroll
                for (int k = 0; k < NC; ++k) {
                    const int c = lane + 32 * k;
                    if (c < D) Ap[k] += pj * __ldg(a.G + (int64_t)j * D + c);
                }
            }
            for (int64_t it = beg; it < end; ++it) {
                const int key = a.keys[it - a.shift];
                const float v = a.vals[it - a.shift];
                const float* qrow = a.Y + (int64_t)key * ld;
                float q[NC], part = 0.f;
#pragma unroll
                for (int k = 0; k < NC; ++k) {
                    const int c = lane + 32 * k;
                    q[k] = c < D ? __ldg(qrow + c) : 0.f;
                    part += p[k] * q[k];
                }
                const float tc = a.alpha * v * warp_sum(part);
#pragma unroll
                for (int k = 0; k < NC; ++k) Ap[k] += tc * q[k];
            }
            float pAp = 0.f;
#pragma unroll
            for (int k = 0; k < NC; ++k) pAp += p[k] * Ap[k];
            pAp = warp_sum(pAp);
            const float al = rs_old / (pAp + a.eps);  // algo.cc:71
            float rs_new = 0.f;
#pragma unroll
            for (int k = 0; k < NC; ++k) {
                x[k] += al * p[k];
                r[k] -= al * Ap[k];
                rs_new += r[k] * r[k];
            }
            rs_new = uni(warp_sum(rs_new));
            if (rs_new < a.tol) break;  // algo.cc:76
            const float beta = rs_new / (rs_old + a.eps);
#pragma unroll
            for (int k = 0; k < NC; ++k) p[k] = r[k] + beta * p[k];
            rs_old = rs_new;
        }
        bool bad = false;
#pragma unroll
        for (int k = 0; k < NC; ++k) bad |= !isfinite(x[k]);
        bad = __any_sync(FULL, bad);  // NaN/Inf guard (cf. als.cu:116-120): zero the row
#pragma unroll
        for (int k = 0; k < NC; ++k) {
            const int c = lane + 32 * k;
            if (c < D) {
                const float v = bad ? 0.f : x[k];
                xrow[c] = v;
                for (int pr = 0; pr < a.n_peer; ++pr) a.peerX[pr][row * ld + c] = v;
            }
        }
        __syncwarp();
        if (DET) {   // every lane holds the row's terms, added in entry order
            if (a.loss && a.compute_loss && lane == 0) {
                a.loss[2 * row] = l_nume;
                a.loss[2 * row + 1] = l_deno;
            }
            l_nume = l_deno = 0.0;
        }
    }
    if (!DET && a.loss && a.compute_loss && lane == 0) {
        atomicAdd(a.loss, l_nume);
        atomicAdd(a.loss + 1, l_deno);
    }
}

// ---------------------------------------------------------------------------------------
// iALS++  (als.cc:211-358): block size <= 32*NC
// ---------------------------------------------------------------------------------------
template <int NC, bool DET = false>
__global__ void __launch_bounds__(GEN_WARPS * 32) als_ialspp_warp_kernel(AlsArgs a) {
    __shared__ float xs_all[GEN_WARPS][NC * 32];
    __shared__ float ps_all[GEN_WARPS][NC * 32];
    const int lane = threadIdx.x & 31, wib = warp_id_uniform();
    float* xs = xs_all[wib];
    float* ps = ps_all[wib];
    const int64_t warp0 = (int64_t)blockIdx.x * GEN_WARPS + wib;
    const int64_t nwarps = (int64_t)gridDim.x * GEN_WARPS;
    const int D = a.D, ld = a.ld;
    const int bs_opt = a.block_size < D ? a.block_size : D;  // als.cc:244
    double l_nume = 0.0, l_deno = 0.0;
    for (int64_t ri = a.row_begin + warp0; ri < a.row_end; ri += nwarps) {
        const int64_t row = uni((long long)(a.row_list ? a.row_list[ri] : ri));
        const int64_t beg = uni((long long)(row == 0 ? 0 : a.indptr[row - 1]));
        const int64_t end = uni((long long)a.indptr[row]);
        const int64_t n = end - beg;
        if (n == 0) continue;  // als.cc:289-292
        float* xrow = a.X + row * ld;
        __syncwarp();
#pragma unroll
        for (int k = 0; k < NC; ++k) {
            const int c = lane + 32 * k;
            xs[c] = c < D ? xrow[c] : 0.f;
        }
        __syncwarp();
        // Yui = x . q_c  (als.cc:256-266) + loss pieces with the pre-update row
        for (int64_t it = beg; it < end; ++it) {
            const int key = a.keys[it - a.shift];
            const float* qrow = a.Y + (int64_t)key * ld;
            float part = 0.f;
#pragma unroll
            for (int k = 0; k < NC; ++k) {
                const int c = lane + 32 * k;
                if (c < D) part += xs[c] * __ldg(qrow + c);
            }
            const float dot = warp_sum(part);
            if (lane == 0) a.yui[it - a.shift] = dot;
            if (a.compute_loss && a.axis == 1) {  // als.cc:310-315
                const float av = a.alpha * a.vals[it - a.shift];
                l_nume -= (double)(dot * dot);
                l_nume += (double)((dot - 1.f) * (dot - 1.f)) * (1.0 + (double)av);
                l_deno += (double)av;
            }
        }
        if (a.compute_loss) {
            float xx = 0.f;
#pragma unroll
            for (int k = 0; k < NC; ++k) {
                const int c = lane + 32 * k;
                if (c < D) xx += xs[c] * xs[c];
            }
            xx = warp_sum(xx);
            const float ada = a.adaptive_reg ? (float)n : 1.0f;
            l_nume += (double)(ada * a.reg * xx);  // als.cc:319-321
            if (a.axis == 1) {                     // als.cc:298-301
                float s = 0.f;
                for (int j = 0; j < D; ++j) {
                    const float xj = xs[j];
#pragma unroll
                    for (int k = 0; k < NC; ++k) {
                        const int c = lane + 32 * k;
                        if (c < D) s += xj * __ldg(a.G + (int64_t)j * D + c) * xs[c];
                    }
                }
                l_nume += (double)warp_sum(s);
                l_deno += (double)a.Y_rows;
            }
        }
        __syncwarp();
        for (int bb = 0; bb < D; bb += bs_opt) {
            const int bs = (bb + bs_opt >= D) ? D - bb : bs_opt;  // als.cc:271-274
            float bv[NC], xv[NC], r[NC], p[NC], Ap[NC];
            // b = x G[:, blk] + reg * x_blk   (als.cc:296)
#pragma unroll
            for (int m = 0; m < NC; ++m) {
                const int j = lane + 32 * m;
                bv[m] = j < bs ? a.reg * xs[bb + j] : 0.f;
            }
            for (int k = 0; k < D; ++k) {
                const float xk = xs[k];
#pragma unroll
                for (int m = 0; m < NC; ++m) {
                    const int j = lane + 32 * m;
                    if (j < bs) bv[m] += xk * __ldg(a.G + (int64_t)k * D + bb + j);
                }
            }
            for (int64_t it = beg; it < end; ++it) {  // als.cc:303-308
                const int key = a.keys[it - a.shift];
                const float v = a.vals[it - a.shift];
                const float cf = (a.yui[it - a.shift] - 1.0f) * v * a.alpha;
                const float* qrow = a.Y + (int64_t)key * ld + bb;
#pragma unroll
                for (int m = 0; m < NC; ++m) {
                    const int j = lane + 32 * m;
                    if (j < bs) bv[m] += cf * __ldg(qrow + j);
                }
            }
            float rs = 0.f;
#pragma unroll
            for (int m = 0; m < NC; ++m) {
                xv[m] = 0.f;
                r[m] = bv[m];
                p[m] = bv[m];
                rs += r[m] * r[m];
            }
            double rsold = (double)uni(warp_sum(rs));
            if (rsold > (double)a.tol) {
                for (int step = 0; step < 3; ++step) {  // als.cc:330
                    __syncwarp();
#pragma unroll
                    for (int m = 0; m < NC; ++m) ps[lane + 32 * m] = p[m];
                    __syncwarp();
#pragma unroll
                    for (int m = 0; m < NC; ++m) Ap[m] = a.reg * p[m];  // A = G[blk,blk] + reg I (als.cc:278)
                    for (int k = 0; k < bs; ++k) {
                        const float pk = ps[k];
#pragma unroll
                        for (int m = 0; m < NC; ++m) {
                            const int j = lane + 32 * m;
                            if (j < bs) Ap[m] += pk * __ldg(a.G + (int64_t)(bb + k) * D + bb + j);
                        }
                    }
                    for (int64_t it = beg; it < end; ++it) {  // als.cc:332-336
                        const int key = a.keys[it - a.shift];
                        const float v = a.vals[it - a.shift];
                        const float* qrow = a.Y + (int64_t)key * ld + bb;
                        float q[NC], part = 0.f;
#pragma unroll
                        for (int m = 0; m < NC; ++m) {
                            const int j = lane + 32 * m;
                            q[m] = j < bs ? __ldg(qrow + j) : 0.f;
                            part += q[m] * p[m];
                        }
                        const float cf = v * a.alpha * warp_sum(part);
#pragma unroll
                        for (int m = 0; m < NC; ++m) Ap[m] += cf * q[m];
                    }
                    float pAp = 0.f;
#pragma unroll
                    for (int m = 0; m < NC; ++m) pAp += p[m] * Ap[m];
                    pAp = warp_sum(pAp);
                    const float step_size = (float)(rsold / (double)pAp);  // als.cc:337 (no eps)
                    float rn = 0.f;
#pragma unroll
                    for (int m = 0; m < NC; ++m) {
                        xv[m] += step_size * p[m];
                        r[m] -= step_size * Ap[m];
                        rn += r[m] * r[m];
                    }
                    const double rsnew = (double)uni(warp_sum(rn));
                    if (rsnew < (double)a.tol) break;  // als.cc:341
                    const float beta = (float)(rsnew / rsold);
#pragma unroll
                    for (int m = 0; m < NC; ++m) p[m] = r[m] + beta * p[m];
                    rsold = rsnew;
                }
            }
            __syncwarp();
#pragma unroll
            for (int m = 0; m < NC; ++m) {
                const int j = lane + 32 * m;
                if (j < bs) xs[bb + j] -= xv[m];  // als.cc:346
            }
            for (int64_t it = beg; it < end; ++it) {  // als.cc:347-350
                const int key = a.keys[it - a.shift];
                const float* qrow = a.Y + (int64_t)key * ld + bb;
                float part = 0.f;
#pragma unroll
                for (int m = 0; m < NC; ++m) {
                    const int j = lane + 32 * m;
                    if (j < bs) part += __ldg(qrow + j) * xv[m];
                }
                const float dot = warp_sum(part);
                if (lane == 0) a.yui[it - a.shift] -= dot;
            }
            __syncwarp();
        }
        bool bad = false;
#pragma unroll
        for (int k = 0; k < NC; ++k) {
            const int c = lane + 32 * k;
            if (c < D) bad |= !isfinite(xs[c]);
        }
        bad = __any_sync(FULL, bad);
#pragma unroll
        for (int k = 0; k < NC; ++k) {
            const int c = lane + 32 * k;
            if (c < D) {
                const float v = bad ? 0.f : xs[c];
                xrow[c] = v;
                for (int pr = 0; pr < a.n_peer; ++pr) a.peerX[pr][row * ld + c] = v;
            }
        }
        if (DET) {   // every lane holds the row's terms, added in entry order
            if (a.loss && a.compute_loss && lane == 0) {
                a.loss[2 * row] = l_nume;
                a.loss[2 * row + 1] = l_deno;
            }
            l_nume = l_deno = 0.0;
        }
    }
    if (!DET && a.loss && a.compute_loss && lane == 0) {
        atomicAdd(a.loss, l_nume);
        atomicAdd(a.loss + 1, l_deno);
    }
}

// ---------------------------------------------------------------------------------------
// llt / ldlt  (lib/algo.cc:52-57 on the system of als.cc:180-202): one CTA per row,
// M = G + a*sum v q q^T + reg*kappa*I built in shared memory, in-CTA Cholesky.  LDL^T is served
// by the same LL^T factorisation: the systems are SPD and both give the exact solve up to fp32
// rounding (Eigen's LDLT additionally pivots).
// dynamic smem: D*(D+1) + 2*D + DIRECT_NB*D floats
// ---------------------------------------------------------------------------------------
constexpr int DIRECT_THREADS = 256;
constexpr int DIRECT_NB = 8;

template <bool DET = false>
__global__ void __launch_bounds__(DIRECT_THREADS) als_direct_cta_kernel(AlsArgs a) {
    extern __shared__ float sm[];
    const int D = a.D, ld = a.ld, P1 = D + 1;
    float* M = sm;                       // [D][D+1]
    float* yv = M + (size_t)D * P1;      // [D]
    float* wv = yv + D;                  // [D]
    float* qb = wv + D;                  // [NB][D]
    __shared__ float s_v[DIRECT_NB];
    __shared__ double s_loss[2];
    __shared__ double s_dn[DET ? DIRECT_NB : 1], s_dav[DET ? DIRECT_NB : 1];   // DET: the loss terms of a batch's entries
    const int tid = threadIdx.x, lane = tid & 31, wid = warp_id_uniform();
    if (tid < 2) s_loss[tid] = 0.0;
    for (int64_t ri = a.row_begin + blockIdx.x; ri < a.row_end; ri += gridDim.x) {
        const int64_t row = a.row_list ? a.row_list[ri] : ri;
        const int64_t beg = row == 0 ? 0 : a.indptr[row - 1];
        const int64_t end = a.indptr[row];
        const int64_t n = end - beg;
        if (n == 0) continue;
        __syncthreads();
        float* xrow = a.X + row * ld;
        const float regk = a.reg * (a.adaptive_reg ? (float)n : 1.0f);
        for (int e = tid; e < D * D; e += DIRECT_THREADS) {
            const int i = e / D, j = e - i * D;
            M[i * P1 + j] = a.G[e] + (i == j ? regk : 0.f);
        }
        for (int i = tid; i < D; i += DIRECT_THREADS) {
            yv[i] = 0.f;
            wv[i] = xrow[i];  // pre-update row (loss)
        }
        __syncthreads();
        double l_nume = 0.0, l_deno = 0.0;
        if (a.compute_loss && wid == 0) {
            // x G x (axis 1) and reg*kappa*|x|^2
            float s = 0.f, xx = 0.f;
            for (int i = lane; i < D; i += 32) {
                float t = 0.f;
                for (int k = 0; k < D; ++k) t += wv[k] * a.G[(int64_t)k * D + i];
                s += wv[i] * t;
                xx += wv[i] * wv[i];
            }
            s = warp_sum(s);
            xx = warp_sum(xx);
            if (lane == 0) {
                if (a.axis == 1) {
                    l_nume += s;
                    l_deno += (double)a.Y_rows;
                }
                l_nume += (double)(regk * xx);
            }
        }
        for (int64_t b0 = beg; b0 < end; b0 += DIRECT_NB) {
            const int nb = (int)((end - b0) < DIRECT_NB ? (end - b0) : DIRECT_NB);
            __syncthreads();
            if (DET && a.compute_loss && a.axis == 1 && tid == 0 && b0 > beg) {
                // the previous (full) batch's terms, in entry order; they are rewritten only after the next barrier
                for (int b = 0; b < DIRECT_NB; ++b) {
                    l_nume += s_dn[b];
                    l_deno += s_dav[b];
                }
            }
            for (int e = tid; e < nb * D; e += DIRECT_THREADS) {
                const int b = e / D, c = e - b * D;
                const int key = a.keys[b0 + b - a.shift];
                qb[b * D + c] = __ldg(a.Y + (int64_t)key * ld + c);
            }
            if (tid < nb) s_v[tid] = a.vals[b0 + tid - a.shift];
            __syncthreads();
            if (a.compute_loss && a.axis == 1 && wid < nb) {
                float part = 0.f;
                for (int c = lane; c < D; c += 32) part += wv[c] * qb[wid * D + c];
                const float dot = warp_sum(part);
                if (lane == 0) {
                    const float av = a.alpha * s_v[wid];
                    double dn = -(double)(dot * dot) + (double)((dot - 1.f) * (dot - 1.f)) * (1.0 + (double)av);
                    if (DET) {   // one term per entry; thread 0 adds them in entry order after the next barrier
                        s_dn[wid] = dn;
                        s_dav[wid] = (double)av;
                    } else {
                        atomicAdd(&s_loss[0], dn);
                        atomicAdd(&s_loss[1], (double)av);
                    }
                }
            }
            for (int e = tid; e < D * D; e += DIRECT_THREADS) {
                const int i = e / D, j = e - i * D;
                float acc = 0.f;
                for (int b = 0; b < nb; ++b) acc += (a.alpha * s_v[b] * qb[b * D + i]) * qb[b * D + j];
                M[i * P1 + j] += acc;
            }
            for (int i = tid; i < D; i += DIRECT_THREADS) {
                float acc = 0.f;
                for (int b = 0; b < nb; ++b) acc += (1.0f + a.alpha * s_v[b]) * qb[b * D + i];
                yv[i] += acc;
            }
        }
        __syncthreads();
        if (DET && a.compute_loss && a.axis == 1 && tid == 0) {   // the last batch's terms
            for (int b = 0; b < (int)((n - 1) % DIRECT_NB) + 1; ++b) {
                l_nume += s_dn[b];
                l_deno += s_dav[b];
            }
        }
        // in-place Cholesky (lower), right-looking
        for (int j = 0; j < D; ++j) {
            if (tid == 0) M[j * P1 + j] = sqrtf(M[j * P1 + j]);
            __syncthreads();
            const float ljj = M[j * P1 + j];
            for (int i = j + 1 + tid; i < D; i += DIRECT_THREADS) M[i * P1 + j] /= ljj;
            __syncthreads();
            const int m = D - j - 1;
            for (int e = tid; e < m * m; e += DIRECT_THREADS) {
                const int ii = e / m, kk = e - ii * m;
                if (kk <= ii) {
                    const int i = j + 1 + ii, k = j + 1 + kk;
                    M[i * P1 + k] -= M[i * P1 + j] * M[k * P1 + j];
                }
            }
            __syncthreads();
        }
        if (wid == 0) {
            // forward: L w = y
            for (int i = 0; i < D; ++i) {
                float part = 0.f;
                for (int k = lane; k < i; k += 32) part += M[i * P1 + k] * wv[k];
                part = warp_sum(part);
                __syncwarp();
                if (lane == 0) wv[i] = (yv[i] - part) / M[i * P1 + i];
                __syncwarp();
            }
            // backward: L^T x = w   (x overwrites yv)
            for (int i = D - 1; i >= 0; --i) {
                float part = 0.f;
                for (int k = i + 1 + lane; k < D; k += 32) part += M[k * P1 + i] * yv[k];
                part = warp_sum(part);
                __syncwarp();
                if (lane == 0) yv[i] = (wv[i] - part) / M[i * P1 + i];
                __syncwarp();
            }
            bool bad = false;
            for (int i = lane; i < D; i += 32) bad |= !isfinite(yv[i]);
            bad = __any_sync(FULL, bad);
            for (int i = lane; i < D; i += 32) {
                const float v = bad ? 0.f : yv[i];
                xrow[i] = v;
                for (int pr = 0; pr < a.n_peer; ++pr) a.peerX[pr][row * ld + i] = v;
            }
            if (DET) {
                if (lane == 0 && a.loss && a.compute_loss) {
                    a.loss[2 * row] = l_nume;
                    a.loss[2 * row + 1] = l_deno;
                }
            } else if (lane == 0 && a.compute_loss) {
                atomicAdd(&s_loss[0], l_nume);
                atomicAdd(&s_loss[1], l_deno);
            }
        }
    }
    __syncthreads();
    if (!DET && a.loss && a.compute_loss && tid < 2) atomicAdd(a.loss + tid, s_loss[tid]);
}

// ---------------------------------------------------------------------------------------
// Gram precompute  FF = F^T F  (als.cc:86-93; the reference GPU path calls cublasSgemm,
// als.cu:315-317).  Two-stage and deterministic: each CTA accumulates a [<=128 x <=128] output
// slab over its share of the rows in registers (8x8 per thread), writes a partial, and a second
// kernel sums the partials in fp64.
// ---------------------------------------------------------------------------------------
// d = a * b + c on both halves of an fp32 pair
__device__ __forceinline__ float2 gram_ffma2(float2 a, float2 b, float2 c) {
    return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}

constexpr int GRAM_TR = 32;       // rows per smem tile
constexpr int GRAM_THREADS = 256;

__global__ void __launch_bounds__(GRAM_THREADS, 2) gram_partial_kernel(const float* __restrict__ F, int64_t rows,
                                                                    int D, int ld, float* __restrict__ partial,
                                                                    int nslab) {
    // blockIdx.y enumerates (si, sj) output slabs of 128x128; blockIdx.x strides over row tiles.
    // The next row tile is fetched into registers (128-bit loads) while the current one is multiplied out of
    // shared memory with packed FMAs; a diagonal slab (always the case for d <= 128) keeps a single copy.
    __shared__ __align__(16) float sa[GRAM_TR][128 + 4];
    __shared__ __align__(16) float sb[GRAM_TR][128 + 4];
    const int si = blockIdx.y / nslab, sj = blockIdx.y % nslab;
    const int i0 = si * 128, j0 = sj * 128;
    const bool diag = si == sj;
    const float(*pb)[128 + 4] = diag ? sa : sb;
    const int tid = threadIdx.x;
    const int ti = tid >> 4, tj = tid & 15;  // 16 x 16 threads, 8x8 outputs each
    const bool vec_ok = (ld & 3) == 0 && (reinterpret_cast<uintptr_t>(F) & 15) == 0;
    float2 acc[8][4];
#pragma unroll
    for (int u = 0; u < 8; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) acc[u][v] = make_float2(0.f, 0.f);
    // thread's four 128-bit pieces of a 32 x 128 tile: piece k = row (tid >> 5) + 8k, columns 4 * (tid & 31)
    const int lr = tid >> 5, lc = (tid & 31) * 4;
    auto fetch = [&](int64_t r0, int c0, float4(&v)[4]) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int64_t gr = r0 + lr + 8 * k;
            float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
            if (gr < rows) {
                const float* src = F + gr * ld + c0 + lc;
                if (vec_ok && c0 + lc + 3 < D) {
                    x = __ldg(reinterpret_cast<const float4*>(src));
                } else {
                    if (c0 + lc + 0 < D) x.x = __ldg(src + 0);
                    if (c0 + lc + 1 < D) x.y = __ldg(src + 1);
                    if (c0 + lc + 2 < D) x.z = __ldg(src + 2);
                    if (c0 + lc + 3 < D) x.w = __ldg(src + 3);
                }
            }
            v[k] = x;
        }
    };
    const int64_t ntiles = (rows + GRAM_TR - 1) / GRAM_TR;
    float4 va[4], vb[4];
    if ((int64_t)blockIdx.x < ntiles) {
        fetch((int64_t)blockIdx.x * GRAM_TR, i0, va);
        if (!diag) fetch((int64_t)blockIdx.x * GRAM_TR, j0, vb);
    }
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            *reinterpret_cast<float4*>(&sa[lr + 8 * k][lc]) = va[k];
            if (!diag) *reinterpret_cast<float4*>(&sb[lr + 8 * k][lc]) = vb[k];
        }
        __syncthreads();
        if (tile + gridDim.x < ntiles) {
            fetch((tile + gridDim.x) * GRAM_TR, i0, va);
            if (!diag) fetch((tile + gridDim.x) * GRAM_TR, j0, vb);
        }
#pragma unroll 4
        for (int r = 0; r < GRAM_TR; ++r) {
            const float4 a0 = *reinterpret_cast<const float4*>(&sa[r][ti * 8]);
            const float4 a1 = *reinterpret_cast<const float4*>(&sa[r][ti * 8 + 4]);
            const float4 b0 = *reinterpret_cast<const float4*>(&pb[r][tj * 8]);
            const float4 b1 = *reinterpret_cast<const float4*>(&pb[r][tj * 8 + 4]);
            const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float2 bv[4] = {make_float2(b0.x, b0.y), make_float2(b0.z, b0.w), make_float2(b1.x, b1.y),
                                  make_float2(b1.z, b1.w)};
#pragma unroll
            for (int u = 0; u < 8; ++u)
#pragma unroll
                for (int v = 0; v < 4; ++v) acc[u][v] = gram_ffma2(make_float2(av[u], av[u]), bv[v], acc[u][v]);
        }
    }
    float* out = partial + ((size_t)blockIdx.x * gridDim.y + blockIdx.y) * 128 * 128;
#pragma unroll
    for (int u = 0; u < 8; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v)
            *reinterpret_cast<float2*>(out + (ti * 8 + u) * 128 + tj * 8 + 2 * v) = acc[u][v];
}

__global__ void gram_reduce_kernel(const float* __restrict__ partial, int nparts, int nslab, int D,
                                   float* __restrict__ G) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= D * D) return;
    const int i = e / D, j = e - i * D;
    const int slab = (i >> 7) * nslab + (j >> 7);
    const int li = i & 127, lj = j & 127;
    double s = 0.0;
    for (int p = 0; p < nparts; ++p)
        s += (double)partial[((size_t)p * nslab * nslab + slab) * 128 * 128 + li * 128 + lj];
    G[e] = (float)s;
}

}  // namespace bfl
