/*
 * buffalo_oracle.c -- CPU restatement of kakao/buffalo's matrix-factorisation
 * training hot path (ALS row solves, BPRMF / WARP negative-sampling SGD).
 *
 * THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load it.  The shipped
 * package (buffalo_b200/, buffalo/) never imports, links or executes it.
 *
 * PARITY UNPINNED: the reference holds no golden vectors / known-answer tests for
 * this path (tests/algo/base.py:83-97 only assert ranking thresholds on a dataset
 * that is an LFS pointer here) and it cannot be compiled in this image (Eigen,
 * json11, spdlog submodules are empty; see DESIGN.md).  This file therefore IS the
 * definition of "reference result"; it is cross-checked by an independent NumPy fp64
 * restatement (oracle/np_mirror.py) in tests/test_oracle.py.
 *
 * Third-party arithmetic the reference delegates to and that is absent from
 * the reference repository: Eigen @ 3147391d (3rd/eigen3, .SUBMODULES.json:9-15) for
 * A.llt().solve / A.ldlt().solve (lib/algo.cc:53,56) and the dense row/GEMM
 * expressions.  Restated here as plain fp32 loops (Cholesky LL^T and unpivoted
 * LDL^T); summation order inside Eigen's kernels is not reproducible and is not
 * part of the contract (tolerance 1e-3 relative on factors, BASELINE.json).
 *
 * Every function cites the reference file:line it follows (paths relative to
 * the reference repository).  Plain C11 + OpenMP; build with oracle/Makefile.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#else
static int omp_get_thread_num(void) { return 0; }
static int omp_get_max_threads(void) { return 1; }
#endif

#define ORC_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------- */
/* Options (flat PODs; the reference re-parses a JSON file per class,         */
/* lib/algo.cc:19-37, lib/algo_impl/als/als.cc:30-69)                          */
/* ------------------------------------------------------------------------- */
typedef struct {
    int32_t d;
    int32_t num_workers;
    int32_t num_cg_max_iters;   /* options.py:80 default 3 */
    int32_t optimizer_code;     /* 0 llt, 1 ldlt, 2 manual_cg, 8 ialspp (als.cc:47-67) */
    int32_t block_size;         /* options.py:81 default 32 */
    int32_t adaptive_reg;
    int32_t compute_loss;       /* compute_loss_on_training */
    float alpha, reg_u, reg_i, eps, cg_tolerance;
} orc_als_opt;

typedef struct {
    int32_t d;
    int32_t num_workers;
    int32_t optimizer;          /* 0 sgd, 1 adagrad, 2 adam */
    int32_t use_bias, update_i, update_j;
    int32_t num_negative_samples;
    int32_t verify_neg;
    int32_t uniform_sampling;   /* sampling_power == 0.0 (bpr.cc:91) */
    int32_t per_coordinate_normalize;
    int32_t max_trials;         /* WARP */
    int32_t score_l2;           /* WARP score_func == "l2" */
    int32_t random_seed;
    int32_t num_iters;
    float reg_u, reg_i, reg_j, reg_b;
    float lr, min_lr, beta1, beta2_unused, threshold;
} orc_sgd_opt;

/* The d>=128 => ialspp rule, als.cc:46.  Returns the effective optimizer code. */
ORC_API int orc_als_effective_optimizer(int d, int requested_code) {
    if (d >= 128) return 8;
    return requested_code;
}

/* ------------------------------------------------------------------------- */
/* ALS: Gram precompute  FF = F^T F   (als.cc:86-93)                           */
/* fp32 result; partial sums are kept in fp64 per thread (Eigen's blocked GEMM */
/* order is not reproducible; fp64 partials keep the oracle order-independent) */
/* ------------------------------------------------------------------------- */
ORC_API void orc_als_precompute(const float* F, int64_t rows, int d, float* FF, int num_workers) {
    int nt = num_workers > 0 ? num_workers : omp_get_max_threads();
    double* acc = (double*)calloc((size_t)nt * d * d, sizeof(double));
#pragma omp parallel num_threads(nt)
    {
        double* a = acc + (size_t)omp_get_thread_num() * d * d;
#pragma omp for schedule(static)
        for (int64_t r = 0; r < rows; ++r) {
            const float* f = F + r * d;
            for (int i = 0; i < d; ++i) {
                double fi = f[i];
                for (int j = i; j < d; ++j) a[i * d + j] += fi * (double)f[j];
            }
        }
    }
    for (int i = 0; i < d; ++i)
        for (int j = i; j < d; ++j) {
            double s = 0.0;
            for (int t = 0; t < nt; ++t) s += acc[(size_t)t * d * d + i * d + j];
            FF[i * d + j] = (float)s;
            FF[j * d + i] = (float)s;
        }
    free(acc);
}

/* ------------------------------------------------------------------------- */
/* Algorithm::_leastsquare  (lib/algo.cc:39-131), codes 0,1,2                  */
/* A: d x d symmetric fp32 (row-major == col-major), y: rhs, x: row of X in place */
/* ------------------------------------------------------------------------- */
static float dotf(const float* a, const float* b, int n) {
    float s = 0.f;
    for (int i = 0; i < n; ++i) s += a[i] * b[i];
    return s;
}

/* code 0: A.llt().solve(y)  (algo.cc:53) -- fp32 Cholesky, lower */
static void solve_llt(float* A, const float* y, float* x, int d, float* w) {
    for (int j = 0; j < d; ++j) {
        float s = A[j * d + j];
        for (int k = 0; k < j; ++k) s -= A[j * d + k] * A[j * d + k];
        float ljj = sqrtf(s);
        A[j * d + j] = ljj;
        for (int i = j + 1; i < d; ++i) {
            float t = A[i * d + j];
            for (int k = 0; k < j; ++k) t -= A[i * d + k] * A[j * d + k];
            A[i * d + j] = t / ljj;
        }
    }
    for (int i = 0; i < d; ++i) {
        float t = y[i];
        for (int k = 0; k < i; ++k) t -= A[i * d + k] * w[k];
        w[i] = t / A[i * d + i];
    }
    for (int i = d - 1; i >= 0; --i) {
        float t = w[i];
        for (int k = i + 1; k < d; ++k) t -= A[k * d + i] * x[k];
        x[i] = t / A[i * d + i];
    }
}

/* code 1: A.ldlt().solve(y)  (algo.cc:56) -- Eigen's LDLT pivots; for the SPD
 * systems on this path the unpivoted fp32 LDL^T below gives the same solution
 * up to rounding. */
static void solve_ldlt(float* A, const float* y, float* x, int d, float* w) {
    for (int j = 0; j < d; ++j) {
        float dj = A[j * d + j];
        for (int k = 0; k < j; ++k) dj -= A[j * d + k] * A[j * d + k] * A[k * d + k];
        A[j * d + j] = dj;
        for (int i = j + 1; i < d; ++i) {
            float t = A[i * d + j];
            for (int k = 0; k < j; ++k) t -= A[i * d + k] * A[j * d + k] * A[k * d + k];
            A[i * d + j] = t / dj;
        }
    }
    for (int i = 0; i < d; ++i) {
        float t = y[i];
        for (int k = 0; k < i; ++k) t -= A[i * d + k] * w[k];
        w[i] = t;
    }
    for (int i = 0; i < d; ++i) w[i] /= A[i * d + i];
    for (int i = d - 1; i >= 0; --i) {
        float t = w[i];
        for (int k = i + 1; k < d; ++k) t -= A[k * d + i] * x[k];
        x[i] = t;
    }
}

/* code 2: manual CG (algo.cc:58-82); warm start, reset test, eps in both quotients */
static void solve_manual_cg(const float* A, const float* y, float* x, int d, int max_iters,
                            float eps, float tol, float* r, float* p, float* Ap) {
    /* r = y - x A   (:62) */
    for (int j = 0; j < d; ++j) {
        float s = 0.f;
        for (int i = 0; i < d; ++i) s += x[i] * A[i * d + j];
        r[j] = y[j] - s;
    }
    /* (:64-67) */
    if (dotf(y, y, d) < dotf(r, r, d)) {
        for (int j = 0; j < d; ++j) { x[j] = 0.f; r[j] = y[j]; }
    }
    memcpy(p, r, sizeof(float) * d);
    float rs_old = dotf(r, r, d);
    for (int it = 0; it < max_iters; ++it) {
        for (int j = 0; j < d; ++j) {
            float s = 0.f;
            for (int i = 0; i < d; ++i) s += p[i] * A[i * d + j];
            Ap[j] = s;
        }
        float alpha = rs_old / (dotf(Ap, p, d) + eps);      /* (:71) */
        for (int j = 0; j < d; ++j) x[j] += alpha * p[j];   /* (:72) */
        for (int j = 0; j < d; ++j) r[j] -= alpha * Ap[j];  /* (:73) */
        float rs_new = dotf(r, r, d);
        if (rs_new < tol) break;                            /* (:76) */
        float beta = rs_new / (rs_old + eps);               /* (:78) */
        for (int j = 0; j < d; ++j) p[j] = r[j] + beta * p[j];
        rs_old = rs_new;
    }
}

/* ------------------------------------------------------------------------- */
/* CALS::_partial_update  (als.cc:107-209), d < 128 / optimizer != ialspp      */
/* X = matrix being updated (P on axis 0, Q on axis 1), Y = opposite, FF = Y^T Y */
/* indptr: GLOBAL exclusive end offsets, no leading zero (als.cc:156-157);     */
/* keys/vals: chunk buffers offset by `shifted` (als.cc:147,181-182).          */
/* ------------------------------------------------------------------------- */
static int als_partial_update_direct(const orc_als_opt* o, float* X, const float* Y, int64_t Y_rows,
                                     const float* FF, int start_x, int next_x, const int64_t* indptr,
                                     const int32_t* keys, const float* vals, int axis,
                                     double* out_nume, double* out_deno) {
    const int D = o->d;
    const float reg = axis == 0 ? o->reg_u : o->reg_i;
    const float alpha = o->alpha;
    const int nt = o->num_workers > 0 ? o->num_workers : 1;
    const int end_loop = next_x - start_x;
    const int64_t shifted = start_x == 0 ? 0 : indptr[start_x - 1];
    double* ln = (double*)calloc(nt, sizeof(double));
    double* ld = (double*)calloc(nt, sizeof(double));
#pragma omp parallel num_threads(nt)
    {
        const int wid = omp_get_thread_num();
        float* m = (float*)malloc(sizeof(float) * D * D);
        float* Fxy = (float*)malloc(sizeof(float) * D);
        float* w1 = (float*)malloc(sizeof(float) * D * 4);
        float* tmp = (float*)malloc(sizeof(float) * D);
#pragma omp for schedule(dynamic, 4)
        for (int i = 0; i < end_loop; ++i) {
            const int x = start_x + i;
            const int64_t beg = x == 0 ? 0 : indptr[x - 1];
            const int64_t end = indptr[x];
            const int64_t data_size = end - beg;
            if (data_size == 0) continue;                   /* (:159-162) skipped, not zeroed */
            float* xu = X + (int64_t)x * D;
            memset(m, 0, sizeof(float) * D * D);
            memset(Fxy, 0, sizeof(float) * D);
            if (o->compute_loss && axis == 1) {             /* (:175-178) */
                /* p . (p FF) */
                float s = 0.f;
                for (int j = 0; j < D; ++j) {
                    float t = 0.f;
                    for (int k = 0; k < D; ++k) t += xu[k] * FF[k * D + j];
                    s += xu[j] * t;
                }
                ln[wid] += s;
                ld[wid] += (double)Y_rows;
            }
            for (int64_t it = beg; it < end; ++it) {
                const int c = keys[it - shifted];
                const float v = vals[it - shifted];
                const float* q = Y + (int64_t)c * D;
                /* Fxy += q * (1.0 + v*alpha)   (:185) -- coefficient formed in double */
                const float coef = (float)(1.0 + (double)(v * alpha));
                for (int j = 0; j < D; ++j) Fxy[j] += q[j] * coef;
                /* FiF = Fs^T Fs2 * alpha with Fs = v*q, Fs2 = q  (:183-184,194) */
                for (int a = 0; a < D; ++a) {
                    const float va = v * q[a];
                    float* mr = m + a * D;
                    for (int b = 0; b < D; ++b) mr[b] += va * q[b];
                }
                if (o->compute_loss && axis == 1) {         /* (:187-192) */
                    float dot = dotf(xu, q, D);
                    ln[wid] -= dot * dot;
                    ln[wid] += (dot - 1) * (dot - 1) * (1.0 + v * alpha);
                    ld[wid] += v * alpha;
                }
            }
            for (int a = 0; a < D * D; ++a) m[a] = FF[a] + m[a] * alpha;   /* (:194-195) */
            const float ada_reg = o->adaptive_reg ? (float)data_size : 1.0f;  /* (:196) */
            if (o->compute_loss) ln[wid] += ada_reg * reg * dotf(xu, xu, D);  /* (:198-200) */
            for (int a = 0; a < D; ++a) m[a * D + a] += reg * ada_reg;     /* (:201-202) */
            /* _leastsquare(P, u, m, Fxy)  (:204) */
            if (o->optimizer_code == 0) {
                solve_llt(m, Fxy, tmp, D, w1);
                memcpy(xu, tmp, sizeof(float) * D);
            } else if (o->optimizer_code == 1) {
                solve_ldlt(m, Fxy, tmp, D, w1);
                memcpy(xu, tmp, sizeof(float) * D);
            } else {
                solve_manual_cg(m, Fxy, xu, D, o->num_cg_max_iters, o->eps, o->cg_tolerance,
                                w1, w1 + D, w1 + 2 * D);
            }
        }
        free(m); free(Fxy); free(w1); free(tmp);
    }
    double a = 0, b = 0;
    for (int t = 0; t < nt; ++t) { a += ln[t]; b += ld[t]; }
    free(ln); free(ld);
    *out_nume = a; *out_deno = b;
    return 0;
}

/* ------------------------------------------------------------------------- */
/* CALS::_partial_update_ialspp  (als.cc:211-358)                              */
/* Reference loops block-major over all rows; rows are independent within a    */
/* half-epoch (Y, FF frozen) so the row-major order below is equivalent.       */
/* Quirk fixed (SURVEY 9-3): Yui is sized per row, not indptr[end_loop-1].     */
/* ------------------------------------------------------------------------- */
static int als_partial_update_ialspp(const orc_als_opt* o, float* X, const float* Y, int64_t Y_rows,
                                     const float* FF, int start_x, int next_x, const int64_t* indptr,
                                     const int32_t* keys, const float* vals, int axis,
                                     double* out_nume, double* out_deno) {
    const int D = o->d;
    const float reg = axis == 0 ? o->reg_u : o->reg_i;
    const float alpha = o->alpha;
    const int nt = o->num_workers > 0 ? o->num_workers : 1;
    const int bs_opt = o->block_size < D ? o->block_size : D;   /* (:244) */
    const int end_loop = next_x - start_x;
    const int64_t shifted = start_x == 0 ? 0 : indptr[start_x - 1];
    const double tol = o->cg_tolerance;
    double* ln = (double*)calloc(nt, sizeof(double));
    double* ld = (double*)calloc(nt, sizeof(double));
#pragma omp parallel num_threads(nt)
    {
        const int wid = omp_get_thread_num();
        int64_t ycap = 1024;
        float* Yui = (float*)malloc(sizeof(float) * ycap);
        float* b = (float*)malloc(sizeof(float) * D * 5);
        float *xv = b + D, *r = b + 2 * D, *p = b + 3 * D, *Ap = b + 4 * D;
#pragma omp for schedule(dynamic, 4)
        for (int i = 0; i < end_loop; ++i) {
            const int x = start_x + i;
            const int64_t beg = x == 0 ? 0 : indptr[x - 1];
            const int64_t end = indptr[x];
            const int64_t n = end - beg;
            if (n == 0) continue;                           /* (:289-292) */
            float* xu = X + (int64_t)x * D;
            if (n > ycap) { ycap = n * 2; free(Yui); Yui = (float*)malloc(sizeof(float) * ycap); }
            /* build Y_ui  (:256-266) */
            for (int64_t k = 0; k < n; ++k)
                Yui[k] = dotf(xu, Y + (int64_t)keys[beg + k - shifted] * D, D);
            /* loss pieces, evaluated at block_beg == 0 with the pre-update row (:298-301,310-315,319-321) */
            if (o->compute_loss && axis == 1) {
                float s = 0.f;
                for (int j = 0; j < D; ++j) {
                    float t = 0.f;
                    for (int k = 0; k < D; ++k) t += xu[k] * FF[k * D + j];
                    s += xu[j] * t;
                }
                ln[wid] += s;
                ld[wid] += (double)Y_rows;
                for (int64_t k = 0; k < n; ++k) {
                    const float val = vals[beg + k - shifted];
                    float dot = dotf(xu, Y + (int64_t)keys[beg + k - shifted] * D, D);
                    ln[wid] -= dot * dot;
                    ln[wid] += (dot - 1) * (dot - 1) * (1.0 + val * alpha);
                    ld[wid] += val * alpha;
                }
            }
            if (o->compute_loss) {
                const float ada_reg = o->adaptive_reg ? (float)n : 1.0f;
                ln[wid] += ada_reg * reg * dotf(xu, xu, D);
            }
            for (int bb = 0; bb < D; bb += bs_opt) {
                int bs = bs_opt;
                if (bb + bs >= D) bs = D - bb;              /* (:271-274) */
                /* b = p * gramian + reg * block_p  (:296); gramian = FF[:, bb:bb+bs] */
                for (int j = 0; j < bs; ++j) {
                    float s = 0.f;
                    for (int k = 0; k < D; ++k) s += xu[k] * FF[k * D + bb + j];
                    b[j] = s + reg * xu[bb + j];
                }
                for (int64_t k = 0; k < n; ++k) {           /* (:303-308) */
                    const float* v = Y + (int64_t)keys[beg + k - shifted] * D + bb;
                    const float val = vals[beg + k - shifted];
                    const float residual = Yui[k] - 1.0f;
                    const float cf = residual * val * alpha;
                    for (int j = 0; j < bs; ++j) b[j] += cf * v[j];
                }
                /* CG update (:324-351): A = FF[bb:bb+bs, bb:bb+bs] + reg*I (:278) */
                for (int j = 0; j < bs; ++j) { xv[j] = 0.f; r[j] = b[j]; p[j] = b[j]; }
                double rsold = dotf(r, r, bs);
                if (rsold > tol) {
                    for (int step = 0; step < 3; ++step) {  /* fixed 3 steps (:330) */
                        for (int j = 0; j < bs; ++j) {
                            float s = 0.f;
                            for (int k = 0; k < bs; ++k) s += FF[(bb + j) * D + bb + k] * p[k];
                            Ap[j] = s + reg * p[j];
                        }
                        for (int64_t k = 0; k < n; ++k) {   /* (:332-336) */
                            const float* v = Y + (int64_t)keys[beg + k - shifted] * D + bb;
                            const float val = vals[beg + k - shifted];
                            const float cf = val * alpha * dotf(v, p, bs);
                            for (int j = 0; j < bs; ++j) Ap[j] += cf * v[j];
                        }
                        const float step_size = (float)(rsold / dotf(p, Ap, bs));  /* (:337) no eps */
                        for (int j = 0; j < bs; ++j) xv[j] += step_size * p[j];
                        for (int j = 0; j < bs; ++j) r[j] -= step_size * Ap[j];
                        double rsnew = dotf(r, r, bs);
                        if (rsnew < tol) break;             /* (:341) */
                        const float beta = (float)(rsnew / rsold);
                        for (int j = 0; j < bs; ++j) p[j] = r[j] + beta * p[j];
                        rsold = rsnew;
                    }
                }
                for (int j = 0; j < bs; ++j) xu[bb + j] -= xv[j];          /* (:346) */
                for (int64_t k = 0; k < n; ++k) {                          /* (:347-350) */
                    const float* v = Y + (int64_t)keys[beg + k - shifted] * D + bb;
                    Yui[k] -= dotf(v, xv, bs);
                }
            }
        }
        free(Yui); free(b);
    }
    double a = 0, c = 0;
    for (int t = 0; t < nt; ++t) { a += ln[t]; c += ld[t]; }
    free(ln); free(ld);
    *out_nume = a; *out_deno = c;
    return 0;
}

/* CALS::partial_update dispatch (als.cc:95-105).  P,Q are the user/item factor
 * matrices; axis selects which one is updated (als.cc:126-134). */
ORC_API int orc_als_partial_update(const orc_als_opt* o, float* P, int64_t P_rows, float* Q, int64_t Q_rows,
                                   const float* FF, int start_x, int next_x, const int64_t* indptr,
                                   const int32_t* keys, const float* vals, int axis,
                                   double* nume, double* deno) {
    *nume = 0.0; *deno = 0.0;
    if (next_x - start_x == 0) return 0;                    /* (:115-118) */
    float* X = axis == 0 ? P : Q;
    const float* Y = axis == 0 ? Q : P;
    const int64_t Y_rows = axis == 0 ? Q_rows : P_rows;
    (void)P_rows;
    if (o->optimizer_code == 8)
        return als_partial_update_ialspp(o, X, Y, Y_rows, FF, start_x, next_x, indptr, keys, vals, axis, nume, deno);
    if (o->optimizer_code == 0 || o->optimizer_code == 1 || o->optimizer_code == 2)
        return als_partial_update_direct(o, X, Y, Y_rows, FF, start_x, next_x, indptr, keys, vals, axis, nume, deno);
    return -1;  /* Eigen iterative solvers (codes 3-7, algo.cc:83-127) are not restated */
}

/* ------------------------------------------------------------------------- */
/* Counter-based RNG shared with the CUDA kernels: Philox4x32-10.              */
/* The reference seeds one std::mt19937 per worker thread (bpr.cc:83,          */
/* warp.cc:111) and hands rows to workers through a racy queue, so its draw     */
/* sequence is schedule-dependent and cannot be pinned.  Oracle and kernels     */
/* instead derive every draw from (seed, epoch, positive index, draw number),   */
/* which makes the WARP and BPR(adagrad/adam) epochs pure functions of their    */
/* inputs and lets tests compare gradients element-wise.                        */
/* ------------------------------------------------------------------------- */
static inline void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                 uint32_t k0, uint32_t k1, uint32_t out[4]) {
    for (int i = 0; i < 10; ++i) {
        uint64_t p0 = (uint64_t)0xD2511F53u * c0;
        uint64_t p1 = (uint64_t)0xCD9E8D57u * c2;
        uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0;
        uint32_t n1 = (uint32_t)p1;
        uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
        uint32_t n3 = (uint32_t)p0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

/* draw #t for positive #idx of epoch #epoch: uniform integer in [0, range) by
 * 32x32->64 multiply-shift (bias <= range/2^32, irrelevant at <= 2^24 items). */
static inline uint32_t draw_u32(uint32_t seed, uint32_t epoch, uint64_t idx, uint32_t t) {
    uint32_t o[4];
    philox4x32_10((uint32_t)idx, (uint32_t)(idx >> 32), t >> 2, epoch, seed, 0x5EEDu, o);
    return o[t & 3];
}
static inline int32_t draw_range(uint32_t seed, uint32_t epoch, uint64_t idx, uint32_t t, uint32_t range) {
    return (int32_t)(((uint64_t)draw_u32(seed, epoch, idx, t) * range) >> 32);
}
ORC_API int32_t orc_draw_range(uint32_t seed, uint32_t epoch, uint64_t idx, uint32_t t, uint32_t range) {
    return draw_range(seed, epoch, idx, t, range);
}

/* binary search in a sorted key segment: is `item` one of the user's positives? */
static inline int seen_sorted(const int32_t* keys, int64_t n, int32_t item) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        int64_t mid = (lo + hi) >> 1;
        if (keys[mid] < item) lo = mid + 1; else hi = mid;
    }
    return lo < n && keys[lo] == item;
}

/* lower_bound on the cumulative popularity table (bpr.cc:111-112) */
static inline int32_t cum_lower_bound(const int64_t* cum, int32_t size, int64_t r) {
    int32_t lo = 0, hi = size;
    while (lo < hi) {
        int32_t mid = (lo + hi) >> 1;
        if (cum[mid] < r) lo = mid + 1; else hi = mid;
    }
    return lo;
}

/* ------------------------------------------------------------------------- */
/* BPR negative sampling (bpr.cc:106-117).  One triple per (positive, k<num_neg). */
/* Rows must hold sorted keys (fileio.hpp:330-341 sorts by (row,col)).         */
/* Deviation (documented): positives are visited in CSR order, duplicates kept; */
/* the reference dedups through an unordered_set and visits in hash order       */
/* (bpr.cc:103-104).                                                            */
/* ------------------------------------------------------------------------- */
ORC_API void orc_bpr_sample(const orc_sgd_opt* o, int32_t num_items, int start_x, int next_x,
                            const int64_t* indptr, const int32_t* keys, const int64_t* cum_table,
                            uint32_t epoch, int32_t* out_u, int32_t* out_pos, int32_t* out_neg) {
    const int64_t shifted = start_x == 0 ? 0 : indptr[start_x - 1];
    const int nn = o->num_negative_samples;
    for (int x = start_x; x < next_x; ++x) {
        const int64_t beg = x == 0 ? 0 : indptr[x - 1];
        const int64_t end = indptr[x];
        const int32_t* row = keys + (beg - shifted);
        for (int64_t it = beg; it < end; ++it) {
            for (int k = 0; k < nn; ++k) {
                const uint64_t sid = (uint64_t)it * nn + k;  /* global sample index */
                int32_t neg = 0;
                for (uint32_t t = 0;; ++t) {
                    if (o->uniform_sampling) {
                        neg = draw_range(o->random_seed, epoch, sid, t, (uint32_t)num_items);
                    } else {
                        const int64_t total = cum_table[num_items - 1];
                        uint64_t r64 = ((uint64_t)draw_u32(o->random_seed, epoch, sid, 2 * t) << 32) |
                                       draw_u32(o->random_seed, epoch, sid, 2 * t + 1);
                        int64_t r = (int64_t)(((__uint128_t)r64 * (uint64_t)total) >> 64);
                        neg = cum_lower_bound(cum_table, num_items, r);
                        if (neg >= num_items) neg = num_items - 1;
                    }
                    if (!o->verify_neg || !seen_sorted(row, end - beg, neg)) break;
                    if (t >= 64) break;  /* guard: a user who has seen (almost) every item */
                }
                const int64_t s = (it - shifted) * nn + k;
                out_u[s] = x; out_pos[s] = keys[it - shifted]; out_neg[s] = neg;
            }
        }
    }
}

/* exp table of CBPRMF::build_exp_table (bpr.cc:57-63, bpr.hpp:17) */
#define ORC_EXP_TABLE_SIZE 1000
#define ORC_MAX_EXP 6
static float g_exp_table[ORC_EXP_TABLE_SIZE];
static int g_exp_ready = 0;
static void build_exp_table(void) {
    if (g_exp_ready) return;
    for (int i = 0; i < ORC_EXP_TABLE_SIZE; ++i) {
        float e = (float)exp((i / (float)ORC_EXP_TABLE_SIZE * 2 - 1) * ORC_MAX_EXP);
        g_exp_table[i] = (float)(1.0 / (e + 1));
    }
    g_exp_ready = 1;
}
/* logit = 1 - sigmoid(x) (bpr.cc:123-131).  use_lut=1 follows the reference's
 * 1000-entry table with its INTEGER scale 1000/6/2 = 83; use_lut=0 is the exact
 * expression the CUDA kernels (and the reference's own bpr.cu:113-116) evaluate. */
static inline float bpr_logit(float x, int use_lut) {
    if (ORC_MAX_EXP < x) return 0.0f;
    if (x < -ORC_MAX_EXP) return 1.0f;
    if (use_lut) return g_exp_table[(int)((x + ORC_MAX_EXP) * (ORC_EXP_TABLE_SIZE / ORC_MAX_EXP / 2))];
    return 1.0f / (1.0f + expf(x));
}

/* ------------------------------------------------------------------------- */
/* CBPRMF::worker body (bpr.cc:119-171) over an explicit triple list, applied   */
/* sequentially (deterministic single-worker order).                            */
/* optimizer sgd: in-place updates with lr (job.alpha); else accumulate grads.  */
/* ------------------------------------------------------------------------- */
ORC_API void orc_bpr_update(const orc_sgd_opt* o, float* P, float* Q, float* Qb,
                            float* gradP, float* gradQ, float* gradQb,
                            int32_t* P_cnt, int32_t* Q_cnt,
                            const int32_t* us, const int32_t* poss, const int32_t* negs, int64_t n,
                            float lr, int use_lut) {
    build_exp_table();
    const int D = o->d;
    for (int64_t s = 0; s < n; ++s) {
        const int u = us[s], pos = poss[s], neg = negs[s];
        float* p = P + (int64_t)u * D;
        float* qi = Q + (int64_t)pos * D;
        float* qj = Q + (int64_t)neg * D;
        float x_uij = 0.f;
        for (int k = 0; k < D; ++k) x_uij += p[k] * (qi[k] - qj[k]);          /* (:119) */
        if (o->use_bias) x_uij += Qb[pos] - Qb[neg];                          /* (:120-121) */
        const float logit = bpr_logit(x_uij, use_lut);
        if (o->optimizer != 0) {                                               /* (:138-156) */
            if (o->per_coordinate_normalize) { Q_cnt[neg] += 1; }
            for (int k = 0; k < D; ++k) gradP[(int64_t)u * D + k] += logit * (qi[k] - qj[k]);
            if (o->update_i) {
                for (int k = 0; k < D; ++k) gradQ[(int64_t)pos * D + k] += logit * p[k];
                if (o->use_bias) gradQb[pos] += logit;
            }
            if (o->update_j) {
                for (int k = 0; k < D; ++k) gradQ[(int64_t)neg * D + k] -= logit * p[k];
                if (o->use_bias) gradQb[neg] -= logit;
            }
            /* (:174-181) once per positive: triples are laid out positive-major, num_neg per positive */
            if (o->per_coordinate_normalize && (s % o->num_negative_samples) == 0) { P_cnt[u] += 1; Q_cnt[pos] += 1; }
        } else {                                                               /* (:157-171) */
            /* g is a LAZY Eigen expression in the reference (auto, :158): it is evaluated
             * at `P_.row(u) += alpha * g` AFTER q_i and q_j were updated. */
            if (o->update_i) {
                for (int k = 0; k < D; ++k) qi[k] += lr * (logit * p[k] - o->reg_i * qi[k]);
                if (o->use_bias) Qb[pos] += lr * (logit - o->reg_b * Qb[pos]);
            }
            if (o->update_j) {
                for (int k = 0; k < D; ++k) qj[k] += lr * (-logit * p[k] - o->reg_j * qj[k]);
                if (o->use_bias) Qb[neg] += lr * (-logit - o->reg_b * Qb[neg]);
            }
            for (int k = 0; k < D; ++k) p[k] += lr * (logit * (qi[k] - qj[k]) - o->reg_u * p[k]);
        }
    }
}

/* "pre-update" variant of the sgd branch: all three rows are updated from the values
 * read before the step (what the reference's own CUDA kernel does, bpr.cu:122-134, and
 * what our kernel does).  Used by the collision-free exactness test. */
ORC_API void orc_bpr_update_preupdate(const orc_sgd_opt* o, float* P, float* Q, float* Qb,
                                      const int32_t* us, const int32_t* poss, const int32_t* negs,
                                      int64_t n, float lr) {
    const int D = o->d;
    float* pu = (float*)malloc(sizeof(float) * D * 3);
    for (int64_t s = 0; s < n; ++s) {
        const int u = us[s], pos = poss[s], neg = negs[s];
        float* p = P + (int64_t)u * D;
        float* qi = Q + (int64_t)pos * D;
        float* qj = Q + (int64_t)neg * D;
        memcpy(pu, p, sizeof(float) * D);
        memcpy(pu + D, qi, sizeof(float) * D);
        memcpy(pu + 2 * D, qj, sizeof(float) * D);
        float x_uij = 0.f;
        for (int k = 0; k < D; ++k) x_uij += p[k] * (qi[k] - qj[k]);
        const float bi = Qb[pos], bj = Qb[neg];
        if (o->use_bias) x_uij += bi - bj;
        const float logit = bpr_logit(x_uij, 0);
        if (o->update_i) {
            for (int k = 0; k < D; ++k) qi[k] += lr * (logit * pu[k] - o->reg_i * pu[D + k]);
            if (o->use_bias) Qb[pos] += lr * (logit - o->reg_b * bi);
        }
        if (o->update_j) {
            for (int k = 0; k < D; ++k) qj[k] += lr * (-logit * pu[k] - o->reg_j * pu[2 * D + k]);
            if (o->use_bias) Qb[neg] += lr * (-logit - o->reg_b * bj);
        }
        for (int k = 0; k < D; ++k) p[k] += lr * (logit * (pu[D + k] - pu[2 * D + k]) - o->reg_u * pu[k]);
    }
    free(pu);
}

/* ------------------------------------------------------------------------- */
/* CWARP::worker (warp.cc:103-173): rank-sampling loop + gradient accumulation. */
/* P,Q are NOT modified inside an epoch (gradients only, warp.cc:156-158).      */
/* Draw numbering: every call of rng() consumes one draw index t = 0,1,2,...    */
/* for the positive (including draws rejected as seen, warp.cc:139-141).        */
/* Deviation (documented): positives visited in CSR order without dedup; the    */
/* "seen" set size is the row length.                                           */
/* out_trials (optional, per positive): final `trial` value, 0 when discarded.  */
/* ------------------------------------------------------------------------- */
static inline float warp_score(const float* u, const float* i, int D, int l2) {
    float s = 0.f;
    if (l2) { for (int k = 0; k < D; ++k) { float df = u[k] - i[k]; s += df * df; } return -s; }   /* warp.cc:25-28 */
    for (int k = 0; k < D; ++k) s += u[k] * i[k];                                                   /* warp.cc:21-23 */
    return s;
}

ORC_API void orc_warp_accumulate(const orc_sgd_opt* o, const float* P, const float* Q, int32_t num_items,
                                 float* gradP, float* gradQ, int32_t* P_cnt, int32_t* Q_cnt,
                                 int start_x, int next_x, const int64_t* indptr, const int32_t* keys,
                                 uint32_t epoch, double* out_loss, int64_t* out_updates,
                                 int32_t* out_trials, int32_t* out_negs) {
    const int D = o->d;
    const int64_t shifted = start_x == 0 ? 0 : indptr[start_x - 1];
    const int max_trial = o->max_trials;
    const float threshold = o->threshold;
    double loss = 0.0;
    int64_t updates = 0;
    for (int x = start_x; x < next_x; ++x) {
        const int64_t beg = x == 0 ? 0 : indptr[x - 1];
        const int64_t end = indptr[x];
        const int32_t* row = keys + (beg - shifted);
        const int64_t n_seen = end - beg;
        const float* p = P + (int64_t)x * D;
        for (int64_t it = beg; it < end; ++it) {
            const int pos = keys[it - shifted];
            const float* qi = Q + (int64_t)pos * D;
            const float ui = warp_score(p, qi, D, o->score_l2);     /* (:133) */
            float uj = 0.f;
            int neg = 0;
            int trial = 1;
            uint32_t t = 0;
            while (trial <= max_trial) {                            /* (:137-148) */
                neg = draw_range(o->random_seed, epoch, (uint64_t)it, t++, (uint32_t)num_items);
                if (seen_sorted(row, n_seen, neg)) {                /* (:140-141) not counted */
                    if (t > (uint32_t)(64 * max_trial + 4096)) { trial = max_trial + 1; break; }  /* guard */
                    continue;
                }
                trial += 1;                                         /* (:142) */
                uj = warp_score(p, Q + (int64_t)neg * D, D, o->score_l2);
                if ((ui - uj) < threshold) break;                   /* (:145-146) */
                trial += 1;                                         /* (:147) */
            }
            if (out_trials) out_trials[it - shifted] = trial >= max_trial ? 0 : trial;
            if (out_negs) out_negs[it - shifted] = trial >= max_trial ? -1 : neg;
            if (trial >= max_trial) continue;                       /* (:149-150) */
            /* Phi = log(max(1, int((Q_rows - seen.size() - 1) / trial)))  (:152)
             * (size_t arithmetic in the reference; rows never exceed num_items here) */
            int64_t ratio = ((int64_t)num_items - n_seen - 1) / trial;
            if (ratio < 1) ratio = 1;
            const float Phi = (float)log((double)(int)ratio);
            const float* qj = Q + (int64_t)neg * D;
            float* gp = gradP + (int64_t)x * D;
            float* gi = gradQ + (int64_t)pos * D;
            float* gj = gradQ + (int64_t)neg * D;
            if (!o->score_l2) {                                     /* dot_deriv (:30-40) */
                for (int k = 0; k < D; ++k) {
                    const float du = Phi * (qi[k] - qj[k]);
                    const float di = Phi * p[k];
                    gp[k] += du - o->reg_u * p[k];                  /* (:156) */
                    gi[k] += di - o->reg_i * qi[k];                 /* (:157) */
                    gj[k] += -di - o->reg_j * qj[k];                /* (:158) */
                }
            } else {                                                /* l2_deriv (:42-52) */
                for (int k = 0; k < D; ++k) {
                    const float du = Phi * 2 * (qi[k] - qj[k]);
                    const float di = Phi * (p[k] - qi[k]);
                    const float dj = -Phi * (p[k] - qj[k]);
                    gp[k] += du - o->reg_u * p[k];
                    gi[k] += di - o->reg_i * qi[k];
                    gj[k] += dj - o->reg_j * qj[k];
                }
            }
            if (o->per_coordinate_normalize) { P_cnt[x] += 1; Q_cnt[pos] += 1; Q_cnt[neg] += 1; }  /* (:159-165) */
            loss += (uj - ui + threshold);                          /* (:166) */
            updates += 1;
        }
    }
    if (out_loss) *out_loss = loss;
    if (out_updates) *out_updates = updates;
}

/* ------------------------------------------------------------------------- */
/* SGDAlgorithm::update_parameters  (lib/algo.cc:382-465) + update_adam        */
/* (:365-375) + update_adagrad (:377-380); beta2 := beta1 quirk (:396);        */
/* gradient buffers end up holding the step and are NOT zeroed (no setZero).   */
/* iters: value of iters_ before the call (incremented by the caller, :464).   */
/* Applied to one matrix (rows x cols) at a time; cols == 1 for the bias.      */
/* ------------------------------------------------------------------------- */
#define ORC_FEPS 1e-10f
ORC_API void orc_sgd_apply(int optimizer, float* theta, float* grad, float* mom, float* vel,
                           const int32_t* cnt, int64_t rows, int cols, double reg, double lr,
                           double beta1, int iters, int per_coordinate_normalize, int num_workers) {
    const double beta2 = beta1;  /* algo.cc:396 reads "beta1" twice */
    const int nt = num_workers > 0 ? num_workers : 1;
    /* Eigen converts the double scalars to the matrices' float Scalar type before use */
    const float b1 = (float)beta1, omb1 = (float)(1.0 - beta1);
    const float b2 = (float)beta2, omb2 = (float)(1.0 - beta2);
    const float bc1 = (float)(1.0 - pow(beta1, iters + 1));
    const float bc2 = (float)(1.0 - pow(beta2, iters + 1));
    const float two_reg = (float)(2 * reg), lrf = (float)lr;
#pragma omp parallel for schedule(static) num_threads(nt)
    for (int64_t r = 0; r < rows; ++r) {
        float* th = theta + r * cols;
        float* g = grad + r * cols;
        if (per_coordinate_normalize && cnt && cnt[r]) {
            for (int k = 0; k < cols; ++k) g[k] /= (float)cnt[r];       /* (:399-401) */
        }
        for (int k = 0; k < cols; ++k) g[k] -= th[k] * two_reg;         /* (:403) */
        if (optimizer == 2) {                                            /* adam (:365-375) */
            float* m = mom + r * cols;
            float* v = vel + r * cols;
            for (int k = 0; k < cols; ++k) {
                m[k] = b1 * m[k] + omb1 * g[k];
                v[k] = b2 * v[k] + omb2 * (g[k] * g[k]);
                const float m_hat = m[k] / bc1;
                const float v_hat = v[k] / bc2;
                g[k] = m_hat / (sqrtf(v_hat) + ORC_FEPS);
            }
        } else {                                                         /* adagrad (:377-380) */
            float* v = vel + r * cols;
            for (int k = 0; k < cols; ++k) {
                v[k] = v[k] + g[k] * g[k];
                g[k] = g[k] / (sqrtf(v[k]) + ORC_FEPS);
            }
        }
        for (int k = 0; k < cols; ++k) th[k] += lrf * g[k];              /* (:405) */
    }
}

/* CWARP::update_parameters tail (warp.cc:194-200): row /= max(1, ||row||) */
ORC_API void orc_warp_project(float* M, int64_t rows, int d, int num_workers) {
    const int nt = num_workers > 0 ? num_workers : 1;
#pragma omp parallel for schedule(static) num_threads(nt)
    for (int64_t r = 0; r < rows; ++r) {
        float* m = M + r * d;
        float nrm = sqrtf(dotf(m, m, d));
        float dv = nrm > 1.0f ? nrm : 1.0f;
        for (int k = 0; k < d; ++k) m[k] /= dv;
    }
}

/* CBPRMF::compute_loss (bpr.cc:227-244): mean log(1 + exp(-x_uij)) over probe triples */
ORC_API double orc_bpr_compute_loss(const float* P, const float* Q, const float* Qb, int d, int use_bias,
                                    const int32_t* us, const int32_t* poss, const int32_t* negs, int32_t n) {
    double l = 0.0;
    for (int i = 0; i < n; ++i) {
        const float* p = P + (int64_t)us[i] * d;
        float a = dotf(p, Q + (int64_t)poss[i] * d, d);
        float b = dotf(p, Q + (int64_t)negs[i] * d, d);
        if (use_bias) { a += Qb[poss[i]]; b += Qb[negs[i]]; }
        const double x = (double)a - (double)b;
        l += log(1.0 + exp(-x));
    }
    return n ? l / (double)n : 0.0;
}

/* CWARP::compute_loss (warp.cc:205-226): fraction of probe triples violating the margin */
ORC_API double orc_warp_compute_loss(const float* P, const float* Q, int d, int l2, double threshold,
                                     const int32_t* us, const int32_t* poss, const int32_t* negs, int32_t n) {
    int cnt = 0;
    for (int i = 0; i < n; ++i) {
        const float* p = P + (int64_t)us[i] * d;
        double a = warp_score(p, Q + (int64_t)poss[i] * d, d, l2);
        double b = warp_score(p, Q + (int64_t)negs[i] * d, d, l2);
        cnt += (a - b) < threshold;
    }
    return n ? (double)cnt / (double)n : 0.0;
}

/* linear lr decay of SGDAlgorithm::progress_manager (algo.cc:284-287) */
ORC_API double orc_lr_decay(double lr0, double min_lr, double processed, double total) {
    double progress = processed / total;
    double a = lr0 - (lr0 - min_lr) * progress;
    return a > min_lr ? a : min_lr;
}

ORC_API int orc_num_threads(void) { return omp_get_max_threads(); }
