// BPRMF / WARP backend: sampling, pairwise update, optimizer and loss kernels + C ABI.
// Replaces bpr::CBPRMF (lib/algo_impl/bpr/bpr.cc), warp::CWARP (lib/algo_impl/warp/warp.cc),
// SGDAlgorithm (lib/algo.cc:133-492) and cuda_bpr::CuBPR (lib/cuda/bpr/bpr.cu).
//
// Work decomposition: the reference packs CSR rows into jobs and feeds worker threads through a
// mutex queue (algo.cc:308-362, concurrent_queue.hpp); here the unit of work is one positive
// (u, pos) of the chunk, one warp each, grid-striding.  Every random draw is a pure function of
// (seed, epoch, global positive index, draw number) -- Philox4x32-10, bit-identical to
// oracle/buffalo_oracle.c -- so WARP epochs and BPR adagrad/adam epochs are reproducible and can be
// compared element-wise with the oracle; plain-SGD BPR is Hogwild (atomics) like the reference.
// The accumulating configurations still add their gradients with atomics, in whatever order the warps arrive; the
// option `deterministic` replaces those with ordered sums (sample records, a user pass, an item pass; see the
// "Deterministic mode" kernels below), so the same seed gives the same bits.
#include "bfl_common.cuh"

using namespace bfl;

namespace {

struct SgdArgs {
    float* P;
    float* Q;
    float* Qb;
    float* gP;
    float* gQ;
    float* gQb;
    int32_t* cP;
    int32_t* cQ;
    const int64_t* indptr;   // global end offsets (device)
    const int32_t* keys;     // element (it - shift)
    const int64_t* cum;      // cumulative popularity table or null
    int32_t* trace_trials;   // optional WARP trace (indexed it - shift)
    int32_t* trace_negs;
    double* stat_loss;       // device double
    unsigned long long* stat_updates;
    int64_t shift;
    int64_t row_begin, row_end;
    int64_t it_begin, it_end;  // global positive index range of the chunk
    int32_t num_items;
    int D, ld;
    int optimizer;  // 0 sgd 1 adagrad 2 adam
    int use_bias, update_i, update_j, num_neg, verify_neg, uniform, pcn, max_trials, score_l2;
    uint32_t seed, epoch;
    float reg_u, reg_i, reg_j, reg_b, lr, threshold;
};

// smallest row r in [lo, hi) with indptr[r] > it
__device__ __forceinline__ int64_t row_of(const int64_t* __restrict__ indptr, int64_t lo, int64_t hi, int64_t it) {
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg(indptr + mid) > it) hi = mid; else lo = mid + 1;
    }
    return lo;
}

__device__ __forceinline__ bool seen_sorted(const int32_t* __restrict__ keys, int64_t n, int32_t item) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg(keys + mid) < item) lo = mid + 1; else hi = mid;
    }
    return lo < n && __ldg(keys + lo) == item;
}

__device__ __forceinline__ int32_t cum_lower_bound(const int64_t* __restrict__ cum, int32_t size, int64_t r) {
    int32_t lo = 0, hi = size;
    while (lo < hi) {
        const int32_t mid = (lo + hi) >> 1;
        if (__ldg(cum + mid) < r) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// BPR negative of sample sid = it * num_neg + k of a row whose sorted positives are rk[0, n_seen) (bpr.cc:106-117)
__device__ __forceinline__ int32_t bpr_draw_negative(const SgdArgs& a, uint64_t sid, const int32_t* rk, int64_t n_seen) {
    int32_t neg = 0;
    for (uint32_t t = 0;; ++t) {
        if (a.uniform) {
            neg = draw_range(a.seed, a.epoch, sid, t, (uint32_t)a.num_items);
        } else {
            const uint64_t tot = (uint64_t)__ldg(a.cum + a.num_items - 1);
            const uint64_t r64 = ((uint64_t)draw_u32(a.seed, a.epoch, sid, 2 * t) << 32) |
                                 draw_u32(a.seed, a.epoch, sid, 2 * t + 1);
            const int64_t r = (int64_t)__umul64hi(r64, tot);
            neg = cum_lower_bound(a.cum, a.num_items, r);
            if (neg >= a.num_items) neg = a.num_items - 1;
        }
        if (!a.verify_neg || !seen_sorted(rk, n_seen, neg)) break;
        if (t >= 64) break;
    }
    return neg;
}

// ---------------------------------------------------------------------------------------
// BPR negative sampling (bpr.cc:106-117; reference GPU: fill_rows + generate_samples,
// bpr.cu:22-87).  One thread per (positive, k < num_neg).
// ---------------------------------------------------------------------------------------
__global__ void bpr_sample_kernel(SgdArgs a, int32_t* __restrict__ out_u, int32_t* __restrict__ out_pos,
                                  int32_t* __restrict__ out_neg) {
    const int64_t total = (a.it_end - a.it_begin) * a.num_neg;
    for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < total; s += (int64_t)gridDim.x * blockDim.x) {
        const int64_t it = a.it_begin + s / a.num_neg;
        const int k = (int)(s % a.num_neg);
        const int64_t row = row_of(a.indptr, a.row_begin, a.row_end, it);
        const int64_t beg = row == 0 ? 0 : __ldg(a.indptr + row - 1);
        const int64_t end = __ldg(a.indptr + row);
        const int32_t* rk = a.keys + (beg - a.shift);
        const uint64_t sid = (uint64_t)it * a.num_neg + k;
        const int32_t neg = bpr_draw_negative(a, sid, rk, end - beg);
        out_u[s] = (int32_t)row;
        out_pos[s] = __ldg(a.keys + (it - a.shift));
        out_neg[s] = neg;
    }
}

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
// L2-coherent read: rows are being updated by atomics from other SMs (and by this warp's previous triple)
__device__ __forceinline__ float4 ld4_cg(const float* p) { return __ldcg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ void red4(float* p, float4 v) { atomicAdd(reinterpret_cast<float4*>(p), v); }

// ---------------------------------------------------------------------------------------
// BPR pairwise step (bpr.cc:119-171; reference GPU update_bpr_kernel bpr.cu:89-146).
// One warp per triple; rows are read/updated as float4 (row pitch ld is a multiple of 4,
// padding columns are zero and stay zero).  NV = ceil(ld / 128).
// sgd: deltas are formed from the values read before the step and applied with vector atomics
// (pre-update form, like bpr.cu:122-134).  adagrad/adam: gradients are accumulated (bpr.cc:138-156).
// ---------------------------------------------------------------------------------------
template <int NV>
__global__ void __launch_bounds__(256) bpr_apply_kernel(SgdArgs a, const int32_t* __restrict__ us,
                                                       const int32_t* __restrict__ poss,
                                                       const int32_t* __restrict__ negs, int64_t n) {
    const int lane = threadIdx.x & 31;
    const int64_t w0 = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp_id_uniform();
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int nv4 = a.ld >> 2;
    // Each warp walks a CONTIGUOUS range of triples one after the other, like a worker thread of the reference
    // walks its job's rows (bpr.cc:103-117): the positives of one user are applied sequentially and concurrent
    // warps work on different users, so only item rows are shared Hogwild-style.
    const int64_t per = (n + nw - 1) / nw;
    const int64_t s_end = (w0 + 1) * per < n ? (w0 + 1) * per : n;
    for (int64_t s = w0 * per; s < s_end; ++s) {
        const int u = __ldg(us + s), pos = __ldg(poss + s), neg = __ldg(negs + s);
        float* pu = a.P + (int64_t)u * a.ld;
        float* qi = a.Q + (int64_t)pos * a.ld;
        float* qj = a.Q + (int64_t)neg * a.ld;
        float4 vp[NV], vi[NV], vj[NV];
        float part = 0.f;
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const int c = lane + 32 * k;
            if (c < nv4) {
                vp[k] = ld4_cg(pu + 4 * c);
                vi[k] = ld4_cg(qi + 4 * c);
                vj[k] = ld4_cg(qj + 4 * c);
                part += vp[k].x * (vi[k].x - vj[k].x) + vp[k].y * (vi[k].y - vj[k].y) +
                        vp[k].z * (vi[k].z - vj[k].z) + vp[k].w * (vi[k].w - vj[k].w);
            }
        }
        float x = warp_sum(part);  // bpr.cc:119
        float bi = 0.f, bj = 0.f;
        if (a.use_bias) {
            bi = __ldcg(a.Qb + pos);
            bj = __ldcg(a.Qb + neg);
            x += bi - bj;  // bpr.cc:120-121
        }
        // logit = 1 - sigmoid(x) with the reference's clamp at +-MAX_EXP = 6 (bpr.cc:123-131; the exact
        // expression of bpr.cu:113-116 instead of the CPU path's 1000-entry table)
        const float logit = x > 6.f ? 0.f : (x < -6.f ? 1.f : 1.0f / (1.0f + __expf(x)));
        if (a.optimizer != 0) {
#pragma unroll
            for (int k = 0; k < NV; ++k) {
                const int c = lane + 32 * k;
                if (c < nv4) {
                    red4(a.gP + (int64_t)u * a.ld + 4 * c,
                         make_float4(logit * (vi[k].x - vj[k].x), logit * (vi[k].y - vj[k].y),
                                     logit * (vi[k].z - vj[k].z), logit * (vi[k].w - vj[k].w)));
                    const float4 g = make_float4(logit * vp[k].x, logit * vp[k].y, logit * vp[k].z, logit * vp[k].w);
                    if (a.update_i) red4(a.gQ + (int64_t)pos * a.ld + 4 * c, g);
                    if (a.update_j) red4(a.gQ + (int64_t)neg * a.ld + 4 * c, make_float4(-g.x, -g.y, -g.z, -g.w));
                }
            }
            if (lane == 0) {
                if (a.use_bias) {
                    if (a.update_i) atomicAdd(a.gQb + pos, logit);
                    if (a.update_j) atomicAdd(a.gQb + neg, -logit);
                }
                if (a.pcn) {  // bpr.cc:140-143 per sample; :174-181 once per positive
                    atomicAdd(a.cQ + neg, 1);
                    if (s % a.num_neg == 0) {
                        atomicAdd(a.cP + u, 1);
                        atomicAdd(a.cQ + pos, 1);
                    }
                }
            }
        } else {
            const float lr = a.lr;
#pragma unroll
            for (int k = 0; k < NV; ++k) {
                const int c = lane + 32 * k;
                if (c < nv4) {
                    if (a.update_i)
                        red4(qi + 4 * c, make_float4(lr * (logit * vp[k].x - a.reg_i * vi[k].x),
                                                     lr * (logit * vp[k].y - a.reg_i * vi[k].y),
                                                     lr * (logit * vp[k].z - a.reg_i * vi[k].z),
                                                     lr * (logit * vp[k].w - a.reg_i * vi[k].w)));
                    if (a.update_j)
                        red4(qj + 4 * c, make_float4(lr * (-logit * vp[k].x - a.reg_j * vj[k].x),
                                                     lr * (-logit * vp[k].y - a.reg_j * vj[k].y),
                                                     lr * (-logit * vp[k].z - a.reg_j * vj[k].z),
                                                     lr * (-logit * vp[k].w - a.reg_j * vj[k].w)));
                    red4(pu + 4 * c, make_float4(lr * (logit * (vi[k].x - vj[k].x) - a.reg_u * vp[k].x),
                                                 lr * (logit * (vi[k].y - vj[k].y) - a.reg_u * vp[k].y),
                                                 lr * (logit * (vi[k].z - vj[k].z) - a.reg_u * vp[k].z),
                                                 lr * (logit * (vi[k].w - vj[k].w) - a.reg_u * vp[k].w)));
                }
            }
            if (lane == 0 && a.use_bias) {
                if (a.update_i) atomicAdd(a.Qb + pos, lr * (logit - a.reg_b * bi));
                if (a.update_j) atomicAdd(a.Qb + neg, lr * (-logit - a.reg_b * bj));
            }
        }
    }
}

// ---------------------------------------------------------------------------------------
// WARP rank sampling + gradient accumulation (warp.cc:103-173).  One warp per positive.
// P and Q are read-only inside an epoch (gradients only, warp.cc:156-158).
// ---------------------------------------------------------------------------------------
template <int NV>
__device__ __forceinline__ float warp_score(const float4 (&vp)[NV], const float* __restrict__ q, int nv4, int lane,
                                            int l2, float4 (&vq)[NV]) {
    float part = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        const int c = lane + 32 * k;
        if (c < nv4) {
            vq[k] = ld4(q + 4 * c);
            if (l2) {
                const float dx = vp[k].x - vq[k].x, dy = vp[k].y - vq[k].y, dz = vp[k].z - vq[k].z,
                            dw = vp[k].w - vq[k].w;
                part -= dx * dx + dy * dy + dz * dz + dw * dw;  // warp.cc:25-28
            } else {
                part += vp[k].x * vq[k].x + vp[k].y * vq[k].y + vp[k].z * vq[k].z + vp[k].w * vq[k].w;  // :21-23
            }
        }
    }
    return warp_sum(part);
}

// Rank sampling of positive `it` (warp.cc:137-148): draws until a violating negative or max_trials; returns the trial
// count, the last negative and its score (row in vj).
template <int NV>
__device__ __forceinline__ int warp_rank_draw(const SgdArgs& a, int64_t it, const int32_t* rk, int64_t n_seen,
                                              const float4 (&vp)[NV], float ui, int nv4, int lane, float4 (&vj)[NV],
                                              int& neg, float& uj) {
    int trial = 1;
    uint32_t t = 0;
    while (trial <= a.max_trials) {  // warp.cc:137-148
        neg = draw_range(a.seed, a.epoch, (uint64_t)it, t++, (uint32_t)a.num_items);
        if (uni(seen_sorted(rk, n_seen, neg))) {  // :140-141, not counted as a trial
            if (t > (uint32_t)(64 * a.max_trials + 4096)) {
                trial = a.max_trials + 1;
                break;
            }
            continue;
        }
        trial += 1;  // :142
        uj = uni(warp_score<NV>(vp, a.Q + (int64_t)neg * a.ld, nv4, lane, a.score_l2, vj));
        if ((ui - uj) < a.threshold) break;  // :145-146
        trial += 1;  // :147
    }
    return trial;
}

template <int NV>
__global__ void __launch_bounds__(256) warp_accumulate_kernel(SgdArgs a) {
    const int lane = threadIdx.x & 31;
    const int64_t w0 = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp_id_uniform();
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int nv4 = a.ld >> 2;
    double loss = 0.0;
    unsigned long long updates = 0;
    for (int64_t it = a.it_begin + w0; it < a.it_end; it += nw) {
        const int64_t row = uni((long long)row_of(a.indptr, a.row_begin, a.row_end, it));
        const int64_t beg = uni((long long)(row == 0 ? 0 : __ldg(a.indptr + row - 1)));
        const int64_t end = uni((long long)__ldg(a.indptr + row));
        const int32_t* rk = a.keys + (beg - a.shift);
        const int64_t n_seen = end - beg;
        const int pos = uni(__ldg(a.keys + (it - a.shift)));
        const float* pu = a.P + row * a.ld;
        const float* qi = a.Q + (int64_t)pos * a.ld;
        float4 vp[NV], vi[NV], vj[NV];
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const int c = lane + 32 * k;
            vp[k] = c < nv4 ? ld4(pu + 4 * c) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        const float ui = uni(warp_score<NV>(vp, qi, nv4, lane, a.score_l2, vi));  // warp.cc:133
        float uj = 0.f;
        int neg = 0;
        const int trial = warp_rank_draw<NV>(a, it, rk, n_seen, vp, ui, nv4, lane, vj, neg, uj);
        const bool discard = trial >= a.max_trials;  // :149-150
        if (lane == 0) {
            if (a.trace_trials) a.trace_trials[it - a.shift] = discard ? 0 : trial;
            if (a.trace_negs) a.trace_negs[it - a.shift] = discard ? -1 : neg;
        }
        if (discard) continue;
        int64_t ratio = ((int64_t)a.num_items - n_seen - 1) / trial;  // :152
        if (ratio < 1) ratio = 1;
        const float Phi = logf((float)(int)ratio);
        float* gp = a.gP + row * a.ld;
        float* gi = a.gQ + (int64_t)pos * a.ld;
        float* gj = a.gQ + (int64_t)neg * a.ld;
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const int c = lane + 32 * k;
            if (c < nv4) {
                float4 du, di, dj;
                if (!a.score_l2) {  // dot_deriv warp.cc:30-40
                    du = make_float4(Phi * (vi[k].x - vj[k].x), Phi * (vi[k].y - vj[k].y), Phi * (vi[k].z - vj[k].z),
                                     Phi * (vi[k].w - vj[k].w));
                    di = make_float4(Phi * vp[k].x, Phi * vp[k].y, Phi * vp[k].z, Phi * vp[k].w);
                    dj = make_float4(-di.x, -di.y, -di.z, -di.w);
                } else {  // l2_deriv warp.cc:42-52
                    du = make_float4(Phi * 2 * (vi[k].x - vj[k].x), Phi * 2 * (vi[k].y - vj[k].y),
                                     Phi * 2 * (vi[k].z - vj[k].z), Phi * 2 * (vi[k].w - vj[k].w));
                    di = make_float4(Phi * (vp[k].x - vi[k].x), Phi * (vp[k].y - vi[k].y), Phi * (vp[k].z - vi[k].z),
                                     Phi * (vp[k].w - vi[k].w));
                    dj = make_float4(-Phi * (vp[k].x - vj[k].x), -Phi * (vp[k].y - vj[k].y),
                                     -Phi * (vp[k].z - vj[k].z), -Phi * (vp[k].w - vj[k].w));
                }
                // grad += deriv - reg * param  (warp.cc:156-158)
                red4(gp + 4 * c, make_float4(du.x - a.reg_u * vp[k].x, du.y - a.reg_u * vp[k].y,
                                             du.z - a.reg_u * vp[k].z, du.w - a.reg_u * vp[k].w));
                red4(gi + 4 * c, make_float4(di.x - a.reg_i * vi[k].x, di.y - a.reg_i * vi[k].y,
                                             di.z - a.reg_i * vi[k].z, di.w - a.reg_i * vi[k].w));
                red4(gj + 4 * c, make_float4(dj.x - a.reg_j * vj[k].x, dj.y - a.reg_j * vj[k].y,
                                             dj.z - a.reg_j * vj[k].z, dj.w - a.reg_j * vj[k].w));
            }
        }
        if (lane == 0 && a.pcn) {  // warp.cc:159-165
            atomicAdd(a.cP + row, 1);
            atomicAdd(a.cQ + pos, 1);
            atomicAdd(a.cQ + neg, 1);
        }
        loss += (double)(uj - ui + a.threshold);  // :166
        updates += 1;
    }
    if (lane == 0 && updates) {
        atomicAdd(a.stat_loss, loss);
        atomicAdd(a.stat_updates, updates);
    }
}

// ---------------------------------------------------------------------------------------
// SGDAlgorithm::update_parameters (algo.cc:382-465): element-wise Adam / Adagrad step.
// beta2 := beta1 (algo.cc:396); the gradient buffer ends up holding the step and is NOT
// cleared (no setZero in the reference).  One thread per element; `cols` = row pitch.
// ---------------------------------------------------------------------------------------
__global__ void sgd_apply_kernel(int optimizer, float* __restrict__ theta, float* __restrict__ grad,
                                 float* __restrict__ mom, float* __restrict__ vel, const int32_t* __restrict__ cnt,
                                 int64_t rows, int cols, float two_reg, float lr, float b1, float omb1, float b2,
                                 float omb2, float bc1, float bc2, int pcn) {
    const int64_t n = rows * cols;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
        float g = grad[e];
        const float th = theta[e];
        if (pcn) {
            const int c = cnt[e / cols];
            if (c) g /= (float)c;  // algo.cc:399-401
        }
        g -= th * two_reg;  // :403
        if (optimizer == 2) {  // update_adam :365-375
            const float m = b1 * mom[e] + omb1 * g;
            const float v = b2 * vel[e] + omb2 * (g * g);
            mom[e] = m;
            vel[e] = v;
            g = (m / bc1) / (sqrtf(v / bc2) + 1e-10f);
        } else {  // update_adagrad :377-380
            const float v = vel[e] + g * g;
            vel[e] = v;
            g = g / (sqrtf(v) + 1e-10f);
        }
        grad[e] = g;
        theta[e] = th + lr * g;  // :405
    }
}

// CWARP::update_parameters tail (warp.cc:194-200): row /= max(1, ||row||).  One warp per row.
__global__ void warp_project_kernel(float* __restrict__ M, int64_t rows, int ld) {
    const int lane = threadIdx.x & 31;
    const int64_t w0 = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp_id_uniform();
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = w0; r < rows; r += nw) {
        float* m = M + r * ld;
        float s = 0.f;
        for (int c = lane; c < ld; c += 32) s += m[c] * m[c];
        s = sqrtf(warp_sum(s));
        if (s > 1.0f)
            for (int c = lane; c < ld; c += 32) m[c] /= s;
    }
}

// loss term of probe triple i: BPR log(1+exp(-x_uij)) (bpr.cc:227-244); WARP 1 if violating (warp.cc:205-226)
__device__ __forceinline__ double probe_term(int kind, const float* __restrict__ P, const float* __restrict__ Q,
                                             const float* __restrict__ Qb, int D, int ld, int use_bias, int l2,
                                             double threshold, const int32_t* __restrict__ us,
                                             const int32_t* __restrict__ ps, const int32_t* __restrict__ ns, int i,
                                             int lane) {
    const float* p = P + (int64_t)us[i] * ld;
    const float* qi = Q + (int64_t)ps[i] * ld;
    const float* qj = Q + (int64_t)ns[i] * ld;
    float sa = 0.f, sb = 0.f;
    for (int c = lane; c < D; c += 32) {
        if (l2) {
            const float da = p[c] - qi[c], db = p[c] - qj[c];
            sa -= da * da;
            sb -= db * db;
        } else {
            sa += p[c] * qi[c];
            sb += p[c] * qj[c];
        }
    }
    sa = warp_sum(sa);
    sb = warp_sum(sb);
    if (kind == BFL_SGD_BPR) {
        if (use_bias) {
            sa += Qb[ps[i]];
            sb += Qb[ns[i]];
        }
        return log(1.0 + exp(-((double)sa - (double)sb)));
    }
    return (((double)sa - (double)sb) < threshold) ? 1.0 : 0.0;
}

// probe losses: BPR mean log(1+exp(-x_uij)) (bpr.cc:227-244); WARP fraction violating (warp.cc:205-226)
__global__ void probe_loss_kernel(int kind, const float* __restrict__ P, const float* __restrict__ Q,
                                  const float* __restrict__ Qb, int D, int ld, int use_bias, int l2,
                                  double threshold, const int32_t* __restrict__ us, const int32_t* __restrict__ ps,
                                  const int32_t* __restrict__ ns, int n, double* out) {
    const int lane = threadIdx.x & 31;
    const int w0 = blockIdx.x * (blockDim.x >> 5) + warp_id_uniform();
    const int nw = (gridDim.x * blockDim.x) >> 5;
    double acc = 0.0;
    for (int i = w0; i < n; i += nw)
        acc += probe_term(kind, P, Q, Qb, D, ld, use_bias, l2, threshold, us, ps, ns, i, lane);
    if (lane == 0 && acc != 0.0) atomicAdd(out, acc);
}

// ---------------------------------------------------------------------------------------
// Deterministic mode (option `deterministic`; WARP, BPR adagrad / adam).  P, Q and Qb are read-only during the
// epoch, so every gradient row is a plain sum over the epoch's samples; here that sum is taken in a fixed order.
//   sample pass  one record per sample s = it * num_neg + k: user, positive i, negative j (-1: WARP discard),
//                coefficient c (BPR logit, WARP Phi); two item entries 2s (i, +c) and 2s + 1 (j, -c)
//   user pass    gP[u] += the user's sample terms in ascending s                     (per add_jobs chunk)
//   item pass    the entries sorted by item (stable, so each item's entries stay in ascending 2s + side order);
//                gQ[i] += and gQb[i] += the item's terms in that order               (once per epoch)
// "In order" means: the element sequence is cut at the multiples of kDetSegment of its global index, each piece is
// summed from zero in element order, the pieces are added in order and the result is added to the gradient row once.
// Every bound depends on the data only, not on the grid, the SM count or the chunking.
// ---------------------------------------------------------------------------------------
constexpr int64_t kDetSegment = 4096;    // elements per segment of the user and item sums
constexpr int64_t kDetLossRange = 4096;  // terms per fixed partial of the loss trees

struct DetRec {
    int32_t* u;      // [N] sample records, N = epoch positives * num_neg
    int32_t* i;
    int32_t* j;
    float* c;
    int32_t* major;  // [2N] item of entry 2s + side, num_items when the entry does not update a row
    float* cval;     // [2N] +c / -c
    float* loss;     // [N] WARP loss term, 0 for discards
};

__device__ __forceinline__ float4 f4_sub(float4 a, float4 b) {
    return make_float4(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y), __fsub_rn(a.z, b.z), __fsub_rn(a.w, b.w));
}
__device__ __forceinline__ float4 f4_add(float4 a, float4 b) {
    return make_float4(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z), __fadd_rn(a.w, b.w));
}
__device__ __forceinline__ float4 f4_scale(float c, float4 a) {
    return make_float4(__fmul_rn(c, a.x), __fmul_rn(c, a.y), __fmul_rn(c, a.z), __fmul_rn(c, a.w));
}

// BPR sample pass: one warp per sample.  The draw, the score and the logit are those of bpr_sample_kernel and
// bpr_apply_kernel; the sample counters of per_coordinate_normalize are integer atomics as there.
template <int NV>
__global__ void __launch_bounds__(256) det_bpr_sample_kernel(SgdArgs a, DetRec r) {
    const int lane = threadIdx.x & 31;
    const int64_t w0 = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp_id_uniform();
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int nv4 = a.ld >> 2;
    const int64_t s_end = a.it_end * a.num_neg;
    for (int64_t s = a.it_begin * a.num_neg + w0; s < s_end; s += nw) {
        const int64_t it = s / a.num_neg;
        const int64_t row = uni((long long)row_of(a.indptr, a.row_begin, a.row_end, it));
        const int64_t beg = row == 0 ? 0 : __ldg(a.indptr + row - 1);
        const int64_t end = __ldg(a.indptr + row);
        const int pos = uni(__ldg(a.keys + (it - a.shift)));
        const int neg = uni(bpr_draw_negative(a, (uint64_t)s, a.keys + (beg - a.shift), end - beg));
        const float* pu = a.P + row * a.ld;
        const float* qi = a.Q + (int64_t)pos * a.ld;
        const float* qj = a.Q + (int64_t)neg * a.ld;
        float part = 0.f;
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const int c = lane + 32 * k;
            if (c < nv4) {
                const float4 vp = ld4(pu + 4 * c), vi = ld4(qi + 4 * c), vj = ld4(qj + 4 * c);
                part += vp.x * (vi.x - vj.x) + vp.y * (vi.y - vj.y) + vp.z * (vi.z - vj.z) + vp.w * (vi.w - vj.w);
            }
        }
        float x = warp_sum(part);
        if (a.use_bias) x += __ldg(a.Qb + pos) - __ldg(a.Qb + neg);
        const float logit = x > 6.f ? 0.f : (x < -6.f ? 1.f : 1.0f / (1.0f + __expf(x)));
        if (lane == 0) {
            r.u[s] = (int32_t)row;
            r.i[s] = pos;
            r.j[s] = neg;
            r.c[s] = logit;
            r.major[2 * s] = a.update_i ? pos : a.num_items;
            r.major[2 * s + 1] = a.update_j ? neg : a.num_items;
            r.cval[2 * s] = logit;
            r.cval[2 * s + 1] = -logit;
            if (a.pcn) {
                atomicAdd(a.cQ + neg, 1);
                if (s % a.num_neg == 0) {
                    atomicAdd(a.cP + row, 1);
                    atomicAdd(a.cQ + pos, 1);
                }
            }
        }
    }
}

// WARP sample pass: warp_accumulate_kernel's rank sampling, trace and counters; the gradient terms become a record.
template <int NV>
__global__ void __launch_bounds__(256) det_warp_sample_kernel(SgdArgs a, DetRec r) {
    const int lane = threadIdx.x & 31;
    const int64_t w0 = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp_id_uniform();
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int nv4 = a.ld >> 2;
    unsigned long long updates = 0;
    for (int64_t it = a.it_begin + w0; it < a.it_end; it += nw) {
        const int64_t row = uni((long long)row_of(a.indptr, a.row_begin, a.row_end, it));
        const int64_t beg = uni((long long)(row == 0 ? 0 : __ldg(a.indptr + row - 1)));
        const int64_t end = uni((long long)__ldg(a.indptr + row));
        const int64_t n_seen = end - beg;
        const int pos = uni(__ldg(a.keys + (it - a.shift)));
        const float* pu = a.P + row * a.ld;
        float4 vp[NV], vi[NV], vj[NV];
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const int c = lane + 32 * k;
            vp[k] = c < nv4 ? ld4(pu + 4 * c) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        const float ui = uni(warp_score<NV>(vp, a.Q + (int64_t)pos * a.ld, nv4, lane, a.score_l2, vi));
        float uj = 0.f;
        int neg = 0;
        const int trial = warp_rank_draw<NV>(a, it, a.keys + (beg - a.shift), n_seen, vp, ui, nv4, lane, vj, neg, uj);
        const bool discard = trial >= a.max_trials;
        float Phi = 0.f;
        if (!discard) {
            int64_t ratio = ((int64_t)a.num_items - n_seen - 1) / trial;
            if (ratio < 1) ratio = 1;
            Phi = logf((float)(int)ratio);
            updates += 1;
        }
        if (lane == 0) {
            if (a.trace_trials) a.trace_trials[it - a.shift] = discard ? 0 : trial;
            if (a.trace_negs) a.trace_negs[it - a.shift] = discard ? -1 : neg;
            r.u[it] = (int32_t)row;
            r.i[it] = pos;
            r.j[it] = discard ? -1 : neg;
            r.c[it] = Phi;
            r.major[2 * it] = discard ? a.num_items : pos;
            r.major[2 * it + 1] = discard ? a.num_items : neg;
            r.cval[2 * it] = Phi;
            r.cval[2 * it + 1] = -Phi;
            r.loss[it] = discard ? 0.f : uj - ui + a.threshold;
            if (!discard && a.pcn) {
                atomicAdd(a.cP + row, 1);
                atomicAdd(a.cQ + pos, 1);
                atomicAdd(a.cQ + neg, 1);
            }
        }
    }
    if (lane == 0 && updates) atomicAdd(a.stat_updates, updates);
}

// One segmented, ordered sum over the elements [e_begin, e_end) of the rows [row_lo, row_hi); row r owns the elements
// [ends[r - 1], ends[r]) * per_row.  User pass (kItem false): element s is sample s, the row is P's.  Item pass: element
// e is the sorted entry code[e] = 2s + side with coefficient cval[e], the row is Q's.
struct DetSum {
    const float* P;
    const float* Q;
    const int32_t* rec_u;
    const int32_t* rec_i;
    const int32_t* rec_j;
    const float* rec_c;
    const int32_t* code;
    const float* cval;
    const int64_t* ends;
    float* out;      // gP or gQ
    float* outb;     // gQb or null
    float* part;     // [segment][2][pitch]: slot 0 the piece of a row begun in an earlier segment, slot 1 the first
                     // piece of a row that goes on into the next segment; the bias partial at column ld
    int64_t row_lo, row_hi, e_begin, e_end;
    int per_row, ld, pitch;
    int warp, l2;
    float reg_u, reg_i, reg_j;
};

// the term of element e (lanes' columns), its bias term (item pass) and whether it counts
template <int NV, bool kItem>
__device__ __forceinline__ bool det_term(const DetSum& a, int64_t e, int nv4, int lane, const float4 (&own)[NV],
                                         float4 (&t)[NV], float& tb) {
    if constexpr (kItem) {
        const int32_t code = __ldg(a.code + e);
        const float cs = __ldg(a.cval + e);
        const float reg = (code & 1) ? a.reg_j : a.reg_i;
        const float* pu = a.P + (int64_t)__ldg(a.rec_u + (code >> 1)) * a.ld;
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const int c = lane + 32 * k;
            if (c < nv4) {
                const float4 vp = ld4(pu + 4 * c);
                if (!a.warp) t[k] = f4_scale(cs, vp);                                        // bpr.cc:150-153
                else if (!a.l2) t[k] = f4_sub(f4_scale(cs, vp), f4_scale(reg, own[k]));      // warp.cc:30-40, :156-158
                else t[k] = f4_sub(f4_scale(cs, f4_sub(vp, own[k])), f4_scale(reg, own[k]));  // warp.cc:42-52
            }
        }
        tb = cs;
        return true;
    } else {
        const int32_t j = __ldg(a.rec_j + e);
        if (j < 0) return false;  // a discarded WARP positive contributes nothing
        const float c0 = __ldg(a.rec_c + e);
        const float cu = (a.warp && a.l2) ? __fmul_rn(c0, 2.f) : c0;
        const float* qi = a.Q + (int64_t)__ldg(a.rec_i + e) * a.ld;
        const float* qj = a.Q + (int64_t)j * a.ld;
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const int c = lane + 32 * k;
            if (c < nv4) {
                const float4 du = f4_scale(cu, f4_sub(ld4(qi + 4 * c), ld4(qj + 4 * c)));
                t[k] = a.warp ? f4_sub(du, f4_scale(a.reg_u, own[k])) : du;
            }
        }
        tb = 0.f;
        return true;
    }
}

// one warp per segment: every row piece of the segment is summed in element order; a row that lies inside the
// segment is added to its gradient row here, the pieces of longer rows go to `part` for det_combine_kernel
template <int NV, bool kItem>
__global__ void __launch_bounds__(256) det_sum_kernel(DetSum a) {
    const int lane = threadIdx.x & 31;
    const int64_t w0 = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp_id_uniform();
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int nv4 = a.ld >> 2;
    const int64_t t_end = (a.e_end + kDetSegment - 1) / kDetSegment;
    for (int64_t t = a.e_begin / kDetSegment + w0; t < t_end; t += nw) {
        const int64_t tb = t * kDetSegment, te = tb + kDetSegment;
        int64_t e = tb > a.e_begin ? tb : a.e_begin;
        const int64_t e1 = te < a.e_end ? te : a.e_end;
        int64_t r = uni((long long)row_of(a.ends, a.row_lo, a.row_hi, e / a.per_row));
        while (e < e1) {
            const int64_t rb = (r == 0 ? 0 : __ldg(a.ends + r - 1)) * a.per_row, re = __ldg(a.ends + r) * a.per_row;
            if (re <= e) {  // empty row
                ++r;
                continue;
            }
            // the row's own factor row: WARP's regularisation terms and l2 score read it
            float4 own[NV];
            const float* orow = (kItem ? a.Q : a.P) + r * a.ld;
#pragma unroll
            for (int k = 0; k < NV; ++k) {
                const int c = lane + 32 * k;
                own[k] = (a.warp && c < nv4) ? ld4(orow + 4 * c) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
            float4 acc[NV];
#pragma unroll
            for (int k = 0; k < NV; ++k) acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            float accb = 0.f;
            const int64_t pe = re < e1 ? re : e1;
            for (; e < pe; ++e) {
                float4 t4[NV];
                float b = 0.f;
                if (det_term<NV, kItem>(a, e, nv4, lane, own, t4, b)) {
#pragma unroll
                    for (int k = 0; k < NV; ++k)
                        if (lane + 32 * k < nv4) acc[k] = f4_add(acc[k], t4[k]);
                    accb = __fadd_rn(accb, b);
                }
            }
            if (rb >= tb && re <= te) {  // the whole row: add it once
                float* o = a.out + r * a.ld;
#pragma unroll
                for (int k = 0; k < NV; ++k) {
                    const int c = lane + 32 * k;
                    if (c < nv4) *reinterpret_cast<float4*>(o + 4 * c) = f4_add(ld4(o + 4 * c), acc[k]);
                }
                if (lane == 0 && a.outb) a.outb[r] = __fadd_rn(a.outb[r], accb);
            } else {
                float* p = a.part + (2 * t + (rb < tb ? 0 : 1)) * a.pitch;
#pragma unroll
                for (int k = 0; k < NV; ++k) {
                    const int c = lane + 32 * k;
                    if (c < nv4) *reinterpret_cast<float4*>(p + 4 * c) = acc[k];
                }
                if (lane == 0) p[a.ld] = accb;
            }
            ++r;
        }
    }
}

// one warp per segment t that holds the first piece of a row going on past it: the row's pieces in segment order,
// then added to its gradient row once
template <int NV>
__global__ void __launch_bounds__(256) det_combine_kernel(DetSum a) {
    const int lane = threadIdx.x & 31;
    const int64_t w0 = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp_id_uniform();
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int nv4 = a.ld >> 2;
    const int64_t t_end = (a.e_end + kDetSegment - 1) / kDetSegment;
    for (int64_t t = a.e_begin / kDetSegment + w0; t < t_end; t += nw) {
        const int64_t tb = t * kDetSegment, te = tb + kDetSegment;
        const int64_t e_last = (te < a.e_end ? te : a.e_end) - 1;
        if (e_last < a.e_begin) continue;
        const int64_t r = uni((long long)row_of(a.ends, a.row_lo, a.row_hi, e_last / a.per_row));
        const int64_t rb = (r == 0 ? 0 : __ldg(a.ends + r - 1)) * a.per_row, re = __ldg(a.ends + r) * a.per_row;
        if (rb < tb || re <= te) continue;
        float4 acc[NV];
        const float* p = a.part + (2 * t + 1) * a.pitch;
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const int c = lane + 32 * k;
            acc[k] = c < nv4 ? ld4(p + 4 * c) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        float accb = p[a.ld];
        for (int64_t t2 = t + 1; t2 * kDetSegment < re; ++t2) {
            const float* q = a.part + 2 * t2 * a.pitch;
#pragma unroll
            for (int k = 0; k < NV; ++k)
                if (lane + 32 * k < nv4) acc[k] = f4_add(acc[k], ld4(q + 4 * (lane + 32 * k)));
            accb = __fadd_rn(accb, q[a.ld]);
        }
        float* o = a.out + r * a.ld;
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const int c = lane + 32 * k;
            if (c < nv4) *reinterpret_cast<float4*>(o + 4 * c) = f4_add(ld4(o + 4 * c), acc[k]);
        }
        if (lane == 0 && a.outb) a.outb[r] = __fadd_rn(a.outb[r], accb);
    }
}

__global__ void det_reset_kernel(int32_t* __restrict__ major, int32_t* __restrict__ iota, int64_t n, int32_t sentinel) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
        major[e] = sentinel;
        if (iota) iota[e] = (int32_t)e;
    }
}

// deterministic probe loss: one term per triple
__global__ void det_probe_terms_kernel(int kind, const float* __restrict__ P, const float* __restrict__ Q,
                                       const float* __restrict__ Qb, int D, int ld, int use_bias, int l2,
                                       double threshold, const int32_t* __restrict__ us,
                                       const int32_t* __restrict__ ps, const int32_t* __restrict__ ns, int n,
                                       double* __restrict__ terms) {
    const int lane = threadIdx.x & 31;
    const int w0 = blockIdx.x * (blockDim.x >> 5) + warp_id_uniform();
    const int nw = (gridDim.x * blockDim.x) >> 5;
    for (int i = w0; i < n; i += nw) {
        const double v = probe_term(kind, P, Q, Qb, D, ld, use_bias, l2, threshold, us, ps, ns, i, lane);
        if (lane == 0) terms[i] = v;
    }
}

// Deterministic loss, stage 1: the terms of the fixed ranges of kDetLossRange, each summed by a fixed tree (fp64).
template <typename T>
__global__ void __launch_bounds__(256) det_loss_partial_kernel(const T* terms, int64_t n, double* part) {
    __shared__ double s[256];
    const int64_t lo = (int64_t)blockIdx.x * kDetLossRange, hi = min(n, lo + kDetLossRange);
    double t = 0.0;
    for (int64_t i = lo + threadIdx.x; i < hi; i += 256) t += (double)terms[i];
    s[threadIdx.x] = t;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) part[blockIdx.x] = s[0];
}

// Deterministic loss, stage 2 (one CTA of 256 threads): the partials by the same tree, added into *loss.
__global__ void __launch_bounds__(256) det_loss_final_kernel(const double* part, int64_t nblk, double* loss) {
    __shared__ double s[256];
    double t = 0.0;
    for (int64_t i = threadIdx.x; i < nblk; i += 256) t += part[i];
    s[threadIdx.x] = t;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) *loss += s[0];
}

// ---------------------------------------------------------------------------------------
// Item fold-in (DESIGN.md 4.16): the item side of training's epoch for rows x that are not in Q, with P, Q and Qb
// frozen.  One warp per new row, grid-striding; the row, its bias and its optimizer state stay in registers for all
// epochs.  Positive (u, x) is history entry `it` of row r, visited in CSR order; its negatives come from the model's
// sampler against user u's row of the training CSR (a.indptr / a.keys).  Draw keys: Philox key (seed, 0x5EED),
// epoch word kFoldInDomain + epoch, index (r << 32) + sample of the row (position * num_neg + k for BPR, the position
// for WARP), draw number t.  No atomics: a row's result depends on its history, start row and index only.
// ---------------------------------------------------------------------------------------
constexpr uint32_t kFoldInDomain = 0xF01D0000u;

struct FoldArgs {
    const int64_t* h_ind;    // history END offsets [n]
    const int32_t* h_users;  // history user ids, ascending within a row
    float* X;                // [n, ld] rows, in / out (padding columns zero)
    float* Xb;               // [n] biases, in / out
    int32_t* trace_negs;     // optional [epochs, nnz * per]: negative of each sample, -1 for a WARP discard
    int32_t* trace_trials;   // optional [epochs, nnz]: WARP trial count, 0 for a discard
    int64_t n, nnz;
    int epochs;
    double inv_epochs, lr0, min_lr, beta1;
};

// warp_score with the row in registers: dot or negative squared distance (warp.cc:21-28)
template <int NV>
__device__ __forceinline__ float fold_score(const float4 (&vp)[NV], const float4 (&x)[NV], int nv4, int lane, int l2) {
    float part = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        if (lane + 32 * k < nv4) {
            if (l2) {
                const float dx = vp[k].x - x[k].x, dy = vp[k].y - x[k].y, dz = vp[k].z - x[k].z, dw = vp[k].w - x[k].w;
                part -= dx * dx + dy * dy + dz * dz + dw * dw;
            } else {
                part += vp[k].x * x[k].x + vp[k].y * x[k].y + vp[k].z * x[k].z + vp[k].w * x[k].w;
            }
        }
    }
    return warp_sum(part);
}

// sgd_apply_kernel's element step on one value: count normalisation, regulariser, adagrad / adam, theta += lr0 * step;
// the gradient accumulator keeps the step, as there
__device__ __forceinline__ void fold_step(const SgdArgs& a, float& th, float& g, float& m, float& v, int cnt,
                                          float two_reg, float lr0, float b1, float omb1, float bc1, float bc2) {
    float s = g;
    if (a.pcn && cnt) s /= (float)cnt;
    s -= th * two_reg;
    if (a.optimizer == 2) {
        m = b1 * m + omb1 * s;
        v = b1 * v + omb1 * (s * s);
        s = (m / bc1) / (sqrtf(v / bc2) + 1e-10f);
    } else {
        v = v + s * s;
        s = s / (sqrtf(v) + 1e-10f);
    }
    g = s;
    th = th + lr0 * s;
}

__device__ __forceinline__ void fold_step4(const SgdArgs& a, float4& th, float4& g, float4& m, float4& v, int cnt,
                                           float two_reg, float lr0, float b1, float omb1, float bc1, float bc2) {
    fold_step(a, th.x, g.x, m.x, v.x, cnt, two_reg, lr0, b1, omb1, bc1, bc2);
    fold_step(a, th.y, g.y, m.y, v.y, cnt, two_reg, lr0, b1, omb1, bc1, bc2);
    fold_step(a, th.z, g.z, m.z, v.z, cnt, two_reg, lr0, b1, omb1, bc1, bc2);
    fold_step(a, th.w, g.w, m.w, v.w, cnt, two_reg, lr0, b1, omb1, bc1, bc2);
}

template <int NV, bool kWarp>
__global__ void __launch_bounds__(256, 2) sgd_fold_in_items_kernel(SgdArgs a, FoldArgs f) {
    const int lane = threadIdx.x & 31;
    const int64_t w0 = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp_id_uniform();
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int nv4 = a.ld >> 2;
    const int per = kWarp ? 1 : a.num_neg;
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int64_t r = w0; r < f.n; r += nw) {
        const int64_t hb = uni((long long)(r == 0 ? 0 : __ldg(f.h_ind + r - 1))), he = uni((long long)__ldg(f.h_ind + r));
        float* xr = f.X + r * a.ld;
        float4 x[NV], g[NV], m[NV], v[NV];
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            x[k] = lane + 32 * k < nv4 ? ld4(xr + 4 * (lane + 32 * k)) : zero;
            g[k] = m[k] = v[k] = zero;
        }
        float xb = f.Xb[r], gb = 0.f, mb = 0.f, vb = 0.f;
        double b1pow = 1.0;  // beta1^(e + 1) of adam's bias correction, as a running product
        for (int e = 0; e < f.epochs; ++e) {
            a.epoch = kFoldInDomain + (uint32_t)e;
            // training's linear decay (run_jobs), over the fold-in's own epochs
            const double lr = f.lr0 - (f.lr0 - f.min_lr) * ((double)e * f.inv_epochs);
            a.lr = (float)(lr > f.min_lr ? lr : f.min_lr);
            int cnt = 0;
            for (int64_t it = hb; it < he; ++it) {
                const int u = uni(__ldg(f.h_users + it));
                const int64_t ub = u == 0 ? 0 : __ldg(a.indptr + u - 1), ue = __ldg(a.indptr + u);
                const int32_t* rk = a.keys + ub;
                const float* pu = a.P + (int64_t)u * a.ld;
                float4 vp[NV];
#pragma unroll
                for (int k = 0; k < NV; ++k) vp[k] = lane + 32 * k < nv4 ? ld4(pu + 4 * (lane + 32 * k)) : zero;
                const uint64_t sid0 = ((uint64_t)r << 32) + (uint64_t)(it - hb) * (uint64_t)per;
                int32_t* tn = f.trace_negs ? f.trace_negs + ((int64_t)e * f.nnz + it) * per : nullptr;
                if constexpr (kWarp) {
                    const float ui = uni(fold_score<NV>(vp, x, nv4, lane, a.score_l2));
                    float4 vj[NV];
                    float uj = 0.f;
                    int neg = 0;
                    const int trial = warp_rank_draw<NV>(a, (int64_t)sid0, rk, ue - ub, vp, ui, nv4, lane, vj, neg, uj);
                    const bool discard = trial >= a.max_trials;  // warp.cc:149-150
                    if (lane == 0 && tn) {
                        tn[0] = discard ? -1 : neg;
                        f.trace_trials[(int64_t)e * f.nnz + it] = discard ? 0 : trial;
                    }
                    if (discard) continue;
                    // :152 in 32 bits (num_items and the row length are int32): no 64-bit division subroutine
                    int ratio = (a.num_items - (int)(ue - ub) - 1) / trial;
                    if (ratio < 1) ratio = 1;
                    const float Phi = logf((float)ratio);
#pragma unroll
                    for (int k = 0; k < NV; ++k) {
                        if (lane + 32 * k < nv4) {
                            float4 di;
                            if (!a.score_l2) di = make_float4(Phi * vp[k].x, Phi * vp[k].y, Phi * vp[k].z, Phi * vp[k].w);
                            else di = make_float4(Phi * (vp[k].x - x[k].x), Phi * (vp[k].y - x[k].y),
                                                  Phi * (vp[k].z - x[k].z), Phi * (vp[k].w - x[k].w));
                            g[k].x += di.x - a.reg_i * x[k].x;  // warp.cc:156-158
                            g[k].y += di.y - a.reg_i * x[k].y;
                            g[k].z += di.z - a.reg_i * x[k].z;
                            g[k].w += di.w - a.reg_i * x[k].w;
                        }
                    }
                    cnt += 1;
                } else {
                    for (int s = 0; s < per; ++s) {
                        const int neg = uni(bpr_draw_negative(a, sid0 + (uint64_t)s, rk, ue - ub));
                        const float* qj = a.Q + (int64_t)neg * a.ld;
                        float part = 0.f;
#pragma unroll
                        for (int k = 0; k < NV; ++k) {
                            if (lane + 32 * k < nv4) {
                                const float4 vj = ld4(qj + 4 * (lane + 32 * k));
                                part += vp[k].x * (x[k].x - vj.x) + vp[k].y * (x[k].y - vj.y) +
                                        vp[k].z * (x[k].z - vj.z) + vp[k].w * (x[k].w - vj.w);
                            }
                        }
                        float xs = warp_sum(part);  // bpr.cc:119-121
                        if (a.use_bias) xs += xb - __ldg(a.Qb + neg);
                        const float logit = xs > 6.f ? 0.f : (xs < -6.f ? 1.f : 1.0f / (1.0f + __expf(xs)));
                        if (lane == 0 && tn) tn[s] = neg;
                        if (a.optimizer == 0) {  // the positive side of bpr_apply_kernel's step, after every sample
#pragma unroll
                            for (int k = 0; k < NV; ++k) {
                                if (lane + 32 * k < nv4) {
                                    x[k].x += a.lr * (logit * vp[k].x - a.reg_i * x[k].x);
                                    x[k].y += a.lr * (logit * vp[k].y - a.reg_i * x[k].y);
                                    x[k].z += a.lr * (logit * vp[k].z - a.reg_i * x[k].z);
                                    x[k].w += a.lr * (logit * vp[k].w - a.reg_i * x[k].w);
                                }
                            }
                            if (a.use_bias) xb += a.lr * (logit - a.reg_b * xb);
                        } else {
#pragma unroll
                            for (int k = 0; k < NV; ++k) {
                                if (lane + 32 * k < nv4) {
                                    g[k].x += logit * vp[k].x;
                                    g[k].y += logit * vp[k].y;
                                    g[k].z += logit * vp[k].z;
                                    g[k].w += logit * vp[k].w;
                                }
                            }
                            gb += logit;
                        }
                    }
                    cnt += 1;  // per_coordinate_normalize counts the positive once (bpr.cc:140-143)
                }
            }
            if (a.optimizer != 0) {  // one step per epoch (apply_optimizer)
                const float b1 = (float)f.beta1, omb1 = (float)(1.0 - f.beta1);
                b1pow *= f.beta1;
                const float bc1 = (float)(1.0 - b1pow), lr0 = (float)f.lr0;
#pragma unroll
                for (int k = 0; k < NV; ++k)
                    if (lane + 32 * k < nv4) fold_step4(a, x[k], g[k], m[k], v[k], cnt, 2.f * a.reg_i, lr0, b1, omb1, bc1, bc1);
                if (!kWarp && a.use_bias) fold_step(a, xb, gb, mb, vb, cnt, 2.f * a.reg_b, lr0, b1, omb1, bc1, bc1);
            }
            if constexpr (kWarp) {  // warp_project_kernel: row /= max(1, ||row||)
                float ss = 0.f;
#pragma unroll
                for (int k = 0; k < NV; ++k)
                    if (lane + 32 * k < nv4) ss += x[k].x * x[k].x + x[k].y * x[k].y + x[k].z * x[k].z + x[k].w * x[k].w;
                const float nrm = sqrtf(warp_sum(ss));
                if (nrm > 1.0f) {
#pragma unroll
                    for (int k = 0; k < NV; ++k)
                        if (lane + 32 * k < nv4) x[k] = make_float4(x[k].x / nrm, x[k].y / nrm, x[k].z / nrm, x[k].w / nrm);
                }
            }
        }
#pragma unroll
        for (int k = 0; k < NV; ++k)
            if (lane + 32 * k < nv4) *reinterpret_cast<float4*>(xr + 4 * (lane + 32 * k)) = x[k];
        if (lane == 0) f.Xb[r] = xb;
    }
}

}  // namespace

struct bfl_sgd : Holder {
    int kind = BFL_SGD_BPR;
    int optimizer = 0;
    bool use_bias = true, update_i = true, update_j = true, verify_neg = true, uniform = true, pcn = false;
    bool compute_loss = true, score_l2 = false;
    int num_neg = 1, max_trials = 500, num_iters = 1;
    uint32_t seed = 0;
    float reg_u = 0, reg_i = 0, reg_j = 0, reg_b = 0, threshold = 1.f;
    double lr0 = 0.05, min_lr = 1e-4, beta1 = 0.9;

    // item biases next to the Holder's P and Q
    float* hostQb = nullptr;
    DevBuf<float> ownQb;
    float* dQb = nullptr;
    DevBuf<float> gP, gQ, gQb, mP, mQ, mQb, vP, vQ, vQb;
    DevBuf<int32_t> cP, cQ;
    DevBuf<int64_t> cum;
    bool cum_set = false;

    DevBuf<int64_t> own_indptr;
    CsrBinding csr;   // keys only: the samplers read no values
    DevBuf<int32_t> stage_keys;
    DevBuf<int32_t> tri_u, tri_p, tri_n;
    DevBuf<int32_t> probe;
    DevBuf<double> d_stat;  // [0] warp loss sum, [1] probe loss
    DevBuf<unsigned long long> d_upd;
    int32_t* trace_trials = nullptr;
    int32_t* trace_negs = nullptr;

    int iters = 0, epoch = 0;
    double processed = 0.0, total = 1.0, cur_lr = 0.0;

    // deterministic mode: the epoch's sample records (DetRec), the sorted item entries and the segment partials
    bool deterministic = false;
    DevBuf<int32_t> det_u, det_i, det_j, det_major, det_iota, det_code;
    DevBuf<float> det_c, det_cval, det_cval_sorted, det_loss, det_part;
    DevBuf<int64_t> det_ends;
    DevBuf<double> det_lpart, det_terms;
    int64_t det_n = 0;         // samples per epoch the buffers are laid out for
    bool det_pending = false;  // records of this epoch wait for the item pass

    int apply_options(const JsonOpt& j) override;
};

int bfl_sgd::apply_options(const JsonOpt& j) {
    d = j.integer("d", kind == BFL_SGD_WARP ? 64 : 20);
    if (d <= 0 || d > 512) BFL_FAIL(BFL_ERR_OPTION, "d must be in [1, 512]");
    vdim = (d + 3) / 4 * 4;
    std::string opt_name = j.string("optimizer", kind == BFL_SGD_WARP ? "adagrad" : "sgd");
    if (opt_name == "sgd") optimizer = 0;
    else if (opt_name == "adagrad") optimizer = 1;
    else if (opt_name == "adam") optimizer = 2;
    else BFL_FAIL(BFL_ERR_OPTION, "optimizer must be one of sgd, adagrad, adam");
    if (kind == BFL_SGD_WARP && optimizer == 0)
        BFL_FAIL(BFL_ERR_OPTION, "WARP accumulates gradients only (warp.cc:156-158): optimizer must be adagrad or adam");
    use_bias = kind == BFL_SGD_WARP ? false : j.flag("use_bias", true);
    update_i = j.flag("update_i", true);
    update_j = j.flag("update_j", true);
    verify_neg = j.flag("verify_neg", true);
    uniform = j.number("sampling_power", 0.0) == 0.0;  // bpr.cc:91
    pcn = j.flag("per_coordinate_normalize", false);
    compute_loss = j.flag("compute_loss_on_training", true);
    std::string sf = j.string("score_func", "dot");
    score_l2 = (sf == "l2" || sf == "L2");
    num_neg = j.integer("num_negative_samples", 1);
    if (num_neg < 1) num_neg = 1;
    max_trials = j.integer("max_trials", 500);
    num_iters = j.integer("num_iters", 1);
    seed = (uint32_t)j.integer("random_seed", 0);
    reg_u = (float)j.number("reg_u", 0.0);
    reg_i = (float)j.number("reg_i", 0.0);
    reg_j = (float)j.number("reg_j", 0.0);
    reg_b = (float)j.number("reg_b", 0.0);
    threshold = (float)j.number("threshold", 1.0);
    lr0 = j.number("lr", 0.05);
    min_lr = j.number("min_lr", 0.0001);
    beta1 = j.number("beta1", 0.9);
    deterministic = j.flag("deterministic", false);
    if (deterministic && optimizer == 0)
        BFL_FAIL(BFL_ERR_OPTION, "deterministic needs optimizer adagrad or adam: plain SGD applies its updates "
                                 "Hogwild-style, in the order the warps reach the rows");
    int rc = attach_device();
    if (rc != BFL_OK) return rc;
    if (BFL_OK != d_stat.reserve(2)) return BFL_ERR_CUDA;
    if (BFL_OK != d_upd.reserve(1)) return BFL_ERR_CUDA;
    BFL_CUDA(cudaMemsetAsync(d_stat.p, 0, 2 * sizeof(double), stream));
    BFL_CUDA(cudaMemsetAsync(d_upd.p, 0, sizeof(unsigned long long), stream));
    cur_lr = lr0;
    opt_set = true;
    return BFL_OK;
}

namespace {

int alloc_state(bfl_sgd* h, int64_t num_total_samples) {
    const size_t np = (size_t)h->P_rows * h->vdim, nq = (size_t)h->Q_rows * h->vdim, nb = (size_t)h->Q_rows;
    cudaStream_t st = h->stream;
    if (h->optimizer != 0) {  // initialize_adam_optimizer algo.cc:221-254
        DevBuf<float>* bufs[] = {&h->gP, &h->gQ, &h->gQb, &h->mP, &h->mQ, &h->mQb, &h->vP, &h->vQ, &h->vQb};
        const size_t sizes[] = {np, nq, nb, np, nq, nb, np, nq, nb};
        for (int i = 0; i < 9; ++i) {
            if (h->optimizer == 1 && i >= 3 && i < 6) continue;  // adagrad needs no momentum
            if (BFL_OK != bufs[i]->reserve(sizes[i])) return BFL_ERR_CUDA;
            BFL_CUDA(cudaMemsetAsync(bufs[i]->p, 0, sizes[i] * sizeof(float), st));
        }
    }
    if (BFL_OK != h->cP.reserve((size_t)h->P_rows)) return BFL_ERR_CUDA;
    if (BFL_OK != h->cQ.reserve((size_t)h->Q_rows)) return BFL_ERR_CUDA;
    BFL_CUDA(cudaMemsetAsync(h->cP.p, 0, sizeof(int32_t) * h->P_rows, st));
    BFL_CUDA(cudaMemsetAsync(h->cQ.p, 0, sizeof(int32_t) * h->Q_rows, st));
    h->iters = 0;
    h->epoch = 0;
    h->processed = 0.0;
    h->total = (double)num_total_samples * (double)h->num_iters;  // algo.cc:174-175
    if (h->total <= 0) h->total = 1.0;
    h->cur_lr = h->lr0;
    h->det_n = 0;  // the deterministic buffers are laid out again by the first chunk
    h->det_pending = false;
    BFL_CUDA(cudaStreamSynchronize(st));
    h->factors_ready = true;
    return BFL_OK;
}

// deterministic mode: samples per positive (WARP draws one negative per positive)
int64_t det_per_row(const bfl_sgd* h) { return h->kind == BFL_SGD_WARP ? 1 : h->num_neg; }

// Lays the deterministic buffers out for epochs of `positives` positives: the records, the item entries and their
// sorted copy, the segment partials and the loss partials.  No entry updates a row until a sample pass writes it.
int det_prepare(bfl_sgd* h, int64_t positives, cudaStream_t st) {
    const int64_t n = positives * det_per_row(h);
    if (n == h->det_n) return BFL_OK;
    if (h->det_pending) BFL_FAIL(BFL_ERR_STATE, "deterministic mode: the number of positives changed within an epoch");
    if (2 * n > (int64_t)INT32_MAX)
        BFL_FAIL(BFL_ERR_ARG, "deterministic mode: an epoch holds at most 2^30 - 1 samples (the item entries are "
                              "indexed by int32 2s + side)");
    const size_t N = (size_t)std::max<int64_t>(n, 1);
    const size_t segs = (2 * N + kDetSegment - 1) / kDetSegment;
    const size_t lparts = std::max<size_t>((N + kDetLossRange - 1) / kDetLossRange, 1);
    if (BFL_OK != h->det_u.reserve(N) || BFL_OK != h->det_i.reserve(N) || BFL_OK != h->det_j.reserve(N) ||
        BFL_OK != h->det_c.reserve(N) || BFL_OK != h->det_major.reserve(2 * N) || BFL_OK != h->det_iota.reserve(2 * N) ||
        BFL_OK != h->det_code.reserve(2 * N) || BFL_OK != h->det_cval.reserve(2 * N) ||
        BFL_OK != h->det_cval_sorted.reserve(2 * N) || BFL_OK != h->det_ends.reserve((size_t)h->Q_rows + 1) ||
        BFL_OK != h->det_part.reserve(segs * 2 * (size_t)(h->vdim + 4)) || BFL_OK != h->det_lpart.reserve(lparts) ||
        (h->kind == BFL_SGD_WARP && BFL_OK != h->det_loss.reserve(N)))
        BFL_FAIL(BFL_ERR_CUDA, "deterministic mode: cannot allocate the sample records and item sort buffers of " +
                                   std::to_string(n) + " samples");
    const int grid = (int)std::min<int64_t>((2 * N + 255) / 256, (int64_t)h->num_sms * 32);
    det_reset_kernel<<<grid, 256, 0, st>>>(h->det_major.p, h->det_iota.p, 2 * (int64_t)N, (int32_t)h->Q_rows);
    BFL_LAUNCHED();
    if (h->kind == BFL_SGD_WARP) BFL_CUDA(cudaMemsetAsync(h->det_loss.p, 0, sizeof(float) * N, st));
    h->det_n = n;
    return BFL_OK;
}

DetSum det_sum_args(const bfl_sgd* h) {
    DetSum s;
    s.P = h->dP; s.Q = h->dQ;
    s.rec_u = h->det_u.p; s.rec_i = h->det_i.p; s.rec_j = h->det_j.p; s.rec_c = h->det_c.p;
    s.code = nullptr; s.cval = nullptr; s.ends = nullptr;
    s.out = nullptr; s.outb = nullptr; s.part = h->det_part.p;
    s.row_lo = s.row_hi = s.e_begin = s.e_end = 0;
    s.per_row = 1; s.ld = h->vdim; s.pitch = h->vdim + 4;
    s.warp = h->kind == BFL_SGD_WARP; s.l2 = h->score_l2;
    s.reg_u = h->reg_u; s.reg_i = h->reg_i; s.reg_j = h->reg_j;
    return s;
}

template <bool kItem>
int launch_det_sum(const bfl_sgd* h, const DetSum& s, cudaStream_t st) {
    if (s.e_end <= s.e_begin) return BFL_OK;
    const int64_t segs = (s.e_end - 1) / kDetSegment - s.e_begin / kDetSegment + 1;
    const int grid = (int)std::min<int64_t>((segs + 7) / 8, (int64_t)h->num_sms * 16);
    const int nv = (h->vdim / 4 + 31) / 32;
    if (nv <= 1) det_sum_kernel<1, kItem><<<grid, 256, 0, st>>>(s);
    else if (nv <= 2) det_sum_kernel<2, kItem><<<grid, 256, 0, st>>>(s);
    else det_sum_kernel<4, kItem><<<grid, 256, 0, st>>>(s);
    BFL_LAUNCHED();
    if (nv <= 1) det_combine_kernel<1><<<grid, 256, 0, st>>>(s);
    else if (nv <= 2) det_combine_kernel<2><<<grid, 256, 0, st>>>(s);
    else det_combine_kernel<4><<<grid, 256, 0, st>>>(s);
    BFL_LAUNCHED();
    return BFL_OK;
}

// fixed-tree fp64 sum of terms[0, n) added into *out
template <typename T>
int det_loss_sum(const bfl_sgd* h, const T* terms, int64_t n, double* out, cudaStream_t st) {
    if (n <= 0) return BFL_OK;
    const int64_t nblk = (n + kDetLossRange - 1) / kDetLossRange;
    det_loss_partial_kernel<T><<<(unsigned)nblk, 256, 0, st>>>(terms, n, h->det_lpart.p);
    BFL_LAUNCHED();
    det_loss_final_kernel<<<1, 256, 0, st>>>(h->det_lpart.p, nblk, out);
    BFL_LAUNCHED();
    return BFL_OK;
}

// sample pass and user pass of one chunk (rows [row_begin, row_end) are whole)
int run_jobs_det(bfl_sgd* h, const SgdArgs& a, cudaStream_t st) {
    const int64_t nn = det_per_row(h);
    const DetRec r = {h->det_u.p, h->det_i.p, h->det_j.p, h->det_c.p, h->det_major.p, h->det_cval.p, h->det_loss.p};
    const int nv = (h->vdim / 4 + 31) / 32;
    const int64_t warps = (a.it_end - a.it_begin) * nn;
    const int grid = (int)std::min<int64_t>((warps + 7) / 8, (int64_t)h->num_sms * 16);
    if (h->kind == BFL_SGD_WARP) {
        if (nv <= 1) det_warp_sample_kernel<1><<<grid, 256, 0, st>>>(a, r);
        else if (nv <= 2) det_warp_sample_kernel<2><<<grid, 256, 0, st>>>(a, r);
        else det_warp_sample_kernel<4><<<grid, 256, 0, st>>>(a, r);
    } else {
        if (nv <= 1) det_bpr_sample_kernel<1><<<grid, 256, 0, st>>>(a, r);
        else if (nv <= 2) det_bpr_sample_kernel<2><<<grid, 256, 0, st>>>(a, r);
        else det_bpr_sample_kernel<4><<<grid, 256, 0, st>>>(a, r);
    }
    BFL_LAUNCHED();
    h->det_pending = true;
    DetSum s = det_sum_args(h);
    s.ends = a.indptr;
    s.out = h->gP.p;
    s.row_lo = a.row_begin; s.row_hi = a.row_end;
    s.e_begin = a.it_begin * nn; s.e_end = a.it_end * nn;
    s.per_row = (int)nn;
    return launch_det_sum<false>(h, s, st);
}

// item pass over the records written since the last one: sort the entries by item, add each item's sum to gQ / gQb;
// the WARP loss terms by the fixed tree into the running loss sum; then no entry updates a row again
int det_flush(bfl_sgd* h, cudaStream_t st) {
    if (!h->deterministic || !h->det_pending) return BFL_OK;
    const int64_t n2 = 2 * h->det_n;
    int rc = bfl_csr_from_triples_device(h->det_major.p, h->det_iota.p, h->det_cval.p, n2, (int32_t)h->Q_rows + 1,
                                         (int32_t)std::max<int64_t>(n2, 1), 0, h->det_ends.p, h->det_code.p,
                                         h->det_cval_sorted.p, st);
    if (rc != BFL_OK) return rc;
    int64_t beg = 0, end = 0;
    rc = read_row_span(h->det_ends.p, 0, h->Q_rows, st, &beg, &end);
    if (rc != BFL_OK) return rc;
    DetSum s = det_sum_args(h);
    s.code = h->det_code.p; s.cval = h->det_cval_sorted.p; s.ends = h->det_ends.p;
    s.out = h->gQ.p;
    s.outb = (h->kind == BFL_SGD_BPR && h->use_bias) ? h->gQb.p : nullptr;
    s.row_lo = 0; s.row_hi = h->Q_rows;
    s.e_begin = 0; s.e_end = end;
    rc = launch_det_sum<true>(h, s, st);
    if (rc != BFL_OK) return rc;
    if (h->kind == BFL_SGD_WARP) {
        rc = det_loss_sum(h, h->det_loss.p, h->det_n, h->d_stat.p, st);
        if (rc != BFL_OK) return rc;
        BFL_CUDA(cudaMemsetAsync(h->det_loss.p, 0, sizeof(float) * (size_t)h->det_n, st));
    }
    const int grid = (int)std::min<int64_t>((n2 + 255) / 256, (int64_t)h->num_sms * 32);
    det_reset_kernel<<<std::max(grid, 1), 256, 0, st>>>(h->det_major.p, nullptr, n2, (int32_t)h->Q_rows);
    BFL_LAUNCHED();
    h->det_pending = false;
    return BFL_OK;
}

void fill_args(bfl_sgd* h, SgdArgs& a, const int32_t* keys, int64_t shift, int64_t row_begin, int64_t row_end,
               int64_t it_begin, int64_t it_end) {
    a.P = h->dP; a.Q = h->dQ; a.Qb = h->dQb;
    a.gP = h->gP.p; a.gQ = h->gQ.p; a.gQb = h->gQb.p;
    a.cP = h->cP.p; a.cQ = h->cQ.p;
    a.indptr = h->csr.indptr; a.keys = keys;
    a.cum = h->cum_set ? h->cum.p : nullptr;
    a.trace_trials = h->trace_trials; a.trace_negs = h->trace_negs;
    a.stat_loss = h->d_stat.p; a.stat_updates = h->d_upd.p;
    a.shift = shift; a.row_begin = row_begin; a.row_end = row_end; a.it_begin = it_begin; a.it_end = it_end;
    a.num_items = (int32_t)h->Q_rows; a.D = h->d; a.ld = h->vdim;
    a.optimizer = h->optimizer; a.use_bias = h->use_bias; a.update_i = h->update_i; a.update_j = h->update_j;
    a.num_neg = h->num_neg; a.verify_neg = h->verify_neg; a.uniform = h->uniform || !h->cum_set; a.pcn = h->pcn;
    a.max_trials = h->max_trials; a.score_l2 = h->score_l2; a.seed = h->seed; a.epoch = (uint32_t)h->epoch;
    a.reg_u = h->reg_u; a.reg_i = h->reg_i; a.reg_j = h->reg_j; a.reg_b = h->reg_b;
    a.lr = (float)h->cur_lr; a.threshold = h->threshold;
}

int launch_bpr_apply(bfl_sgd* h, const SgdArgs& a, const int32_t* u, const int32_t* p, const int32_t* n, int64_t cnt,
                     cudaStream_t st) {
    if (cnt <= 0) return BFL_OK;
    // >= 16 consecutive triples per warp, at most 32 warps per SM (staleness grows with the number of triples in flight)
    const int grid = (int)std::min<int64_t>((cnt + 127) / 128, (int64_t)h->num_sms * 4);
    const int nv = (h->vdim / 4 + 31) / 32;
    if (nv <= 1) bpr_apply_kernel<1><<<grid, 256, 0, st>>>(a, u, p, n, cnt);
    else if (nv <= 2) bpr_apply_kernel<2><<<grid, 256, 0, st>>>(a, u, p, n, cnt);
    else bpr_apply_kernel<4><<<grid, 256, 0, st>>>(a, u, p, n, cnt);
    BFL_LAUNCHED();
    return BFL_OK;
}

// process rows [row_begin,row_end) whose positives are keys[it - shift], it in [it_begin, it_end)
int run_jobs(bfl_sgd* h, const int32_t* keys, int64_t shift, int64_t row_begin, int64_t row_end, int64_t it_begin,
             int64_t it_end, cudaStream_t st) {
    const int64_t npos = it_end - it_begin;
    // job.alpha = lr_ at job creation (algo.cc:351,359); linear decay by processed fraction (:284-287)
    double lr = h->lr0 - (h->lr0 - h->min_lr) * (h->processed / h->total);
    h->cur_lr = lr > h->min_lr ? lr : h->min_lr;
    if (npos <= 0) return BFL_OK;
    SgdArgs a;
    fill_args(h, a, keys, shift, row_begin, row_end, it_begin, it_end);
    if (h->deterministic) {
        int rc = run_jobs_det(h, a, st);
        if (rc != BFL_OK) return rc;
    } else if (h->kind == BFL_SGD_WARP) {
        const int grid = (int)std::min<int64_t>((npos + 7) / 8, (int64_t)h->num_sms * 16);
        const int nv = (h->vdim / 4 + 31) / 32;
        if (nv <= 1) warp_accumulate_kernel<1><<<grid, 256, 0, st>>>(a);
        else if (nv <= 2) warp_accumulate_kernel<2><<<grid, 256, 0, st>>>(a);
        else warp_accumulate_kernel<4><<<grid, 256, 0, st>>>(a);
        BFL_LAUNCHED();
    } else {
        // sample + apply in slabs so the triple buffers stay bounded (<= 64M samples)
        const int64_t slab_pos = std::max<int64_t>(1, (int64_t)(1 << 26) / h->num_neg);
        for (int64_t b = it_begin; b < it_end; b += slab_pos) {
            const int64_t e = std::min(it_end, b + slab_pos);
            const int64_t cnt = (e - b) * h->num_neg;
            if (BFL_OK != h->tri_u.reserve((size_t)cnt)) return BFL_ERR_CUDA;
            if (BFL_OK != h->tri_p.reserve((size_t)cnt)) return BFL_ERR_CUDA;
            if (BFL_OK != h->tri_n.reserve((size_t)cnt)) return BFL_ERR_CUDA;
            SgdArgs s = a;
            s.it_begin = b;
            s.it_end = e;
            const int grid = (int)std::min<int64_t>((cnt + 255) / 256, (int64_t)h->num_sms * 32);
            bpr_sample_kernel<<<grid, 256, 0, st>>>(s, h->tri_u.p, h->tri_p.p, h->tri_n.p);
            BFL_LAUNCHED();
            int rc = launch_bpr_apply(h, s, h->tri_u.p, h->tri_p.p, h->tri_n.p, cnt, st);
            if (rc != BFL_OK) return rc;
        }
    }
    h->processed += (double)npos;
    return BFL_OK;
}

int apply_optimizer(bfl_sgd* h, cudaStream_t st) {
    if (h->optimizer != 0) {
        const double beta2 = h->beta1;  // algo.cc:396
        const float b1 = (float)h->beta1, omb1 = (float)(1.0 - h->beta1);
        const float b2 = (float)beta2, omb2 = (float)(1.0 - beta2);
        const float bc1 = (float)(1.0 - pow(h->beta1, h->iters + 1));
        const float bc2 = (float)(1.0 - pow(beta2, h->iters + 1));
        struct Item { float* th; float* g; float* m; float* v; const int32_t* c; int64_t rows; int cols; double reg; };
        Item items[3] = {{h->dP, h->gP.p, h->mP.p, h->vP.p, h->cP.p, h->P_rows, h->vdim, h->reg_u},
                         {h->dQ, h->gQ.p, h->mQ.p, h->vQ.p, h->cQ.p, h->Q_rows, h->vdim, h->reg_i},
                         {h->dQb, h->gQb.p, h->mQb.p, h->vQb.p, h->cQ.p, h->Q_rows, 1, h->reg_b}};
        const int nitems = (h->use_bias && h->kind == BFL_SGD_BPR) ? 3 : 2;
        for (int i = 0; i < nitems; ++i) {
            const Item& it = items[i];
            const int64_t n = it.rows * it.cols;
            const int grid = (int)std::min<int64_t>((n + 255) / 256, (int64_t)h->num_sms * 32);
            sgd_apply_kernel<<<grid, 256, 0, st>>>(h->optimizer, it.th, it.g, it.m, it.v, it.c, it.rows, it.cols,
                                                   (float)(2 * it.reg), (float)h->lr0, b1, omb1, b2, omb2, bc1, bc2,
                                                   h->pcn ? 1 : 0);
            BFL_LAUNCHED();
        }
        if (h->pcn) {  // algo.cc:424-427
            BFL_CUDA(cudaMemsetAsync(h->cP.p, 0, sizeof(int32_t) * h->P_rows, st));
            BFL_CUDA(cudaMemsetAsync(h->cQ.p, 0, sizeof(int32_t) * h->Q_rows, st));
        }
    }
    if (h->kind == BFL_SGD_WARP) {  // warp.cc:192-201
        const int gq = (int)std::min<int64_t>((h->Q_rows + 7) / 8, (int64_t)h->num_sms * 16);
        warp_project_kernel<<<gq, 256, 0, st>>>(h->dQ, h->Q_rows, h->vdim);
        BFL_LAUNCHED();
        const int gp = (int)std::min<int64_t>((h->P_rows + 7) / 8, (int64_t)h->num_sms * 16);
        warp_project_kernel<<<gp, 256, 0, st>>>(h->dP, h->P_rows, h->vdim);
        BFL_LAUNCHED();
    }
    h->iters += 1;  // algo.cc:464
    h->epoch += 1;
    return BFL_OK;
}

int sync_to_host(bfl_sgd* h) {
    if (!h->hostP) return BFL_OK;
    BFL_CUDA(cudaMemcpyAsync(h->hostP, h->dP, sizeof(float) * (size_t)h->P_rows * h->vdim, cudaMemcpyDeviceToHost, h->stream));
    BFL_CUDA(cudaMemcpyAsync(h->hostQ, h->dQ, sizeof(float) * (size_t)h->Q_rows * h->vdim, cudaMemcpyDeviceToHost, h->stream));
    BFL_CUDA(cudaMemcpyAsync(h->hostQb, h->dQb, sizeof(float) * (size_t)h->Q_rows, cudaMemcpyDeviceToHost, h->stream));
    BFL_CUDA(cudaStreamSynchronize(h->stream));
    return BFL_OK;
}

}  // namespace

extern "C" {

bfl_sgd_t* bfl_sgd_create(int kind) {
    if (kind != BFL_SGD_BPR && kind != BFL_SGD_WARP) return nullptr;
    bfl_sgd* h = new (std::nothrow) bfl_sgd();
    if (h) h->kind = kind;
    return h;
}

void bfl_sgd_destroy(bfl_sgd_t* h) { delete h; }

int bfl_sgd_init(bfl_sgd_t* h, const char* opt_path) { return init_holder(h, opt_path, true); }

int bfl_sgd_init_json(bfl_sgd_t* h, const char* json_text) { return init_holder(h, json_text, false); }

int bfl_sgd_get_vdim(bfl_sgd_t* h) { return h ? h->vdim : 0; }

int bfl_sgd_initialize_model(bfl_sgd_t* h, float* P, int32_t P_rows, float* Q, int32_t Q_rows, float* Qb,
                             int64_t num_total_samples) {
    if (!h || !h->opt_set) BFL_FAIL(BFL_ERR_STATE, "init() must succeed before initialize_model()");
    if (!Qb) BFL_FAIL(BFL_ERR_ARG, "bad factor arguments");
    int rc = h->mirror_factors(P, P_rows, Q, Q_rows);
    if (rc != BFL_OK) return rc;
    h->hostQb = Qb;
    if (BFL_OK != h->ownQb.reserve((size_t)Q_rows)) return BFL_ERR_CUDA;
    h->dQb = h->ownQb.p;
    BFL_CUDA(cudaMemcpyAsync(h->dP, P, sizeof(float) * (size_t)P_rows * h->vdim, cudaMemcpyHostToDevice, h->stream));
    BFL_CUDA(cudaMemcpyAsync(h->dQ, Q, sizeof(float) * (size_t)Q_rows * h->vdim, cudaMemcpyHostToDevice, h->stream));
    BFL_CUDA(cudaMemcpyAsync(h->dQb, Qb, sizeof(float) * (size_t)Q_rows, cudaMemcpyHostToDevice, h->stream));
    return alloc_state(h, num_total_samples);
}

int bfl_sgd_bind_factors_device(bfl_sgd_t* h, float* dP, int64_t P_rows, float* dQ, int64_t Q_rows, float* dQb,
                                int64_t num_total_samples) {
    if (!h || !h->opt_set) BFL_FAIL(BFL_ERR_STATE, "init() must succeed before binding factors");
    if (!dQb) BFL_FAIL(BFL_ERR_ARG, "bad factor arguments");
    int rc = h->borrow_factors(dP, P_rows, dQ, Q_rows);
    if (rc != BFL_OK) return rc;
    h->hostQb = nullptr;
    h->ownQb.release();
    h->dQb = dQb;
    return alloc_state(h, num_total_samples);
}

int bfl_sgd_set_cumulative_table(bfl_sgd_t* h, const int64_t* cum_table, int32_t size) {
    if (!h || !h->opt_set) BFL_FAIL(BFL_ERR_STATE, "init() must precede set_cumulative_table()");
    if (!cum_table || size <= 0) BFL_FAIL(BFL_ERR_ARG, "bad cumulative table");
    if (BFL_OK != h->cum.reserve((size_t)size)) return BFL_ERR_CUDA;
    BFL_CUDA(cudaMemcpyAsync(h->cum.p, cum_table, sizeof(int64_t) * size, cudaMemcpyHostToDevice, h->stream));
    BFL_CUDA(cudaStreamSynchronize(h->stream));
    // an all-zero table (sampling_power == 0, bpr.py:101-111) means uniform sampling
    h->cum_set = cum_table[size - 1] > 0;
    return BFL_OK;
}

int bfl_sgd_set_placeholder(bfl_sgd_t* h, const int64_t* indptr, size_t batch_size) {
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "initialize_model() must precede set_placeholder()");
    if (!indptr) BFL_FAIL(BFL_ERR_ARG, "null indptr");
    if (BFL_OK != h->own_indptr.reserve((size_t)h->P_rows)) return BFL_ERR_CUDA;
    BFL_CUDA(cudaMemcpyAsync(h->own_indptr.p, indptr, sizeof(int64_t) * h->P_rows, cudaMemcpyHostToDevice, h->stream));
    h->csr.indptr = h->own_indptr.p;
    if (batch_size && BFL_OK != h->stage_keys.reserve(batch_size)) return BFL_ERR_CUDA;
    BFL_CUDA(cudaStreamSynchronize(h->stream));
    return BFL_OK;
}

int bfl_sgd_bind_csr_device(bfl_sgd_t* h, const int64_t* d_indptr, const int32_t* d_keys, int64_t rows, int64_t nnz) {
    if (!h || !h->opt_set) BFL_FAIL(BFL_ERR_STATE, "init() must precede bind_csr");
    return h->csr.bind(d_indptr, d_keys, nullptr, rows, nnz, false);
}

int bfl_sgd_launch_workers(bfl_sgd_t* h) {
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "initialize_model() must precede launch_workers()");
    return BFL_OK;
}

int bfl_sgd_wait_until_done(bfl_sgd_t* h) {
    if (!h) BFL_FAIL(BFL_ERR_ARG, "null handle");
    if (h->stream) BFL_CUDA(cudaStreamSynchronize(h->stream));
    return BFL_OK;
}

int bfl_sgd_join(bfl_sgd_t* h, double* out) {
    if (out) *out = 0.0;
    if (!h) BFL_FAIL(BFL_ERR_ARG, "null handle");
    if (h->stream) BFL_CUDA(cudaStreamSynchronize(h->stream));
    return sync_to_host(h);
}

int bfl_sgd_add_jobs(bfl_sgd_t* h, int32_t start_x, int32_t next_x, const int64_t* indptr, const int32_t* keys) {
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "initialize_model() must precede add_jobs()");
    if (next_x - start_x == 0) return BFL_OK;  // algo.cc:314-317
    if (start_x < 0 || next_x > h->P_rows || next_x < start_x || !indptr || !keys) BFL_FAIL(BFL_ERR_ARG, "bad chunk arguments");
    if (h->csr.indptr != h->own_indptr.p || !h->own_indptr.p) {
        if (BFL_OK != h->own_indptr.reserve((size_t)h->P_rows)) return BFL_ERR_CUDA;
        BFL_CUDA(cudaMemcpyAsync(h->own_indptr.p, indptr, sizeof(int64_t) * h->P_rows, cudaMemcpyHostToDevice, h->stream));
        h->csr.indptr = h->own_indptr.p;
    }
    const int64_t beg = start_x == 0 ? 0 : indptr[start_x - 1];
    const int64_t end = indptr[next_x - 1];
    const int64_t n = end - beg;
    if (h->deterministic) {
        int rc = det_prepare(h, indptr[h->P_rows - 1], h->stream);
        if (rc != BFL_OK) return rc;
    }
    if (n > 0) {
        if (BFL_OK != h->stage_keys.reserve((size_t)n)) return BFL_ERR_CUDA;
        BFL_CUDA(cudaMemcpyAsync(h->stage_keys.p, keys, sizeof(int32_t) * n, cudaMemcpyHostToDevice, h->stream));
    }
    int rc = run_jobs(h, h->stage_keys.p, beg, start_x, next_x, beg, end, h->stream);
    if (rc != BFL_OK) return rc;
    // the staging buffer is reused by the next chunk: drain before returning
    BFL_CUDA(cudaStreamSynchronize(h->stream));
    return BFL_OK;
}

int bfl_sgd_add_jobs_device(bfl_sgd_t* h, int64_t row_begin, int64_t row_end, void* stream) {
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "factors not bound");
    if (!h->csr.indptr || (!h->csr.keys && h->csr.nnz > 0)) BFL_FAIL(BFL_ERR_STATE, "no device CSR bound");
    int rc = h->csr.check_range(row_begin, row_end);
    if (rc != BFL_OK) return rc;
    if (row_end == row_begin) return BFL_OK;
    int64_t beg = 0, end = 0;
    rc = read_row_span(h->csr.indptr, row_begin, row_end, (cudaStream_t)stream, &beg, &end);
    if (rc != BFL_OK) return rc;
    if (h->deterministic) {
        rc = det_prepare(h, h->csr.nnz, (cudaStream_t)stream);
        if (rc != BFL_OK) return rc;
    }
    return run_jobs(h, h->csr.keys, 0, row_begin, row_end, beg, end, (cudaStream_t)stream);
}

int bfl_sgd_reduce_items_device(bfl_sgd_t* h, void* stream) {
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "factors not bound");
    if (!h->deterministic) BFL_FAIL(BFL_ERR_STATE, "the item pass serves the deterministic option only");
    return det_flush(h, (cudaStream_t)stream);
}

int bfl_sgd_segment_len(void) { return (int)kDetSegment; }

int bfl_sgd_update_parameters(bfl_sgd_t* h) {
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "initialize_model() must precede update_parameters()");
    int rc = det_flush(h, h->stream);
    if (rc != BFL_OK) return rc;
    rc = apply_optimizer(h, h->stream);
    if (rc != BFL_OK) return rc;
    return sync_to_host(h);  // cuda/_bpr.pyx:60-61
}

int bfl_sgd_update_parameters_device(bfl_sgd_t* h, void* stream) {
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "factors not bound");
    int rc = det_flush(h, (cudaStream_t)stream);
    if (rc != BFL_OK) return rc;
    return apply_optimizer(h, (cudaStream_t)stream);
}

int bfl_sgd_synchronize(bfl_sgd_t* h, int device_to_host) {
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "initialize_model() must precede synchronize()");
    if (device_to_host) return sync_to_host(h);
    if (!h->hostP) return BFL_OK;
    BFL_CUDA(cudaMemcpyAsync(h->dP, h->hostP, sizeof(float) * (size_t)h->P_rows * h->vdim, cudaMemcpyHostToDevice, h->stream));
    BFL_CUDA(cudaMemcpyAsync(h->dQ, h->hostQ, sizeof(float) * (size_t)h->Q_rows * h->vdim, cudaMemcpyHostToDevice, h->stream));
    BFL_CUDA(cudaMemcpyAsync(h->dQb, h->hostQb, sizeof(float) * (size_t)h->Q_rows, cudaMemcpyHostToDevice, h->stream));
    BFL_CUDA(cudaStreamSynchronize(h->stream));
    return BFL_OK;
}

int bfl_sgd_compute_loss(bfl_sgd_t* h, int32_t n, const int32_t* users, const int32_t* positives,
                         const int32_t* negatives, double* out_loss) {
    if (out_loss) *out_loss = 0.0;
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "initialize_model() must precede compute_loss()");
    if (n <= 0) return BFL_OK;
    if (!users || !positives || !negatives) BFL_FAIL(BFL_ERR_ARG, "null probe arrays");
    if (BFL_OK != h->probe.reserve((size_t)3 * n)) return BFL_ERR_CUDA;
    BFL_CUDA(cudaMemcpyAsync(h->probe.p, users, sizeof(int32_t) * n, cudaMemcpyHostToDevice, h->stream));
    BFL_CUDA(cudaMemcpyAsync(h->probe.p + n, positives, sizeof(int32_t) * n, cudaMemcpyHostToDevice, h->stream));
    BFL_CUDA(cudaMemcpyAsync(h->probe.p + 2 * n, negatives, sizeof(int32_t) * n, cudaMemcpyHostToDevice, h->stream));
    BFL_CUDA(cudaMemsetAsync(h->d_stat.p + 1, 0, sizeof(double), h->stream));
    const int grid = std::min((n + 7) / 8, h->num_sms * 4);
    if (h->deterministic) {  // per-triple terms, summed by the fixed tree
        if (BFL_OK != h->det_terms.reserve((size_t)n)) return BFL_ERR_CUDA;
        if (BFL_OK != h->det_lpart.reserve((size_t)(n + kDetLossRange - 1) / kDetLossRange)) return BFL_ERR_CUDA;
        det_probe_terms_kernel<<<grid, 256, 0, h->stream>>>(h->kind, h->dP, h->dQ, h->dQb, h->d, h->vdim,
                                                            h->use_bias, h->score_l2, (double)h->threshold, h->probe.p,
                                                            h->probe.p + n, h->probe.p + 2 * n, n, h->det_terms.p);
        BFL_LAUNCHED();
        int rc = det_loss_sum(h, h->det_terms.p, n, h->d_stat.p + 1, h->stream);
        if (rc != BFL_OK) return rc;
    } else {
        probe_loss_kernel<<<grid, 256, 0, h->stream>>>(h->kind, h->dP, h->dQ, h->dQb, h->d, h->vdim, h->use_bias,
                                                       h->score_l2, (double)h->threshold, h->probe.p, h->probe.p + n,
                                                       h->probe.p + 2 * n, n, h->d_stat.p + 1);
        BFL_LAUNCHED();
    }
    double v = 0.0;
    BFL_CUDA(cudaMemcpyAsync(&v, h->d_stat.p + 1, sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    BFL_CUDA(cudaStreamSynchronize(h->stream));
    if (out_loss) *out_loss = v / (double)n;
    return BFL_OK;
}

int bfl_sgd_apply_triples_device(bfl_sgd_t* h, const int32_t* d_users, const int32_t* d_pos, const int32_t* d_neg,
                                 int64_t n, float lr, void* stream) {
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "factors not bound");
    if (h->kind != BFL_SGD_BPR) BFL_FAIL(BFL_ERR_STATE, "explicit triples are a BPR hook");
    if (h->deterministic) BFL_FAIL(BFL_ERR_STATE, "explicit triples add their gradients with atomics: not in deterministic mode");
    SgdArgs a;
    fill_args(h, a, nullptr, 0, 0, 0, 0, 0);
    a.lr = lr;
    return launch_bpr_apply(h, a, d_users, d_pos, d_neg, n, (cudaStream_t)stream);
}

int bfl_sgd_sample_device(bfl_sgd_t* h, int64_t row_begin, int64_t row_end, int32_t* d_users, int32_t* d_pos,
                          int32_t* d_neg, void* stream) {
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "factors not bound");
    if (!h->csr.indptr || !h->csr.keys) BFL_FAIL(BFL_ERR_STATE, "no device CSR bound");
    if (row_end == row_begin) BFL_FAIL(BFL_ERR_ARG, "bad row range");
    int rc = h->csr.check_range(row_begin, row_end);
    if (rc != BFL_OK) return rc;
    int64_t beg = 0, end = 0;
    rc = read_row_span(h->csr.indptr, row_begin, row_end, (cudaStream_t)stream, &beg, &end);
    if (rc != BFL_OK) return rc;
    SgdArgs a;
    fill_args(h, a, h->csr.keys, 0, row_begin, row_end, beg, end);
    const int64_t cnt = (end - beg) * h->num_neg;
    if (cnt <= 0) return BFL_OK;
    const int grid = (int)std::min<int64_t>((cnt + 255) / 256, (int64_t)h->num_sms * 32);
    bpr_sample_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(a, d_users, d_pos, d_neg);
    BFL_LAUNCHED();
    return BFL_OK;
}

float* bfl_sgd_grad_device(bfl_sgd_t* h, int which) {
    if (!h) return nullptr;
    return which == 0 ? h->gP.p : (which == 1 ? h->gQ.p : h->gQb.p);
}

int32_t* bfl_sgd_count_device(bfl_sgd_t* h, int which) {
    if (!h) return nullptr;
    return which == 0 ? h->cP.p : h->cQ.p;
}

int bfl_sgd_set_trace_device(bfl_sgd_t* h, int32_t* d_trials, int32_t* d_negs) {
    if (!h) BFL_FAIL(BFL_ERR_ARG, "null handle");
    h->trace_trials = d_trials;
    h->trace_negs = d_negs;
    return BFL_OK;
}

int bfl_sgd_fold_in_items_device(bfl_sgd_t* h, const float* dP, int64_t P_rows, const float* dQ, const float* dQb,
                                 int64_t Q_rows, const int64_t* d_train_indptr, const int32_t* d_train_keys,
                                 const int64_t* d_cum, const int64_t* d_hist_indptr, const int32_t* d_hist_users,
                                 int64_t n, int64_t hist_nnz, float* dX, float* dXb, int epochs,
                                 int32_t* d_trace_negs, int32_t* d_trace_trials, void* stream) {
    if (!h || !h->opt_set) BFL_FAIL(BFL_ERR_STATE, "init() must precede fold_in_items");
    if (epochs < 1) BFL_FAIL(BFL_ERR_ARG, "fold_in_items: epochs must be >= 1");
    if (n < 0 || n > (int64_t)INT32_MAX || hist_nnz < 0) BFL_FAIL(BFL_ERR_ARG, "fold_in_items: bad row count");
    if (P_rows < 1 || Q_rows < 1 || Q_rows > (int64_t)INT32_MAX) BFL_FAIL(BFL_ERR_ARG, "fold_in_items: bad factor shapes");
    if (n == 0) return BFL_OK;
    if (!dP || !dQ || !dQb || !d_train_indptr || !d_train_keys || !d_hist_indptr || !d_hist_users || !dX || !dXb)
        BFL_FAIL(BFL_ERR_ARG, "fold_in_items: null array");
    if (h->kind == BFL_SGD_WARP && (d_trace_negs == nullptr) != (d_trace_trials == nullptr))
        BFL_FAIL(BFL_ERR_ARG, "fold_in_items: a WARP trace needs both the negatives and the trial counts");
    SgdArgs a;
    fill_args(h, a, d_train_keys, 0, 0, P_rows, 0, 0);
    a.P = const_cast<float*>(dP); a.Q = const_cast<float*>(dQ); a.Qb = const_cast<float*>(dQb);
    a.gP = a.gQ = a.gQb = nullptr; a.cP = a.cQ = nullptr;
    a.indptr = d_train_indptr;
    a.cum = d_cum;
    a.uniform = h->uniform || !d_cum;
    a.trace_trials = a.trace_negs = nullptr;
    a.num_items = (int32_t)Q_rows;
    FoldArgs f;
    f.h_ind = d_hist_indptr; f.h_users = d_hist_users; f.X = dX; f.Xb = dXb;
    f.trace_negs = d_trace_negs; f.trace_trials = d_trace_trials;
    f.n = n; f.nnz = hist_nnz; f.epochs = epochs; f.inv_epochs = 1.0 / (double)epochs;
    f.lr0 = h->lr0; f.min_lr = h->min_lr; f.beta1 = h->beta1;
    const int grid = (int)std::min<int64_t>((n + 7) / 8, (int64_t)h->num_sms * 16);
    const int nv = (h->vdim / 4 + 31) / 32;
    cudaStream_t st = (cudaStream_t)stream;
    if (h->kind == BFL_SGD_WARP) {
        if (nv <= 1) sgd_fold_in_items_kernel<1, true><<<grid, 256, 0, st>>>(a, f);
        else if (nv <= 2) sgd_fold_in_items_kernel<2, true><<<grid, 256, 0, st>>>(a, f);
        else sgd_fold_in_items_kernel<4, true><<<grid, 256, 0, st>>>(a, f);
    } else {
        if (nv <= 1) sgd_fold_in_items_kernel<1, false><<<grid, 256, 0, st>>>(a, f);
        else if (nv <= 2) sgd_fold_in_items_kernel<2, false><<<grid, 256, 0, st>>>(a, f);
        else sgd_fold_in_items_kernel<4, false><<<grid, 256, 0, st>>>(a, f);
    }
    BFL_LAUNCHED();
    return BFL_OK;
}

int bfl_sgd_epoch(bfl_sgd_t* h) { return h ? h->epoch : -1; }
double bfl_sgd_current_lr(bfl_sgd_t* h) { return h ? h->cur_lr : 0.0; }

int bfl_sgd_read_stats(bfl_sgd_t* h, double* loss_sum, int64_t* num_updates) {
    if (!h || !h->opt_set) BFL_FAIL(BFL_ERR_STATE, "init() first");
    double l = 0.0;
    unsigned long long u = 0;
    BFL_CUDA(cudaDeviceSynchronize());
    BFL_CUDA(cudaMemcpy(&l, h->d_stat.p, sizeof(double), cudaMemcpyDeviceToHost));
    BFL_CUDA(cudaMemcpy(&u, h->d_upd.p, sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    if (loss_sum) *loss_sum = l;
    if (num_updates) *num_updates = (int64_t)u;
    return BFL_OK;
}

}  // extern "C"
