// pLSI backend: EM pass, normalisation and initialisation kernels + C ABI.
// Replaces plsi::CPLSI (lib/algo_impl/plsi/plsi.cc) behind CyPLSI (buffalo/algo/_plsi.pyx:13-57).
//
// One EM iteration is reset -> update over the rowwise CSR -> normalize -> swap (buffalo/algo/plsi.py:132-160).
// The update is one pass over the rows: every nonzero (x, c, v) gathers the current item row Q[c], forms
// latent = max(P[x] * Q[c], 1e-10) over the d real columns, and adds v * latent / sum(latent) into the new user row
// and into the new item row.  Only row x's warp reads P[x] during the pass, so the new user row overwrites P[x] in
// place; the new item rows go to the library-owned accumulator Qacc through float4 atomics.  A per-row flag records
// which user rows the pass wrote: a row the pass never reached counts as zero in normalize, as the reference's
// zeroed accumulator would.
//
// Deterministic mode (option `deterministic`): the atomics go.  An item pass over the colwise CSR runs first and
// builds every new item row with plain stores from the current P and Q (one warp per item, or per fixed segment of a
// long item, whose partial rows a second kernel adds in segment order); the row pass then runs without the item
// accumulation, and the loss is per-row fp64 partials summed by a fixed tree.  The same inputs give the same bits.
//
// Layout: factor rows have pitch vdim = ceil4(d) on the device; padding columns stay zero.  The holder entry points
// take the caller's [rows x d] host arrays (plsi.py:107-111 does not pad) and copy with a pitch conversion.
#include <algorithm>
#include <cmath>
#include <new>
#include <vector>

#include "bfl_common.cuh"

using namespace bfl;

namespace {

constexpr float kLatentFloor = 1e-10f;   // plsi.cc:95
constexpr int kColsumBlocks = 512;       // fixed partial count: the column sums do not depend on the device
// Entries per segment of a long item row in the deterministic item pass.  A compile-time constant, so the order of
// every item sum depends on the data only, not on the grid, the SM count or the chunking.
constexpr int64_t kItemSegment = 4096;

__device__ __forceinline__ void red4(float* p, float4 v) { atomicAdd(reinterpret_cast<float4*>(p), v); }

__device__ __forceinline__ float4 ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// latent of one float4 slice starting at column col; columns >= d are padding and contribute nothing
__device__ __forceinline__ float4 latent4(float4 p, float4 q, int col, int d) {
    float4 l;
    l.x = col + 0 < d ? fmaxf(p.x * q.x, kLatentFloor) : 0.f;
    l.y = col + 1 < d ? fmaxf(p.y * q.y, kLatentFloor) : 0.f;
    l.z = col + 2 < d ? fmaxf(p.z * q.z, kLatentFloor) : 0.f;
    l.w = col + 3 < d ? fmaxf(p.w * q.w, kLatentFloor) : 0.f;
    return l;
}

struct EmArgs {
    float* P;                // [P_rows x vdim]: current rows in, new (unnormalised) rows out
    const float* Q;          // [Q_rows x vdim] current item factors (read only during the pass)
    float* Qacc;             // [Q_rows x vdim] new item factors, accumulated with atomics
    uint8_t* visited;        // [P_rows] set for every row the pass writes
    const int64_t* ends;     // ends[i] = end offset of row row_begin + i; ends[-1] is valid when row_begin > 0
    const int32_t* keys;     // entry j at keys[j - shift]
    const float* vals;
    int64_t shift;
    int64_t row_begin, n_rows;
    double* loss;            // += -sum v * log(norm) (nullable)
    int d, vdim;
    double* row_loss;        // kDet: row_loss[i] = -sum v * log(norm) of row row_begin + i (nullable)
};

// One warp per user row.  A row is split into float4 slices; G lanes (a group) cover one entry's slices, NV slices
// per lane when a row has more than 32 slices, and the 32 / G groups of the warp take different entries.  Keys and
// values are loaded 32 at a time, coalesced, and broadcast by shuffles; each group keeps U item rows in flight.
// kDet: no item accumulation (the item pass built Qacc) and the loss goes to row_loss instead of an atomic.
template <int G, int NV, int U, bool kDet = false>
__global__ void __launch_bounds__(256) plsi_em_kernel(const EmArgs a) {
    constexpr int NG = 32 / G;
    __shared__ double s_loss[8];
    const int lane = threadIdx.x & 31, g = lane / G, gl = lane % G;
    const int nv4 = a.vdim >> 2;
    const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    double lacc = 0.0;
    for (int64_t i = warp0; i < a.n_rows; i += nwarps) {
        if constexpr (kDet) lacc = 0.0;
        const int64_t x = a.row_begin + i;
        const int64_t beg = (x == 0) ? 0 : a.ends[i - 1];
        const int64_t end = a.ends[i];
        float* prow = a.P + x * a.vdim;
        float4 p[NV], acc[NV];
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const int s = gl + G * k;
            p[k] = s < nv4 ? *reinterpret_cast<const float4*>(prow + 4 * s) : make_float4(0.f, 0.f, 0.f, 0.f);
            acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        for (int64_t base = beg; base < end; base += 32) {
            const int cnt = (int)min((int64_t)32, end - base);
            const int my_key = lane < cnt ? __ldg(a.keys + (base + lane - a.shift)) : 0;
            const float my_val = lane < cnt ? __ldg(a.vals + (base + lane - a.shift)) : 0.f;
            for (int t = 0; t < cnt; t += NG * U) {
                int c[U];
                float v[U];
                bool ok[U];
                float4 q[U][NV];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const int e = t + u * NG + g;
                    ok[u] = e < cnt;
                    c[u] = __shfl_sync(FULL, my_key, e & 31);
                    v[u] = __shfl_sync(FULL, my_val, e & 31);
#pragma unroll
                    for (int k = 0; k < NV; ++k) {
                        const int s = gl + G * k;
                        q[u][k] = (ok[u] && s < nv4) ? ld4(a.Q + (int64_t)c[u] * a.vdim + 4 * s)
                                                     : make_float4(0.f, 0.f, 0.f, 0.f);
                    }
                }
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    float4 l[NV];
                    float ps = 0.f;
#pragma unroll
                    for (int k = 0; k < NV; ++k) {
                        l[k] = latent4(p[k], q[u][k], 4 * (gl + G * k), a.d);
                        ps += (l[k].x + l[k].y) + (l[k].z + l[k].w);
                    }
#pragma unroll
                    for (int o = G / 2; o > 0; o >>= 1) ps += __shfl_xor_sync(FULL, ps, o);
                    // lanes past the chunk's end add zeros to acc and skip the atomics
                    const float w = ok[u] ? v[u] / ps : 0.f;
                    if (ok[u] && gl == 0) lacc -= (double)v[u] * (double)logf(ps);
                    if constexpr (kDet) {
                        // the rounding of the default instantiation (a product, then a sum: its product also
                        // feeds the atomic, so it is not contracted), spelled out so that no FMA forms here
#pragma unroll
                        for (int k = 0; k < NV; ++k) {
                            acc[k].x = __fadd_rn(acc[k].x, __fmul_rn(l[k].x, w));
                            acc[k].y = __fadd_rn(acc[k].y, __fmul_rn(l[k].y, w));
                            acc[k].z = __fadd_rn(acc[k].z, __fmul_rn(l[k].z, w));
                            acc[k].w = __fadd_rn(acc[k].w, __fmul_rn(l[k].w, w));
                        }
                    } else {
                        float* qrow = a.Qacc + (int64_t)c[u] * a.vdim;
#pragma unroll
                        for (int k = 0; k < NV; ++k) {
                            const int s = gl + G * k;
                            const float4 ctb = make_float4(l[k].x * w, l[k].y * w, l[k].z * w, l[k].w * w);
                            acc[k].x += ctb.x; acc[k].y += ctb.y; acc[k].z += ctb.z; acc[k].w += ctb.w;
                            if (ok[u] && s < nv4) red4(qrow + 4 * s, ctb);
                        }
                    }
                }
            }
        }
        // the groups of the warp hold partial sums of the same row: fold them into group 0
#pragma unroll
        for (int k = 0; k < NV; ++k) {
#pragma unroll
            for (int o = G; o < 32; o <<= 1) {
                acc[k].x += __shfl_xor_sync(FULL, acc[k].x, o);
                acc[k].y += __shfl_xor_sync(FULL, acc[k].y, o);
                acc[k].z += __shfl_xor_sync(FULL, acc[k].z, o);
                acc[k].w += __shfl_xor_sync(FULL, acc[k].w, o);
            }
            const int s = gl + G * k;
            if (g == 0 && s < nv4) *reinterpret_cast<float4*>(prow + 4 * s) = acc[k];
        }
        if (lane == 0) a.visited[x] = 1;
        if constexpr (kDet) {
            if (a.row_loss) {
                const double r = warp_sum_d(lacc);
                if (lane == 0) a.row_loss[i] = r;
            }
        }
    }
    if constexpr (!kDet) {
        if (a.loss) {
            lacc = warp_sum_d(lacc);
            if (lane == 0) s_loss[threadIdx.x >> 5] = lacc;
            __syncthreads();
            if (threadIdx.x == 0) {
                double s = 0.0;
                for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += s_loss[w];
                if (s != 0.0) atomicAdd(a.loss, s);
            }
        }
    }
}

struct FoldArgs {
    const float* Q;          // [Q_rows x vdim] item factors, fixed
    const int64_t* ends;     // END offsets of the history rows (row 0 starts at entry 0)
    const int32_t* keys;     // item of each entry
    const float* vals;
    float* X;                // [n_rows x vdim]: start rows in, folded rows out
    int64_t n_rows;
    int iters, d, vdim;
    float a1;                // alpha1 / d, as normalize_all passes it to the row normalisation
};

// Folding-in (Hofmann): EM on one user row with the item factors fixed.  One warp per history row, the lane layout of
// plsi_em_kernel (G lanes per entry, NV float4 slices per lane, U item rows in flight per group).  The row stays in
// registers for all `iters` iterations; each iteration streams the row's keys, values and item rows, accumulates as
// the deterministic row pass does (a product, then a sum, in entry order per group; groups folded by a butterfly, so
// every group holds the same bits), and divides (acc + a1) by its sum over the d real columns with the rounding of
// plsi_normalize_rows_kernel.  No atomics and no shared state: the result depends on the row's own data only.  Rows
// without entries keep their start row.  Only the final row is stored.
template <int G, int NV, int U>
__global__ void __launch_bounds__(256) plsi_fold_in_kernel(const FoldArgs a) {
    constexpr int NG = 32 / G;
    const int lane = threadIdx.x & 31, g = lane / G, gl = lane % G;
    const int nv4 = a.vdim >> 2;
    const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t x = warp0; x < a.n_rows; x += nwarps) {
        const int64_t beg = (x == 0) ? 0 : a.ends[x - 1];
        const int64_t end = a.ends[x];
        if (end <= beg) continue;
        float* xrow = a.X + x * a.vdim;
        float4 p[NV], acc[NV];
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const int s = gl + G * k;
            p[k] = s < nv4 ? *reinterpret_cast<const float4*>(xrow + 4 * s) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        for (int it = 0; it < a.iters; ++it) {
#pragma unroll
            for (int k = 0; k < NV; ++k) acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int64_t base = beg; base < end; base += 32) {
                const int cnt = (int)min((int64_t)32, end - base);
                const int my_key = lane < cnt ? __ldg(a.keys + base + lane) : 0;
                const float my_val = lane < cnt ? __ldg(a.vals + base + lane) : 0.f;
                for (int t = 0; t < cnt; t += NG * U) {
                    bool ok[U];
                    float v[U];
                    float4 q[U][NV];
#pragma unroll
                    for (int u = 0; u < U; ++u) {
                        const int e = t + u * NG + g;
                        ok[u] = e < cnt;
                        const int c = __shfl_sync(FULL, my_key, e & 31);
                        v[u] = __shfl_sync(FULL, my_val, e & 31);
#pragma unroll
                        for (int k = 0; k < NV; ++k) {
                            const int s = gl + G * k;
                            q[u][k] = (ok[u] && s < nv4) ? ld4(a.Q + (int64_t)c * a.vdim + 4 * s)
                                                         : make_float4(0.f, 0.f, 0.f, 0.f);
                        }
                    }
#pragma unroll
                    for (int u = 0; u < U; ++u) {
                        float4 l[NV];
                        float ps = 0.f;
#pragma unroll
                        for (int k = 0; k < NV; ++k) {
                            l[k] = latent4(p[k], q[u][k], 4 * (gl + G * k), a.d);
                            ps += (l[k].x + l[k].y) + (l[k].z + l[k].w);
                        }
#pragma unroll
                        for (int o = G / 2; o > 0; o >>= 1) ps += __shfl_xor_sync(FULL, ps, o);
                        const float w = ok[u] ? v[u] / ps : 0.f;
#pragma unroll
                        for (int k = 0; k < NV; ++k) {
                            acc[k].x = __fadd_rn(acc[k].x, __fmul_rn(l[k].x, w));
                            acc[k].y = __fadd_rn(acc[k].y, __fmul_rn(l[k].y, w));
                            acc[k].z = __fadd_rn(acc[k].z, __fmul_rn(l[k].z, w));
                            acc[k].w = __fadd_rn(acc[k].w, __fmul_rn(l[k].w, w));
                        }
                    }
                }
            }
            float ps = 0.f;
#pragma unroll
            for (int k = 0; k < NV; ++k) {
#pragma unroll
                for (int o = G; o < 32; o <<= 1) {
                    acc[k].x += __shfl_xor_sync(FULL, acc[k].x, o);
                    acc[k].y += __shfl_xor_sync(FULL, acc[k].y, o);
                    acc[k].z += __shfl_xor_sync(FULL, acc[k].z, o);
                    acc[k].w += __shfl_xor_sync(FULL, acc[k].w, o);
                }
                const int col = 4 * (gl + G * k);
                if (gl + G * k < nv4)
                    ps += (col + 0 < a.d ? acc[k].x + a.a1 : 0.f) + (col + 1 < a.d ? acc[k].y + a.a1 : 0.f) +
                          (col + 2 < a.d ? acc[k].z + a.a1 : 0.f) + (col + 3 < a.d ? acc[k].w + a.a1 : 0.f);
            }
#pragma unroll
            for (int o = G / 2; o > 0; o >>= 1) ps += __shfl_xor_sync(FULL, ps, o);
#pragma unroll
            for (int k = 0; k < NV; ++k) {
                const int col = 4 * (gl + G * k);
                p[k].x = col + 0 < a.d ? (acc[k].x + a.a1) / ps : 0.f;
                p[k].y = col + 1 < a.d ? (acc[k].y + a.a1) / ps : 0.f;
                p[k].z = col + 2 < a.d ? (acc[k].z + a.a1) / ps : 0.f;
                p[k].w = col + 3 < a.d ? (acc[k].w + a.a1) / ps : 0.f;
            }
        }
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const int s = gl + G * k;
            if (g == 0 && s < nv4) *reinterpret_cast<float4*>(xrow + 4 * s) = p[k];
        }
    }
}

struct ItemArgs {
    const float* P;          // [P_rows x vdim] current user rows (read only during the pass)
    const float* Q;          // [Q_rows x vdim] current item rows (read only)
    float* Qacc;             // [Q_rows x vdim] new item rows, written with plain stores
    float* part;             // [n_segs x vdim] partial rows of the long items' segments
    const int64_t* ends;     // ends[i] = end offset of item item_begin + i; ends[-1] is valid when item_begin > 0
    const int32_t* keys;     // entry j (a user row) at keys[j - shift]
    const float* vals;
    int64_t shift;
    int64_t item_begin, n_items;
    const int32_t* seg;      // segment tasks: seg[2s] = item, seg[2s + 1] = segment index within the item
    int64_t n_segs;
    int d, vdim;
};

// Deterministic item pass: one warp per item of at most kItemSegment entries (tasks [0, n_items)) and one per segment
// of a longer item (tasks [n_items, n_items + n_segs)).  The lane layout, latent4 and the norm reduction are those of
// plsi_em_kernel, with Q[item] held in registers and the user rows gathered, so every norm is bitwise the one the row
// pass computes for the same entry.  Each group sums its entries in order, the groups fold by a fixed butterfly, and
// the row goes out with plain stores: to Qacc, or to the segment's partial row.
template <int G, int NV, int U>
__global__ void __launch_bounds__(256) plsi_item_kernel(const ItemArgs a) {
    constexpr int NG = 32 / G;
    const int lane = threadIdx.x & 31, g = lane / G, gl = lane % G;
    const int nv4 = a.vdim >> 2;
    const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t task = warp0; task < a.n_items + a.n_segs; task += nwarps) {
        int64_t item, beg, end;
        float* out;
        if (task < a.n_items) {
            item = a.item_begin + task;
            beg = (item == 0) ? 0 : a.ends[task - 1];
            end = a.ends[task];
            if (end - beg > kItemSegment) continue;          // its segments write partial rows
            out = a.Qacc + item * a.vdim;
        } else {
            const int64_t s = task - a.n_items;
            item = a.seg[2 * s];
            const int64_t t = item - a.item_begin;
            beg = ((item == 0) ? 0 : a.ends[t - 1]) + (int64_t)a.seg[2 * s + 1] * kItemSegment;
            end = min(a.ends[t], beg + kItemSegment);
            out = a.part + s * a.vdim;
        }
        const float* qrow = a.Q + item * a.vdim;
        float4 q[NV], acc[NV];
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const int s = gl + G * k;
            q[k] = s < nv4 ? ld4(qrow + 4 * s) : make_float4(0.f, 0.f, 0.f, 0.f);
            acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        for (int64_t base = beg; base < end; base += 32) {
            const int cnt = (int)min((int64_t)32, end - base);
            const int my_key = lane < cnt ? __ldg(a.keys + (base + lane - a.shift)) : 0;
            const float my_val = lane < cnt ? __ldg(a.vals + (base + lane - a.shift)) : 0.f;
            for (int t = 0; t < cnt; t += NG * U) {
                int r[U];
                float v[U];
                bool ok[U];
                float4 p[U][NV];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const int e = t + u * NG + g;
                    ok[u] = e < cnt;
                    r[u] = __shfl_sync(FULL, my_key, e & 31);
                    v[u] = __shfl_sync(FULL, my_val, e & 31);
#pragma unroll
                    for (int k = 0; k < NV; ++k) {
                        const int s = gl + G * k;
                        p[u][k] = (ok[u] && s < nv4) ? ld4(a.P + (int64_t)r[u] * a.vdim + 4 * s)
                                                     : make_float4(0.f, 0.f, 0.f, 0.f);
                    }
                }
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    float4 l[NV];
                    float ps = 0.f;
#pragma unroll
                    for (int k = 0; k < NV; ++k) {
                        l[k] = latent4(p[u][k], q[k], 4 * (gl + G * k), a.d);
                        ps += (l[k].x + l[k].y) + (l[k].z + l[k].w);
                    }
#pragma unroll
                    for (int o = G / 2; o > 0; o >>= 1) ps += __shfl_xor_sync(FULL, ps, o);
                    const float w = ok[u] ? v[u] / ps : 0.f;
#pragma unroll
                    for (int k = 0; k < NV; ++k) {
                        acc[k].x = __fadd_rn(acc[k].x, __fmul_rn(l[k].x, w));
                        acc[k].y = __fadd_rn(acc[k].y, __fmul_rn(l[k].y, w));
                        acc[k].z = __fadd_rn(acc[k].z, __fmul_rn(l[k].z, w));
                        acc[k].w = __fadd_rn(acc[k].w, __fmul_rn(l[k].w, w));
                    }
                }
            }
        }
#pragma unroll
        for (int k = 0; k < NV; ++k) {
#pragma unroll
            for (int o = G; o < 32; o <<= 1) {
                acc[k].x += __shfl_xor_sync(FULL, acc[k].x, o);
                acc[k].y += __shfl_xor_sync(FULL, acc[k].y, o);
                acc[k].z += __shfl_xor_sync(FULL, acc[k].z, o);
                acc[k].w += __shfl_xor_sync(FULL, acc[k].w, o);
            }
            const int s = gl + G * k;
            if (g == 0 && s < nv4) *reinterpret_cast<float4*>(out + 4 * s) = acc[k];
        }
    }
}

// Long items: Qacc[item] = the item's segment partial rows added in segment order.  One thread per (item, column);
// long_off[L] .. long_off[L + 1] are item long_items[L]'s rows of `part`.
__global__ void __launch_bounds__(256) plsi_item_combine_kernel(const float* part, const int32_t* long_items,
                                                                const int64_t* long_off, int64_t n_long, int vdim,
                                                                float* Qacc) {
    const int64_t n = n_long * vdim;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t L = e / vdim;
        const int col = (int)(e % vdim);
        const int64_t s0 = long_off[L], s1 = long_off[L + 1];
        float t = part[s0 * vdim + col];
        for (int64_t s = s0 + 1; s < s1; ++s) t += part[s * vdim + col];
        Qacc[(int64_t)long_items[L] * vdim + col] = t;
    }
}

// P rows: (row + alpha1) / sum(row + alpha1) over the d real columns (plsi.cc:115-119).  A row the last pass did not
// write is the reference's zeroed accumulator row.  visited == null: every row is taken as it is.  G lanes per row.
template <int G>
__global__ void __launch_bounds__(256) plsi_normalize_rows_kernel(float* P, const uint8_t* visited, int64_t rows,
                                                                  int d, int vdim, float alpha1) {
    const int lane = threadIdx.x & 31, gl = lane % G;
    const int nv4 = vdim >> 2;
    const int64_t grp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / G;
    const int64_t ngrp = ((int64_t)gridDim.x * blockDim.x) / G;
    const int64_t span = (rows + (32 / G) - 1) / (32 / G) * (32 / G);   // whole warps iterate together
    for (int64_t x = grp0; x < span; x += ngrp) {
        const bool live = x < rows;
        const bool zero = live && visited && !visited[x];
        float* row = P + (live ? x : 0) * vdim;
        float ps = 0.f;
        for (int s = gl; s < nv4; s += G) {
            float4 v = (live && !zero) ? *reinterpret_cast<const float4*>(row + 4 * s) : make_float4(0.f, 0.f, 0.f, 0.f);
            const int col = 4 * s;
            ps += (col + 0 < d ? v.x + alpha1 : 0.f) + (col + 1 < d ? v.y + alpha1 : 0.f) +
                  (col + 2 < d ? v.z + alpha1 : 0.f) + (col + 3 < d ? v.w + alpha1 : 0.f);
        }
#pragma unroll
        for (int o = G / 2; o > 0; o >>= 1) ps += __shfl_xor_sync(FULL, ps, o);
        if (!live) continue;
        for (int s = gl; s < nv4; s += G) {
            float4 v = zero ? make_float4(0.f, 0.f, 0.f, 0.f) : *reinterpret_cast<const float4*>(row + 4 * s);
            const int col = 4 * s;
            v.x = col + 0 < d ? (v.x + alpha1) / ps : 0.f;
            v.y = col + 1 < d ? (v.y + alpha1) / ps : 0.f;
            v.z = col + 2 < d ? (v.z + alpha1) / ps : 0.f;
            v.w = col + 3 < d ? (v.w + alpha1) / ps : 0.f;
            *reinterpret_cast<float4*>(row + 4 * s) = v;
        }
    }
}

// Q columns, stage 1: per-CTA fp64 partial column sums over a fixed contiguous item range.
__global__ void __launch_bounds__(256) plsi_colsum_partial_kernel(const float* Q, int64_t rows, int vdim,
                                                                  int64_t rows_per_blk, double* part) {
    __shared__ double s_part[1024];
    const int nv4 = vdim >> 2;
    const int par = blockDim.x / nv4;             // rows summed side by side
    const int r = threadIdx.x / nv4, s = threadIdx.x % nv4;
    const int64_t lo = (int64_t)blockIdx.x * rows_per_blk, hi = min(rows, lo + rows_per_blk);
    double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
    if (r < par) {
        for (int64_t i = lo + r; i < hi; i += par) {
            const float4 v = *reinterpret_cast<const float4*>(Q + i * vdim + 4 * s);
            a0 += v.x; a1 += v.y; a2 += v.z; a3 += v.w;
        }
        double* dst = s_part + r * vdim + 4 * s;
        dst[0] = a0; dst[1] = a1; dst[2] = a2; dst[3] = a3;
    }
    __syncthreads();
    for (int k = threadIdx.x; k < vdim; k += blockDim.x) {
        double t = 0.0;
        for (int j = 0; j < par; ++j) t += s_part[j * vdim + k];
        part[(int64_t)blockIdx.x * vdim + k] = t;
    }
}

// Q columns, stage 2: the partials in block order, plus rows * alpha2 (the reference adds alpha2 to every entry).
__global__ void plsi_colsum_final_kernel(const double* part, int nblk, int vdim, int64_t rows, float alpha2,
                                         double* colsum) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= vdim) return;
    double t = 0.0;
    for (int b = 0; b < nblk; ++b) t += part[(int64_t)b * vdim + k];
    colsum[k] = t + (double)rows * (double)alpha2;
}

// Q columns, stage 3: (q + alpha2) / column sum (plsi.cc:120-124); padding columns stay zero.
__global__ void __launch_bounds__(256) plsi_scale_cols_kernel(float* Q, int64_t rows, int d, int vdim, float alpha2,
                                                              const double* colsum) {
    const int nv4 = vdim >> 2;
    const int64_t n = rows * nv4;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
        const int s = (int)(e % nv4);
        const int col = 4 * s;
        float4* p = reinterpret_cast<float4*>(Q) + e;
        float4 v = *p;
        v.x = col + 0 < d ? (float)((double)(v.x + alpha2) / colsum[col + 0]) : 0.f;
        v.y = col + 1 < d ? (float)((double)(v.y + alpha2) / colsum[col + 1]) : 0.f;
        v.z = col + 2 < d ? (float)((double)(v.z + alpha2) / colsum[col + 2]) : 0.f;
        v.w = col + 3 < d ? (float)((double)(v.w + alpha2) / colsum[col + 3]) : 0.f;
        *p = v;
    }
}

// |N(0, 1/d)| per real column (plsi.cc:51-64), from Philox4x32-10 keyed by (seed, matrix, element): Box-Muller on
// the first two words.  Padding columns are zero.
__global__ void __launch_bounds__(256) plsi_init_kernel(float* F, int64_t rows, int d, int vdim, uint32_t seed,
                                                        uint32_t matrix) {
    const int64_t n = rows * vdim;
    const float sd = 1.0f / (float)d;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = e / vdim;
        const int col = (int)(e % vdim);
        float v = 0.f;
        if (col < d) {
            const uint64_t idx = (uint64_t)r * (uint64_t)d + (uint64_t)col;
            uint32_t o[4];
            philox4x32_10((uint32_t)idx, (uint32_t)(idx >> 32), matrix, 0x504C5349u, seed, 0x5EEDu, o);
            const float u1 = ((float)(o[0] >> 8) + 1.0f) * (1.0f / 16777216.0f);   // (0, 1]
            const float u2 = (float)(o[1] >> 8) * (1.0f / 16777216.0f);
            v = fabsf(sqrtf(-2.0f * logf(u1)) * cospif(2.0f * u2)) * sd;
        }
        F[e] = v;
    }
}

}  // namespace

// The items of a colwise CSR longer than one segment, ascending: items[L] owns segments off[L] .. off[L + 1] - 1, and
// seg holds the (item, segment index) pair of every segment.
struct LongItems {
    std::vector<int32_t> items;
    std::vector<int64_t> off{0};
    std::vector<int32_t> seg;
    // indptr: HOST global END offsets; items [item_begin, item_end)
    void build(const int64_t* indptr, int64_t item_begin, int64_t item_end) {
        items.clear(); seg.clear(); off.assign(1, 0);
        for (int64_t x = item_begin; x < item_end; ++x) {
            const int64_t len = indptr[x] - (x == 0 ? 0 : indptr[x - 1]);
            if (len <= kItemSegment) continue;
            const int64_t n = (len + kItemSegment - 1) / kItemSegment;
            items.push_back((int32_t)x);
            for (int64_t k = 0; k < n; ++k) {
                seg.push_back((int32_t)x);
                seg.push_back((int32_t)k);
            }
            off.push_back(off.back() + n);
        }
    }
    int64_t n_segs() const { return off.back(); }
};

// the Holder's hostP/hostQ are the caller's [rows x d] arrays (holder path), ownP/ownQ the library's device copies
struct bfl_plsi : Holder {
    uint32_t seed = 0;

    DevBuf<float> Qacc;                         // new item factors of the running iteration
    DevBuf<uint8_t> visited;
    DevBuf<double> colpart, colsum, d_loss;

    DevBuf<int64_t> stage_ends;
    DevBuf<int32_t> stage_keys;
    DevBuf<float> stage_vals;
    CsrBinding csr;

    // deterministic mode
    bool deterministic = false;
    bool rows_done = false;                     // a row pass ran since the last reset / swap: P is overwritten
    DevBuf<double> row_loss, loss_part;
    DevBuf<float> seg_part;                     // partial rows of the long items' segments
    CsrBinding ccsr;                            // the bound colwise CSR (rows == Q_rows)
    LongItems bound_long;                       // its long items, built once per binding
    DevBuf<int32_t> d_seg, d_long_items;        // the long-item table on the device (bound or the chunk's)
    DevBuf<int64_t> d_long_off;
    bool long_bound = false;                    // the device table is bound_long (a chunk's replaces it)

    int apply_options(const JsonOpt& j) override;
};

int bfl_plsi::apply_options(const JsonOpt& j) {
    d = j.integer("d", 20);
    if (d <= 0 || d > 512) BFL_FAIL(BFL_ERR_OPTION, "d must be in [1, 512]");
    vdim = (d + 3) / 4 * 4;
    seed = (uint32_t)j.integer("random_seed", 0);
    deterministic = j.flag("deterministic", false);
    int rc = attach_device();
    if (rc != BFL_OK) return rc;
    if (BFL_OK != d_loss.reserve(1)) return BFL_ERR_CUDA;
    opt_set = true;
    return BFL_OK;
}

namespace {

int grid_for(const bfl_plsi* h, int64_t work, int per_block, int blocks_per_sm) {
    return (int)std::max<int64_t>(1, std::min<int64_t>((work + per_block - 1) / per_block,
                                                       (int64_t)h->num_sms * blocks_per_sm));
}

// zero the accumulator and the row flags (plsi.cc:40-42)
int reset_acc(bfl_plsi* h, cudaStream_t st) {
    BFL_CUDA(cudaMemsetAsync(h->Qacc.p, 0, sizeof(float) * (size_t)h->Q_rows * h->vdim, st));
    BFL_CUDA(cudaMemsetAsync(h->visited.p, 0, (size_t)h->P_rows, st));
    h->rows_done = false;
    return BFL_OK;
}

int alloc_state(bfl_plsi* h) {
    if (BFL_OK != h->Qacc.reserve((size_t)h->Q_rows * h->vdim)) return BFL_ERR_CUDA;
    if (BFL_OK != h->visited.reserve((size_t)h->P_rows)) return BFL_ERR_CUDA;
    if (BFL_OK != h->colpart.reserve((size_t)kColsumBlocks * h->vdim)) return BFL_ERR_CUDA;
    if (BFL_OK != h->colsum.reserve((size_t)h->vdim)) return BFL_ERR_CUDA;
    if (h->deterministic) {
        if (BFL_OK != h->row_loss.reserve((size_t)std::max<int64_t>(1, h->P_rows))) return BFL_ERR_CUDA;
        if (BFL_OK != h->loss_part.reserve((size_t)std::max<int64_t>(1, (h->P_rows + kLossRows - 1) / kLossRows)))
            return BFL_ERR_CUDA;
    }
    return reset_acc(h, h->stream);
}

// The deterministic row pass at 64 < d <= 128 keeps 3 item rows in flight, not 4: with 4, ptxas holds that
// instantiation to 64 registers and spills.  U does not change any sum: group g still takes entries g, g + NG, ...
// in order, so the rows and the loss are those of U = 4 bit for bit.
template <bool kDet>
void launch_em_kernel(int nv4, int grid, const EmArgs& a, cudaStream_t st) {
    if (nv4 <= 1) plsi_em_kernel<1, 1, 2, kDet><<<grid, 256, 0, st>>>(a);
    else if (nv4 <= 2) plsi_em_kernel<2, 1, 2, kDet><<<grid, 256, 0, st>>>(a);
    else if (nv4 <= 4) plsi_em_kernel<4, 1, 2, kDet><<<grid, 256, 0, st>>>(a);
    else if (nv4 <= 8) plsi_em_kernel<8, 1, 2, kDet><<<grid, 256, 0, st>>>(a);
    else if (nv4 <= 16) plsi_em_kernel<16, 1, 4, kDet><<<grid, 256, 0, st>>>(a);
    else if (nv4 <= 32) plsi_em_kernel<32, 1, kDet ? 3 : 4, kDet><<<grid, 256, 0, st>>>(a);
    else if (nv4 <= 64) plsi_em_kernel<32, 2, 4, kDet><<<grid, 256, 0, st>>>(a);
    else plsi_em_kernel<32, 4, 2, kDet><<<grid, 256, 0, st>>>(a);
}

// The row pass.  Deterministic mode: no item accumulation, and the loss (when a.loss is set) is the row losses of
// the range summed by the fixed tree of loss_tree_*_kernel (bfl_common.cuh), added into a.loss[0] by one thread.
int launch_em(bfl_plsi* h, EmArgs a, cudaStream_t st) {
    h->rows_done = true;
    if (a.n_rows <= 0) return BFL_OK;
    const int grid = grid_for(h, a.n_rows, 8, 16);
    const int nv4 = h->vdim / 4;
    if (!h->deterministic) {
        a.row_loss = nullptr;
        launch_em_kernel<false>(nv4, grid, a, st);
        BFL_LAUNCHED();
        return BFL_OK;
    }
    a.row_loss = a.loss ? h->row_loss.p : nullptr;
    launch_em_kernel<true>(nv4, grid, a, st);
    BFL_LAUNCHED();
    if (a.loss) {
        const int64_t nblk = (a.n_rows + kLossRows - 1) / kLossRows;
        loss_tree_partial_kernel<1><<<(unsigned)nblk, 256, 0, st>>>(h->row_loss.p, a.n_rows, h->loss_part.p);
        BFL_LAUNCHED();
        loss_tree_final_kernel<1><<<1, 256, 0, st>>>(h->loss_part.p, nblk, a.loss);
        BFL_LAUNCHED();
    }
    return BFL_OK;
}

// uploads a long-item table and sizes the segment partial rows for it
int upload_long(bfl_plsi* h, const LongItems& t, cudaStream_t st) {
    const size_t n_long = t.items.size();
    if (BFL_OK != h->d_long_off.reserve(n_long + 1)) return BFL_ERR_CUDA;
    BFL_CUDA(cudaMemcpyAsync(h->d_long_off.p, t.off.data(), sizeof(int64_t) * (n_long + 1), cudaMemcpyHostToDevice, st));
    if (n_long == 0) return BFL_OK;
    if (BFL_OK != h->d_long_items.reserve(n_long)) return BFL_ERR_CUDA;
    if (BFL_OK != h->d_seg.reserve(t.seg.size())) return BFL_ERR_CUDA;
    if (BFL_OK != h->seg_part.reserve((size_t)t.n_segs() * h->vdim)) return BFL_ERR_CUDA;
    BFL_CUDA(cudaMemcpyAsync(h->d_long_items.p, t.items.data(), sizeof(int32_t) * n_long, cudaMemcpyHostToDevice, st));
    BFL_CUDA(cudaMemcpyAsync(h->d_seg.p, t.seg.data(), sizeof(int32_t) * t.seg.size(), cudaMemcpyHostToDevice, st));
    return BFL_OK;
}

// The item pass over items [a.item_begin, a.item_begin + a.n_items); long items la .. lb - 1 of the uploaded table t
// are the range's.
int launch_items(bfl_plsi* h, ItemArgs a, const LongItems& t, int64_t la, int64_t lb, cudaStream_t st) {
    if (h->rows_done)
        BFL_FAIL(BFL_ERR_STATE, "the item pass must run before the row pass of the same iteration (P is overwritten)");
    if (a.n_items <= 0) return BFL_OK;
    const int64_t s0 = t.off[la], s1 = t.off[lb];
    a.seg = h->d_seg.p + 2 * s0;
    a.n_segs = s1 - s0;
    a.part = h->seg_part.p + s0 * h->vdim;
    a.d = h->d;
    a.vdim = h->vdim;
    const int grid = grid_for(h, a.n_items + a.n_segs, 8, 16);
    const int nv4 = h->vdim / 4;
    if (nv4 <= 1) plsi_item_kernel<1, 1, 2><<<grid, 256, 0, st>>>(a);
    else if (nv4 <= 2) plsi_item_kernel<2, 1, 2><<<grid, 256, 0, st>>>(a);
    else if (nv4 <= 4) plsi_item_kernel<4, 1, 2><<<grid, 256, 0, st>>>(a);
    else if (nv4 <= 8) plsi_item_kernel<8, 1, 2><<<grid, 256, 0, st>>>(a);
    else if (nv4 <= 16) plsi_item_kernel<16, 1, 4><<<grid, 256, 0, st>>>(a);
    else if (nv4 <= 32) plsi_item_kernel<32, 1, 4><<<grid, 256, 0, st>>>(a);
    else if (nv4 <= 64) plsi_item_kernel<32, 2, 4><<<grid, 256, 0, st>>>(a);
    else plsi_item_kernel<32, 4, 2><<<grid, 256, 0, st>>>(a);
    BFL_LAUNCHED();
    if (lb > la) {
        plsi_item_combine_kernel<<<grid_for(h, (lb - la) * h->vdim, 256, 16), 256, 0, st>>>(
            h->seg_part.p, h->d_long_items.p + la, h->d_long_off.p + la, lb - la, h->vdim, a.Qacc);
        BFL_LAUNCHED();
    }
    return BFL_OK;
}

int normalize_rows(bfl_plsi* h, float* P, const uint8_t* visited, float alpha1, cudaStream_t st) {
    const int nv4 = h->vdim / 4;
    const int G = nv4 <= 1 ? 1 : nv4 <= 2 ? 2 : nv4 <= 4 ? 4 : nv4 <= 8 ? 8 : nv4 <= 16 ? 16 : 32;
    const int grid = grid_for(h, h->P_rows, 256 / G, 32);
    switch (G) {
        case 1: plsi_normalize_rows_kernel<1><<<grid, 256, 0, st>>>(P, visited, h->P_rows, h->d, h->vdim, alpha1); break;
        case 2: plsi_normalize_rows_kernel<2><<<grid, 256, 0, st>>>(P, visited, h->P_rows, h->d, h->vdim, alpha1); break;
        case 4: plsi_normalize_rows_kernel<4><<<grid, 256, 0, st>>>(P, visited, h->P_rows, h->d, h->vdim, alpha1); break;
        case 8: plsi_normalize_rows_kernel<8><<<grid, 256, 0, st>>>(P, visited, h->P_rows, h->d, h->vdim, alpha1); break;
        case 16: plsi_normalize_rows_kernel<16><<<grid, 256, 0, st>>>(P, visited, h->P_rows, h->d, h->vdim, alpha1); break;
        default: plsi_normalize_rows_kernel<32><<<grid, 256, 0, st>>>(P, visited, h->P_rows, h->d, h->vdim, alpha1); break;
    }
    BFL_LAUNCHED();
    return BFL_OK;
}

int normalize_cols(bfl_plsi* h, float* Q, float alpha2, cudaStream_t st) {
    const int64_t rpb = std::max<int64_t>(1, (h->Q_rows + kColsumBlocks - 1) / kColsumBlocks);
    const int nblk = (int)((h->Q_rows + rpb - 1) / rpb);
    plsi_colsum_partial_kernel<<<nblk, 256, 0, st>>>(Q, h->Q_rows, h->vdim, rpb, h->colpart.p);
    BFL_LAUNCHED();
    plsi_colsum_final_kernel<<<(h->vdim + 127) / 128, 128, 0, st>>>(h->colpart.p, nblk, h->vdim, h->Q_rows, alpha2,
                                                                     h->colsum.p);
    BFL_LAUNCHED();
    plsi_scale_cols_kernel<<<grid_for(h, h->Q_rows * (h->vdim / 4), 256, 16), 256, 0, st>>>(Q, h->Q_rows, h->d, h->vdim,
                                                                                           alpha2, h->colsum.p);
    BFL_LAUNCHED();
    return BFL_OK;
}

// plsi.cc:108-125: alpha1 /= d, alpha2 /= num_items (in float, as the reference)
int normalize_all(bfl_plsi* h, float alpha1, float alpha2, cudaStream_t st) {
    const float a1 = alpha1 / (float)h->d, a2 = alpha2 / (float)h->Q_rows;
    int rc = normalize_rows(h, h->dP, h->visited.p, a1, st);
    if (rc != BFL_OK) return rc;
    return normalize_cols(h, h->Qacc.p, a2, st);
}

int copy_rows(float* dst, size_t dpitch, const float* src, size_t spitch, int64_t rows, int d, cudaMemcpyKind kind,
              cudaStream_t st) {
    if (rows <= 0) return BFL_OK;
    BFL_CUDA(cudaMemcpy2DAsync(dst, dpitch * sizeof(float), src, spitch * sizeof(float), sizeof(float) * d, (size_t)rows,
                               kind, st));
    return BFL_OK;
}

// holder path: device copies of the caller's [rows x d] arrays, padding columns zeroed
int adopt_host(bfl_plsi* h, float* P, int32_t P_rows, float* Q, int32_t Q_rows) {
    if (!h || !h->opt_set) BFL_FAIL(BFL_ERR_STATE, "init() must succeed before initialize_model()");
    int rc = h->mirror_factors(P, P_rows, Q, Q_rows);
    if (rc != BFL_OK) return rc;
    h->factors_ready = false;
    return alloc_state(h);
}

// Copies one host chunk, major rows [start_x, next_x) of a CSR with global END offsets `indptr`, into the staging
// buffers: the chunk's end offsets preceded by the previous row's end when start_x > 0 (*lead = 1), its keys and
// values.  *beg is the chunk's first global entry.
int stage_chunk(bfl_plsi* h, int64_t start_x, int64_t next_x, const int64_t* indptr, const int32_t* keys,
                const float* vals, int64_t* beg, int64_t* lead) {
    *beg = start_x == 0 ? 0 : indptr[start_x - 1];
    const int64_t n = indptr[next_x - 1] - *beg;
    if (n > 0 && (!keys || !vals)) BFL_FAIL(BFL_ERR_ARG, "null keys / vals");
    cudaStream_t st = h->stream;
    *lead = start_x > 0 ? 1 : 0;
    const int64_t n_ends = next_x - start_x + *lead;
    if (BFL_OK != h->stage_ends.reserve((size_t)n_ends)) return BFL_ERR_CUDA;
    BFL_CUDA(cudaMemcpyAsync(h->stage_ends.p, indptr + start_x - *lead, sizeof(int64_t) * n_ends, cudaMemcpyHostToDevice,
                             st));
    if (n > 0) {
        if (BFL_OK != h->stage_keys.reserve((size_t)n)) return BFL_ERR_CUDA;
        if (BFL_OK != h->stage_vals.reserve((size_t)n)) return BFL_ERR_CUDA;
        BFL_CUDA(cudaMemcpyAsync(h->stage_keys.p, keys, sizeof(int32_t) * n, cudaMemcpyHostToDevice, st));
        BFL_CUDA(cudaMemcpyAsync(h->stage_vals.p, vals, sizeof(float) * n, cudaMemcpyHostToDevice, st));
    }
    return BFL_OK;
}

int download(bfl_plsi* h) {
    int rc = copy_rows(h->hostP, h->d, h->dP, h->vdim, h->P_rows, h->d, cudaMemcpyDeviceToHost, h->stream);
    if (rc != BFL_OK) return rc;
    rc = copy_rows(h->hostQ, h->d, h->dQ, h->vdim, h->Q_rows, h->d, cudaMemcpyDeviceToHost, h->stream);
    if (rc != BFL_OK) return rc;
    BFL_CUDA(cudaStreamSynchronize(h->stream));
    return BFL_OK;
}

}  // namespace

extern "C" {

bfl_plsi_t* bfl_plsi_create(void) { return new (std::nothrow) bfl_plsi(); }

void bfl_plsi_destroy(bfl_plsi_t* h) { delete h; }

int bfl_plsi_init(bfl_plsi_t* h, const char* opt_path) { return init_holder(h, opt_path, true); }

int bfl_plsi_init_json(bfl_plsi_t* h, const char* json_text) { return init_holder(h, json_text, false); }

int bfl_plsi_get_vdim(bfl_plsi_t* h) { return h ? h->vdim : 0; }

int bfl_plsi_initialize_model(bfl_plsi_t* h, float* P, int32_t P_rows, float* Q, int32_t Q_rows) {
    int rc = adopt_host(h, P, P_rows, Q, Q_rows);
    if (rc != BFL_OK) return rc;
    cudaStream_t st = h->stream;
    plsi_init_kernel<<<grid_for(h, (int64_t)P_rows * h->vdim, 256, 16), 256, 0, st>>>(h->dP, P_rows, h->d, h->vdim,
                                                                                      h->seed, 0u);
    BFL_LAUNCHED();
    plsi_init_kernel<<<grid_for(h, (int64_t)Q_rows * h->vdim, 256, 16), 256, 0, st>>>(h->dQ, Q_rows, h->d, h->vdim,
                                                                                      h->seed, 1u);
    BFL_LAUNCHED();
    if (BFL_OK != (rc = normalize_rows(h, h->dP, nullptr, 0.f, st))) return rc;
    if (BFL_OK != (rc = normalize_cols(h, h->dQ, 0.f, st))) return rc;
    if (BFL_OK != (rc = download(h))) return rc;
    h->factors_ready = true;
    return BFL_OK;
}

int bfl_plsi_set_model(bfl_plsi_t* h, float* P, int32_t P_rows, float* Q, int32_t Q_rows) {
    int rc = adopt_host(h, P, P_rows, Q, Q_rows);
    if (rc != BFL_OK) return rc;
    cudaStream_t st = h->stream;
    BFL_CUDA(cudaMemsetAsync(h->dP, 0, sizeof(float) * (size_t)P_rows * h->vdim, st));
    BFL_CUDA(cudaMemsetAsync(h->dQ, 0, sizeof(float) * (size_t)Q_rows * h->vdim, st));
    if (BFL_OK != (rc = copy_rows(h->dP, h->vdim, P, h->d, P_rows, h->d, cudaMemcpyHostToDevice, st))) return rc;
    if (BFL_OK != (rc = copy_rows(h->dQ, h->vdim, Q, h->d, Q_rows, h->d, cudaMemcpyHostToDevice, st))) return rc;
    BFL_CUDA(cudaStreamSynchronize(st));
    h->factors_ready = true;
    return BFL_OK;
}

int bfl_plsi_reset(bfl_plsi_t* h) {
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "initialize_model() must precede reset()");
    int rc = reset_acc(h, h->stream);
    if (rc != BFL_OK) return rc;
    BFL_CUDA(cudaStreamSynchronize(h->stream));
    return BFL_OK;
}

int bfl_plsi_partial_update(bfl_plsi_t* h, int32_t start_x, int32_t next_x, const int64_t* indptr,
                            const int32_t* keys, const float* vals, double* loss) {
    if (loss) *loss = 0.0;
    if (!h || !h->factors_ready || !h->hostP) BFL_FAIL(BFL_ERR_STATE, "initialize_model() must precede partial_update()");
    if (next_x == start_x) return BFL_OK;
    if (start_x < 0 || next_x > h->P_rows || next_x < start_x || !indptr) BFL_FAIL(BFL_ERR_ARG, "bad chunk arguments");
    int64_t beg = 0, lead = 0;
    int rc = stage_chunk(h, start_x, next_x, indptr, keys, vals, &beg, &lead);
    if (rc != BFL_OK) return rc;
    cudaStream_t st = h->stream;
    BFL_CUDA(cudaMemsetAsync(h->d_loss.p, 0, sizeof(double), st));
    EmArgs a;
    a.P = h->dP; a.Q = h->dQ; a.Qacc = h->Qacc.p; a.visited = h->visited.p;
    a.ends = h->stage_ends.p + lead; a.keys = h->stage_keys.p; a.vals = h->stage_vals.p; a.shift = beg;
    a.row_begin = start_x; a.n_rows = next_x - start_x; a.loss = h->d_loss.p; a.d = h->d; a.vdim = h->vdim;
    rc = launch_em(h, a, st);
    if (rc != BFL_OK) return rc;
    double out = 0.0;
    BFL_CUDA(cudaMemcpyAsync(&out, h->d_loss.p, sizeof(double), cudaMemcpyDeviceToHost, st));
    BFL_CUDA(cudaStreamSynchronize(st));   // the staging buffers are reused by the next chunk
    if (loss) *loss = out;
    return BFL_OK;
}

int bfl_plsi_partial_update_items(bfl_plsi_t* h, int32_t start_x, int32_t next_x, const int64_t* indptr,
                                  const int32_t* keys, const float* vals) {
    if (!h || !h->factors_ready || !h->hostP)
        BFL_FAIL(BFL_ERR_STATE, "initialize_model() must precede partial_update_items()");
    if (!h->deterministic) BFL_FAIL(BFL_ERR_STATE, "the item pass needs the deterministic option");
    if (h->rows_done)
        BFL_FAIL(BFL_ERR_STATE, "the item pass must run before the row pass of the same iteration (P is overwritten)");
    if (next_x == start_x) return BFL_OK;
    if (start_x < 0 || next_x > h->Q_rows || next_x < start_x || !indptr) BFL_FAIL(BFL_ERR_ARG, "bad chunk arguments");
    int64_t beg = 0, lead = 0;
    int rc = stage_chunk(h, start_x, next_x, indptr, keys, vals, &beg, &lead);
    if (rc != BFL_OK) return rc;
    cudaStream_t st = h->stream;
    LongItems t;
    t.build(indptr, start_x, next_x);
    if (BFL_OK != (rc = upload_long(h, t, st))) return rc;
    h->long_bound = false;
    ItemArgs a;
    a.P = h->dP; a.Q = h->dQ; a.Qacc = h->Qacc.p;
    a.ends = h->stage_ends.p + lead; a.keys = h->stage_keys.p; a.vals = h->stage_vals.p; a.shift = beg;
    a.item_begin = start_x; a.n_items = next_x - start_x;
    if (BFL_OK != (rc = launch_items(h, a, t, 0, (int64_t)t.items.size(), st))) return rc;
    BFL_CUDA(cudaStreamSynchronize(st));   // the staging buffers are reused by the next chunk
    return BFL_OK;
}

int bfl_plsi_item_segment_len(void) { return (int)kItemSegment; }

int bfl_plsi_normalize(bfl_plsi_t* h, float alpha1, float alpha2) {
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "initialize_model() must precede normalize()");
    int rc = normalize_all(h, alpha1, alpha2, h->stream);
    if (rc != BFL_OK) return rc;
    BFL_CUDA(cudaStreamSynchronize(h->stream));
    return BFL_OK;
}

int bfl_plsi_swap(bfl_plsi_t* h) {
    if (!h || !h->factors_ready || !h->hostP) BFL_FAIL(BFL_ERR_STATE, "initialize_model() must precede swap()");
    // the normalised accumulator becomes the current item matrix; the old one is the next accumulator
    std::swap(h->ownQ.p, h->Qacc.p);
    std::swap(h->ownQ.cap, h->Qacc.cap);
    h->dQ = h->ownQ.p;
    h->rows_done = false;
    return download(h);
}

int bfl_plsi_release(bfl_plsi_t* h) {
    if (!h) BFL_FAIL(BFL_ERR_ARG, "null handle");
    if (h->stream) BFL_CUDA(cudaStreamSynchronize(h->stream));
    h->ownP.release(); h->ownQ.release(); h->Qacc.release(); h->visited.release();
    h->colpart.release(); h->colsum.release();
    h->stage_ends.release(); h->stage_keys.release(); h->stage_vals.release();
    h->row_loss.release(); h->loss_part.release(); h->seg_part.release();
    h->d_seg.release(); h->d_long_items.release(); h->d_long_off.release();
    h->ccsr = CsrBinding();
    h->bound_long = LongItems();
    h->long_bound = false;
    h->rows_done = false;
    h->hostP = h->hostQ = nullptr;
    h->dP = h->dQ = nullptr;
    h->P_rows = h->Q_rows = 0;
    h->factors_ready = false;
    return BFL_OK;
}

int bfl_plsi_bind_factors_device(bfl_plsi_t* h, float* dP, int64_t P_rows, float* dQ, int64_t Q_rows) {
    if (!h || !h->opt_set) BFL_FAIL(BFL_ERR_STATE, "init() must succeed before binding factors");
    int rc = h->borrow_factors(dP, P_rows, dQ, Q_rows);
    if (rc != BFL_OK) return rc;
    rc = alloc_state(h);
    if (rc != BFL_OK) return rc;
    BFL_CUDA(cudaStreamSynchronize(h->stream));
    h->factors_ready = true;
    return BFL_OK;
}

int bfl_plsi_bind_csr_device(bfl_plsi_t* h, const int64_t* d_indptr, const int32_t* d_keys, const float* d_vals,
                             int64_t rows, int64_t nnz) {
    if (!h || !h->opt_set) BFL_FAIL(BFL_ERR_STATE, "init() must precede bind_csr");
    return h->csr.bind(d_indptr, d_keys, d_vals, rows, nnz, true);
}

int bfl_plsi_update_device(bfl_plsi_t* h, int64_t row_begin, int64_t row_end, double* d_loss, void* stream) {
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "factors not bound");
    if (!h->csr.indptr) BFL_FAIL(BFL_ERR_STATE, "no device CSR bound");
    if (h->csr.rows != h->P_rows) BFL_FAIL(BFL_ERR_STATE, "the bound CSR and P disagree on the number of rows");
    int rc = h->csr.check_range(row_begin, row_end);
    if (rc != BFL_OK) return rc;
    EmArgs a;
    a.P = h->dP; a.Q = h->dQ; a.Qacc = h->Qacc.p; a.visited = h->visited.p;
    a.ends = h->csr.indptr + row_begin; a.keys = h->csr.keys; a.vals = h->csr.vals; a.shift = 0;
    a.row_begin = row_begin; a.n_rows = row_end - row_begin; a.loss = d_loss; a.d = h->d; a.vdim = h->vdim;
    return launch_em(h, a, (cudaStream_t)stream);
}

int bfl_plsi_normalize_device(bfl_plsi_t* h, float alpha1, float alpha2, void* stream) {
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "factors not bound");
    return normalize_all(h, alpha1, alpha2, (cudaStream_t)stream);
}

int bfl_plsi_swap_device(bfl_plsi_t* h, void* stream) {
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "factors not bound");
    cudaStream_t st = (cudaStream_t)stream;
    BFL_CUDA(cudaMemcpyAsync(h->dQ, h->Qacc.p, sizeof(float) * (size_t)h->Q_rows * h->vdim, cudaMemcpyDeviceToDevice, st));
    return reset_acc(h, st);
}

int bfl_plsi_bind_colwise_csr_device(bfl_plsi_t* h, const int64_t* d_indptr, const int32_t* d_keys,
                                     const float* d_vals, int64_t rows, int64_t nnz) {
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "factors must be bound before the colwise CSR");
    if (!h->deterministic) BFL_FAIL(BFL_ERR_STATE, "the colwise CSR serves the deterministic option only");
    if (rows != h->Q_rows) BFL_FAIL(BFL_ERR_ARG, "the colwise CSR must have Q_rows rows");
    int rc = h->ccsr.bind(d_indptr, d_keys, d_vals, rows, nnz, true);
    if (rc != BFL_OK) return rc;
    // the long-item table, from a host copy of the END offsets
    std::vector<int64_t> ends((size_t)rows);
    BFL_CUDA(cudaMemcpyAsync(ends.data(), d_indptr, sizeof(int64_t) * (size_t)rows, cudaMemcpyDeviceToHost, h->stream));
    BFL_CUDA(cudaStreamSynchronize(h->stream));
    h->bound_long.build(ends.data(), 0, rows);
    if (BFL_OK != (rc = upload_long(h, h->bound_long, h->stream))) return rc;
    BFL_CUDA(cudaStreamSynchronize(h->stream));
    h->long_bound = true;
    return BFL_OK;
}

int bfl_plsi_update_items_device(bfl_plsi_t* h, int64_t item_begin, int64_t item_end, void* stream) {
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "factors not bound");
    if (!h->deterministic) BFL_FAIL(BFL_ERR_STATE, "the item pass needs the deterministic option");
    if (!h->ccsr.indptr) BFL_FAIL(BFL_ERR_STATE, "no colwise CSR bound");
    if (h->ccsr.rows != h->Q_rows) BFL_FAIL(BFL_ERR_STATE, "the bound colwise CSR and Q disagree on the number of rows");
    int rc = h->ccsr.check_range(item_begin, item_end);
    if (rc != BFL_OK) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (!h->long_bound) {
        if (BFL_OK != (rc = upload_long(h, h->bound_long, st))) return rc;
        h->long_bound = true;
    }
    const std::vector<int32_t>& li = h->bound_long.items;
    const int64_t la = std::lower_bound(li.begin(), li.end(), (int32_t)item_begin) - li.begin();
    const int64_t lb = std::lower_bound(li.begin(), li.end(), (int32_t)item_end) - li.begin();
    ItemArgs a;
    a.P = h->dP; a.Q = h->dQ; a.Qacc = h->Qacc.p;
    a.ends = h->ccsr.indptr + item_begin; a.keys = h->ccsr.keys; a.vals = h->ccsr.vals; a.shift = 0;
    a.item_begin = item_begin; a.n_items = item_end - item_begin;
    return launch_items(h, a, h->bound_long, la, lb, st);
}

int bfl_plsi_fold_in_device(bfl_plsi_t* h, const float* d_Q, int64_t Q_rows, const int64_t* d_indptr,
                            const int32_t* d_keys, const float* d_vals, int64_t rows, int64_t nnz, float* d_X, int iters,
                            float alpha1, void* stream) {
    if (!h || !h->opt_set) BFL_FAIL(BFL_ERR_STATE, "init() must succeed before fold_in");
    if (rows < 0 || nnz < 0 || Q_rows <= 0 || iters < 1) BFL_FAIL(BFL_ERR_ARG, "bad fold_in sizes (rows, nnz, Q_rows, iters)");
    if (rows == 0) return BFL_OK;
    if (!d_Q || !d_indptr || !d_X || (nnz > 0 && (!d_keys || !d_vals))) BFL_FAIL(BFL_ERR_ARG, "null fold_in argument");
    if (((uintptr_t)d_Q | (uintptr_t)d_X) & 15) BFL_FAIL(BFL_ERR_ARG, "d_Q and d_X must be 16-byte aligned");
    FoldArgs a;
    a.Q = d_Q; a.ends = d_indptr; a.keys = d_keys; a.vals = d_vals; a.X = d_X; a.n_rows = rows;
    a.iters = iters; a.d = h->d; a.vdim = h->vdim;
    a.a1 = alpha1 / (float)h->d;                                   // normalize_all's alpha1 /= d
    const int grid = grid_for(h, rows, 8, 16);
    const int nv4 = h->vdim / 4;
    cudaStream_t st = (cudaStream_t)stream;
    // (G, NV, U) of plsi_em_kernel's default instantiations; U, the item rows in flight per group, changes no sum
    if (nv4 <= 1) plsi_fold_in_kernel<1, 1, 2><<<grid, 256, 0, st>>>(a);
    else if (nv4 <= 2) plsi_fold_in_kernel<2, 1, 2><<<grid, 256, 0, st>>>(a);
    else if (nv4 <= 4) plsi_fold_in_kernel<4, 1, 2><<<grid, 256, 0, st>>>(a);
    else if (nv4 <= 8) plsi_fold_in_kernel<8, 1, 2><<<grid, 256, 0, st>>>(a);
    else if (nv4 <= 16) plsi_fold_in_kernel<16, 1, 3><<<grid, 256, 0, st>>>(a);   // U = 4 spills 4 bytes here
    else if (nv4 <= 32) plsi_fold_in_kernel<32, 1, 4><<<grid, 256, 0, st>>>(a);
    else if (nv4 <= 64) plsi_fold_in_kernel<32, 2, 4><<<grid, 256, 0, st>>>(a);
    else plsi_fold_in_kernel<32, 4, 2><<<grid, 256, 0, st>>>(a);
    BFL_LAUNCHED();
    return BFL_OK;
}

}  // extern "C"
