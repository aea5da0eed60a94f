// Tuned iALS++ row-solve kernel for sm_90a (the d >= 128 path, lib/algo_impl/als/als.cc:211-358, and any
// d % 32 == 0, d <= 256, with block_size 32).
//
// Work decomposition
//   * rows are binned by length; a TEAM of W warps (W = 1..16) owns one row at a time, a CTA of 16 warps
//     holds 16/W teams, the grid is persistent (one CTA per SM) and strides over the class's row list;
//   * inside a warp the lane id splits as lane = b + 4*a: `a` (0..7) selects an nnz inside a tile of 32
//     gathered rows (slots a, a+8, a+16, a+24), `b` (0..3) selects 8 of the 32 columns of the current
//     column block (the four b-lanes of a row are adjacent lanes, so a 128-bit gather touches few lines).  A
//     lane therefore holds a 4 x 8 register patch of the tile and every per-nnz operation of the block solve
//     (q.p dot, axpy into the block vector) is pure register FMA work:
//        - a dot product over the block's 32 columns finishes with 2 shuffles (over b),
//        - a tile's contribution to a 32-vector finishes with a 7-shuffle transposed reduction (over a)
//          that leaves column 8b + a in lane (a, b);
//   * the Yui pass streams the gathered opposite-factor rows with two 128-bit loads per slot and block straight
//     into registers; the block passes are fed by lane-private cp.async staging of the next block's 128-byte
//     segments (L2 hits) and keep K tiles per warp in registers for the whole block (b, 3 CG steps, Yui update)
//     when the row fits the team (n <= 32*W*K); the long-row class keeps a third tile in its staging cells and
//     rows beyond that re-gather per pass;
//   * the dense terms x.G[:,blk] and A p are expressed as extra "pseudo-nnz" tiles whose rows come from the
//     Gram matrix (in shared memory for d <= 128, through L1/L2 above), distributed over the team's warps;
//   * per-row state (x, Yui, alpha*v, keys) lives in shared memory; every warp contributes its tiles' partial
//     of a team-wide 32-vector, the team's first warp (the solver) adds the partials up, runs the CG scalar
//     recurrences and publishes the next direction -- two named barriers per reduction, no replicated algebra
//     (the shuffles and shared-memory reads of that algebra, not the FMAs, are what the team kernels are bound by).
#pragma once
#include <algorithm>
#include <map>

#include "als_explicit.cuh"
#include "als_generic.cuh"
#include "als_tc.cuh"
#include "bfl_common.cuh"

namespace bfl {

constexpr int FAST_WARPS = 16;   // 512 threads x 128 registers: two register tiles per warp (fewer warps per row = less redundant work)
constexpr int FAST_THREADS = FAST_WARPS * 32;
constexpr int FAST_NCLASS = 8;
constexpr int FAST_NR_CAP = 12288;  // longest row the non-resident class accepts (smem for Yui/w/keys)

// class -> (W, K, resident, max nnz)
struct FastClass { int W, K, res, cap; };
__host__ __device__ inline FastClass fast_class(int c) {
    switch (c) {
        case 0: return {1, 1, 1, 32};
        case 1: return {1, 2, 1, 64};
        case 2: return {2, 2, 1, 128};
        case 3: return {4, 2, 1, 256};
        case 4: return {8, 2, 1, 512};
        case 5: return {16, 3, 1, 1536};  // 2 register tiles + 1 shared-memory tile per warp
        case 6: return {16, 1, 0, FAST_NR_CAP};
        default: return {0, 0, 0, 0x7fffffff};  // class 7: too long for the tuned kernels -> generic kernel
    }
}
__host__ __device__ inline int fast_class_of(int64_t n) {
    if (n <= 32) return 0;
    if (n <= 64) return 1;
    if (n <= 128) return 2;
    if (n <= 256) return 3;
    if (n <= 512) return 4;
    if (n <= 1536) return 5;
    if (n <= FAST_NR_CAP) return 6;
    return 7;
}

// ---- binning ------------------------------------------------------------------------------
// long_regather: rows of 513..1536 nnz are sent to the re-gathering class (6) instead of the staged class (5)
__host__ __device__ inline int fast_route(int64_t n, int long_regather) {
    const int c = fast_class_of(n);
    return (long_regather && c == 5) ? 6 : c;
}

__global__ void fast_count_kernel(const int64_t* __restrict__ indptr, int64_t row_begin, int64_t row_end,
                                  unsigned int* __restrict__ counts, int long_regather) {
    __shared__ unsigned int c[FAST_NCLASS];
    if (threadIdx.x < FAST_NCLASS) c[threadIdx.x] = 0;
    __syncthreads();
    for (int64_t r = row_begin + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < row_end;
         r += (int64_t)gridDim.x * blockDim.x) {
        const int64_t n = indptr[r] - (r == 0 ? 0 : indptr[r - 1]);
        if (n > 0) atomicAdd(&c[fast_route(n, long_regather)], 1u);
    }
    __syncthreads();
    if (threadIdx.x < FAST_NCLASS && c[threadIdx.x]) atomicAdd(counts + threadIdx.x, c[threadIdx.x]);
}

__global__ void fast_fill_kernel(const int64_t* __restrict__ indptr, int64_t row_begin, int64_t row_end,
                                 unsigned int* __restrict__ cursors, int32_t* __restrict__ lists, int long_regather) {
    for (int64_t r = row_begin + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < row_end;
         r += (int64_t)gridDim.x * blockDim.x) {
        const int64_t n = indptr[r] - (r == 0 ? 0 : indptr[r - 1]);
        if (n > 0) {
            const unsigned int pos = atomicAdd(cursors + fast_route(n, long_regather), 1u);
            lists[pos] = (int32_t)r;
        }
    }
}

// ---- device helpers -------------------------------------------------------------------------
template <int W>
__device__ __forceinline__ void team_sync(int team) {
    if (W == 1) {
        __syncwarp();
    } else {
        asm volatile("bar.sync %0, %1;" ::"r"(team + 1), "r"(32 * W) : "memory");
    }
}

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 lds4(const float* p) { return *reinterpret_cast<const float4*>(p); }

// fp32 pairs: d = a * b + c on both halves (sm_90 has no packed fp32 FMA; two FFMAs, same rounding)
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
    return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }

// a lane's 8 columns as 4 packed pairs
struct V8 { float2 v[4]; };

__device__ __forceinline__ V8 v8_zero() {
    V8 r;
#pragma unroll
    for (int k = 0; k < 4; ++k) r.v[k] = make_float2(0.f, 0.f);
    return r;
}
__device__ __forceinline__ V8 v8_from(float4 lo, float4 hi) {
    V8 r;
    r.v[0] = make_float2(lo.x, lo.y); r.v[1] = make_float2(lo.z, lo.w);
    r.v[2] = make_float2(hi.x, hi.y); r.v[3] = make_float2(hi.z, hi.w);
    return r;
}
__device__ __forceinline__ V8 v8_lds(const float* p) { return v8_from(lds4(p), lds4(p + 4)); }
__device__ __forceinline__ V8 v8_ldg(const float* p) { return v8_from(ldg4(p), ldg4(p + 4)); }
__device__ __forceinline__ float v8_dot(const V8& q, const V8& x) {
    float2 s = fmul2(q.v[0], x.v[0]);
#pragma unroll
    for (int k = 1; k < 4; ++k) s = ffma2(q.v[k], x.v[k], s);
    return s.x + s.y;
}
__device__ __forceinline__ void v8_axpy(V8& acc, float cf, const V8& q) {
    const float2 c2 = make_float2(cf, cf);
#pragma unroll
    for (int k = 0; k < 4; ++k) acc.v[k] = ffma2(c2, q.v[k], acc.v[k]);
}

// sum of the 8 a-lanes' acc for column b*8+k; lane (a,b) ends up with column b*8 + a (the a-lanes sit 4 apart)
__device__ __forceinline__ float transposed_reduce8(const V8& acc, int la) {
    const bool h4 = la & 4, h2 = la & 2, h1 = la & 1;
    // first step (a bit 2): keep one float4 half, send the other
    const float2 s0 = h4 ? acc.v[0] : acc.v[2], s1 = h4 ? acc.v[1] : acc.v[3];
    const float2 k0 = h4 ? acc.v[2] : acc.v[0], k1 = h4 ? acc.v[3] : acc.v[1];
    float2 v0, v1;
    v0.x = k0.x + __shfl_xor_sync(FULL, s0.x, 16);
    v0.y = k0.y + __shfl_xor_sync(FULL, s0.y, 16);
    v1.x = k1.x + __shfl_xor_sync(FULL, s1.x, 16);
    v1.y = k1.y + __shfl_xor_sync(FULL, s1.y, 16);
    // second step (a bit 1)
    const float2 s = h2 ? v0 : v1, k = h2 ? v1 : v0;
    float2 u;
    u.x = k.x + __shfl_xor_sync(FULL, s.x, 8);
    u.y = k.y + __shfl_xor_sync(FULL, s.y, 8);
    // last step
    return (h1 ? u.y : u.x) + __shfl_xor_sync(FULL, h1 ? u.x : u.y, 4);
}

// finish a block dot over the 4 b-lanes (lane bits 0,1)
__device__ __forceinline__ float sum_over_b(float s) {
    s += __shfl_xor_sync(FULL, s, 1);
    s += __shfl_xor_sync(FULL, s, 2);
    return s;
}

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// dynamic smem layout:
//   [GSM ? Gs[D*(D+4)] : -] | staging: 16 warps x (K+KS)*8 chunks x 32 lanes x 16 B (RES only) |
//   per team: xs[D] red[2*W*32] pvec[32] (W*32 reserved) dl[32] (96 reserved) yui[cap] wv[cap] ks[cap]
__host__ __device__ inline size_t fast_team_floats(int D, int W, int cap) { return (size_t)D + 96 * W + 96 + 3 * (size_t)cap; }
__host__ __device__ inline size_t fast_smem_bytes(int D, int W, int K, int KS, bool res, bool gsm, int cap) {
    return sizeof(float) * ((gsm ? (size_t)D * (D + 4) : 0) + (res ? (size_t)FAST_WARPS * (K + KS) * 8 * 128 : 0) +
                            (FAST_WARPS / W) * fast_team_floats(D, W, cap));
}

// W warps per row, K register-resident tiles per warp, KS extra tiles per warp kept in shared memory,
// RES=false: nothing resident, every pass re-gathers (rows longer than 32*W*(K+KS)); GSM: Gram matrix in smem.
// DET: a row's loss terms are reduced inside each warp of the team (the lanes' terms come from a fixed tile -> lane map),
// added across the team's warps in warp order and stored at loss[2 row] (AlsArgs::loss), instead of atomics on loss[0 .. 2).
template <int W, int K, int KS, bool RES, bool GSM, bool DET = false>
__global__ void __launch_bounds__(FAST_THREADS, 1) als_ialspp_team_kernel(AlsArgs a, int cap) {
    extern __shared__ __align__(16) float smem[];
    constexpr int TEAMS = FAST_WARPS / W;
    constexpr int KT = K + KS;
    const int D = a.D, ld = a.ld, GP = GSM ? D + 4 : D, NB = D >> 5;
    const int tid = threadIdx.x, lane = tid & 31;
    // broadcast through lane 0 so the compiler knows the warp index (and everything derived from it: team, row
    // loop, trip counts) is warp-uniform; otherwise every shuffle below is compiled as a WARPSYNC.COLLECTIVE call
    const int warp = __shfl_sync(FULL, tid >> 5, 0);
    const int team = warp / W, wt = warp % W;
    // lane = b + 4*a: the four column-group lanes of one gathered row are ADJACENT lanes, so a quarter-warp of a
    // 128-bit gather touches 2 cache lines (not 8) -- the L1/LSU wavefront count of the gathers drops 4x
    const int la = lane >> 2, lb = lane & 3;
    const int mycol = lb * 8 + la;   // the column of the 32-vector this lane owns after a transposed reduction
    float* Gs = smem;
    float* stg_all = smem + (GSM ? (size_t)D * (D + 4) : 0);
    float* stg = stg_all + (size_t)warp * KT * 8 * 128;      // [KT*8 chunks][32 lanes][4 floats]
    float* tb = stg_all + (RES ? (size_t)FAST_WARPS * KT * 8 * 128 : 0) + (size_t)team * fast_team_floats(D, W, cap);
    float* xs = tb;
    float* red = xs + D;                 // [2][W][32]
    float* pvec = red + 64 * W;          // the CG direction, published by the solver warp
    float* dl = red + 96 * W;            // the block's solution delta
    float* yui = red + 96 * W + 96;
    float* wv = yui + cap;
    int32_t* ks = reinterpret_cast<int32_t*>(wv + cap);
    const float* Gp = GSM ? Gs : a.G;    // pseudo-nnz rows come from smem or (long-row class) from L1/L2

    if (GSM) {
        for (int e = tid * 4; e < D * D; e += FAST_THREADS * 4) {
            const float4 g = ldg4(a.G + e);
            const int r = e / D, c = e - r * D;
            *reinterpret_cast<float4*>(Gs + r * GP + c) = g;
        }
        __syncthreads();
    }

    double l_nume = 0.0, l_deno = 0.0;
    const float tol = a.tol;
    // Team-wide sum of one 32-vector (one element per lane), deterministic (fixed warp order): every warp stores its
    // partial, and after a team barrier the solver warp (wt == 0) adds them up.
    // W <= 2: red[w][lane].  W >= 4: partials grouped by four warps, red[w/4][lane][w%4], so that the solver
    // collects the W partials with W/4 128-bit loads (the scalar store is a 4-way bank conflict, once per warp).
    auto store_partial = [&](float v) {
        if (W == 1) return;
        if (W >= 4) red[((wt >> 2) * 32 + lane) * 4 + (wt & 3)] = v;
        else red[wt * 32 + lane] = v;
    };
    auto solver_total = [&](float v) -> float {
        if (W == 1) return v;
        float tot = 0.f;
        if (W >= 4) {
#pragma unroll
            for (int g = 0; g < W / 4; ++g) {
                const float4 p4 = lds4(red + (g * 32 + lane) * 4);
                tot += (p4.x + p4.y) + (p4.z + p4.w);
            }
        } else {
#pragma unroll
            for (int w = 0; w < W; ++w) tot += red[w * 32 + lane];
        }
        return tot;
    };
    const int64_t stride = (int64_t)gridDim.x * TEAMS;

    // issue the async copies of this lane's patch of column block B; reg_tiles / smem_tiles select the tiles.  The
    // staging cells of a register tile are free as soon as the block has read them back, those of a shared-memory
    // tile only after the block's last pass.
    auto stage_block = [&](int B, int ntiles, bool reg_tiles, bool smem_tiles) {
#pragma unroll
        for (int kk = 0; kk < KT; ++kk) {
            if (kk < K ? !reg_tiles : !smem_tiles) continue;
            const int t = wt + kk * W;
            if (kk < K || t < ntiles) {   // register tiles: always (padded slots gather a valid row, weight 0)
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float* src = a.Y + (int64_t)ks[t * 32 + la + 8 * i] * ld + B * 32 + lb * 8;
                    float* dst = stg + ((kk * 4 + i) * 2) * 128 + lane * 4;
                    cp_async16(dst, src);
                    cp_async16(dst + 128, src + 4);
                }
            }
        }
        cp_async_commit();
    };

    for (int64_t ri = a.row_begin + (int64_t)blockIdx.x * TEAMS + team; ri < a.row_end; ri += stride) {
        const int row = __shfl_sync(FULL, a.row_list[ri], 0);
        const int64_t beg = row == 0 ? 0 : a.indptr[row - 1];
        const int n = __shfl_sync(FULL, (int)(a.indptr[row] - beg), 0);
        const int ntiles = (n + 31) >> 5;
        float* xrow = a.X + (int64_t)row * ld;
        team_sync<W>(team);  // the previous row's readers are done with the team's smem
        {
            const int32_t k0 = a.keys[beg - a.shift];
            const int npad = RES ? cap : ntiles * 32;
            for (int c = wt * 32 + lane; c < npad; c += 32 * W) {
                const bool ok = c < n;
                ks[c] = ok ? a.keys[beg - a.shift + c] : k0;          // padded slots gather a valid row ...
                wv[c] = ok ? a.vals[beg - a.shift + c] * a.alpha : 0.f;  // ... with weight 0
                if (!ok) yui[c] = 0.f;
            }
        }
        for (int j = wt * 32 + lane; j < D; j += 32 * W) xs[j] = xrow[j];
        team_sync<W>(team);
        if (RES) stage_block(0, ntiles, true, true);   // block 0's segments fly while the Yui pass streams the rows

        // ---- Yui = x . q_c over all D columns (als.cc:256-266), loss pieces with the pre-update row ----
        for (int t = wt; t < ntiles; t += W) {
            float2 part2[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) part2[i] = make_float2(0.f, 0.f);
            const float* rowp[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) rowp[i] = a.Y + (int64_t)ks[t * 32 + la + 8 * i] * ld + lb * 8;
            for (int B = 0; B < NB; ++B) {
                V8 q0[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) q0[i] = v8_ldg(rowp[i] + B * 32);
                const V8 x0 = v8_lds(xs + B * 32 + lb * 8);
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int k = 0; k < 4; ++k) part2[i] = ffma2(q0[i].v[k], x0.v[k], part2[i]);
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float dot = sum_over_b(part2[i].x + part2[i].y);
                const int slot = t * 32 + la + 8 * i;
                if (lb == 0 && slot < n) {
                    yui[slot] = dot;
                    if (a.compute_loss && a.axis == 1) {  // als.cc:310-315
                        const float av = wv[slot];
                        l_nume += -(double)(dot * dot) + (double)((dot - 1.f) * (dot - 1.f)) * (1.0 + (double)av);
                        l_deno += (double)av;
                    }
                }
            }
        }
        // pull the next row's gathered rows towards L2 while this row is being solved
        if (W <= 8 && ri + stride < a.row_end) {   // long rows: the in-flight working set already fills L2
            const int64_t row2 = a.row_list[ri + stride];
            const int64_t beg2 = row2 == 0 ? 0 : a.indptr[row2 - 1];
            const int n2 = (int)(a.indptr[row2] - beg2);
            for (int c = wt * 32 + lane; c < n2 * NB; c += 32 * W) {
                const int s2 = c / NB, l2 = c - s2 * NB;
                prefetch_l2(a.Y + (int64_t)a.keys[beg2 - a.shift + s2] * ld + l2 * 32);
            }
        }
        if (a.compute_loss) {
            // reg * kappa * |x|^2 (als.cc:319-321) and, item side, x G x (als.cc:298-301); team-strided over j
            float xx = 0.f, xgx = 0.f;
            for (int j = wt * 32 + lane; j < D; j += 32 * W) {
                const float xj = xs[j];
                xx += xj * xj;
                if (a.axis == 1) {
                    float s = 0.f;
                    for (int k = 0; k < D; ++k) s = fmaf(xs[k], Gp[k * GP + j], s);
                    xgx += xj * s;
                }
            }
            xx = warp_sum(xx);
            xgx = warp_sum(xgx);
            if (lane == 0) {
                l_nume += (double)((a.adaptive_reg ? (float)n : 1.0f) * a.reg * xx);
                if (a.axis == 1) {
                    l_nume += (double)xgx;
                    if (wt == 0) l_deno += (double)a.Y_rows;
                }
            }
            if (DET && a.loss) {
                l_nume = warp_sum_d(l_nume);
                l_deno = warp_sum_d(l_deno);
                if (lane == 0) {
                    if (W == 1) {
                        a.loss[2 * (int64_t)row] = l_nume;
                        a.loss[2 * (int64_t)row + 1] = l_deno;
                    } else {   // [W][2] doubles in the half of `red` that no partial uses
                        double* lred = reinterpret_cast<double*>(red + 32 * W);
                        lred[2 * wt] = l_nume;
                        lred[2 * wt + 1] = l_deno;
                    }
                }
            }
            if (DET) l_nume = l_deno = 0.0;
        }
        team_sync<W>(team);
        if (DET && W > 1 && a.compute_loss && a.loss && wt == 0 && lane == 0) {   // rewritten only after this row's later barriers
            const double* lred = reinterpret_cast<const double*>(red + 32 * W);
            double sn = lred[0], sd = lred[1];
#pragma unroll
            for (int w = 1; w < W; ++w) {
                sn += lred[2 * w];
                sd += lred[2 * w + 1];
            }
            a.loss[2 * (int64_t)row] = sn;
            a.loss[2 * (int64_t)row + 1] = sd;
        }

        // ---- column blocks (als.cc:268-352) ----
        for (int B = 0; B < NB; ++B) {
            const int col0 = B * 32 + lb * 8;
            V8 q[K][4];
            if (RES) {
                cp_async_wait_all();   // each lane reads back only what it copied itself: no barrier needed
#pragma unroll
                for (int kk = 0; kk < K; ++kk)
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const float* src = stg + ((kk * 4 + i) * 2) * 128 + lane * 4;
                        q[kk][i] = v8_from(lds4(src), lds4(src + 128));
                    }
                if (B + 1 < NB) stage_block(B + 1, ntiles, true, false);   // prefetch the next block behind the math
            }
            // per-pass visitor over this warp's tiles: register tiles, smem-resident tiles, or re-gathered tiles
            auto for_tiles = [&](auto&& body) {
                if (RES) {
#pragma unroll
                    for (int kk = 0; kk < K; ++kk) body(wt + kk * W, q[kk]);   // branch-free: padding has weight 0
#pragma unroll
                    for (int kk = K; kk < KT; ++kk) {
                        const int t = wt + kk * W;
                        if (t < ntiles) {
                            V8 qs[4];
#pragma unroll
                            for (int i = 0; i < 4; ++i) {
                                const float* src = stg + ((kk * 4 + i) * 2) * 128 + lane * 4;
                                qs[i] = v8_from(lds4(src), lds4(src + 128));
                            }
                            body(t, qs);
                        }
                    }
                } else {
                    for (int t = wt; t < ntiles; t += W) {
                        V8 qs[4];
#pragma unroll
                        for (int i = 0; i < 4; ++i) qs[i] = v8_ldg(a.Y + (int64_t)ks[t * 32 + la + 8 * i] * ld + col0);
                        body(t, qs);
                    }
                }
            };

            // b = x G[:,blk] + reg x_blk + sum (Yui - 1) v a q_blk   (als.cc:296,303-308)
            V8 acc = v8_zero();
            for_tiles([&](int t, const V8(&qq)[4]) {
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int slot = t * 32 + la + 8 * i;
                    v8_axpy(acc, (yui[slot] - 1.0f) * wv[slot], qq[i]);
                }
            });
            for (int pt = 0; pt < NB; ++pt) {  // pseudo tiles: rows of G[:, blk], coefficient x_i
                if ((W - 1 - (pt % W)) != wt) continue;
#pragma unroll
                for (int m = 0; m < 4; ++m) {
                    const int i = pt * 32 + la + 8 * m;
                    v8_axpy(acc, xs[i], GSM ? v8_lds(Gp + i * GP + col0) : v8_ldg(Gp + i * GP + col0));
                }
            }
            const float gpart = transposed_reduce8(acc, la);
            store_partial(gpart);
            team_sync<W>(team);

            // ---- 3 CG steps on (A + sum v a q q^T) delta = g, A = G[blk,blk] + reg I (als.cc:278,324-345) ----
            // The reference skips the solve when rsold <= tol and leaves the loop when rsnew < tol (als.cc:329,341).
            // Here the three steps always run and those conditions only mask the updates: identical results, no
            // data-dependent branch around the shuffles / team barriers.  The recurrences live in the solver warp.
            float xv = 0.f, r = 0.f, p = 0.f, rsold = 0.f;
            bool act = false;
            if (wt == 0) {
                const float g = solver_total(gpart) + a.reg * xs[B * 32 + mycol];
                r = g;
                p = g;
                rsold = warp_sum(r * r);
                act = rsold > tol;
                pvec[mycol] = p;
            }
            team_sync<W>(team);
#pragma unroll 1
            for (int step = 0; step < 3; ++step) {
                const V8 pc = v8_lds(pvec + lb * 8);
                acc = v8_zero();
                for_tiles([&](int t, const V8(&qq)[4]) {
                    float dots[4];
#pragma unroll
                    for (int i = 0; i < 4; ++i) dots[i] = v8_dot(qq[i], pc);
#pragma unroll
                    for (int i = 0; i < 4; ++i) dots[i] = sum_over_b(dots[i]);
#pragma unroll
                    for (int i = 0; i < 4; ++i) v8_axpy(acc, wv[t * 32 + la + 8 * i] * dots[i], qq[i]);
                });
                if (wt == W - 1) {  // pseudo tile: rows of G[blk, blk], coefficient p_i
#pragma unroll
                    for (int m = 0; m < 4; ++m) {
                        const int i = la + 8 * m;
                        const float* gr = Gp + (B * 32 + i) * GP + col0;
                        v8_axpy(acc, pvec[i], GSM ? v8_lds(gr) : v8_ldg(gr));
                    }
                }
                const float part = transposed_reduce8(acc, la);
                store_partial(part);
                team_sync<W>(team);   // all partials stored, and everybody has read this step's direction
                if (wt == 0) {
                    const float Ap = solver_total(part) + a.reg * p;
                    const float pAp = warp_sum(p * Ap);
                    // als.cc:337 (no eps): the reference divides a double holding a float by a float and rounds to
                    // float; the fast fp32 division (reciprocal + multiply, <= 2 ulp) is far inside the parity bar
                    const float step_size = act ? __fdividef(rsold, pAp) : 0.f;
                    xv = fmaf(step_size, p, xv);
                    r = fmaf(-step_size, Ap, r);
                    const float rsnew = warp_sum(r * r);
                    act = act && !(rsnew < tol);                          // als.cc:341
                    if (act) p = fmaf(__fdividef(rsnew, rsold), p, r);   // predicated update
                    rsold = act ? rsnew : rsold;
                    if (step < 2) {
                        pvec[mycol] = p;
                    } else {   // x_blk -= delta (als.cc:346)
                        dl[mycol] = xv;
                        xs[B * 32 + mycol] -= xv;
                    }
                }
                team_sync<W>(team);   // the next direction (or the block's delta) is published
            }
            // ---- Yui -= q_blk . delta  (als.cc:347-350) ----
            const V8 xc = v8_lds(dl + lb * 8);
            if (B + 1 < NB) {   // Yui is not read again after the last block
                for_tiles([&](int t, const V8(&qq)[4]) {
                    float dots[4];
#pragma unroll
                    for (int i = 0; i < 4; ++i) dots[i] = v8_dot(qq[i], xc);
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const float dot = sum_over_b(dots[i]);
                        if (lb == 0) yui[t * 32 + la + 8 * i] -= dot;
                    }
                });
            }
            if (RES && KS > 0 && B + 1 < NB) stage_block(B + 1, ntiles, false, true);   // smem-resident tiles are free only now
            __syncwarp();   // the next block reads Yui slots written by other lanes of this warp
        }
        // NaN/Inf guard (cf. als.cu:116-120), then write the row back
        bool bad = false;
        for (int j = lane; j < D; j += 32) bad |= !isfinite(xs[j]);
        bad = __any_sync(FULL, bad);
        for (int j = wt * 32 + lane; j < D; j += 32 * W) {
            const float v = bad ? 0.f : xs[j];
            xrow[j] = v;
            // fused exchange: the same 128-byte segments go straight into the peers' replicas over NVLink
            for (int pr = 0; pr < a.n_peer; ++pr) a.peerX[pr][(int64_t)row * ld + j] = v;
        }
    }
    if (!DET && a.loss && a.compute_loss) {
        l_nume = warp_sum_d(l_nume);
        l_deno = warp_sum_d(l_deno);
        if (lane == 0 && (l_nume != 0.0 || l_deno != 0.0)) {
            atomicAdd(a.loss, l_nume);
            atomicAdd(a.loss + 1, l_deno);
        }
    }
}

// ---- host side --------------------------------------------------------------------------------
struct FastBins {
    DevBuf<int32_t> lists;           // all classes back to back
    DevBuf<unsigned int> counters;   // [0..7] counts, [8..15] cursors
    unsigned int count[FAST_NCLASS] = {0};
    unsigned int offset[FAST_NCLASS + 1] = {0};
    // split-row work items of class 7 (rows beyond FAST_NR_CAP): triples (row, chunk, slot), see als_tc.cuh
    DevBuf<int32_t> items;
    DevBuf<unsigned long long> item_counter;
    int64_t n_items = -1;
    int items_split_class = -1;
    // deterministic mode: items in list order; END offsets of the list rows' chunks (device and host) and the batches
    // (list row bounds) of the last scratch budget
    bool items_det = false;
    DevBuf<long long> chunk_end;
    std::vector<long long> h_chunk_end;
    std::vector<int64_t> det_batches;
    size_t det_batches_budget = 0;
};
// nnz per chunk of a split row.  The tensor core's fp32 accumulator truncates (measured: -0.5 ulp per accumulating MMA on
// average, 3 MMAs per 8 entries => ~1.1e-5 relative after 1000 entries), so no accumulator is allowed to run longer
// than ~2000 entries: longer rows are summed from 2048-entry partial matrices with ordinary rounded fp32 adds.
constexpr int64_t TC_SPLIT = 2048;
struct FastBinKey {
    const void* indptr; int64_t b, e;
    bool operator<(const FastBinKey& o) const {
        if (indptr != o.indptr) return indptr < o.indptr;
        if (b != o.b) return b < o.b;
        return e < o.e;
    }
};
struct FastCache {
    std::map<FastBinKey, FastBins*> bins;
    DevBuf<float> scratch;   // partial matrices of the split rows (als_tc.cuh PARTIAL mode), one slot per row
    // deterministic mode: one slot per chunk of the batch in flight; budget in bytes for a batch's chunk + row slots
    // (0: a quarter of the free device memory at first use, at most 2 GiB)
    DevBuf<float> chunk_scratch;
    size_t det_budget = 0;
    void clear() {
        for (auto& kv : bins) delete kv.second;
        bins.clear();
    }
    ~FastCache() { clear(); }
};

inline bool fast_als_applicable(int optimizer_code, int d, int vdim, int block_size) {
    // d <= 128: the Gram matrix lives in shared memory; 128 < d <= 256: it is read through L1/L2 (GSM = false)
    return optimizer_code == 8 && d % 32 == 0 && d <= 256 && vdim == d && block_size == 32;
}

template <int W, int K, int KS, bool RES, bool GSM, bool DET = false>
int fast_launch_class(const AlsArgs& a, int cap, int num_sms, cudaStream_t st) {
    const size_t smem = fast_smem_bytes(a.D, W, K, KS, RES, GSM, cap);
    constexpr int SMEM_MAX = 227 * 1024;
    // per device/context attribute: set it on every launch (a process may drive several GPUs)
    BFL_CUDA(cudaFuncSetAttribute(als_ialspp_team_kernel<W, K, KS, RES, GSM, DET>,
                                  cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_MAX));
    if (smem > (size_t)SMEM_MAX) BFL_FAIL(BFL_ERR_STATE, "tuned ALS kernel: shared memory budget exceeded");
    const int64_t nrows = a.row_end - a.row_begin;
    constexpr int TEAMS = FAST_WARPS / W;
    const int grid = (int)std::min<int64_t>((nrows + TEAMS - 1) / TEAMS, (int64_t)num_sms);
    als_ialspp_team_kernel<W, K, KS, RES, GSM, DET><<<grid, FAST_THREADS, smem, st>>>(a, cap);
    BFL_LAUNCHED();
    return BFL_OK;
}
// det_loss: a.loss takes per-row terms (the DET instantiation)
template <int W, int K, int KS, bool RES, bool GSM>
int fast_launch_class(const AlsArgs& a, int cap, int num_sms, cudaStream_t st, bool det_loss) {
    return det_loss ? fast_launch_class<W, K, KS, RES, GSM, true>(a, cap, num_sms, st)
                    : fast_launch_class<W, K, KS, RES, GSM>(a, cap, num_sms, st);
}

// explicit-matrix solve of the rows list[0 .. nrows) from their row slots scratch[0 .. nrows); det_loss: a0.loss takes
// per-row terms (the DET instantiation)
inline int launch_explicit_solve(const AlsArgs& a0, const int32_t* list, int64_t nrows, const float* scratch, bool det_loss,
                                 int num_sms, cudaStream_t st) {
    ExplicitArgs ea;
    ea.a = a0;
    ea.a.row_list = list;
    ea.a.row_begin = 0;
    ea.a.row_end = nrows;
    ea.scratch = scratch;
    const int ge = (int)std::min<int64_t>(nrows, (int64_t)num_sms * 4);
    if (a0.D == 128) {
        if (det_loss) als_explicit_solve_kernel<128, true><<<ge, 128, 0, st>>>(ea);
        else als_explicit_solve_kernel<128><<<ge, 128, 0, st>>>(ea);
    } else {
        if (det_loss) als_explicit_solve_kernel<256, true><<<ge, 256, 0, st>>>(ea);
        else als_explicit_solve_kernel<256><<<ge, 256, 0, st>>>(ea);
    }
    BFL_LAUNCHED();
    return BFL_OK;
}

// Deterministic split rows: the long rows list7[0 .. n7) in batches of whole rows whose chunk and row slots fit the
// budget (a batch always takes at least one row).  Per batch: chunk matrices by plain stores, the ordered sum of each
// row's chunks, the explicit-matrix solve.  The items follow list7, so the chunks of list row i are the items
// first[i] .. first[i] + nc_i of an exclusive scan; list7 itself is filled through fast_fill_kernel's atomic cursor, so
// the item order, the slot of a chunk and the batch bounds differ between handles.  No bit depends on them: a row is
// summed on its own in chunk order and its loss terms are stored by row.  Scratch that cannot be allocated is an error.
template <int D>
int fast_split_rows_det(const AlsArgs& a0, FastCache& cache, FastBins* fb, const int32_t* list7, int64_t n7,
                        int split_min_class, bool det_loss, int num_sms, cudaStream_t st) {
    if (fb->n_items < 0 || fb->items_split_class != split_min_class || !fb->items_det) {
        const int g7 = (int)std::min<int64_t>((n7 + 127) / 128, 1024);
        if (BFL_OK != fb->chunk_end.reserve((size_t)n7)) return BFL_ERR_CUDA;
        tc::tc_chunk_counts_kernel<<<g7, 128, 0, st>>>(a0.indptr, list7, n7, TC_SPLIT, fb->chunk_end.p);
        BFL_LAUNCHED();
        int rc = inclusive_scan_i64(fb->chunk_end.p, fb->chunk_end.p, n7, st);
        if (rc != BFL_OK) return rc;
        fb->h_chunk_end.resize((size_t)n7);
        BFL_CUDA(cudaMemcpyAsync(fb->h_chunk_end.data(), fb->chunk_end.p, sizeof(long long) * (size_t)n7, cudaMemcpyDeviceToHost, st));
        BFL_CUDA(cudaStreamSynchronize(st));
        const long long total = fb->h_chunk_end.back();
        if (BFL_OK != fb->items.reserve(3 * (size_t)total)) return BFL_ERR_CUDA;
        tc::tc_fill_items_scanned_kernel<<<g7, 128, 0, st>>>(list7, n7, fb->chunk_end.p, fb->items.p);
        BFL_LAUNCHED();
        fb->n_items = (int64_t)total;
        fb->items_split_class = split_min_class;
        fb->items_det = true;
        fb->det_batches.clear();
    }
    const size_t sf = tc::scratch_floats<D>(), sfb = sf * sizeof(float);
    if (!cache.det_budget) {
        size_t free_b = 0, total_b = 0;
        BFL_CUDA(cudaMemGetInfo(&free_b, &total_b));
        cache.det_budget = std::max<size_t>(std::min<size_t>(free_b / 4, (size_t)2 << 30), 2 * sfb);
    }
    const long long* ce = fb->h_chunk_end.data();
    if (fb->det_batches.empty() || fb->det_batches_budget != cache.det_budget) {
        fb->det_batches.assign(1, 0);
        size_t used = 0;
        for (int64_t i = 0; i < n7; ++i) {
            const size_t cost = (size_t)(ce[i] - (i ? ce[i - 1] : 0) + 1) * sfb;
            if (used && used + cost > cache.det_budget) {
                fb->det_batches.push_back(i);
                used = 0;
            }
            used += cost;
        }
        fb->det_batches.push_back(n7);
        fb->det_batches_budget = cache.det_budget;
    }
    int64_t max_rows = 0, max_chunks = 0;
    for (size_t b = 0; b + 1 < fb->det_batches.size(); ++b) {
        const int64_t i = fb->det_batches[b], j = fb->det_batches[b + 1];
        max_rows = std::max(max_rows, j - i);
        max_chunks = std::max<int64_t>(max_chunks, ce[j - 1] - (i ? ce[i - 1] : 0));
    }
    if (BFL_OK != cache.scratch.reserve(sf * (size_t)max_rows) || BFL_OK != cache.chunk_scratch.reserve(sf * (size_t)max_chunks))
        BFL_FAIL(BFL_ERR_CUDA, "deterministic ALS: cannot allocate the split-row scratch (" +
                                   std::to_string((sfb * (size_t)(max_rows + max_chunks)) >> 20) +
                                   " MB); lower _b200_det_scratch_mb or free device memory");
    const int nf4 = (int)((a0.compute_loss && a0.axis == 1 ? sf : (size_t)D * D + D) / 4);
    for (size_t b = 0; b + 1 < fb->det_batches.size(); ++b) {
        const int64_t i = fb->det_batches[b], j = fb->det_batches[b + 1];
        const int64_t chunk0 = i ? ce[i - 1] : 0, nchunks = ce[j - 1] - chunk0;
        int rc = tc::tc_launch_partial<D>(a0, fb->items.p + 3 * chunk0, nchunks, cache.chunk_scratch.p, nchunks, TC_SPLIT,
                                          num_sms, st, true);
        if (rc != BFL_OK) return rc;
        for (int64_t r = i; r < j; r += 65535) {   // grid.y limit
            const dim3 grid((nf4 + 255) / 256, (unsigned)std::min<int64_t>(65535, j - r));
            tc::tc_chunk_reduce_kernel<<<grid, 256, 0, st>>>(cache.chunk_scratch.p, fb->chunk_end.p, r, chunk0, sf, nf4,
                                                             cache.scratch.p + (size_t)(r - i) * sf);
            BFL_LAUNCHED();
        }
        rc = launch_explicit_solve(a0, list7 + i, j - i, cache.scratch.p, det_loss, num_sms, st);
        if (rc != BFL_OK) return rc;
    }
    return BFL_OK;
}

// bins rows [row_begin,row_end) of a.indptr by length (cached per (indptr,row range)) and launches one
// kernel per non-empty class; class 7 (n > FAST_NR_CAP) is returned to the caller through `leftover`.
// Tensor-core kernel (als_tc.cuh): classes tc_min_class .. split_min_class-1 are solved by ONE fused launch over their
// contiguous part of the binned list; classes >= split_min_class (rows of any length) go through the split-row mode
// (chunk matrices summed in global memory + explicit-matrix solve).  FAST_NCLASS disables either.
inline int fast_als_launch(const AlsArgs& a0, FastCache& cache, int num_sms, cudaStream_t st,
                           const int32_t** leftover_rows, int64_t* leftover_count, int tc_min_class, int split_min_class,
                           int long_regather = 0, bool det = false) {
    // deterministic mode: split rows through fast_split_rows_det, and the kernels that store per-row loss terms
    const bool det_loss = det && a0.loss && a0.compute_loss;
    *leftover_rows = nullptr;
    *leftover_count = 0;
    const int64_t nrows = a0.row_end - a0.row_begin;
    FastBinKey key{a0.indptr, a0.row_begin, a0.row_end};
    FastBins* fb = nullptr;
    auto it = cache.bins.find(key);
    if (it == cache.bins.end()) {
        if (cache.bins.size() >= 256) cache.clear();
        fb = new FastBins();
        if (BFL_OK != fb->lists.reserve((size_t)nrows) || BFL_OK != fb->counters.reserve(2 * FAST_NCLASS)) {
            delete fb;
            return BFL_ERR_CUDA;
        }
        BFL_CUDA(cudaMemsetAsync(fb->counters.p, 0, 2 * FAST_NCLASS * sizeof(unsigned int), st));
        const int grid = (int)std::min<int64_t>((nrows + 255) / 256, (int64_t)num_sms * 8);
        fast_count_kernel<<<grid, 256, 0, st>>>(a0.indptr, a0.row_begin, a0.row_end, fb->counters.p, long_regather);
        BFL_LAUNCHED();
        BFL_CUDA(cudaMemcpyAsync(fb->count, fb->counters.p, FAST_NCLASS * sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
        BFL_CUDA(cudaStreamSynchronize(st));
        fb->offset[0] = 0;
        for (int c = 0; c < FAST_NCLASS; ++c) fb->offset[c + 1] = fb->offset[c] + fb->count[c];
        BFL_CUDA(cudaMemcpyAsync(fb->counters.p + FAST_NCLASS, fb->offset, FAST_NCLASS * sizeof(unsigned int),
                                 cudaMemcpyHostToDevice, st));
        fast_fill_kernel<<<grid, 256, 0, st>>>(a0.indptr, a0.row_begin, a0.row_end, fb->counters.p + FAST_NCLASS,
                                               fb->lists.p, long_regather);
        BFL_LAUNCHED();
        cache.bins[key] = fb;
    } else {
        fb = it->second;
    }
    tc_min_class = std::min(tc_min_class, split_min_class);
    const bool has_split = split_min_class < FAST_NCLASS && fb->offset[FAST_NCLASS] > fb->offset[split_min_class];
    if (has_split && det) {
        const int64_t n7 = fb->offset[FAST_NCLASS] - fb->offset[split_min_class];
        const int32_t* list7 = fb->lists.p + fb->offset[split_min_class];
        const int rc = a0.D == 128
                           ? fast_split_rows_det<128>(a0, cache, fb, list7, n7, split_min_class, det_loss, num_sms, st)
                           : fast_split_rows_det<256>(a0, cache, fb, list7, n7, split_min_class, det_loss, num_sms, st);
        if (rc != BFL_OK) return rc;
    }
    if (has_split && !det) {
        // long rows (any length): cut into chunks spread over the SMs, partial matrices summed in global memory, then the
        // explicit-matrix solve
        const int64_t n7 = fb->offset[FAST_NCLASS] - fb->offset[split_min_class];
        const int32_t* list7 = fb->lists.p + fb->offset[split_min_class];
        if (fb->n_items < 0 || fb->items_split_class != split_min_class) {
            if (BFL_OK != fb->item_counter.reserve(2)) return BFL_ERR_CUDA;
            BFL_CUDA(cudaMemsetAsync(fb->item_counter.p, 0, 2 * sizeof(unsigned long long), st));
            const int g7 = (int)std::min<int64_t>((n7 + 127) / 128, 1024);
            tc::tc_count_items_kernel<<<g7, 128, 0, st>>>(a0.indptr, list7, n7, TC_SPLIT, fb->item_counter.p);
            BFL_LAUNCHED();
            unsigned long long total = 0;
            BFL_CUDA(cudaMemcpyAsync(&total, fb->item_counter.p, sizeof(total), cudaMemcpyDeviceToHost, st));
            BFL_CUDA(cudaStreamSynchronize(st));
            if (BFL_OK != fb->items.reserve(3 * (size_t)total)) return BFL_ERR_CUDA;
            tc::tc_fill_items_kernel<<<g7, 128, 0, st>>>(a0.indptr, list7, n7, TC_SPLIT, fb->item_counter.p + 1, fb->items.p);
            BFL_LAUNCHED();
            fb->n_items = (int64_t)total;
            fb->items_split_class = split_min_class;
        }
        const size_t sf = a0.D == 128 ? tc::scratch_floats<128>() : tc::scratch_floats<256>();
        if (BFL_OK != cache.scratch.reserve(sf * (size_t)n7)) return BFL_ERR_CUDA;
        int rc = a0.D == 128
                     ? tc::tc_launch_partial<128>(a0, fb->items.p, fb->n_items, cache.scratch.p, n7, TC_SPLIT, num_sms, st)
                     : tc::tc_launch_partial<256>(a0, fb->items.p, fb->n_items, cache.scratch.p, n7, TC_SPLIT, num_sms, st);
        if (rc != BFL_OK) return rc;
        rc = launch_explicit_solve(a0, list7, n7, cache.scratch.p, false, num_sms, st);
        if (rc != BFL_OK) return rc;
    }
    if (tc_min_class < split_min_class && fb->offset[split_min_class] > fb->offset[tc_min_class]) {
        AlsArgs a = a0;
        a.row_list = fb->lists.p;
        a.row_begin = fb->offset[tc_min_class];
        a.row_end = fb->offset[split_min_class];
        const int rc = tc::tc_launch(a, num_sms, st, det_loss);
        if (rc != BFL_OK) return rc;
    }
    for (int c = 0; c < std::min(FAST_NCLASS - 1, tc_min_class); ++c) {
        if (!fb->count[c]) continue;
        AlsArgs a = a0;
        a.row_list = fb->lists.p;
        a.row_begin = fb->offset[c];
        a.row_end = fb->offset[c + 1];
        const FastClass fc = fast_class(c);
        int rc = BFL_OK;
        const bool gsm = a.D <= 128;   // d x (d+4) floats of Gram fit next to the staging buffers only up to d = 128
        switch (c) {
            case 0: rc = gsm ? fast_launch_class<1, 1, 0, true, true>(a, fc.cap, num_sms, st, det_loss)
                             : fast_launch_class<1, 1, 0, true, false>(a, fc.cap, num_sms, st, det_loss); break;
            case 1: rc = gsm ? fast_launch_class<1, 2, 0, true, true>(a, fc.cap, num_sms, st, det_loss)
                             : fast_launch_class<1, 2, 0, true, false>(a, fc.cap, num_sms, st, det_loss); break;
            case 2: rc = gsm ? fast_launch_class<2, 2, 0, true, true>(a, fc.cap, num_sms, st, det_loss)
                             : fast_launch_class<2, 2, 0, true, false>(a, fc.cap, num_sms, st, det_loss); break;
            case 3: rc = gsm ? fast_launch_class<4, 2, 0, true, true>(a, fc.cap, num_sms, st, det_loss)
                             : fast_launch_class<4, 2, 0, true, false>(a, fc.cap, num_sms, st, det_loss); break;
            case 4: rc = gsm ? fast_launch_class<8, 2, 0, true, true>(a, fc.cap, num_sms, st, det_loss)
                             : fast_launch_class<8, 2, 0, true, false>(a, fc.cap, num_sms, st, det_loss); break;
            case 5: rc = fast_launch_class<16, 2, 1, true, false>(a, fc.cap, num_sms, st, det_loss); break;
            case 6: rc = gsm ? fast_launch_class<16, 1, 0, false, true>(a, fc.cap, num_sms, st, det_loss)
                             : fast_launch_class<16, 1, 0, false, false>(a, fc.cap, num_sms, st, det_loss); break;
        }
        if (rc != BFL_OK) return rc;
    }
    if (split_min_class >= FAST_NCLASS && fb->count[FAST_NCLASS - 1]) {
        *leftover_rows = fb->lists.p + fb->offset[FAST_NCLASS - 1];
        *leftover_count = fb->count[FAST_NCLASS - 1];
    }
    return BFL_OK;
}

}  // namespace bfl
