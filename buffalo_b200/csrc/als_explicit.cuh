// Explicit-matrix iALS++ row solve for rows whose matrix  S = sum_c w_c q_c q_c^T  and vectors  b = sum_c w_c q_c,
// sum_c q_c, sum_c w_c  were accumulated in global memory by the split-row (PARTIAL) mode of the tensor-core kernel
// (als_tc.cuh).  Same algebra as that kernel's epilogue (lib/algo_impl/als/als.cc:268-352 with Yui_c == x.q_c):
//   M = G + reg I + S;  h = M x - b;  for each 32-column block B: 3-step CG on M[B,B] delta = h[B], x[B] -= delta,
//   h[later] -= M[later, B] delta.
// One CTA of D threads per row; thread j owns column j of the (symmetric) matrix, so every global read of a matrix
// row is coalesced across the CTA.
// DET: the row's loss terms are reduced inside each warp, added across the CTA's warps in warp order and stored at
// loss[2 row] (AlsArgs::loss) instead of being added to loss[0 .. 2) with atomics.
#pragma once
#include "als_generic.cuh"
#include "bfl_common.cuh"

namespace bfl {

struct ExplicitArgs {
    AlsArgs a;              // row_list[row_begin..row_end): the long rows, scratch slot i for list entry row_begin + i
    const float* scratch;   // per slot: D*D matrix, D (b), D (sum q), 4 (sum w, pad)
};

template <int D, bool DET = false>
__global__ void __launch_bounds__(D) als_explicit_solve_kernel(ExplicitArgs ea) {
    static_assert(D % 32 == 0 && D <= 256, "d % 32 == 0, d <= 256");
    const AlsArgs& a = ea.a;
    __shared__ float xs[D];
    __shared__ float pv[32];
    __shared__ float dl[2][32];
    __shared__ int badf[D / 32];
    __shared__ double lred[DET ? D / 32 : 1][2];
    const int j = threadIdx.x, lane = j & 31, q = j >> 5;
    const size_t SF = (size_t)D * D + 2 * D + 4;
    double l_nume = 0.0, l_deno = 0.0;
    for (int64_t it = blockIdx.x; it < a.row_end - a.row_begin; it += gridDim.x) {
        const int row = a.row_list[a.row_begin + it];
        const int64_t beg = row == 0 ? 0 : a.indptr[row - 1];
        const int64_t n = a.indptr[row] - beg;
        const float* Ms = ea.scratch + (size_t)it * SF;
        const float bj = Ms[(size_t)D * D + j];
        const float xj = a.X[(int64_t)row * a.ld + j];
        __syncthreads();   // previous row's readers of xs are done
        xs[j] = xj;
        __syncthreads();
        float hG = 0.f, hD = 0.f;
#pragma unroll 4
        for (int i = 0; i < D; ++i) {
            const float xi = xs[i];
            hD = fmaf(Ms[(size_t)i * D + j], xi, hD);
            hG = fmaf(__ldg(a.G + (size_t)i * D + j), xi, hG);
        }
        hG = fmaf(a.reg, xj, hG);
        if (a.compute_loss) {
            const float kappa = a.adaptive_reg ? (float)n : 1.0f;
            double t = (double)(kappa * a.reg * xj * xj);
            if (a.axis == 1) {
                const float sq = Ms[(size_t)D * D + D + j], ws = Ms[(size_t)D * D + 2 * D];
                t += (double)xj * (double)(hG - a.reg * xj) + (double)xj * (double)hD -
                     2.0 * (double)xj * ((double)bj + (double)sq);
                if (j == 0) {
                    t += (double)n + (double)ws;
                    l_deno += (double)a.Y_rows + (double)ws;
                }
            }
            l_nume += t;
            if (DET) {
                l_nume = warp_sum_d(l_nume);
                l_deno = warp_sum_d(l_deno);
                if (lane == 0) {
                    lred[q][0] = l_nume;
                    lred[q][1] = l_deno;
                }
                l_nume = l_deno = 0.0;
            }
        }
        float h = hG + hD - bj;
        const float tol = a.tol;
#pragma unroll 1
        for (int B = 0; B < D / 32; ++B) {
            if (q == B) {
                float md[32];
#pragma unroll
                for (int i = 0; i < 32; ++i)
                    md[i] = Ms[(size_t)(B * 32 + i) * D + j] + __ldg(a.G + (size_t)(B * 32 + i) * D + j) +
                            (i == lane ? a.reg : 0.f);
                float r = h, p = h, xv = 0.f;
                float rsold = warp_sum(r * r);
                bool act = rsold > tol;
#pragma unroll 1
                for (int step = 0; step < 3; ++step) {
                    pv[lane] = p;
                    __syncwarp();
                    float a0 = 0.f, a1 = 0.f;
#pragma unroll
                    for (int i = 0; i < 32; i += 2) {
                        a0 = fmaf(md[i], pv[i], a0);
                        a1 = fmaf(md[i + 1], pv[i + 1], a1);
                    }
                    __syncwarp();
                    const float Ap = a0 + a1;
                    const float pAp = warp_sum(p * Ap);
                    const float ss = act ? __fdividef(rsold, pAp) : 0.f;
                    xv = fmaf(ss, p, xv);
                    r = fmaf(-ss, Ap, r);
                    const float rsnew = warp_sum(r * r);
                    act = act && !(rsnew < tol);
                    if (act) p = fmaf(__fdividef(rsnew, rsold), p, r);
                    rsold = act ? rsnew : rsold;
                }
                dl[B & 1][lane] = xv;
                xs[j] -= xv;
            }
            __syncthreads();
            if (q > B) {
                float u = 0.f;
#pragma unroll 8
                for (int i = 0; i < 32; ++i)
                    u = fmaf(Ms[(size_t)(B * 32 + i) * D + j] + __ldg(a.G + (size_t)(B * 32 + i) * D + j), dl[B & 1][i], u);
                h -= u;
            }
        }
        float v = xs[j];
        const bool badw = __any_sync(FULL, !isfinite(v));
        if (lane == 0) badf[q] = badw;
        __syncthreads();
        bool bad = false;
#pragma unroll
        for (int w = 0; w < D / 32; ++w) bad |= badf[w] != 0;
        v = bad ? 0.f : v;
        if (DET && a.loss && a.compute_loss && j == 0) {   // lred: written before the block loop's barriers
            double sn = lred[0][0], sd = lred[0][1];
#pragma unroll
            for (int w = 1; w < D / 32; ++w) {
                sn += lred[w][0];
                sd += lred[w][1];
            }
            a.loss[2 * (int64_t)row] = sn;
            a.loss[2 * (int64_t)row + 1] = sd;
        }
        a.X[(int64_t)row * a.ld + j] = v;
        for (int pr = 0; pr < a.n_peer; ++pr) a.peerX[pr][(int64_t)row * a.ld + j] = v;
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

}  // namespace bfl
