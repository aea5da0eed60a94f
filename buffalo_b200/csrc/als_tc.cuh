// Tensor-core iALS++ row solve for sm_90a (d = 128, block_size 32): the Hopper-native path of
// lib/algo_impl/als/als.cc:211-358.
//
// Algebra.  With M = G + reg*I + sum_c w_c q_c q_c^T (w = alpha*v) and b = sum_c w_c q_c, the reference's block
// right-hand side (als.cc:296,303-308) is  g_B = (x M)[B] - b[B]  for the CURRENT x (Yui_c == x.q_c at every point of
// its loop), its CG operator (als.cc:278,330-336) is M[B,B], and "p_blk -= x; Yui -= q_blk.x" (als.cc:346-350) keeps
// that invariant.  So one row is: form the explicit d x d matrix once, then run the block Gauss-Seidel sweep with the
// fixed 3-step CG on 32 x 32 diagonal blocks -- O(d^2) work per row that does not depend on the row length, and the
// per-nnz work collapses into one rank-1 update  M += (sqrt(w) q)(sqrt(w) q)^T, a dense contraction: tensor cores.
//
// Precision.  The contraction runs on wgmma (fp16 operands, fp32 accumulator) with a two-term fp16 split of the scaled
// operand t = 2^e sqrt|w| q = head + tail (head: 11 significant bits, tail: the next 11): head.head + head.tail +
// tail.head leaves a relative error of ~2^-21 per product, fp32-grade like the reference's arithmetic, at twice the
// tensor rate and half the shared-memory traffic per entry of the equivalent 3xTF32 scheme (K = 16 per instruction
// instead of 8).  The power of two 2^e (tc_scale_kernel: from max|Y| and max|w| of the launch) places the largest
// operand just below 2^15, so nothing overflows fp16 and entries down to 2^-20 of the largest keep a normal tail; the
// accumulator starts a row at 2^2e (G + reg I) and is multiplied by 2^-2e (exact) when it is read.  b and the loss
// pieces are accumulated in plain fp32 from the unscaled rows.
//
// Pipeline of one persistent CTA (one per SM, 13 warps, warp-specialised, mbarrier hand-offs only, one elected arrival
// per warp; hand-offs are per GROUP of two consecutive tiles of the CTA's tile stream):
//   planner warp     : walks the CTA's rows; every level of the dependent load chain (row id -> offsets -> keys / values)
//                     is issued whole rows ahead of its use; per tile of 32 entries it writes the gather plan (keys,
//                     2^e sqrt|w|, w, count / flags) into a 16-slot ring -- it runs up to 8 groups ahead;
//   4 convert warps  : (a) gathers: one hand-off ahead of its use, warp cw copies the rows cw, cw + 4, ... of a planned
//                     tile with one coalesced 16-byte-per-lane cp.async per 512 bytes (SASS LDGSTS) into a three-stage
//                     ring (commit / wait groups + one mbarrier arrival per warp);
//                     (b) convert: thread = feature m: reads column m of the raw tile (conflict-free), scales, splits,
//                     and writes 16-byte groups of 8 consecutive k into the K-major un-swizzled operand slabs (8 x 16 B
//                     core matrices, conflict-free) over the group's rows in the same stage; accumulates b_m = sum w q_m (exact fp32) and the loss pieces in
//                     registers; groups of two full tiles take a branch-free straight-line path;
//   MMA warpgroup    : executes the generic -> async proxy fence for the group it has acquired, then issues wgmma
//                     (SASS HGMMA) for the two 64-row halves of the row's matrix, accumulating in registers: rows 64..127
//                     over all 128 columns (m64n128k16), rows 0..63 only over columns 0..63 (m64n64k16; the matrix is
//                     symmetric -- split-row chunks accumulate full blocks); entries with negative weight travel in
//                     their own tiles and are subtracted with the negate-A immediate.  At a row's end it waits for the
//                     MMAs, stores 2^-2e x accumulator (and the transpose of rows 64..127 x columns 0..63) into the
//                     shared-memory matrix of the epilogue and starts the next row from the CTA's shared-memory copy of
//                     2^2e (G + reg I);
//   4 epilogue warps : a systolic pipeline over the row's blocks.  Thread j owns matrix row j, warp q column block q:
//                     h = M x - b from the shared matrix; then warp q folds the deltas of blocks 0..q-1 into its h as
//                     they are published, runs the 3-step CG of its own 32 x 32 block and publishes its delta.  Nothing in
//                     a row's sweep is a group-wide barrier, so warp 0 is already waiting for the next row while warp 3
//                     finishes this one; the MMA warpgroup fills the next row's accumulator meanwhile.
// Rows of any length stream through (no per-nnz state), which removes the long-row cliff of the SIMT classes; rows
// longer than the split threshold are cut into chunks whose partial matrices are summed in global memory and solved
// by als_explicit_solve_kernel (als_explicit.cuh).
#pragma once
#include "als_generic.cuh"
#include "bfl_common.cuh"
#include <type_traits>

#include "sm90_ptx.cuh"

namespace bfl {
namespace tc {

using namespace sm90;

// 16 warps = 4 warpgroups: epilogue 0..3 (warp q owns matrix rows 32q..32q+31), MMA 4..7, convert 8..11, planner 12
// (warps 13..15 only hand their registers back).  Launched at 128 registers per thread; setmaxnreg then moves registers
// from the planner's warpgroup to the MMA warpgroup, whose 128 x 128 fp32 accumulator needs 128 of them by itself.  Every
// SM sub-partition runs one warp of each warpgroup, so the four budgets must sum to 4 x 128.
constexpr int N_CONV = 4, KH = N_CONV / 4;
constexpr int W_EPI = 0, W_MMA = 4, W_CONV = 8, W_PLAN = W_CONV + N_CONV;
constexpr int WARPS = 16, THREADS = WARPS * 32;
constexpr int REG_MMA = 200, REG_PLAN = 4 * 128 - 128 - 128 - REG_MMA;   // 56: the planner keeps a few row pointers
constexpr int NXS = 8;     // x buffers of the epilogue pipeline (a fast warp publishes row r + 1 while a slow one reads row r - 3)
// Hand-offs are per GROUP of PT consecutive tiles of the CTA's tile stream (a group may span rows: every tile carries its own
// flags): the barrier round trips of a one-tile hand-off cost as much as the math of a tile.
constexpr int PT = 2;      // tiles per hand-off group
// Ring of stages (groups): a group's gathered fp32 rows and its operand slabs are both 32 KB and share one stage, which
// holds the rows of group g + 1 (being gathered), then group g (converted in place), then group g - 1 (read by wgmma)
constexpr int NS = 3;
constexpr int GATHER_AHEAD = 1;   // groups between a convert warp's gather issue and its use of the group (< NS - 1)
constexpr int NPG = 8, NP = NPG * PT;   // gather-plan ring (small slots): the planner runs up to NPG groups ahead
constexpr int NBV = 8;     // ring of per-row vectors handed from the convert warps to the epilogue
// d = 128: 32 gathered rows per stage; d = 256 (split-row mode only): 16 rows per stage, and the chunk matrix is
// accumulated in three launches (passes) of 128 x 128 blocks: rows / columns 0..127, rows 0..127 x columns 128..255
// (its transpose is the remaining quadrant), rows / columns 128..255
template <int D>
struct Cfg {
    static constexpr int TILE = D == 128 ? 32 : 16;      // gathered rows per stage
    static constexpr int NF = D / 128;                    // features per convert thread
    static constexpr int LBO = D * 16;                    // bytes between the 8-k chunks of an operand slab
    static constexpr int OP_BYTES = TILE * D * 2;         // head (or tail) slab of one stage
};
constexpr uint32_t F_FIRST = 1u << 8, F_LAST = 1u << 9, F_NEG = 1u << 10, F_STOP = 1u << 11;

// column c of the epilogue's matrix is stored as 128 floats, row r at (r ^ msw(c)): the MMA warpgroup's fragment stores
// and the epilogue's reads (thread j reads row j of one column) are both free of bank conflicts
__device__ __forceinline__ int msw(int c) { return ((c >> 1) & 3) << 3; }

// 2^2e (G + reg I) of a fused launch, packed: the 8 x 8 blocks (R, C) with R >= C, block (R, C) at float
// 64 (R (R + 1) / 2 + C), element (r, c) at 8 (r % 8) + c % 8 in it (the diagonal blocks are stored whole)
constexpr int G_FLOATS = 16 * 17 / 2 * 64;
__device__ __forceinline__ int g_block(int R, int C) { return (R * (R + 1) / 2 + C) * 64; }

template <int D>
union Stage {
    // operand slab: element (feature m, entry k) at byte (k/8)*LBO + (m/8)*128 + (m%8)*16 + (k%8)*2
    unsigned char op[PT][2][Cfg<D>::OP_BYTES];        // [tile of the group][head|tail]
    float raw[PT][Cfg<D>::TILE * D];                   // gathered rows, pitch D
};
static_assert(sizeof(Stage<128>::op) == sizeof(Stage<128>::raw) && sizeof(Stage<256>::op) == sizeof(Stage<256>::raw),
              "a group's rows and its slabs fill the same stage");

template <int D>
struct Smem {
    static constexpr int TILE = Cfg<D>::TILE;
    alignas(1024) Stage<D> st[NS];
    alignas(128) float mat[128 * 128];                 // fused mode: M of the row being solved (column-major, msw)
    alignas(16) float g[G_FLOATS];                     // fused mode: 2^2e (G + reg I), loaded once per CTA
    alignas(16) float bvec[NBV][KH][D];                // b = sum w q
    alignas(16) float sumq[NBV][KH][D];                // sum q (loss only)
    alignas(16) float xs[NXS][D];                      // 128-bit reads: every vector below is 16-byte aligned
    alignas(16) float pv[4][32];                       // CG direction of the warp that owns the block
    alignas(16) float dl[4][32];                       // [block]: the block's solution delta
    alignas(16) float sws[NP][TILE];                   // gather plan: 2^e sqrt|w| per slot
    alignas(16) float wv[NP][TILE];                    //              w per slot
    alignas(16) int32_t keys[NP][TILE];                //              gathered row per slot
    float wsum[NBV][KH];                               // sum w (loss only)
    uint32_t meta_raw[NP];                             //              count | flags
    uint32_t meta_op[NS][PT];
    int badrow[NXS];
    // per stage: raw_full (the group's rows have landed), op_full (converted), st_empty (the MMAs are done with it)
    alignas(8) uint64_t plan_full[NPG], plan_empty[NPG], raw_full[NS], op_full[NS], st_empty[NS];
    alignas(8) uint64_t acc_full, acc_empty, x_full[NXS], d_full[4];
};
// deterministic loss of the fused mode: the epilogue warps' terms of a row, handed to the last block's warp
template <int D>
struct SmemDet : Smem<D> {
    double lossp[NXS][4][2];
};
// one CTA per SM: 227 KB of shared memory per block on sm_90
static_assert(sizeof(SmemDet<128>) <= 232448 && sizeof(SmemDet<256>) <= 232448, "shared memory of als_tc_kernel");

// PARTIAL = false: rows of a.row_list[row_begin..row_end) are solved in place.
// PARTIAL = true : the list holds chunk items of long rows (pairs: row, chunk index); the chunk's matrix and vectors are
//                  added to scratch[slot] (slot = items[3*i+2]) and solved later by als_explicit_solve_kernel.
// DET (deterministic mode, separate instantiations):
//   PARTIAL: a scratch slot belongs to a CHUNK (slot = the item's index in this launch) and is written with plain stores;
//            tc_chunk_reduce_kernel then adds the chunk slots of a row in ascending chunk order.  Every element of a chunk
//            slot is stored exactly once, so the slots need no memset:
//              matrix, d = 128 (r0 = c0 = 0): d0 holds rows 0..63, d1 rows 64..127, each over all 128 columns (N0 = 128); a
//                thread's (n, h, i) enumerate distinct (r, c) and the four MMA warps own disjoint rows 16 wq + 0..15 (+ 64);
//              matrix, d = 256: pass 0 stores rows / columns 0..127, pass 2 rows / columns 128..255, pass 1 rows 0..127 x
//                columns 128..255 and (r0 != c0) the mirrored element (c, r) of each, i.e. rows 128..255 x columns 0..127:
//                four disjoint quadrants, each element once;
//              vectors (pass 0 only): b[0..D) and, with LOSS1, sum q[0..D) and the four floats (sum w, 0, 0, 0) by the
//                epilogue thread j (and j + 128 at d = 256).  Without LOSS1 only matrix + b are written, and only those read.
//   fused:   the loss terms of a row are reduced inside each epilogue warp, handed through shared memory along the
//            delta hand-offs (d_full) to the warp of the last block, added there in warp order and stored at loss[2 row].
struct TcArgs {
    AlsArgs a;
    const int32_t* items;   // PARTIAL: triples (row, chunk, scratch slot)
    float* scratch;         // PARTIAL: per slot D*D matrix + D (b) + D (sum q) + 4 (sum w, ...) floats
    int64_t split;          // PARTIAL: chunk length in nnz
    int pass;               // PARTIAL, d = 256: which 128 x 128 block of the chunk matrix this launch accumulates (0..2)
    int debug;              // BFL_TC_DEBUG (timing experiments only; results are wrong): 1 no gathers, 2 no MMAs, 4 no convert math, 8 no epilogue math, 16 planner only,
                            // 32 fused rows start from a zero accumulator instead of 2^2e (G + reg I) (values only: the start is read from shared memory either way)
};

template <int D>
__host__ __device__ constexpr size_t scratch_floats() { return (size_t)D * D + 2 * D + 4; }

// operand scaling of one launch: out[0] = 2^e, out[1] = 2^-2e with 2^e max|Y| sqrt(max|w|) in [2^14, 2^15)
__global__ void tc_absmax_kernel(const float* __restrict__ p, size_t n, unsigned int* __restrict__ out) {
    float m = 0.f;
    const size_t gtid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, gsz = (size_t)gridDim.x * blockDim.x;
    const size_t lead = min(n, (size_t)(((16 - ((uintptr_t)p & 15)) & 15) / 4));   // scalars up to 16-byte alignment
    const size_t n4 = (n - lead) / 4;
    const float4* p4 = reinterpret_cast<const float4*>(p + lead);
    for (size_t i = gtid; i < n4; i += gsz) {
        const float4 v = __ldg(p4 + i);
        m = fmaxf(fmaxf(m, fmaxf(fabsf(v.x), fabsf(v.y))), fmaxf(fabsf(v.z), fabsf(v.w)));
    }
    for (size_t i = gtid; i < lead; i += gsz) m = fmaxf(m, fabsf(p[i]));
    for (size_t i = lead + n4 * 4 + gtid; i < n; i += gsz) m = fmaxf(m, fabsf(p[i]));
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(FULL, m, o));
    // non-negative floats order like their bit patterns (fmaxf drops NaNs; an Inf input ends up as scale 2^-60, the rows
    // it touches come out non-finite and are zeroed by the guard, like the reference's GPU path)
    if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(out, __float_as_uint(m));
}
__global__ void tc_scale_kernel(const unsigned int* __restrict__ ymax, const unsigned int* __restrict__ vmax, float alpha,
                                float* __restrict__ out) {
    const float y = __uint_as_float(*ymax), w = __uint_as_float(*vmax) * fabsf(alpha);
    const float top = y * sqrtf(w);
    int e = 0;
    if (top > 0.f && isfinite(top)) {
        int ex;
        frexpf(top, &ex);          // top = f * 2^ex, f in [0.5, 1)
        e = 15 - ex;               // 2^e top in [2^14, 2^15)
    }
    e = max(-60, min(60, e));
    out[0] = ldexpf(1.f, e);
    out[1] = ldexpf(1.f, -2 * e);
}

// LOSS1: compute_loss on the item axis (the convert warps also hand sum q / sum w to the epilogue); a template parameter so
// that the common case keeps a branch-free convert loop
template <int D, bool PARTIAL, bool LOSS1, bool DET = false>
__global__ void __launch_bounds__(THREADS, 1) als_tc_kernel(TcArgs ta) {
    static_assert(D == 128 || (D == 256 && PARTIAL), "fused row solve: d = 128; split-row mode: d = 128 or 256");
    constexpr int TILE = Cfg<D>::TILE, NF = Cfg<D>::NF, LBO = Cfg<D>::LBO;
    extern __shared__ __align__(1024) unsigned char smem_raw_[];
    Smem<D>& S = *reinterpret_cast<Smem<D>*>(smem_raw_);
    [[maybe_unused]] SmemDet<D>& SD = *reinterpret_cast<SmemDet<D>*>(smem_raw_);   // DET instantiations only
    const AlsArgs& a = ta.a;
    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(FULL, tid >> 5, 0);

    if (tid == 0) {
        for (int i = 0; i < NS; ++i) {
            // every barrier counts WARPS, not threads: an arrive executed by 32 lanes is 32 serial barrier updates
            mbar_init(&S.raw_full[i], N_CONV);
            mbar_init(&S.op_full[i], N_CONV);
            mbar_init(&S.st_empty[i], 4);
        }
        for (int i = 0; i < NPG; ++i) {
            mbar_init(&S.plan_full[i], 1);
            mbar_init(&S.plan_empty[i], N_CONV);
        }
        mbar_init(&S.acc_full, 4);
        mbar_init(&S.acc_empty, 4);
        for (int b = 0; b < 4; ++b) mbar_init(&S.d_full[b], 1);
        for (int i = 0; i < NXS; ++i) {
            mbar_init(&S.x_full[i], 4);
            S.badrow[i] = 0;
        }
        mbar_init_fence();
    }
    const float scale = __ldg(a.tc_scales), inv2 = __ldg(a.tc_scales + 1);
    if (!PARTIAL) {
        // the fused rows' accumulator start, the same fp32 values for every row of the launch.  Only the lower block
        // triangle is kept: G from the Gram kernel is symmetric bit for bit ((i, j) and (j, i) are the same FMAs in the
        // same order)
        const float s2 = scale * scale;
        const bool zero = ta.debug & 32;
        for (int e = tid; e < 128 * 128; e += THREADS) {
            const int r = e >> 7, c = e & 127;
            if ((r >> 3) >= (c >> 3)) {
                float g = zero ? 0.f : __ldg(a.G + e);
                g += r == c && !zero ? a.reg : 0.f;
                S.g[g_block(r >> 3, c >> 3) + 8 * (r & 7) + (c & 7)] = g * s2;
            }
        }
    }
    __syncthreads();

    const int64_t nitems = a.row_end - a.row_begin;
    const int64_t my_first = (int64_t)blockIdx.x;
    const int64_t stride = gridDim.x;

    // item -> (row, first entry, count)
    auto item_info = [&](int64_t it, int& row, int64_t& beg, int64_t& n, int& slot) {
        if (PARTIAL) {
            const int32_t* p = ta.items + 3 * (a.row_begin + it);
            row = p[0];
            const int64_t rb = row == 0 ? 0 : a.indptr[row - 1];
            const int64_t rn = a.indptr[row] - rb;
            beg = rb + (int64_t)p[1] * ta.split;
            n = min(ta.split, rn - (int64_t)p[1] * ta.split);
            slot = DET ? (int)it : p[2];
        } else {
            row = a.row_list[a.row_begin + it];
            beg = row == 0 ? 0 : a.indptr[row - 1];
            n = a.indptr[row] - beg;
            slot = 0;
        }
    };

    if (warp >= W_PLAN) {
        setmaxnreg_dec<REG_PLAN>();
        if (warp != W_PLAN) return;   // nothing after this point waits for the CTA as a whole
        // ================= planner: gather plans =================
        uint32_t gsl = 0, rph = 0, pe = 0;   // group slot, phase of plan_empty, tile within the group
        // begin a tile: its plan slot (the group's slots are claimed when its first tile starts)
        auto tile_begin = [&]() -> uint32_t {
            if (pe == 0) mbar_wait_idle(&S.plan_empty[gsl], rph ^ 1u);
            return gsl * PT + pe;
        };
        // finish a tile (after __syncwarp): the group is published with its last tile
        auto tile_end = [&]() {
            if (++pe == PT) {
                if (lane == 0) mbar_arrive(&S.plan_full[gsl]);
                pe = 0;
                if (++gsl == NPG) { gsl = 0; rph ^= 1u; }
            }
        };
        auto emit = [&](unsigned mask, uint32_t flags, int32_t key, float w) {
            const int cnt = __popc(mask);
            const int slot = __popc(mask & ((1u << lane) - 1u));
            const uint32_t rs = tile_begin();
            if ((mask >> lane) & 1u) {
                S.keys[rs][slot] = key;
                S.sws[rs][slot] = sqrtf(fabsf(w)) * scale;
                S.wv[rs][slot] = w;
            } else {   // the lanes without an entry zero the scale / weight of the unused slots cnt .. TILE-1
                const int zslot = cnt + lane - slot;
                if (zslot < TILE) {
                    S.sws[rs][zslot] = 0.f;
                    S.wv[rs][zslot] = 0.f;
                }
            }
            if (lane == 0) S.meta_raw[rs] = (uint32_t)cnt | flags;
            __syncwarp();
            tile_end();
        };
        // Software pipeline over the CTA's items.  Every level of the dependent load chain  item -> row offsets -> entries
        // is issued whole rows ahead of its use (a gathered tile takes ~700 cycles to issue, a global load ~1-2 thousand
        // cycles under load: with a one-tile look-ahead every tile paid that latency):
        //   item i+4: row id            item i+3: offsets            item i+2: first super-chunk of entries (keys, weights)
        // and inside a long row the next super-chunk (SC tiles) is loaded while the current one is being emitted.
        // The planner is one warp on the critical path of every tile (with all the math switched off the kernel still
        // needed ~1000 cycles per tile for the plan hand-offs alone): inside a row everything is 32-bit, and a super-chunk
        // without negative weights -- the normal case -- takes the short path: slot == lane, no ballots, no prefix sums.
        constexpr int SC = 4, SCN = SC * TILE;
        const bool inl = lane < TILE;
        auto load_id = [&](int64_t it, int& row, int& chunk) {
            row = -1;
            chunk = 0;
            if (it < nitems) {
                if (PARTIAL) {
                    const int32_t* p = ta.items + 3 * (a.row_begin + it);
                    row = p[0];
                    chunk = p[1];
                } else {
                    row = a.row_list[a.row_begin + it];
                }
            }
        };
        auto load_span = [&](int row, int chunk, const int32_t*& kp, const float*& vp, int& n) {
            kp = a.keys;
            vp = a.vals;
            n = 0;
            if (row >= 0) {
                const int64_t rb = row == 0 ? 0 : a.indptr[row - 1];
                const int64_t rn = a.indptr[row] - rb;
                int64_t beg = rb;
                n = (int)rn;            // fused rows are binned below 2^31 entries, chunks are `split` long
                if (PARTIAL) {
                    beg = rb + (int64_t)chunk * ta.split;
                    n = (int)min(ta.split, rn - (int64_t)chunk * ta.split);
                }
                kp = a.keys + (beg - a.shift);
                vp = a.vals + (beg - a.shift);
            }
        };
        auto load_sc = [&](const int32_t* kp, const float* vp, int n, int c0, int32_t (&key)[SC], float (&w)[SC]) {
#pragma unroll
            for (int s = 0; s < SC; ++s) {
                const int idx = c0 + s * TILE + lane;
                const bool ok = inl && idx < n;
                key[s] = ok ? kp[idx] : 0;
                w[s] = ok ? vp[idx] * a.alpha : 0.f;
            }
        };
        auto emit_sc = [&](int n, int c0, const int32_t (&key)[SC], const float (&w)[SC]) {
            bool neg = false;
#pragma unroll
            for (int s = 0; s < SC; ++s) neg |= w[s] < 0.f;
            if (!__any_sync(FULL, neg)) {
#pragma unroll
                for (int s = 0; s < SC; ++s) {
                    const int t0 = c0 + s * TILE;
                    if (t0 < n) {
                        const uint32_t meta = (uint32_t)min(TILE, n - t0) | (t0 == 0 ? F_FIRST : 0u) | (t0 + TILE >= n ? F_LAST : 0u);
                        const uint32_t rs = tile_begin();
                        if (inl) {   // lanes beyond the row's end carry key 0, weight 0: the unused slots are zero-filled
                            float sq;
                            asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(sq) : "f"(w[s]));
                            S.keys[rs][lane] = key[s];
                            S.sws[rs][lane] = sq * scale;
                            S.wv[rs][lane] = w[s];
                        }
                        if (lane == 0) S.meta_raw[rs] = meta;
                        __syncwarp();
                        tile_end();
                    }
                }
            } else {
#pragma unroll
                for (int s = 0; s < SC; ++s) {
                    const int t0 = c0 + s * TILE;
                    if (t0 < n) {
                        const bool valid = inl && t0 + lane < n;
                        const unsigned pm = __ballot_sync(FULL, valid && !(w[s] < 0.f));
                        const unsigned nm = __ballot_sync(FULL, valid && (w[s] < 0.f));
                        const bool lastc = t0 + TILE >= n;
                        uint32_t fl = (t0 == 0 ? F_FIRST : 0u);
                        if (pm) {
                            emit(pm, fl | ((lastc && !nm) ? F_LAST : 0u), key[s], w[s]);
                            fl = 0u;
                        }
                        if (nm) emit(nm, fl | F_NEG | (lastc ? F_LAST : 0u), key[s], w[s]);
                    }
                }
            }
        };
        const int32_t *kp0, *kp1, *kp2, *kp3;
        const float *vp0, *vp1, *vp2, *vp3;
        int n0, n1, n2, n3;
        int row_t, ch_t, row4, ch4;
        int32_t k0[SC], k1[SC], k2[SC], nk[SC];
        float w0[SC], w1[SC], w2[SC], nw[SC];
        load_id(my_first, row_t, ch_t);
        load_span(row_t, ch_t, kp0, vp0, n0);
        load_sc(kp0, vp0, n0, 0, k0, w0);
        load_id(my_first + stride, row_t, ch_t);
        load_span(row_t, ch_t, kp1, vp1, n1);
        load_sc(kp1, vp1, n1, 0, k1, w1);
        load_id(my_first + 2 * stride, row_t, ch_t);
        load_span(row_t, ch_t, kp2, vp2, n2);
        load_id(my_first + 3 * stride, row4, ch4);
        for (int64_t it = my_first; it < nitems; it += stride) {
            // issue the look-ahead loads (their results are first touched one item later)
            load_sc(kp2, vp2, n2, 0, k2, w2);
            load_span(row4, ch4, kp3, vp3, n3);
            load_id(it + 4 * stride, row4, ch4);
            for (int c0 = 0; c0 < n0; c0 += SCN) {
                const bool more = c0 + SCN < n0;
                if (more) load_sc(kp0, vp0, n0, c0 + SCN, nk, nw);
                emit_sc(n0, c0, k0, w0);
                if (more) {
#pragma unroll
                    for (int s = 0; s < SC; ++s) { k0[s] = nk[s]; w0[s] = nw[s]; }
                }
            }
#pragma unroll
            for (int s = 0; s < SC; ++s) { k0[s] = k1[s]; w0[s] = w1[s]; k1[s] = k2[s]; w1[s] = w2[s]; }
            kp0 = kp1; vp0 = vp1; n0 = n1; kp1 = kp2; vp1 = vp2; n1 = n2; kp2 = kp3; vp2 = vp3; n2 = n3;
        }
        // stop marker: fills the rest of the current group (or one more group)
        do {
            const uint32_t rs = tile_begin();
            if (lane == 0) S.meta_raw[rs] = F_STOP;
            __syncwarp();
            tile_end();
        } while (pe != 0);
    } else if (warp >= W_MMA && warp < W_MMA + 4) {
        setmaxnreg_inc<REG_MMA>();
        // ================= MMA warpgroup =================
        // The accumulated block: feature rows [r0, r0 + 128) x feature columns [c0, c0 + 128); d0 holds rows r0 .. r0 + 63,
        // d1 rows r0 + 64 .. r0 + 127 (fragment layout: sm90_ptx.cuh).  Fused mode: the row's matrix is symmetric, so d0
        // only accumulates columns 0 .. 63 (m64n64: a quarter of the tensor-core work and of its shared-memory operand
        // reads saved); its columns 64 .. 127 are the transpose of d1's columns 0 .. 63 and are stored from there.
        const int r0 = (D == 256 && ta.pass == 2) ? 128 : 0, c0 = (D == 256 && ta.pass > 0) ? 128 : 0;
        const int wq = warp - W_MMA;
        const int fr = 16 * wq + (lane >> 2), fc = 2 * (lane & 3);   // fragment row / column of register 0
        constexpr int N0 = PARTIAL ? 128 : 64;                        // columns accumulated in d0
        float d0[N0 / 2], d1[64];
        auto mma0 = [&](auto neg, uint64_t adesc, uint64_t bdesc) {
            constexpr bool NEG = decltype(neg)::value;
            if constexpr (PARTIAL) wgmma_m64n128k16_f16<NEG>(d0, adesc, bdesc);
            else wgmma_m64n64k16_f16<NEG>(d0, adesc, bdesc);
        };
        // A new row's accumulator: 2^2e (G + reg I) in fused mode (so that the epilogue reads one matrix), 0 for chunks.
        // acc_init_nh sets the registers of (n, h): elements (fr + 8 h, 8 n + fc + i) of d0 and (fr + 8 h + 64, ...) of d1,
        // from S.g; an element above the block diagonal is read from its mirror.  The block row of fr is warp-uniform.
        const int rb = 2 * wq;
        const int g_lo = 8 * (lane >> 2) + fc, g_up = 8 * fc + (lane >> 2);   // offsets in a block below / above
        auto g_pair = [&](int R, int C) -> float2 {   // elements (8 R + lane / 4, 8 C + fc + {0, 1})
            const bool low = R >= C;
            const float* p = S.g + (low ? g_block(R, C) + g_lo : g_block(C, R) + g_up);
            return make_float2(p[0], p[low ? 1 : 8]);
        };
        auto acc_init_nh = [&](const int n, const int h) {
            if constexpr (PARTIAL) {
                d0[4 * n + 2 * h] = 0.f; d0[4 * n + 2 * h + 1] = 0.f;
                d1[4 * n + 2 * h] = 0.f; d1[4 * n + 2 * h + 1] = 0.f;
            } else {
                if (8 * n < N0) {
                    const float2 g0 = g_pair(rb + h, n);
                    d0[4 * n + 2 * h] = g0.x; d0[4 * n + 2 * h + 1] = g0.y;
                }
                const float2 g1 = n < 8 ? *reinterpret_cast<const float2*>(S.g + g_block(8 + rb + h, n) + g_lo)
                                        : g_pair(8 + rb + h, n);
                d1[4 * n + 2 * h] = g1.x; d1[4 * n + 2 * h + 1] = g1.y;
            }
        };
        auto acc_init = [&]() {
#pragma unroll
            for (int n = 0; n < 16; ++n)
#pragma unroll
                for (int h = 0; h < 2; ++h) acc_init_nh(n, h);
        };
        uint32_t os = 0, oph = 0, aph = 0;
        int64_t seq = 0;   // rows (items) finished so far
        bool stop = false;
        acc_init();
        while (!stop) {
            mbar_wait(&S.op_full[os], oph);
            fence_proxy_async_smem();   // the convert warps' generic-proxy operand stores -> visible to the tensor core's reads
#pragma unroll 1
            for (int e = 0; e < PT; ++e) {
                const uint32_t meta = S.meta_op[os][e];
                if (meta & F_STOP) {
                    stop = true;
                    break;
                }
                const int ksteps = (ta.debug & 2) ? 0 : (int)(meta & 0xffu);
                const uint32_t hi = s32(&S.st[os].op[e][0][0]), lo = s32(&S.st[os].op[e][1][0]);
                wgmma_fence();
#pragma unroll 1
                for (int ks = 0; ks < ksteps; ++ks) {
                    // K = 16 = two 8-k chunks LBO apart; neighbouring 8-feature core matrices 128 B apart (SBO); the
                    // features f of an operand start f / 8 core matrices into the slab
                    const uint32_t k0 = ks * 2 * LBO;
                    const uint64_t ah0 = smem_desc(hi + k0 + r0 * 16, LBO, 128), ah1 = smem_desc(hi + k0 + (r0 + 64) * 16, LBO, 128);
                    const uint64_t al0 = smem_desc(lo + k0 + r0 * 16, LBO, 128), al1 = smem_desc(lo + k0 + (r0 + 64) * 16, LBO, 128);
                    const uint64_t bh = smem_desc(hi + k0 + c0 * 16, LBO, 128), bl = smem_desc(lo + k0 + c0 * 16, LBO, 128);
                    if (meta & F_NEG) {
                        mma0(std::true_type{}, ah0, bh);
                        mma0(std::true_type{}, ah0, bl);
                        mma0(std::true_type{}, al0, bh);
                        wgmma_m64n128k16_f16<true>(d1, ah1, bh);
                        wgmma_m64n128k16_f16<true>(d1, ah1, bl);
                        wgmma_m64n128k16_f16<true>(d1, al1, bh);
                    } else {
                        mma0(std::false_type{}, ah0, bh);
                        mma0(std::false_type{}, ah0, bl);
                        mma0(std::false_type{}, al0, bh);
                        wgmma_m64n128k16_f16<false>(d1, ah1, bh);
                        wgmma_m64n128k16_f16<false>(d1, ah1, bl);
                        wgmma_m64n128k16_f16<false>(d1, al1, bh);
                    }
                }
                wgmma_commit();
                if (meta & F_LAST) {
                    wgmma_wait<0>();
#pragma unroll
                    for (int i = 0; i < 64; ++i) { if (i < N0 / 2) acc_fence(d0[i]); acc_fence(d1[i]); }
                    mbar_wait_idle(&S.acc_empty, aph ^ 1u);   // the epilogue is done with the previous row
                    if constexpr (PARTIAL) {
                        // the chunk of item my_first + seq * stride; pass 1 of d = 256 also writes the transposed block.
                        // Default: float atomics into the row's slot (the chunks of one row are summed in arrival order);
                        // DET: plain stores into the chunk's own slot
                        const int slot = DET ? (int)(my_first + seq * stride) : ta.items[3 * (a.row_begin + my_first + seq * stride) + 2];
                        float* sc = ta.scratch + (size_t)slot * scratch_floats<D>();
#pragma unroll
                        for (int n = 0; n < 16; ++n)
#pragma unroll
                            for (int h = 0; h < 2; ++h)
#pragma unroll
                                for (int i = 0; i < 2; ++i) {
                                    const int r = r0 + fr + 8 * h, c = c0 + 8 * n + fc + i;
                                    const float v0 = d0[4 * n + 2 * h + i] * inv2, v1 = d1[4 * n + 2 * h + i] * inv2;
                                    if constexpr (DET) {
                                        sc[(size_t)r * D + c] = v0;
                                        sc[(size_t)(r + 64) * D + c] = v1;
                                        if (r0 != c0) {
                                            sc[(size_t)c * D + r] = v0;
                                            sc[(size_t)c * D + r + 64] = v1;
                                        }
                                    } else {
                                        atomicAdd(sc + (size_t)r * D + c, v0);
                                        atomicAdd(sc + (size_t)(r + 64) * D + c, v1);
                                        if (r0 != c0) {
                                            atomicAdd(sc + (size_t)c * D + r, v0);
                                            atomicAdd(sc + (size_t)c * D + r + 64, v1);
                                        }
                                    }
                                }
                        acc_init();
                    } else {
                        // the next row's start is loaded into each register pair right after its last store, so that the
                        // shared-memory loads overlap the stores
#pragma unroll
                        for (int n = 0; n < 16; ++n)
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
#pragma unroll
                                for (int i = 0; i < 2; ++i) {
                                    const int r = fr + 8 * h, c = 8 * n + fc + i;
                                    const float v1 = d1[4 * n + 2 * h + i] * inv2;
                                    S.mat[c * 128 + ((r + 64) ^ msw(c))] = v1;
                                    if (8 * n < N0) {   // (r, c) from d0, and (c, r + 64) = (r + 64, c) by symmetry
                                        S.mat[c * 128 + (r ^ msw(c))] = d0[4 * n + 2 * h + i] * inv2;
                                        S.mat[(r + 64) * 128 + (c ^ msw(r + 64))] = v1;
                                    }
                                }
                                acc_init_nh(n, h);
                            }
                    }
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&S.acc_full);
                    aph ^= 1u;
                    ++seq;
                }
            }
            wgmma_wait<0>();   // the group's operand reads are done
#pragma unroll
            for (int i = 0; i < 64; ++i) { if (i < N0 / 2) acc_fence(d0[i]); acc_fence(d1[i]); }
            __syncwarp();
            if (lane == 0) mbar_arrive(&S.st_empty[os]);   // (after a stop nobody waits for it any more)
            if (++os == NS) { os = 0; oph ^= 1u; }
        }
    } else if (warp >= W_CONV && warp < W_CONV + N_CONV) {
        // ================= convert: raw fp32 -> scaled fp16 head/tail operand slabs =================
        // thread ct owns features m = ct + 128 f: a warp reads 32 consecutive floats of one gathered row (conflict-free)
        // and writes 32 consecutive 16-byte groups of a core-matrix column (conflict-free).
        const int cta = tid - W_CONV * 32;
        const int ct = cta & 127;          // feature(s) of this thread
        const int kh = cta >> 7;           // which part of a tile's entries this convert set takes
        constexpr int CHS = TILE / 8 / KH; // 8-entry chunks per tile and set
        uint32_t rs = 0, rph = 0, bslot = 0;   // stage of the group being converted
        float2 bacc[NF], qacc[NF];
        float wacc = 0.f;
#pragma unroll
        for (int f = 0; f < NF; ++f) { bacc[f] = make_float2(0.f, 0.f); qacc[f] = make_float2(0.f, 0.f); }
        // Gathers.  The convert warps issue the gathers themselves, GATHER_AHEAD groups before they consume the group:
        // warp cw copies the TILE / N_CONV rows cw, cw + N_CONV, ... of a planned tile with one coalesced 16-byte-per-lane
        // cp.async per 512 bytes (SASS LDGSTS; a whole warp instruction moves a full row segment, so the issue cost is a
        // few instructions per row -- a TMA bulk copy per gathered row would serialise on one issuing thread) as one
        // commit group per group; before converting a group a warp waits for its own copies (cp.async.wait_group) and
        // posts one arrival on the stage's mbarrier.
        const int cw = cta >> 5;
        uint32_t gs = 0, gph = 0, grs = 0, grph = 0;   // plan group slot / stage of the next group to gather
        bool plan_end = false;
        auto gather = [&]() {
            if (plan_end) {
                cp_async_commit();   // keep one commit group per iteration so that wait_group counts groups to the very end
                return;
            }
            mbar_wait(&S.plan_full[gs], gph);
            mbar_wait(&S.st_empty[grs], grph ^ 1u);   // the MMAs are done with the group that used this stage
            const uint32_t gm0 = S.meta_raw[gs * PT], gm1 = S.meta_raw[gs * PT + 1];
            if (PT == 2 && !(ta.debug & 1) && ((gm0 | gm1) & F_STOP) == 0 && (gm0 & 0xffu) == TILE && (gm1 & 0xffu) == TILE) {
                // two full tiles (the common case): straight-line copies, no per-row predicates
                int32_t kk[PT][TILE / N_CONV];
#pragma unroll
                for (int e = 0; e < PT; ++e)
#pragma unroll
                    for (int i = 0; i < TILE / N_CONV; ++i) kk[e][i] = S.keys[gs * PT + e][cw + N_CONV * i];
#pragma unroll
                for (int e = 0; e < PT; ++e)
#pragma unroll
                    for (int i = 0; i < TILE / N_CONV; ++i) {
                        const float* src = a.Y + (int64_t)kk[e][i] * a.ld + lane * 4;
                        float* dst = &S.st[grs].raw[e][(cw + N_CONV * i) * D + lane * 4];
#pragma unroll
                        for (int c = 0; c < D / 128; ++c) cp_async16_cg(dst + c * 128, src + c * 128);
                    }
            } else
#pragma unroll
            for (int e = 0; e < PT; ++e) {
                const uint32_t gmeta = S.meta_raw[gs * PT + e];
                if (gmeta & F_STOP) {
                    plan_end = true;
                } else {
                    const int gcnt = (ta.debug & 1) ? 0 : (int)(gmeta & 0xffu);
#pragma unroll
                    for (int i = 0; i < TILE / N_CONV; ++i) {
                        const int slot = cw + N_CONV * i;
                        if (slot < gcnt) {
                            const float* src = a.Y + (int64_t)S.keys[gs * PT + e][slot] * a.ld + lane * 4;
                            float* dst = &S.st[grs].raw[e][slot * D + lane * 4];
#pragma unroll
                            for (int c = 0; c < D / 128; ++c) cp_async16_cg(dst + c * 128, src + c * 128);
                        }
                    }
                }
            }
            cp_async_commit();
            if (++gs == NPG) { gs = 0; gph ^= 1u; }
            if (++grs == NS) { grs = 0; grph ^= 1u; }
        };
        uint32_t cs = 0;   // plan group slot of the group being converted
        bool done = false;
        if (ta.debug & 16) {   // timing experiment: consume the plans as fast as they come, nothing else
            uint32_t ph = 0;
            for (;;) {
                mbar_wait(&S.plan_full[cs], ph);
                const bool stop = (S.meta_raw[cs * PT] | S.meta_raw[cs * PT + 1]) & F_STOP;
                __syncwarp();
                if (lane == 0) mbar_arrive(&S.plan_empty[cs]);
                if (stop) break;
                if (++cs == NPG) { cs = 0; ph ^= 1u; }
            }
            if (cta == 0) S.meta_op[0][0] = F_STOP;
            __syncwarp();
            if (lane == 0) mbar_arrive(&S.op_full[0]);
            done = true;
        }
#pragma unroll 1
        for (int i = 0; i < GATHER_AHEAD && !done; ++i) gather();
        while (!done) {
            gather();
            cp_async_wait_group<GATHER_AHEAD>();   // this warp's rows of the group about to be converted have landed
            __syncwarp();
            if (lane == 0) mbar_arrive(&S.raw_full[rs]);
            mbar_wait(&S.raw_full[rs], rph);        // ... and everybody else's
            // all of this thread's values of the group are read up front (independent loads, one exposed latency per group instead
            // of one per 8-entry chunk); unused slots read stale data that the guarded path zeroes
            float qv[PT][CHS * 8 * NF];
#pragma unroll
            for (int e = 0; e < PT; ++e)
#pragma unroll
                for (int c = 0; c < CHS; ++c)
#pragma unroll
                    for (int i = 0; i < 8; ++i)
#pragma unroll
                        for (int f = 0; f < NF; ++f)
                            qv[e][(c * 8 + i) * NF + f] = S.st[rs].raw[e][((kh * CHS + c) * 8 + i) * D + ct + 128 * f];
            // the slabs overwrite the rows in place: every convert thread has read its rows of the group first
            named_bar_sync(1, N_CONV * 32);
            const uint32_t cm0 = S.meta_raw[cs * PT], cm1 = S.meta_raw[cs * PT + 1];
            const bool fast2 = PT == 2 && !(ta.debug & 4) && ((cm0 | cm1) & F_STOP) == 0 && (cm0 & 0xffu) == TILE &&
                               (cm1 & 0xffu) == TILE;
            if (fast2) {
                // Two full tiles: one straight-line block (the row bookkeeping is branch-free: the accumulators are reset by
                // selects on F_FIRST, the partial sums are stored after EVERY tile and the slot only advances on F_LAST), so
                // that the compiler can interleave the four chunks' load -> scale -> split -> store chains.
#pragma unroll
                for (int e = 0; e < PT; ++e) {
                    const uint32_t meta = e == 0 ? cm0 : cm1;
                    const uint32_t psl = cs * PT + e;
                    const bool first = (meta & F_FIRST) != 0;
#pragma unroll
                    for (int f = 0; f < NF; ++f) {
                        bacc[f].x = first ? 0.f : bacc[f].x; bacc[f].y = first ? 0.f : bacc[f].y;
                        qacc[f].x = first ? 0.f : qacc[f].x; qacc[f].y = first ? 0.f : qacc[f].y;
                    }
                    wacc = first ? 0.f : wacc;
                    unsigned char* hi = &S.st[rs].op[e][0][0];
                    unsigned char* lo = &S.st[rs].op[e][1][0];
#pragma unroll
                    for (int c = 0; c < CHS; ++c) {
                        const int kc = kh * CHS + c, k0 = kc * 8;
                        const float4 sa = *reinterpret_cast<const float4*>(&S.sws[psl][k0]);
                        const float4 sb = *reinterpret_cast<const float4*>(&S.sws[psl][k0 + 4]);
                        const float4 wa = *reinterpret_cast<const float4*>(&S.wv[psl][k0]);
                        const float4 wb = *reinterpret_cast<const float4*>(&S.wv[psl][k0 + 4]);
                        if (LOSS1) wacc += ((wa.x + wa.y) + (wa.z + wa.w)) + ((wb.x + wb.y) + (wb.z + wb.w));
#pragma unroll
                        for (int f = 0; f < NF; ++f) {
                            const int m = ct + 128 * f;
                            const float* q = &qv[e][0];
                            const float2 q01 = make_float2(q[(c * 8 + 0) * NF + f], q[(c * 8 + 1) * NF + f]);
                            const float2 q23 = make_float2(q[(c * 8 + 2) * NF + f], q[(c * 8 + 3) * NF + f]);
                            const float2 q45 = make_float2(q[(c * 8 + 4) * NF + f], q[(c * 8 + 5) * NF + f]);
                            const float2 q67 = make_float2(q[(c * 8 + 6) * NF + f], q[(c * 8 + 7) * NF + f]);
                            uint4 h4, l4;
                            split_f16x2(f2mul(q01, make_float2(sa.x, sa.y)), h4.x, l4.x);
                            split_f16x2(f2mul(q23, make_float2(sa.z, sa.w)), h4.y, l4.y);
                            split_f16x2(f2mul(q45, make_float2(sb.x, sb.y)), h4.z, l4.z);
                            split_f16x2(f2mul(q67, make_float2(sb.z, sb.w)), h4.w, l4.w);
                            const int off = kc * LBO + (m >> 3) * 128 + (m & 7) * 16;
                            *reinterpret_cast<uint4*>(hi + off) = h4;
                            *reinterpret_cast<uint4*>(lo + off) = l4;
                            bacc[f] = f2fma(make_float2(wa.x, wa.y), q01, bacc[f]);
                            bacc[f] = f2fma(make_float2(wa.z, wa.w), q23, bacc[f]);
                            bacc[f] = f2fma(make_float2(wb.x, wb.y), q45, bacc[f]);
                            bacc[f] = f2fma(make_float2(wb.z, wb.w), q67, bacc[f]);
                            if (LOSS1) {
                                qacc[f].x += (q01.x + q23.x) + (q45.x + q67.x);
                                qacc[f].y += (q01.y + q23.y) + (q45.y + q67.y);
                            }
                        }
                    }
#pragma unroll
                    for (int f = 0; f < NF; ++f) {
                        S.bvec[bslot][kh][ct + 128 * f] = bacc[f].x + bacc[f].y;
                        if (LOSS1) S.sumq[bslot][kh][ct + 128 * f] = qacc[f].x + qacc[f].y;
                    }
                    if (LOSS1 && ct == 0) S.wsum[bslot][kh] = wacc;
                    bslot = (bslot + ((meta & F_LAST) ? 1u : 0u)) & (NBV - 1);
                    if (cta == 0) S.meta_op[rs][e] = (uint32_t)(TILE / 16) | (meta & (F_FIRST | F_LAST | F_NEG));
                }
            } else
#pragma unroll
            for (int e = 0; e < PT; ++e) {
                if (done) continue;
                const uint32_t psl = cs * PT + e;   // the tile's plan slot
                const uint32_t meta = S.meta_raw[psl];
                if (meta & F_STOP) {
                    if (cta == 0) S.meta_op[rs][e] = F_STOP;
                    done = true;
                    continue;
                }
                const int cnt = (int)(meta & 0xffu), ksteps = (cnt + 15) >> 4;
                if (meta & F_FIRST) {
#pragma unroll
                    for (int f = 0; f < NF; ++f) { bacc[f] = make_float2(0.f, 0.f); qacc[f] = make_float2(0.f, 0.f); }
                    wacc = 0.f;
                }
                unsigned char* hi = &S.st[rs].op[e][0][0];
                unsigned char* lo = &S.st[rs].op[e][1][0];
                // one chunk = 8 consecutive entries k of this thread's feature(s): a 16-byte group of the head and of the
                // tail slab.  GUARD: the tile is not full -- slots >= cnt hold stale rows (scale and weight 0 from the
                // planner; the value is zeroed as well so that a stale Inf/NaN cannot leak into an unrelated row).
                auto chunk = [&](auto guard, const int c) {
                    constexpr bool GUARD = decltype(guard)::value;
                    const int kc = kh * CHS + c, k0 = kc * 8;
                    const float4 sa = *reinterpret_cast<const float4*>(&S.sws[psl][k0]);
                    const float4 sb = *reinterpret_cast<const float4*>(&S.sws[psl][k0 + 4]);
                    const float4 wa = *reinterpret_cast<const float4*>(&S.wv[psl][k0]);
                    const float4 wb = *reinterpret_cast<const float4*>(&S.wv[psl][k0 + 4]);
                    if (LOSS1) wacc += ((wa.x + wa.y) + (wa.z + wa.w)) + ((wb.x + wb.y) + (wb.z + wb.w));
#pragma unroll
                    for (int f = 0; f < NF; ++f) {
                        const int m = ct + 128 * f;
                        float q[8];
#pragma unroll
                        for (int i = 0; i < 8; ++i) q[i] = qv[e][(c * 8 + i) * NF + f];
                        if (GUARD) {
#pragma unroll
                            for (int i = 0; i < 8; ++i) q[i] = (k0 + i < cnt) ? q[i] : 0.f;
                        }
                        const float2 q01 = make_float2(q[0], q[1]), q23 = make_float2(q[2], q[3]);
                        const float2 q45 = make_float2(q[4], q[5]), q67 = make_float2(q[6], q[7]);
                        uint4 h4, l4;
                        split_f16x2(f2mul(q01, make_float2(sa.x, sa.y)), h4.x, l4.x);
                        split_f16x2(f2mul(q23, make_float2(sa.z, sa.w)), h4.y, l4.y);
                        split_f16x2(f2mul(q45, make_float2(sb.x, sb.y)), h4.z, l4.z);
                        split_f16x2(f2mul(q67, make_float2(sb.z, sb.w)), h4.w, l4.w);
                        const int off = kc * LBO + (m >> 3) * 128 + (m & 7) * 16;
                        *reinterpret_cast<uint4*>(hi + off) = h4;
                        *reinterpret_cast<uint4*>(lo + off) = l4;
                        bacc[f] = f2fma(make_float2(wa.x, wa.y), q01, bacc[f]);
                        bacc[f] = f2fma(make_float2(wa.z, wa.w), q23, bacc[f]);
                        bacc[f] = f2fma(make_float2(wb.x, wb.y), q45, bacc[f]);
                        bacc[f] = f2fma(make_float2(wb.z, wb.w), q67, bacc[f]);
                        if (LOSS1) {
                            qacc[f].x += (q[0] + q[2]) + (q[4] + q[6]);
                            qacc[f].y += (q[1] + q[3]) + (q[5] + q[7]);
                        }
                    }
                };
                if (ta.debug & 4) {
                } else if (cnt == TILE) {   // full tile: straight-line code
#pragma unroll
                    for (int c = 0; c < CHS; ++c) chunk(std::false_type{}, c);
                } else {
#pragma unroll
                    for (int c = 0; c < CHS; ++c)
                        if (kh * CHS + c < 2 * ksteps) chunk(std::true_type{}, c);
                }
                if (meta & F_LAST) {
#pragma unroll
                    for (int f = 0; f < NF; ++f) {
                        S.bvec[bslot][kh][ct + 128 * f] = bacc[f].x + bacc[f].y;
                        if (LOSS1) S.sumq[bslot][kh][ct + 128 * f] = qacc[f].x + qacc[f].y;
                    }
                    if (LOSS1 && ct == 0) S.wsum[bslot][kh] = wacc;
                    bslot = (bslot + 1) & (NBV - 1);
                }
                if (cta == 0) S.meta_op[rs][e] = (uint32_t)ksteps | (meta & (F_FIRST | F_LAST | F_NEG));
            }
            // (no proxy fence here: FENCE.VIEW.ASYNC in a thread with cp.async / global loads in flight waits for them -- the
            // next groups' gathers -- so the generic->async proxy fence is executed by the MMA-issuing warp after it has
            // acquired the group through op_full)
            __syncwarp();
            if (lane == 0) {   // one arrival per warp on each of the two hand-offs of a group
                mbar_arrive(&S.plan_empty[cs]);
                mbar_arrive(&S.op_full[rs]);
            }
            cs = (cs + 1) & (NPG - 1);
            if (++rs == NS) { rs = 0; rph ^= 1u; }
        }
    } else {
        // ================= epilogue: explicit-matrix block Gauss-Seidel / CG, systolic over the blocks of a row =================
        const int q = warp & 3;                  // column block owned by this warp
        const int j = q * 32 + lane;             // matrix row
        float* pv = S.pv[q];
        double l_nume = 0.0, l_deno = 0.0;
        const float tol = a.tol;
        if constexpr (PARTIAL) {
            // the chunk's matrix went to scratch straight from the MMA warpgroup; add its vectors (once per chunk: pass 0)
            int row = 0, slot = 0, nrow = 0, nslot = 0;
            int64_t beg, n = 0, nbeg, nn = 0;
            if (my_first < nitems) item_info(my_first, row, beg, n, slot);
            for (int64_t seq = 0; my_first + seq * stride < nitems; ++seq) {
                const int64_t nit = my_first + (seq + 1) * stride;
                if (nit < nitems) item_info(nit, nrow, nbeg, nn, nslot);
                const uint32_t aph = (uint32_t)(seq & 1);
                const uint32_t bs = (uint32_t)(seq & (NBV - 1));
                mbar_wait_idle(&S.acc_full, aph);
                float* sc = ta.scratch + (size_t)slot * scratch_floats<D>();
                if constexpr (DET) {
                    if (ta.pass == 0) {
                        for (int jj = j; jj < D; jj += 128) {
                            sc[(size_t)D * D + jj] = S.bvec[bs][0][jj] + (KH == 2 ? S.bvec[bs][KH - 1][jj] : 0.f);
                            if (LOSS1) sc[(size_t)D * D + D + jj] = S.sumq[bs][0][jj] + (KH == 2 ? S.sumq[bs][KH - 1][jj] : 0.f);
                        }
                        if (LOSS1 && j < 4)
                            sc[(size_t)D * D + 2 * D + j] = j == 0 ? S.wsum[bs][0] + (KH == 2 ? S.wsum[bs][KH - 1] : 0.f) : 0.f;
                    }
                } else if (ta.pass == 0) {
                    for (int jj = j; jj < D; jj += 128) {
                        atomicAdd(sc + (size_t)D * D + jj, S.bvec[bs][0][jj] + (KH == 2 ? S.bvec[bs][KH - 1][jj] : 0.f));
                        if (LOSS1) atomicAdd(sc + (size_t)D * D + D + jj, S.sumq[bs][0][jj] + (KH == 2 ? S.sumq[bs][KH - 1][jj] : 0.f));
                    }
                    if (LOSS1 && j == 0) atomicAdd(sc + (size_t)D * D + 2 * D, S.wsum[bs][0] + (KH == 2 ? S.wsum[bs][KH - 1] : 0.f));
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&S.acc_empty);
                row = nrow; slot = nslot; n = nn;
            }
        } else {
            // Row pipeline registers: x_j of rows seq (xj), seq + 1 (x1), and the row ids of seq + 1, seq + 2; the loads
            // for seq + 2 / seq + 3 are issued one iteration before they are touched.
            auto row_of = [&](int64_t sq) -> int {
                const int64_t it = my_first + sq * stride;
                return it < nitems ? a.row_list[a.row_begin + it] : -1;
            };
            auto len_of = [&](int row) -> float {   // only for the adaptive-reg loss term
                if (row < 0 || !a.compute_loss) return 0.f;
                return (float)(a.indptr[row] - (row == 0 ? 0 : a.indptr[row - 1]));
            };
            int row = (ta.debug & 16) ? -1 : row_of(0), row1 = row_of(1), row2 = row_of(2);
            float xj = row >= 0 ? a.X[(int64_t)row * a.ld + j] : 0.f;
            float x1 = row1 >= 0 ? a.X[(int64_t)row1 * a.ld + j] : 0.f;
            float nlen = len_of(row), nlen1 = len_of(row1);
            if (row >= 0) {   // publish row 0's x
                S.xs[0][j] = xj;
                __syncwarp();
                if (lane == 0) mbar_arrive(&S.x_full[0]);
            }
            // element (j, c) of the row's matrix
            auto mat = [&](int c) -> float { return S.mat[c * 128 + (j ^ msw(c))]; };
            for (int64_t seq = 0; row >= 0; ++seq) {
                // look-ahead loads
                const int row3 = row_of(seq + 3);
                const float x2 = row2 >= 0 ? a.X[(int64_t)row2 * a.ld + j] : 0.f;
                const float nlen2 = len_of(row2);
                if (row1 >= 0) {   // publish the next row's x: by the time a warp gets there everybody has
                    S.xs[(seq + 1) & (NXS - 1)][j] = x1;
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&S.x_full[(seq + 1) & (NXS - 1)]);
                }
                const uint32_t aph = (uint32_t)(seq & 1);
                const uint32_t bs = (uint32_t)(seq & (NBV - 1));
                const uint32_t xsl = (uint32_t)(seq & (NXS - 1));
                const float* xs = S.xs[xsl];
                mbar_wait(&S.x_full[xsl], (uint32_t)((seq / NXS) & 1));
                mbar_wait_idle(&S.acc_full, aph);
                if (ta.debug & 8) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&S.acc_empty);
                    row = row1; row1 = row2; row2 = row3;
                    xj = x1; x1 = x2;
                    continue;
                }
                const float bj = S.bvec[bs][0][j] + (KH == 2 ? S.bvec[bs][KH - 1][j] : 0.f);
                double ln_row = 0.0, ld_row = 0.0;   // DET: this warp's loss terms of the row
                // ---- h = M x - b; keep the diagonal block of M in registers ----
                float hM = 0.f;
                float md[32];
#pragma unroll
                for (int c = 0; c < D / 32; ++c) {
                    float h0 = 0.f, h1 = 0.f;
#pragma unroll
                    for (int i = 0; i < 32; i += 4) {
                        const float4 x4 = *reinterpret_cast<const float4*>(xs + c * 32 + i);
                        const float m0 = mat(c * 32 + i), m1 = mat(c * 32 + i + 1), m2 = mat(c * 32 + i + 2), m3 = mat(c * 32 + i + 3);
                        h0 = fmaf(m0, x4.x, h0); h1 = fmaf(m1, x4.y, h1);
                        h0 = fmaf(m2, x4.z, h0); h1 = fmaf(m3, x4.w, h1);
                        if (c == q) { md[i] = m0; md[i + 1] = m1; md[i + 2] = m2; md[i + 3] = m3; }
                    }
                    hM += h0 + h1;
                }
                if (a.compute_loss) {
                    // als.cc:298-321 with the pre-update row: reg*kappa*|x|^2 (both axes); item side additionally
                    // x G x + sum_obs[(1+w)(yhat-1)^2 - yhat^2] = x G x + x D x - 2 x.(b + sum q) + (n + sum w),
                    // where x (G + D) x = x M x - reg |x|^2
                    const float kappa = a.adaptive_reg ? nlen : 1.0f;
                    double t = (double)(kappa * a.reg * xj * xj);
                    if (a.axis == 1) {
                        t += (double)xj * (double)hM - (double)(a.reg * xj * xj) -
                             2.0 * (double)xj * ((double)bj + (double)S.sumq[bs][0][j] + (KH == 2 ? (double)S.sumq[bs][KH - 1][j] : 0.0));
                        if (j == 0) {
                            const double ws = (double)S.wsum[bs][0] + (KH == 2 ? (double)S.wsum[bs][KH - 1] : 0.0);
                            t += (double)nlen + ws;
                            l_deno += (double)a.Y_rows + ws;
                        }
                    }
                    if constexpr (DET) {
                        // the denominator only ever has thread 0's term (warp 0, lane 0): nothing to reduce
                        ln_row = warp_sum_d(t);
                        ld_row = l_deno;
                        l_deno = 0.0;
                        if (q < 3 && lane == 0) {   // published by this warp's d_full arrival below
                            SD.lossp[xsl][q][0] = ln_row;
                            SD.lossp[xsl][q][1] = ld_row;
                        }
                    } else {
                        l_nume += t;
                    }
                }
                float h = hM - bj;
                // ---- fold in the deltas of the earlier blocks as they appear: h -= M[j, B] . delta_B ----
#pragma unroll 1
                for (int B = 0; B < q; ++B) {
                    float mv[32];
#pragma unroll
                    for (int i = 0; i < 32; ++i) mv[i] = mat(B * 32 + i);
                    mbar_wait(&S.d_full[B], aph);
                    float u0 = 0.f, u1 = 0.f;
#pragma unroll
                    for (int i = 0; i < 32; i += 4) {
                        const float4 d4 = *reinterpret_cast<const float4*>(&S.dl[B][i]);
                        u0 = fmaf(mv[i], d4.x, u0);
                        u1 = fmaf(mv[i + 1], d4.y, u1);
                        u0 = fmaf(mv[i + 2], d4.z, u0);
                        u1 = fmaf(mv[i + 3], d4.w, u1);
                    }
                    h -= u0 + u1;
                }
                if constexpr (DET) {
                    // the waits on d_full[0 .. 2] above acquired the earlier warps' terms: add them in warp order
                    if (q == 3 && lane == 0 && a.loss && a.compute_loss) {
                        double sn = SD.lossp[xsl][0][0], sd = SD.lossp[xsl][0][1];
#pragma unroll
                        for (int w = 1; w < 3; ++w) {
                            sn += SD.lossp[xsl][w][0];
                            sd += SD.lossp[xsl][w][1];
                        }
                        a.loss[2 * (int64_t)row] = sn + ln_row;
                        a.loss[2 * (int64_t)row + 1] = sd + ld_row;
                    }
                }
                // this warp's reads of the matrix are done
                __syncwarp();
                if (lane == 0) mbar_arrive(&S.acc_empty);
                // ---- 3-step CG on the own diagonal block (als.cc:324-345) ----
                float xv = 0.f;
                {
                    float r = h, p = h;
                    float rsold = warp_sum(r * r);
                    bool act = rsold > tol;            // als.cc:329
#pragma unroll 1
                    for (int step = 0; step < 3; ++step) {
                        pv[lane] = p;
                        __syncwarp();
                        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
                        for (int i = 0; i < 32; i += 4) {
                            const float4 p4 = *reinterpret_cast<const float4*>(pv + i);
                            a0 = fmaf(md[i], p4.x, a0); a1 = fmaf(md[i + 1], p4.y, a1);
                            a2 = fmaf(md[i + 2], p4.z, a2); a3 = fmaf(md[i + 3], p4.w, a3);
                        }
                        __syncwarp();
                        const float Ap = (a0 + a1) + (a2 + a3);
                        const float pAp = warp_sum(p * Ap);
                        const float ss = act ? __fdividef(rsold, pAp) : 0.f;   // als.cc:337 (no eps)
                        xv = fmaf(ss, p, xv);
                        r = fmaf(-ss, Ap, r);
                        const float rsnew = warp_sum(r * r);
                        act = act && !(rsnew < tol);                            // als.cc:341
                        if (act) p = fmaf(__fdividef(rsnew, rsold), p, r);
                        rsold = act ? rsnew : rsold;
                    }
                }
                float v = xj - xv;                      // als.cc:346
                const bool badw = __any_sync(FULL, !isfinite(v));
                // write the own block (and the peers' replicas, fused exchange) BEFORE publishing the delta: the warp of the
                // last block may overwrite the row (NaN/Inf guard, cf. als.cu:116-120) and must come after these stores
                a.X[(int64_t)row * a.ld + j] = v;
                for (int pr = 0; pr < a.n_peer; ++pr) a.peerX[pr][(int64_t)row * a.ld + j] = v;
                if (q < 3) {
                    S.dl[q][lane] = xv;
                    if (badw && lane == 0) atomicOr(&S.badrow[xsl], 1);
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&S.d_full[q]);
                }
                // the warp of the last block has seen every earlier block's flag (set before that block's delta was
                // published) and zeroes the whole row if any block came out non-finite
                if (q == 3) {
                    const bool bad = badw || (S.badrow[xsl] != 0);
                    if (bad) {
#pragma unroll
                        for (int c = 0; c < 4; ++c) {
                            a.X[(int64_t)row * a.ld + c * 32 + lane] = 0.f;
                            for (int pr = 0; pr < a.n_peer; ++pr) a.peerX[pr][(int64_t)row * a.ld + c * 32 + lane] = 0.f;
                        }
                        __syncwarp();
                        if (lane == 0) S.badrow[xsl] = 0;
                    }
                }
                row = row1; row1 = row2; row2 = row3;
                xj = x1; x1 = x2;
                nlen = nlen1; nlen1 = nlen2;
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
    }
}

// ---- host side ---------------------------------------------------------------------------------
inline bool tc_applicable(int optimizer_code, int d, int vdim, int block_size) {
    return optimizer_code == 8 && d == 128 && vdim == 128 && block_size == 32;
}
// split-row mode (rows beyond the SIMT kernels' cap): d = 128 and d = 256
inline bool tc_split_applicable(int optimizer_code, int d, int vdim, int block_size) {
    return optimizer_code == 8 && (d == 128 || d == 256) && vdim == d && block_size == 32;
}

// device-side operand scale of the next tensor-core launches: maxes[0] = bits of max|Y| (noted at Gram time),
// maxes[1] = bits of max|v| over the values of this launch
inline int tc_note_absmax(const float* p, size_t n, unsigned int* out, int num_sms, cudaStream_t st) {
    BFL_CUDA(cudaMemsetAsync(out, 0, sizeof(unsigned int), st));
    if (n == 0) return BFL_OK;
    const int grid = (int)std::min<size_t>((n / 4 + 255) / 256 + 1, (size_t)num_sms * 8);
    tc_absmax_kernel<<<grid, 256, 0, st>>>(p, n, out);
    BFL_LAUNCHED();
    return BFL_OK;
}
inline int tc_update_scale(const unsigned int* ymax, const unsigned int* vmax, float alpha, float* scales, cudaStream_t st) {
    tc_scale_kernel<<<1, 1, 0, st>>>(ymax, vmax, alpha, scales);
    BFL_LAUNCHED();
    return BFL_OK;
}

// split-row items: every row of list[0..nrows) is cut into chunks of `split` entries -> triples (row, chunk, slot)
__global__ void tc_count_items_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ list, int64_t nrows,
                                      int64_t split, unsigned long long* total) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nrows; i += (int64_t)gridDim.x * blockDim.x) {
        const int row = list[i];
        const int64_t n = indptr[row] - (row == 0 ? 0 : indptr[row - 1]);
        atomicAdd(total, (unsigned long long)((n + split - 1) / split));
    }
}
__global__ void tc_fill_items_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ list, int64_t nrows,
                                     int64_t split, unsigned long long* cursor, int32_t* __restrict__ items) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nrows; i += (int64_t)gridDim.x * blockDim.x) {
        const int row = list[i];
        const int64_t n = indptr[row] - (row == 0 ? 0 : indptr[row - 1]);
        const int64_t nc = (n + split - 1) / split;
        const unsigned long long pos = atomicAdd(cursor, (unsigned long long)nc);
        for (int64_t c = 0; c < nc; ++c) {
            items[3 * (pos + c) + 0] = row;
            items[3 * (pos + c) + 1] = (int32_t)c;
            items[3 * (pos + c) + 2] = (int32_t)i;
        }
    }
}

// Deterministic mode: chunk counts of the long rows (scanned by the caller into END offsets) and items in list order, so
// that the chunks of list row i are the items first[i] .. first[i] + nc_i (first = exclusive prefix) -- no atomic cursor.
__global__ void tc_chunk_counts_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ list, int64_t nrows,
                                       int64_t split, long long* __restrict__ counts) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nrows; i += (int64_t)gridDim.x * blockDim.x) {
        const int row = list[i];
        const int64_t n = indptr[row] - (row == 0 ? 0 : indptr[row - 1]);
        counts[i] = (n + split - 1) / split;
    }
}
__global__ void tc_fill_items_scanned_kernel(const int32_t* __restrict__ list, int64_t nrows,
                                             const long long* __restrict__ chunk_end, int32_t* __restrict__ items) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nrows; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t pos = i == 0 ? 0 : chunk_end[i - 1], nc = chunk_end[i] - pos;
        for (int64_t c = 0; c < nc; ++c) {
            items[3 * (pos + c) + 0] = list[i];
            items[3 * (pos + c) + 1] = (int32_t)c;
            items[3 * (pos + c) + 2] = (int32_t)i;
        }
    }
}

// Deterministic mode: row slot i of `rows_out` = chunk slot first .. last of list row row0 + i, added in ascending chunk
// order with rounded fp32 adds, starting from the first chunk.  chunk_end: END offsets of the whole list's chunks,
// chunk0: the first chunk held by `chunks`.  blockIdx.y = row of the batch; threads run over the slot in 16-byte pieces
// (nf4 of them: matrix + b, or the whole slot when the loss vectors were written), so every access is coalesced.
__global__ void __launch_bounds__(256) tc_chunk_reduce_kernel(const float* __restrict__ chunks, const long long* __restrict__ chunk_end,
                                                              int64_t row0, int64_t chunk0, size_t slot_floats, int nf4,
                                                              float* __restrict__ rows_out) {
    const int64_t i = row0 + blockIdx.y;
    const int64_t c0 = (i == 0 ? 0 : chunk_end[i - 1]) - chunk0, c1 = chunk_end[i] - chunk0;
    float4* out = reinterpret_cast<float4*>(rows_out + (size_t)blockIdx.y * slot_floats);
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < nf4; e += gridDim.x * blockDim.x) {
        float4 acc = __ldg(reinterpret_cast<const float4*>(chunks + (size_t)c0 * slot_floats) + e);
        for (int64_t c = c0 + 1; c < c1; ++c) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(chunks + (size_t)c * slot_floats) + e);
            acc.x = __fadd_rn(acc.x, v.x);
            acc.y = __fadd_rn(acc.y, v.y);
            acc.z = __fadd_rn(acc.z, v.z);
            acc.w = __fadd_rn(acc.w, v.w);
        }
        out[e] = acc;
    }
}

// chunk matrices of the split rows; a.row_begin/row_end index `items`.  Default: added into one slot per row of
// `scratch`, which is zeroed here.  det: stored into one slot per item, no memset (see the kernel's DET notes)
template <int D>
int tc_launch_partial(const AlsArgs& a, const int32_t* items, int64_t nitems, float* scratch, int64_t nslots,
                      int64_t split, int num_sms, cudaStream_t st, bool det = false) {
    if (nitems <= 0) return BFL_OK;
    if (!a.tc_scales) BFL_FAIL(BFL_ERR_STATE, "tensor-core ALS kernel: operand scale not prepared");
    TcArgs ta;
    ta.a = a;
    ta.a.row_begin = 0;
    ta.a.row_end = nitems;
    ta.items = items;
    ta.scratch = scratch;
    ta.split = split;
    ta.debug = 0;
    if (!det) BFL_CUDA(cudaMemsetAsync(scratch, 0, sizeof(float) * scratch_floats<D>() * (size_t)nslots, st));
    const size_t smem = sizeof(Smem<D>);
    const int grid = (int)std::min<int64_t>(nitems, (int64_t)num_sms);
    for (ta.pass = 0; ta.pass < (D == 128 ? 1 : 3); ++ta.pass) {
        if (det && a.compute_loss && a.axis == 1) {
            BFL_CUDA(cudaFuncSetAttribute(als_tc_kernel<D, true, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            als_tc_kernel<D, true, true, true><<<grid, THREADS, smem, st>>>(ta);
        } else if (det) {
            BFL_CUDA(cudaFuncSetAttribute(als_tc_kernel<D, true, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            als_tc_kernel<D, true, false, true><<<grid, THREADS, smem, st>>>(ta);
        } else if (a.compute_loss && a.axis == 1) {
            BFL_CUDA(cudaFuncSetAttribute(als_tc_kernel<D, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            als_tc_kernel<D, true, true><<<grid, THREADS, smem, st>>>(ta);
        } else {
            BFL_CUDA(cudaFuncSetAttribute(als_tc_kernel<D, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            als_tc_kernel<D, true, false><<<grid, THREADS, smem, st>>>(ta);
        }
        BFL_LAUNCHED();
    }
    return BFL_OK;
}

// solves the rows a.row_list[a.row_begin .. a.row_end) (any length > 0) with the fused tensor-core kernel; det_loss:
// a.loss takes per-row terms (the DET instantiations)
inline int tc_launch(const AlsArgs& a, int num_sms, cudaStream_t st, bool det_loss = false) {
    const int64_t nrows = a.row_end - a.row_begin;
    if (nrows <= 0) return BFL_OK;
    if (!a.tc_scales) BFL_FAIL(BFL_ERR_STATE, "tensor-core ALS kernel: operand scale not prepared");
    TcArgs ta;
    ta.a = a;
    ta.items = nullptr;
    ta.scratch = nullptr;
    ta.split = 0;
    ta.pass = 0;
    ta.debug = getenv("BFL_TC_DEBUG") ? atoi(getenv("BFL_TC_DEBUG")) : 0;
    const size_t smem = sizeof(Smem<128>);
    const int grid = (int)std::min<int64_t>(nrows, (int64_t)num_sms);
    if (det_loss) {
        const size_t smem_det = sizeof(SmemDet<128>);
        if (a.axis == 1) {
            BFL_CUDA(cudaFuncSetAttribute(als_tc_kernel<128, false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_det));
            als_tc_kernel<128, false, true, true><<<grid, THREADS, smem_det, st>>>(ta);
        } else {
            BFL_CUDA(cudaFuncSetAttribute(als_tc_kernel<128, false, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_det));
            als_tc_kernel<128, false, false, true><<<grid, THREADS, smem_det, st>>>(ta);
        }
    } else if (a.compute_loss && a.axis == 1) {
        BFL_CUDA(cudaFuncSetAttribute(als_tc_kernel<128, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        als_tc_kernel<128, false, true><<<grid, THREADS, smem, st>>>(ta);
    } else {
        BFL_CUDA(cudaFuncSetAttribute(als_tc_kernel<128, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        als_tc_kernel<128, false, false><<<grid, THREADS, smem, st>>>(ta);
    }
    BFL_LAUNCHED();
    return BFL_OK;
}

}  // namespace tc
}  // namespace bfl
