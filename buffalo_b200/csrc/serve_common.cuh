// The batch serving kernel's building blocks (DESIGN.md 4.9), shared by serve.cu and the IVF search of ivf.cu: the
// CTA shape, the register-tile scoring that reproduces topk_score_slice's per-pair order bit for bit, the warp-scope
// radix select and the shared-memory budget of one 32-query x 1024-candidate slice.  Everything is in an unnamed
// namespace: each translation unit compiles its own copy.
#pragma once
#include "seen_common.cuh"

namespace {

using namespace bfl;

constexpr int SV_THREADS = 256;
constexpr int SV_QR = 4;                            // queries per warp (register tile rows)
constexpr int SV_QT = SV_QR * (SV_THREADS / 32);    // queries per CTA
constexpr int SV_SLICE = 1024;                      // candidates per CTA
constexpr int SV_DMAX = 256;                        // widest d of the batch kernel (shared memory)
constexpr int SV_BATCH_MAX = 16384;                 // queries per internal batch
constexpr size_t SV_CAND_BYTES = (size_t)1 << 30;   // candidate scratch aimed at per batch

// row pitch of a staged tile in floats: pitch / 4 is odd, so the float4 reads of 8 consecutive lanes (one row each) fall
// into 8 different bank groups
__host__ __device__ inline int tile_pitch(int dpad) { return ((dpad >> 2) & 1) ? dpad : dpad + 4; }

// words of a warp's selection scratch in the tile buffers once scoring is done: 256 histogram counters, then with
// seen items 32 words of seen bitmask (one bit per candidate of the slice)
__host__ __device__ constexpr int sel_words(bool seen) { return seen ? 256 + SV_SLICE / 32 : 256; }

struct ScoreCtx {
    const float* q;      // the warp's SV_QR query rows in shared memory, pitch dpad
    const float* t;      // the lane's first tile row; its b-th row is t + b * 32 * pitch
    int dpad, pitch, d;
    bool vec;
};

// Lane l's partial sum of topk_score_slice for every (query, item) of the register tile: the same columns in the same
// order with the same fmaf nesting.
template <int IR>
__device__ __forceinline__ void leaf(const ScoreCtx& s, int l, float (&p)[SV_QR][IR]) {
#pragma unroll
    for (int a = 0; a < SV_QR; ++a)
#pragma unroll
        for (int b = 0; b < IR; ++b) p[a][b] = 0.f;
    if (s.vec) {
        for (int c = l * 4; c < s.d; c += 128) {
            float4 x[SV_QR], v[IR];
#pragma unroll
            for (int a = 0; a < SV_QR; ++a) x[a] = *reinterpret_cast<const float4*>(s.q + a * s.dpad + c);
#pragma unroll
            for (int b = 0; b < IR; ++b) v[b] = *reinterpret_cast<const float4*>(s.t + b * 32 * s.pitch + c);
#pragma unroll
            for (int a = 0; a < SV_QR; ++a)
#pragma unroll
                for (int b = 0; b < IR; ++b)
                    p[a][b] = fmaf(v[b].x, x[a].x, fmaf(v[b].y, x[a].y, fmaf(v[b].z, x[a].z, fmaf(v[b].w, x[a].w, p[a][b]))));
        }
    } else {
        for (int c = l; c < s.d; c += 32) {
            float x[SV_QR], v[IR];
#pragma unroll
            for (int a = 0; a < SV_QR; ++a) x[a] = s.q[a * s.dpad + c];
#pragma unroll
            for (int b = 0; b < IR; ++b) v[b] = s.t[b * 32 * s.pitch + c];
#pragma unroll
            for (int a = 0; a < SV_QR; ++a)
#pragma unroll
                for (int b = 0; b < IR; ++b) p[a][b] = fmaf(v[b], x[a], p[a][b]);
        }
    }
}

// warp_sum's butterfly (offsets 16, 8, 4, 2, 1) as an expression tree over the 32 lane partials: the sum over the lanes
// whose low NB bits are X is the sum of the two halves that differ in bit NB.  tree<0, 0> is lane 0's warp_sum.
template <int NB, int X, int IR>
__device__ __forceinline__ void tree(const ScoreCtx& s, float (&out)[SV_QR][IR]) {
    if constexpr (NB == 5) {
        leaf<IR>(s, X, out);
    } else {
        float hi[SV_QR][IR];
        tree<NB + 1, X, IR>(s, out);
        tree<NB + 1, X | (1 << NB), IR>(s, hi);
#pragma unroll
        for (int a = 0; a < SV_QR; ++a)
#pragma unroll
            for (int b = 0; b < IR; ++b) out[a][b] = out[a][b] + hi[a][b];
    }
}

// One warp: the k largest of vals[0..n) -> (out_v, out_i)[0..k) unordered, index = idx0 + position, ties at the k-th
// value to the smaller position.  The selection of block_select (topk.cu) at warp scope, so that the 8 warps of a CTA
// select for 8 queries at once with no block barrier.  hist: 256 counters of the warp.
// SEEN: position i does not exist for the selection when bit i of seen[0..32) is set (n <= 1024, no bit at or past n);
// the min(k, unseen) selected go to out_key as rank keys, unordered, and their number to *out_cnt.
template <bool SEEN>
__device__ void warp_select(const float* vals, int idx0, int n, int k, float* out_v, int32_t* out_i, unsigned* hist,
                            const uint32_t* seen = nullptr, unsigned long long* out_key = nullptr,
                            int32_t* out_cnt = nullptr) {
    const int lane = threadIdx.x & 31;
    auto live = [&](int i) { return !SEEN || !((seen[i >> 5] >> (i & 31)) & 1u); };
    if constexpr (SEEN) {
        const int nv = n - (int)__reduce_add_sync(FULL, (unsigned)__popc(seen[lane]));
        if (lane == 0) *out_cnt = nv < k ? nv : k;
        if (nv <= k) {
            unsigned base = 0;
            for (int i0 = 0; i0 < n; i0 += 32) {
                const int i = i0 + lane;
                const bool keep = i < n && live(i);
                const unsigned bal = __ballot_sync(FULL, keep);
                if (keep) out_key[base + __popc(bal & ((1u << lane) - 1u))] = rank_key(vals[i], idx0 + i);
                base += __popc(bal);
            }
            return;
        }
    } else if (n <= k) {
        for (int i = lane; i < k; i += 32) {
            out_v[i] = i < n ? vals[i] : -INFINITY;
            out_i[i] = i < n ? idx0 + i : -1;
        }
        return;
    }
    uint32_t prefix = 0, mask = 0;
    unsigned kk = (unsigned)k;
    for (int shift = 24; shift >= 0; shift -= 8) {
#pragma unroll
        for (int j = 0; j < 8; ++j) hist[lane + 32 * j] = 0;
        __syncwarp();
        for (int i = lane; i < n; i += 32) {
            const uint32_t u = ord_of(vals[i]);
            if ((u & mask) == prefix && live(i)) atomicAdd(&hist[(u >> shift) & 255u], 1u);
        }
        __syncwarp();
        // lane owns bins 8 lane .. 8 lane + 7; suf = matches in its bins and all higher ones
        unsigned loc[8], own = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            loc[j] = hist[8 * lane + j];
            own += loc[j];
        }
        unsigned suf = own;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned t = __shfl_down_sync(FULL, suf, o);
            if (lane + o < 32) suf += t;
        }
        // the k-th largest is in the one lane with (suf - own) < kk <= suf
        const bool mine = suf - own < kk && kk <= suf;
        unsigned bin = 0, left = 0;
        if (mine) {
            unsigned cum = suf - own;
            int b = 7;
            for (; b > 0; --b) {
                if (cum + loc[b] >= kk) break;
                cum += loc[b];
            }
            bin = 8u * lane + b;
            left = kk - cum;                        // still needed inside the bin
        }
        const int src = __ffs(__ballot_sync(FULL, mine)) - 1;
        bin = __shfl_sync(FULL, bin, src);
        kk = __shfl_sync(FULL, left, src);
        prefix |= bin << shift;
        mask |= 255u << shift;
        __syncwarp();
    }
    const uint32_t T = prefix;                      // kk ties to take; k - kk elements are strictly larger
    unsigned n_gt = 0, n_tie = 0;
    const unsigned below = (1u << lane) - 1u;
    for (int i0 = 0; i0 < n; i0 += 32) {
        const int i = i0 + lane;
        const float v = i < n ? vals[i] : 0.f;
        const uint32_t u = ord_of(v);
        const bool ok = i < n && live(i);
        const bool gt = ok && u > T, tie = ok && u == T;
        const unsigned bg = __ballot_sync(FULL, gt), bt = __ballot_sync(FULL, tie);
        if (gt) {
            const unsigned pos = n_gt + __popc(bg & below);
            if constexpr (SEEN) {
                out_key[pos] = rank_key(v, idx0 + i);
            } else {
                out_v[pos] = v;
                out_i[pos] = idx0 + i;
            }
        }
        const unsigned r = n_tie + __popc(bt & below);
        if (tie && r < kk) {
            if constexpr (SEEN) {
                out_key[(k - kk) + r] = rank_key(v, idx0 + i);
            } else {
                out_v[(k - kk) + r] = v;
                out_i[(k - kk) + r] = idx0 + i;
            }
        }
        n_gt += __popc(bg);
        n_tie += __popc(bt);
    }
}

size_t slice_smem_bytes(int d, int IR, bool seen, int* tile_floats) {
    const int dpad = (d + 3) & ~3;
    int tf = 32 * IR * tile_pitch(dpad);
    const int sel = (SV_THREADS / 32) * sel_words(seen);
    if (2 * tf < sel) tf = sel / 2;                 // room for the select histograms (and seen bitmasks)
    *tile_floats = tf;
    return sizeof(float) * ((size_t)SV_QT * SV_SLICE + (size_t)SV_QT * dpad + 2 * (size_t)tf);
}

}  // namespace

namespace bfl {
// dst[r] = src[idx[r]] for n rows of d floats (pitch ld on both sides, padding columns zero; an index outside
// [0, n_src) gives a zero row), stream-ordered; serve.cu
int serve_gather_rows(const float* src, int64_t n_src, int ld, const int32_t* idx, int64_t n, int d, float* dst,
                      cudaStream_t st);

// A device CSR of END offsets read per query: query q of a batch reads row row[q], or row base + q without `row`.
struct CandRows {
    const int64_t* indptr;
    const int32_t* keys;
    const int32_t* row;
    int64_t base;
};
// candidates.cu, stream-ordered.  cand_plan: the work list of a batch of nb queries with candidate lists `cand`:
// unit_end / key_end [nb] become the inclusive sums of each query's units (slices of up to 1024 list positions) and of
// its rank-key slots.  cand_batch: per query q, the k best of its list (scores and ties of bfl_serve_topk with the list
// as the pool), without the items of its sorted seen row when seen.indptr is set -> out_idx (item ids, -1 pads) /
// out_val (nullable; 0.0f pads) [nb x k].  cand_key / cand_cnt hold key_end[nb - 1] keys and n_units counts.
int cand_plan(CandRows cand, int64_t nb, int k, long long* unit_end, long long* key_end, cudaStream_t st);
int cand_batch(const float* queries, int64_t n_q, int ldq, const int32_t* qidx, int64_t nb, const float* items, int ldi,
               const float* bias, int d, int k, CandRows cand, CandRows seen, const long long* unit_end,
               const long long* key_end, long long n_units, unsigned long long* cand_key, int32_t* cand_cnt,
               int32_t* out_idx, float* out_val, cudaStream_t st);
// rerank.cu, stream-ordered: the MMR re-ranking of n rows of m candidates (item ids, -1 pads; scores) against the item
// rows (pitch ld, first d columns) -> out_idx / out_val [n x k].  1 <= k <= m <= 256, 0 <= diversify <= 1.
int mmr_rerank(const float* items, int ld, int d, const int32_t* cand_idx, const float* cand_val, int64_t n, int m,
               int k, float diversify, int32_t* out_idx, float* out_val, cudaStream_t st);
}  // namespace bfl
