// Per-category caps over ranked lists (DESIGN.md 4.18): the device path of ParALS / ParBPRMF
// topk_recommendation(categories=..., category_cap=...) and buffalo_b200.parallel.cap_categories.  Per row, the
// candidates are walked best first and an item is accepted when its category is -1 or fewer than the category's cap
// items of it are accepted already, until topk are accepted.  A row's walk can span several calls (rounds), each over
// the next part of the row's ranking: the accepted count, the accepted items and a table of (category, count) persist
// in the caller's buffers between them.
//   category_walk_kernel: one warp per row, 32 candidates per step.  __match_any_sync groups the lanes of one category;
//                         a lane's rank in its group plus the category's count so far decides its cap test, and a
//                         ballot prefix over the lanes that pass decides the topk limit, so a step accepts exactly what
//                         the sequential walk accepts.  The table is open-addressed (linear probing) with at least
//                         2 topk slots, and only categories with an accepted item enter it, so it is never more than
//                         half full.  New categories are inserted one lane at a time in lane order.  -1 entries are
//                         skipped wherever they stand.
// A row's state and output depend on that row's candidates alone.  No atomics.
#include <climits>

#include "bfl_common.cuh"

using namespace bfl;

namespace {

constexpr int CW_WARPS = 4;

__device__ __forceinline__ int cw_hash(int32_t g, unsigned mask) {
    return (int)(((uint32_t)g * 0x9E3779B1u) >> 7) & (int)mask;
}

// Slot of category g in tab (pairs of (g + 1, count); 0 marks an empty slot): its own slot, or the empty one where it
// would go.
__device__ __forceinline__ int cw_probe(const int32_t* tab, int32_t g, unsigned mask) {
    int s = cw_hash(g, mask);
    for (;;) {
        const int32_t key = tab[2 * s];
        if (key == 0 || key == g + 1) return s;
        s = (s + 1) & (int)mask;
    }
}

// state row: [0] accepted count, then `slots` pairs (category + 1, count).
__global__ void __launch_bounds__(32 * CW_WARPS) category_walk_kernel(
    const int32_t* __restrict__ cand_idx, const float* __restrict__ cand_val, int64_t n, int m,
    const int32_t* __restrict__ rows, const int32_t* __restrict__ categories, const int32_t* __restrict__ caps,
    int cap_all, int topk, int slots, int32_t* __restrict__ state, int32_t* __restrict__ out_idx,
    float* __restrict__ out_val) {
    const int lane = threadIdx.x & 31;
    const int64_t r = (int64_t)blockIdx.x * CW_WARPS + (threadIdx.x >> 5);
    if (r >= n) return;
    const int64_t row = rows ? rows[r] : r;
    int32_t* st = state + row * (1 + 2 * (int64_t)slots);
    int32_t* tab = st + 1;
    const unsigned mask = (unsigned)slots - 1u;
    const unsigned lt = (1u << lane) - 1u;
    int acc = st[0];
    const int32_t* ci = cand_idx + r * m;
    const float* cv = cand_val + r * m;
    int32_t* oi = out_idx + row * topk;
    float* ov = out_val + row * topk;
    for (int s0 = 0; s0 < m && acc < topk; s0 += 32) {
        const int j = s0 + lane;
        const int32_t c = j < m ? ci[j] : -1;
        const bool valid = c >= 0;
        const int32_t g = valid ? categories[c] : -1;
        const bool capped = g >= 0;
        int slot = 0, cnt = 0, cap = INT_MAX;
        if (capped) {
            slot = cw_probe(tab, g, mask);
            cnt = tab[2 * slot] ? tab[2 * slot + 1] : 0;
            cap = caps ? caps[g] : cap_all;
        }
        // uncapped and invalid lanes form groups of their own kind; only the capped lanes' ranks are read
        const unsigned grp = __match_any_sync(FULL, valid ? g : INT_MIN);
        const int rank = __popc(grp & lt);
        const bool pass = valid && (!capped || cnt + rank < cap);
        const unsigned pass_mask = __ballot_sync(FULL, pass);
        const bool take = pass && acc + __popc(pass_mask & lt) < topk;
        const unsigned take_mask = __ballot_sync(FULL, take);
        if (take) {
            const int at = acc + __popc(take_mask & lt);
            oi[at] = c;
            ov[at] = cv[j];
        }
        // the first taken lane of each capped group writes the group's new count
        const unsigned taken = grp & take_mask;
        const bool leader = capped && take && (taken & lt) == 0;
        if (leader && tab[2 * slot]) tab[2 * slot + 1] = cnt + __popc(taken);
        unsigned fresh = __ballot_sync(FULL, leader && !tab[2 * slot]);
        while (fresh) {
            const int l = __ffs(fresh) - 1;
            if (lane == l) {
                const int s = cw_probe(tab, g, mask);   // again: an earlier lane may have taken the slot
                tab[2 * s] = g + 1;
                tab[2 * s + 1] = __popc(taken);
            }
            __syncwarp();
            fresh &= fresh - 1;
        }
        acc += __popc(take_mask);
    }
    if (lane == 0) st[0] = acc;
}

}  // namespace

extern "C" {

int bfl_category_walk_device(const int32_t* d_cand_idx, const float* d_cand_val, int64_t n, int m,
                             const int32_t* d_rows, const int32_t* d_categories, const int32_t* d_caps, int cap_all,
                             int topk, int slots, int32_t* d_state, int32_t* d_out_idx, float* d_out_val,
                             void* stream) {
    if (BFL_OK != require_device()) return BFL_ERR_CUDA;
    if (n < 0 || m < 1 || topk < 1 || !d_categories || !d_state || !d_out_idx || !d_out_val ||
        (n && (!d_cand_idx || !d_cand_val)) || (!d_caps && cap_all < 0))
        BFL_FAIL(BFL_ERR_ARG, "category walk: bad arguments");
    if (slots < 2 * topk || slots > (1 << 30) || (slots & (slots - 1)))
        BFL_FAIL(BFL_ERR_ARG, "category walk: slots must be a power of two of at least 2 topk");
    if ((n + CW_WARPS - 1) / CW_WARPS > INT_MAX) BFL_FAIL(BFL_ERR_ARG, "category walk: too many rows in one call");
    if (n == 0) return BFL_OK;
    const unsigned blocks = (unsigned)((n + CW_WARPS - 1) / CW_WARPS);
    category_walk_kernel<<<blocks, 32 * CW_WARPS, 0, (cudaStream_t)stream>>>(
        d_cand_idx, d_cand_val, n, m, d_rows, d_categories, d_caps, cap_all, topk, slots, d_state, d_out_idx, d_out_val);
    BFL_LAUNCHED();
    return BFL_OK;
}

}  // extern "C"
