// ALS explanations (explain.cu, DESIGN.md 4.11): the launcher behind bfl_als_explain_device.
#pragma once
#include "bfl_common.cuh"

namespace bfl {

constexpr int EXPLAIN_DMAX = 256;      // the packed lower triangle of A_r fits in shared memory up to here
constexpr int EXPLAIN_KMAX = 4096;     // targets per history row (the serve handle's largest k)
constexpr int EXPLAIN_TOPM_MAX = 64;   // contributions kept per (row, target)

struct ExplainArgs {
    const float* G;          // d x d Gram Q'Q (row-major)
    const float* Q;          // [Q_rows, ld] item factors
    int64_t Q_rows;
    int D, ld;
    float alpha, reg;        // alpha and reg_u of the user half-epoch
    bool adaptive_reg;       // reg * (entries of the row)
    const int64_t* indptr;   // [n] END offsets of the history rows
    const int32_t* keys;     // items in [0, Q_rows), ascending within a row (duplicates adjacent)
    const float* vals;
    int64_t n;
    const int32_t* targets;  // [n, k] item indexes, -1 (or anything outside [0, Q_rows)) for no target
    int k, topm;
    float* scores;           // [n, k]
    int32_t* out_keys;       // [n, k, topm]
    float* out_contrib;      // [n, k, topm]
};

// a.n rows on `st`; arguments are checked by the caller (k, topm and D within the limits above)
int explain_launch(const ExplainArgs& a, int num_sms, cudaStream_t st);

}  // namespace bfl
