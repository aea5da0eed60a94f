/*
 * buffalo_b200.h -- C ABI of the H100-native matrix-factorisation training backend.
 *
 * This is the drop-in boundary: every entry point below replaces one method of the
 * reference's Cython holder classes (the `self.obj` object driven by
 * buffalo/algo/{als,bpr,warp,plsi}.py).  Plain pointers and sizes only -- no torch, numpy or
 * C++ types cross the boundary.  INTEGRATION.md shows the ctypes / Cython stub a
 * reference maintainer would add to bind it.  All file:line citations are relative to
 * the reference repository root.
 *
 * Conventions
 *  - every function returning `int` returns 0 on success and a non-zero code on failure;
 *    bfl_last_error() then returns a thread-local human-readable message.  (The reference
 *    throws std::runtime_error through CHECK_CUDA, include/buffalo/cuda/utils.cuh:24-31;
 *    `init` returns false on an unreadable/invalid option file, lib/algo.cc:22-34.)
 *  - factor matrices are float32 row-major with row pitch `vdim` = bfl_*_get_vdim()
 *    (the reference pads to a multiple of 32, lib/cuda/als/als.cu:251-252; we pad to a
 *    multiple of 4 so rows are 16-byte aligned); padding columns must be zero.
 *  - CSR layout contract (buffalo/data/base.py:187-192): `indptr[x]` is the EXCLUSIVE END
 *    offset of row x (no leading zero), int64; `keys` int32 zero-based opposite index;
 *    `vals` float32.
 *  - "host" entry points take host pointers and perform the H2D/D2H copies themselves,
 *    exactly like the reference CUDA backend (als.cu:361-364,403); "device" entry points
 *    take device pointers (e.g. torch CUDA tensor storage) and run entirely on `stream`.
 *  - there is no CPU fallback: every entry point fails loudly when no sm_90 device is
 *    present.
 */
#ifndef BUFFALO_B200_H_
#define BUFFALO_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BFL_OK 0
#define BFL_ERR_OPTION 1   /* option file missing / not parseable / unsupported value */
#define BFL_ERR_CUDA 2     /* a CUDA runtime call failed */
#define BFL_ERR_STATE 3    /* call sequence violated (e.g. update before initialize_model) */
#define BFL_ERR_ARG 4      /* bad argument */

const char* bfl_last_error(void);
/* library/ABI version and the SM architecture the kernels were compiled for (90) */
int bfl_abi_version(void);
int bfl_compiled_sm(void);
/* BFL_OK when a CUDA device of compute capability 9.0 is current, else BFL_ERR_CUDA with the "no CPU fallback" error:
 * the check every device call makes first, for callers that want it before their own device work */
int bfl_require_device(void);
/* number of kernels this library launched since load (bench.py's gpu_launches claim) */
int64_t bfl_kernel_launch_count(void);
/* Map another process's device allocation into this process with the CURRENT device as accessor
 * (cudaIpcOpenMemHandle + lazy peer access): `handle64` is the 64-byte cudaIpcMemHandle_t exported by the owner.
 * Returns the base address of the allocation (NULL on failure, see bfl_last_error).  Used by the fused multi-GPU
 * exchange; a handle must be opened at most once per process. */
void* bfl_ipc_open(const void* handle64);
int bfl_ipc_close(void* base);
/* Device allocations that can be exported to other processes (plain cudaMalloc, so the IPC handle refers to
 * exactly this buffer): used for the factor replicas of the fused multi-GPU exchange. */
void* bfl_dev_alloc(size_t bytes);
int bfl_dev_free(void* p);
int bfl_ipc_export(void* dev_ptr, void* out_handle64);

/* ======================================================================================
 * ALS  -- replaces CyALS (buffalo/algo/_als.pyx:28-63 -> als::CALS, lib/algo_impl/als/als.cc)
 *         and the CUDA holder (buffalo/algo/cuda/_als.pyx:25-67 -> cuda_als::CuALS,
 *         lib/cuda/als/als.cu)
 * ====================================================================================== */
typedef struct bfl_als bfl_als_t;

/* CyALS.__cinit__ / __dealloc__ (_als.pyx:32-37) */
bfl_als_t* bfl_als_create(void);
void bfl_als_destroy(bfl_als_t* h);

/* CALS::init(opt_path) (als.cc:30-69; CuALS::init als.cu:230-267).  `opt_path` is the JSON
 * option file the Python layer writes (buffalo/algo/base.py:18-24).  Applies the
 * d >= 128 => "ialspp" rule (als.cc:46).  Optimizers: llt, ldlt, manual_cg, ialspp;
 * the Eigen iterative solvers (eigen_cg...eigen_minres, lib/algo.cc:83-127) are rejected
 * with BFL_ERR_OPTION. */
int bfl_als_init(bfl_als_t* h, const char* opt_path);
/* same, from JSON text already in memory */
int bfl_als_init_json(bfl_als_t* h, const char* json_text);

/* CuALS::get_vdim (als.cu:338-340) */
int bfl_als_get_vdim(bfl_als_t* h);

/* CALS::initialize_model(P, P_rows, Q, Q_rows) (als.cc:76-83; CuALS als.cu:269-289).
 * HOST pointers, [rows x vdim] float32.  The pointers are retained (reference semantics):
 * bfl_als_partial_update writes the updated rows back into them. */
int bfl_als_initialize_model(bfl_als_t* h, float* P, int32_t P_rows, float* Q, int32_t Q_rows);

/* CuALS::set_placeholder(lindptr, rindptr, batch_size) (als.cu:291-307): copies both
 * end-offset arrays to the device and sizes the key/value staging buffers. */
int bfl_als_set_placeholder(bfl_als_t* h, const int64_t* lindptr, const int64_t* rindptr, size_t batch_size);

/* CALS::precompute(axis) (als.cc:86-93; als.cu:310-319): FF = Y^T Y of the opposite
 * factor matrix (axis 0 -> Q^T Q). */
int bfl_als_precompute(bfl_als_t* h, int axis);

/* CALS::partial_update(start_x, next_x, indptr, keys, vals, axis) -> pair<double,double>
 * (als.cc:95-105 -> _partial_update :107-209 | _partial_update_ialspp :211-358;
 * CuALS::partial_update als.cu:342-406).  HOST buffers: `indptr` is the global end-offset
 * array, `keys`/`vals` are the chunk buffers starting at row start_x.  Copies the chunk to
 * the device, solves rows [start_x, next_x), copies the updated rows back into the host
 * factor matrix given to initialize_model, returns the loss numerator / denominator. */
int bfl_als_partial_update(bfl_als_t* h, int32_t start_x, int32_t next_x, const int64_t* indptr,
                           const int32_t* keys, const float* vals, int axis,
                           double* loss_nume, double* loss_deno);

/* ---- device-resident path (no reference counterpart: the reference re-uploads every
 * chunk, als.cu:361-364).  Pointers are DEVICE pointers owned by the caller. ---- */
int bfl_als_bind_factors_device(bfl_als_t* h, float* dP, int64_t P_rows, float* dQ, int64_t Q_rows);
/* bind one CSR orientation (axis 0: rowwise/users, 1: colwise/items) resident on device */
int bfl_als_bind_csr_device(bfl_als_t* h, int axis, const int64_t* d_indptr, const int32_t* d_keys,
                            const float* d_vals, int64_t rows, int64_t nnz);
/* FF = Y^T Y on `stream` */
int bfl_als_precompute_device(bfl_als_t* h, int axis, void* stream);
/* partial FF over rows [row_begin,row_end) of the opposite factor (axis 0: rows of Q) -- a row-sharded run computes
 * the Gram of its own freshly solved rows and all-reduces the d x d result (bfl_als_gram_device_mut) instead of every
 * rank recomputing the full matrix (als.cc:86-93 restricted to a row range; SURVEY 8e). */
int bfl_als_precompute_rows_device(bfl_als_t* h, int axis, int64_t row_begin, int64_t row_end, void* stream);
/* solve rows [row_begin, row_end) of the bound CSR `axis` on `stream`; adds the loss pieces
 * into d_loss[0] (numerator), d_loss[1] (denominator) (device doubles, may be NULL). */
int bfl_als_update_device(bfl_als_t* h, int axis, int64_t row_begin, int64_t row_end,
                          double* d_loss, void* stream);
/* multi-GPU fused exchange (no reference counterpart; the reference is single-device): DEVICE pointers, valid in
 * this process (CUDA IPC / peer access), of the OTHER ranks' replicas of the matrix updated on `axis` (P for axis
 * 0, Q for axis 1).  Every solved row is then also stored into those replicas from inside the solve kernel, so the
 * all-gather of the updated shard overlaps the solve row by row; the caller only needs a stream-ordered barrier
 * between half-epochs.  n_peers = 0 switches the fused exchange off.  At most 15 peers. */
int bfl_als_set_peer_replicas(bfl_als_t* h, int axis, int n_peers, float* const* peer_ptrs);

/* Explanations of the exact row solve (csrc/explain.cu, DESIGN.md 4.11).  For n history rows (DEVICE CSR: d_indptr
 * int64 END offsets, d_keys int32 items in [0, Q_rows) ascending within a row (not checked), d_vals float32) and d_targets
 * int32 [n, k] (item indexes; -1 for no target), with A_r = Q'Q + alpha sum v_j q_j q_j' + reg_u kappa I and
 * b_r = sum (1 + alpha v_j) q_j (kappa = the row's entry count with adaptive_reg, else 1), writes
 *   d_scores [n, k]            q_i' A_r^-1 b_r,
 *   d_out_keys [n, k, topm]    the topm history items with the largest (q_i' A_r^-1 q_j)(1 + alpha v_j), entries of
 *                              one item summed, descending, ties to the smaller item; -1 pads,
 *   d_out_contrib [n, k, topm] those contributions; 0.0 pads.
 * A -1 target or an empty row gives score 0.0 and keys -1.  A non-positive Cholesky pivot of A_r gives NaN scores and
 * keys -1 for that row only.  Reads the bound Q, the Gram of the last bfl_als_precompute_device(axis 0) (else
 * BFL_ERR_STATE), alpha, reg_u and adaptive_reg.  k in [1, 4096], topm in [1, 64], d <= 256, else BFL_ERR_ARG.  No
 * atomics: a row's outputs do not depend on the other rows of the call. */
int bfl_als_explain_device(bfl_als_t* h, const int64_t* d_indptr, const int32_t* d_keys, const float* d_vals, int64_t n,
                           const int32_t* d_targets, int k, int topm, float* d_scores, int32_t* d_out_keys,
                           float* d_out_contrib, void* stream);

/* Posterior draws of the exact row solve (csrc/explain.cu, DESIGN.md 4.17).  For n history rows (DEVICE CSR: d_indptr
 * int64 END offsets, d_keys int32 items in [0, Q_rows) ascending within a row (not checked), d_vals float32), with
 * A_r = Q'Q + alpha sum v_j q_j q_j' + reg_u kappa I = L L' (kappa = the row's entry count with adaptive_reg, else 1;
 * an empty row gives Q'Q + reg_u kappa I), writes
 *   d_out [n, ld]              d_mean[r] + scale L^-T z_r in columns [0, d) (columns d..ld-1 are not written),
 * where ld >= d is the row pitch of d_mean and d_out only (Q is read at the handle's own pitch),
 * one draw from N(mean_r, scale^2 A_r^-1).  z_r ~ N(0, I) is Box-Muller on the Philox words
 * draw_u32(seed, 0x54530417, d_draw_keys[r], t) (int64 [n], non-negative), so a row's draw depends only on the seed,
 * its key, its history, its mean, Q, the Gram and the options, not on the other rows of the call.  d_out may be d_mean.
 * scale = 0 copies the mean.  A row whose A_r meets a non-positive or NaN Cholesky pivot is written as its mean and
 * counted: *d_failed (a device int64) += the number of such rows.  Reads the bound Q, the Gram of the last
 * bfl_als_precompute_device(axis 0) (else BFL_ERR_STATE), alpha, reg_u and adaptive_reg.  d <= 256, ld >= d and a
 * finite scale >= 0, else BFL_ERR_ARG.  No atomics. */
int bfl_als_posterior_sample_device(bfl_als_t* h, const int64_t* d_indptr, const int32_t* d_keys, const float* d_vals,
                                    int64_t n, const float* d_mean, int ld, const int64_t* d_draw_keys, uint32_t seed,
                                    float scale, float* d_out, int64_t* d_failed, void* stream);

/* device pointer of the current Gram matrix [d x d] (tests) */
const float* bfl_als_gram_device(bfl_als_t* h);
/* multi-GPU: when several ranks each computed the Gram of their shard of Y, the host
 * all-reduces this buffer (d*d floats) before bfl_als_update_device. */
float* bfl_als_gram_device_mut(bfl_als_t* h);

/* ======================================================================================
 * BPRMF / WARP -- replaces CyBPRMF / CyWARP (buffalo/algo/_bpr.pyx:34-92, _warp.pyx:34-92 ->
 * bpr::CBPRMF lib/algo_impl/bpr/bpr.cc, warp::CWARP lib/algo_impl/warp/warp.cc, both on
 * SGDAlgorithm lib/algo.cc:133-492) and the CUDA holder CyBPR (buffalo/algo/cuda/_bpr.pyx:27-80
 * -> cuda_bpr::CuBPR lib/cuda/bpr/bpr.cu).  The reference has no CUDA WARP (warp.py:30-32).
 * ====================================================================================== */
typedef struct bfl_sgd bfl_sgd_t;

#define BFL_SGD_BPR 0
#define BFL_SGD_WARP 1

bfl_sgd_t* bfl_sgd_create(int kind);
void bfl_sgd_destroy(bfl_sgd_t* h);

/* CBPRMF::init / CWARP::init (bpr.cc:39-47, warp.cc:71-88) */
int bfl_sgd_init(bfl_sgd_t* h, const char* opt_path);
int bfl_sgd_init_json(bfl_sgd_t* h, const char* json_text);
int bfl_sgd_get_vdim(bfl_sgd_t* h);

/* SGDAlgorithm::initialize_model(P, P_rows, Q, Q_rows, Qb, num_total_samples)
 * (algo.cc:148-176; CuBPR bpr.cu:284-312).  HOST pointers; retained; synchronised back by
 * bfl_sgd_synchronize(h, 1) / bfl_sgd_update_parameters.  Allocates gradient / momentum /
 * velocity state unless optimizer == "sgd" (algo.cc:221-254). */
int bfl_sgd_initialize_model(bfl_sgd_t* h, float* P, int32_t P_rows, float* Q, int32_t Q_rows,
                             float* Qb, int64_t num_total_samples);
/* device-resident variant: caller-owned DEVICE pointers, nothing is copied back */
int bfl_sgd_bind_factors_device(bfl_sgd_t* h, float* dP, int64_t P_rows, float* dQ, int64_t Q_rows,
                                float* dQb, int64_t num_total_samples);

/* CBPRMF::set_cumulative_table(cum_table, size) (bpr.cc:66-70): HOST int64[size]; copied. */
int bfl_sgd_set_cumulative_table(bfl_sgd_t* h, const int64_t* cum_table, int32_t size);

/* CuBPR::set_placeholder(indptr, batch_size) (bpr.cu:314-325) */
int bfl_sgd_set_placeholder(bfl_sgd_t* h, const int64_t* indptr, size_t batch_size);
/* bind a device-resident rowwise CSR (keys only) */
int bfl_sgd_bind_csr_device(bfl_sgd_t* h, const int64_t* d_indptr, const int32_t* d_keys,
                            int64_t rows, int64_t nnz);

/* SGDAlgorithm::launch_workers / wait_until_done / join (algo.cc:211-219,467-492): the GPU
 * path is stream-ordered, so these only synchronise. */
int bfl_sgd_launch_workers(bfl_sgd_t* h);
int bfl_sgd_wait_until_done(bfl_sgd_t* h);
int bfl_sgd_join(bfl_sgd_t* h, double* out);

/* SGDAlgorithm::add_jobs(start_x, next_x, indptr, positives) (algo.cc:308-362) followed by
 * the work CBPRMF::worker / CWARP::worker would do for those rows (bpr.cc:72-188,
 * warp.cc:103-173; CuBPR::partial_update bpr.cu:350-430).  HOST buffers. */
int bfl_sgd_add_jobs(bfl_sgd_t* h, int32_t start_x, int32_t next_x, const int64_t* indptr,
                     const int32_t* keys);
/* same over rows [row_begin,row_end) of the bound device CSR, on `stream` */
int bfl_sgd_add_jobs_device(bfl_sgd_t* h, int64_t row_begin, int64_t row_end, void* stream);

/* SGDAlgorithm::update_parameters (algo.cc:382-465) + CWARP projection (warp.cc:192-201);
 * on the host-pointer path it also copies P,Q,Qb back (cuda/_bpr.pyx:60-61). */
int bfl_sgd_update_parameters(bfl_sgd_t* h);
int bfl_sgd_update_parameters_device(bfl_sgd_t* h, void* stream);
/* CuBPR::synchronize(device_to_host) (bpr.cu:327-348) */
int bfl_sgd_synchronize(bfl_sgd_t* h, int device_to_host);

/* CBPRMF::compute_loss / CWARP::compute_loss (bpr.cc:227-244, warp.cc:205-226).  HOST int32[n]. */
int bfl_sgd_compute_loss(bfl_sgd_t* h, int32_t n, const int32_t* users, const int32_t* positives,
                         const int32_t* negatives, double* out_loss);

/* ---- test hooks (deterministic parity): explicit triples, gradient read-back ---- */
/* apply the BPR update to explicit DEVICE triples (what add_jobs does after sampling) */
int bfl_sgd_apply_triples_device(bfl_sgd_t* h, const int32_t* d_users, const int32_t* d_pos,
                                 const int32_t* d_neg, int64_t n, float lr, void* stream);
/* sample BPR triples for rows [row_begin,row_end) of the bound CSR into DEVICE arrays */
int bfl_sgd_sample_device(bfl_sgd_t* h, int64_t row_begin, int64_t row_end, int32_t* d_users,
                          int32_t* d_pos, int32_t* d_neg, void* stream);
/* device pointers of the gradient accumulators (NULL for optimizer == sgd) */
float* bfl_sgd_grad_device(bfl_sgd_t* h, int which /*0 P, 1 Q, 2 Qb*/);
/* device pointers of the per-row sample counters used by per_coordinate_normalize (algo.cc:398-413; int32[rows]).
 * Together with the gradient accumulators these are what a row-sharded multi-GPU epoch all-reduces before
 * update_parameters (SURVEY 8e). */
int32_t* bfl_sgd_count_device(bfl_sgd_t* h, int which /*0 P rows, 1 Q rows*/);
/* WARP: per-positive trial counts / chosen negatives of the last add_jobs (device int32[nnz]) */
int bfl_sgd_set_trace_device(bfl_sgd_t* h, int32_t* d_trials, int32_t* d_negs);
/* current epoch counter / decayed learning rate (algo.cc:284-287) */
int bfl_sgd_epoch(bfl_sgd_t* h);
double bfl_sgd_current_lr(bfl_sgd_t* h);
int bfl_sgd_read_stats(bfl_sgd_t* h, double* loss_sum, int64_t* num_updates);
/* Deterministic mode (option `deterministic`): the item pass over the samples recorded since the last one -- adds every
 * item's gradient sum to the Q / Qb accumulators in the fixed order and the WARP loss terms to the running loss sum.
 * update_parameters runs it first, so it is only needed to read the epoch's accumulators before the optimizer step
 * (or to all-reduce them across ranks).  BFL_ERR_STATE without the option. */
int bfl_sgd_reduce_items_device(bfl_sgd_t* h, void* stream);
/* samples / item entries per segment of the deterministic user and item sums */
int bfl_sgd_segment_len(void);
/* Item fold-in (DESIGN.md 4.16): `epochs` epochs of the item side of training for n new rows, with the trained factors
 * frozen.  Uses the holder's options only (init() must have succeeded; no factors need to be bound).  All arrays are
 * DEVICE memory:
 *   dP [P_rows, vdim], dQ [Q_rows, vdim], dQb [Q_rows]     the trained factors, read only;
 *   d_train_indptr int64 [P_rows] END offsets, d_train_keys  the training data's rowwise CSR, each row ascending
 *                                                          (the negatives' seen check);
 *   d_cum int64 [Q_rows] or NULL                           BPR popularity table (NULL: uniform negatives);
 *   d_hist_indptr int64 [n] END offsets, d_hist_users int32 [hist_nnz]   the new rows' users, ascending per row;
 *   dX [n, vdim], dXb [n]                                  start rows and biases in, folded rows and biases out.
 * d_trace_negs (int32 [epochs, hist_nnz * samples per positive]) and, for WARP, d_trace_trials (int32 [epochs,
 * hist_nnz]) are optional records of the draws: the negative of each sample (-1 for a WARP discard) and WARP's trial
 * count (0 for a discard).  Each row's result depends only on its history, start row and index: no atomics. */
int bfl_sgd_fold_in_items_device(bfl_sgd_t* h, const float* dP, int64_t P_rows, const float* dQ, const float* dQb,
                                 int64_t Q_rows, const int64_t* d_train_indptr, const int32_t* d_train_keys,
                                 const int64_t* d_cum, const int64_t* d_hist_indptr, const int32_t* d_hist_users,
                                 int64_t n, int64_t hist_nnz, float* dX, float* dXb, int epochs,
                                 int32_t* d_trace_negs, int32_t* d_trace_trials, void* stream);

/* ======================================================================================
 * PLSI -- replaces CyPLSI (buffalo/algo/_plsi.pyx:13-57 -> plsi::CPLSI, lib/algo_impl/plsi/plsi.cc)
 *
 * One iteration is reset -> partial_update per rowwise chunk -> normalize -> swap (buffalo/algo/plsi.py:132-160).
 * The new user rows are written over the current ones on the device as the pass goes (only a row's own update
 * reads it); the new item rows accumulate in a library-owned matrix.  Each user row must be updated at most once
 * between reset and normalize; a row the pass never reached counts as zero in normalize, like the reference's
 * zeroed accumulator.  The holder path keeps its own device copy of the factors: changes the caller makes to the
 * host arrays take effect through bfl_plsi_set_model.
 * ====================================================================================== */
typedef struct bfl_plsi bfl_plsi_t;

/* CyPLSI.__cinit__ / __dealloc__ */
bfl_plsi_t* bfl_plsi_create(void);
void bfl_plsi_destroy(bfl_plsi_t* h);
/* CPLSI::init(opt_path) (plsi.cc:21-30): d in [1, 512] (else BFL_ERR_OPTION), random_seed */
int bfl_plsi_init(bfl_plsi_t* h, const char* opt_path);
int bfl_plsi_init_json(bfl_plsi_t* h, const char* json_text);
/* device row pitch of the factor matrices: ceil4(d) */
int bfl_plsi_get_vdim(bfl_plsi_t* h);
/* CPLSI::initialize_model(P, P_rows, Q, Q_rows) (plsi.cc:44-70).  HOST pointers, [rows x d] float32 (not padded),
 * retained.  Fills them with |N(0, 1/d)| drawn on the device from Philox4x32-10 keyed by (random_seed, matrix,
 * element), then divides every P row by its sum and every Q column by its sum. */
int bfl_plsi_initialize_model(bfl_plsi_t* h, float* P, int32_t P_rows, float* Q, int32_t Q_rows);
/* retain and upload the caller's current [rows x d] arrays without drawing (no reference counterpart: the
 * reference reads the caller's arrays directly, so inherited or replaced factors need this here) */
int bfl_plsi_set_model(bfl_plsi_t* h, float* P, int32_t P_rows, float* Q, int32_t Q_rows);
/* CPLSI::reset (plsi.cc:40-42): zero the item accumulator and the record of updated rows */
int bfl_plsi_reset(bfl_plsi_t* h);
/* CPLSI::partial_update(start_x, next_x, indptr, keys, vals) (plsi.cc:72-106).  HOST buffers: `indptr` is the
 * global end-offset array, `keys` / `vals` the chunk starting at row start_x.  *loss receives -sum v log(norm) of
 * the chunk (fp64). */
int bfl_plsi_partial_update(bfl_plsi_t* h, int32_t start_x, int32_t next_x, const int64_t* indptr,
                            const int32_t* keys, const float* vals, double* loss);
/* Deterministic mode (option "deterministic": true): the same inputs give bitwise the same factors and loss.  An
 * iteration is reset -> partial_update_items per colwise chunk -> partial_update per rowwise chunk -> normalize ->
 * swap.  The item pass builds the new item rows from the colwise CSR and the CURRENT P and Q, so it must come before
 * the row pass of its iteration (after it: BFL_ERR_STATE); partial_update then leaves the item rows alone, and its
 * *loss is a fixed-order sum.  HOST buffers with the conventions of partial_update: `indptr` is the global colwise
 * end-offset array, `keys` (user rows) / `vals` the chunk starting at item start_x.  Without the option: BFL_ERR_STATE. */
int bfl_plsi_partial_update_items(bfl_plsi_t* h, int32_t start_x, int32_t next_x, const int64_t* indptr,
                                  const int32_t* keys, const float* vals);
/* entries per segment of a long item row in the deterministic item pass (a compile-time constant) */
int bfl_plsi_item_segment_len(void);
/* CPLSI::normalize(alpha1, alpha2) (plsi.cc:108-125): alpha1 /= d, alpha2 /= num_items, then every P row
 * (+alpha1) and every Q column (+alpha2) is divided by its sum.  Column sums are fp64 and deterministic. */
int bfl_plsi_normalize(bfl_plsi_t* h, float alpha1, float alpha2);
/* CPLSI::swap (plsi.cc:127-130): the new factors become current and are copied into the retained host arrays */
int bfl_plsi_swap(bfl_plsi_t* h);
/* CPLSI::release (plsi.cc:36-38): free the device state */
int bfl_plsi_release(bfl_plsi_t* h);

/* ---- device-resident path: caller-owned DEVICE pointers, [rows x vdim] factors, work on `stream` ---- */
int bfl_plsi_bind_factors_device(bfl_plsi_t* h, float* dP, int64_t P_rows, float* dQ, int64_t Q_rows);
/* the rowwise CSR (rows == P_rows) */
int bfl_plsi_bind_csr_device(bfl_plsi_t* h, const int64_t* d_indptr, const int32_t* d_keys, const float* d_vals,
                             int64_t rows, int64_t nnz);
/* update rows [row_begin, row_end); adds -sum v log(norm) into d_loss[0] (device double, may be NULL).  In
 * deterministic mode the row pass leaves the item rows alone and the loss is a fixed-order sum over the range. */
int bfl_plsi_update_device(bfl_plsi_t* h, int64_t row_begin, int64_t row_end, double* d_loss, void* stream);
/* deterministic mode: the colwise CSR (rows == Q_rows, else BFL_ERR_ARG), bound after the factors.  Its END offsets
 * are read once here to list the items longer than one segment and to size their partial rows. */
int bfl_plsi_bind_colwise_csr_device(bfl_plsi_t* h, const int64_t* d_indptr, const int32_t* d_keys,
                                     const float* d_vals, int64_t rows, int64_t nnz);
/* deterministic mode: the item pass over items [item_begin, item_end) of the colwise CSR; runs before
 * bfl_plsi_update_device in each iteration (after it: BFL_ERR_STATE until swap_device) */
int bfl_plsi_update_items_device(bfl_plsi_t* h, int64_t item_begin, int64_t item_end, void* stream);
int bfl_plsi_normalize_device(bfl_plsi_t* h, float alpha1, float alpha2, void* stream);
/* copy the new item factors into dQ and zero the accumulator for the next iteration (no separate reset) */
int bfl_plsi_swap_device(bfl_plsi_t* h, void* stream);
/* Folding-in (DESIGN.md 4.10): `iters` EM iterations on each of `rows` user rows with the item factors fixed.  Per
 * iteration a row becomes the row pass's sum of v * l / sum(l), l = max(x * q, 1e-10), then (acc + alpha1 / d) divided
 * by its sum over the d columns, as bfl_plsi_normalize does (alpha1 is passed undivided, like there).  DEVICE arrays,
 * stream-ordered: d_Q [Q_rows x vdim] and d_X [rows x vdim] 16-byte aligned, padding columns zero; d_indptr[rows] END
 * offsets from 0, d_keys items in [0, Q_rows) (not checked), d_vals.  d_X holds the start rows in and the results out;
 * rows without entries keep their start row.  Uses only the handle's options (d), not its factors or CSR; no atomics,
 * so the same inputs give the same bits. */
int bfl_plsi_fold_in_device(bfl_plsi_t* h, const float* d_Q, int64_t Q_rows, const int64_t* d_indptr,
                            const int32_t* d_keys, const float* d_vals, int64_t rows, int64_t nnz, float* d_X, int iters,
                            float alpha1, void* stream);

/* =====================================================================================
 * Evaluation top-k (SURVEY.md 8(f-2)); replaces the host quickselect behind Evaluable.get_topk /
 * Algo._get_topk_recommendation (buffalo/evaluate/base.py:31-42, buffalo/parallel/_core.hpp:69-142):
 * scores = queries . items^T (+ item_bias), the k best item indices per query, best first; ties go to the
 * smaller index; -1 pads when there are fewer than k items.  k <= 4096.
 * ===================================================================================== */
/* device pointers, stream-ordered */
int bfl_topk_device(const float* d_queries, int64_t nq, int ldq, const float* d_items, int64_t n_items, int ldi,
                    const float* d_item_bias /* nullable */, int d, int k, int32_t* d_out_idx, float* d_out_val,
                    void* stream);
/* host pointers (copies in, runs, copies out); out_val may be NULL */
int bfl_topk_host(const float* queries, int64_t nq, int ldq, const float* items, int64_t n_items, int ldi,
                  const float* item_bias /* nullable */, int d, int k, int32_t* out_idx, float* out_val);

/* =====================================================================================
 * Batch serving top-k (DESIGN.md 4.9); the device path of buffalo.parallel's ParALS / ParBPRMF
 * (dot_topn, buffalo/parallel/_core.hpp:88-142).  A handle keeps the item factors (and bias) and the query factors
 * resident on the device and answers "the k best items for these n query rows" for any n:
 *  - score = query . item (+ item_bias), best first, ties to the smaller item id, -1 / 0.0f where fewer than k
 *    candidates exist; k <= 4096, row counts < 2^31.  Keys and scores are bitwise those of bfl_topk_device on the same
 *    rows (same row pitches).
 *  - set_items / set_queries upload HOST arrays once; bind_*_device borrow caller-owned DEVICE memory that must stay
 *    valid while the handle uses it.  Items first: setting or binding the items clears the pool AND the queries (topk
 *    is BFL_ERR_STATE until the queries are set again); the queries must have at least the items' width.  Device item
 *    rows of a multiple of 4 floats (ld and d) must be 16-byte aligned.  set_queries with the very array given to
 *    set_items (same rows, same ld) shares the resident copy (most_similar).
 *  - set_pool restricts the candidates to HOST indices into the item matrix (any order, duplicates allowed: candidates
 *    rank as the rows of items[pool] would, ties to the smaller pool position); results carry item ids.  NULL removes
 *    the pool; an empty pool or an index outside the items is BFL_ERR_ARG.
 *  - topk: HOST query_idx[n] (rows of the query matrix), HOST out_idx [n x k] and out_val [n x k] (nullable).  The call
 *    is cut into batches; a batch's result is copied out through two pinned buffers while the next batch runs.
 *  - topk_device: DEVICE arrays, stream-ordered on `stream`; indices outside the query matrix read as zero rows.
 *  A handle serves one call at a time: topk and topk_device use scratch buffers the handle owns and grows on demand, so
 *  calls on one handle must not overlap, on any stream or thread (use one handle per concurrent caller).
 *  The handle owns two streams and its pinned buffers and starts no thread; destroy releases all of it.
 * ===================================================================================== */
typedef struct bfl_serve bfl_serve_t;
bfl_serve_t* bfl_serve_create(void);
void bfl_serve_destroy(bfl_serve_t* h);
int bfl_serve_set_items(bfl_serve_t* h, const float* items, int64_t n_items, int ld, int d,
                        const float* item_bias /* nullable */);
int bfl_serve_bind_items_device(bfl_serve_t* h, const float* d_items, int64_t n_items, int ld, int d,
                                const float* d_item_bias /* nullable */);
int bfl_serve_set_queries(bfl_serve_t* h, const float* queries, int64_t n_q, int ld);
int bfl_serve_bind_queries_device(bfl_serve_t* h, const float* d_queries, int64_t n_q, int ld);
int bfl_serve_set_pool(bfl_serve_t* h, const int32_t* pool_idx /* nullable */, int64_t n_pool);
int bfl_serve_topk(bfl_serve_t* h, const int32_t* query_idx, int64_t n, int k, int32_t* out_idx,
                   float* out_val /* nullable */);
int bfl_serve_topk_device(bfl_serve_t* h, const int32_t* d_query_idx, int64_t n, int k, int32_t* d_out_idx,
                          float* d_out_val, void* stream);

/* =====================================================================================
 * Batch serving top-k without each query's seen items (DESIGN.md 4.9), on a serve handle: what bfl_serve_topk /
 * bfl_serve_topk_device return with the query's seen items left out of its candidates (with a pool: the pool's
 * candidates whose item is seen).  The survivors keep their order, keys and score bits; -1 / 0.0f pad when fewer
 * than k candidates remain.  The seen rows are arguments of the call, so nothing of them stays on the handle.
 *  - seen_topk: HOST arrays.  seen_indptr[n] END offsets (row i holds the items of query i: seen_keys[seen_indptr[i - 1]
 *    .. seen_indptr[i]), from 0), keys in [0, n_items), any order, duplicates allowed.  Each batch's rows are staged
 *    through two pinned buffers and uploaded next to it; rows not in ascending order are sorted on the device.  A
 *    batch also holds at most 2^24 seen keys (a longer row is a batch of its own).  Non-monotone offsets or a key out
 *    of range is BFL_ERR_ARG before any device work.
 *  - seen_topk_device: DEVICE arrays, stream-ordered; query q reads row d_seen_row[q] of the CSR (END offsets, rows
 *    non-decreasing: the caller sorts them, e.g. with bfl_csr_from_triples_device).
 * ===================================================================================== */
int bfl_seen_topk(bfl_serve_t* h, const int32_t* query_idx, int64_t n, int k, const int64_t* seen_indptr,
                  const int32_t* seen_keys, int32_t* out_idx, float* out_val /* nullable */);
int bfl_seen_topk_device(bfl_serve_t* h, const int32_t* d_query_idx, int64_t n, int k, const int64_t* d_seen_indptr,
                         const int32_t* d_seen_keys, const int32_t* d_seen_row, int32_t* d_out_idx, float* d_out_val,
                         void* stream);

/* =====================================================================================
 * Batch serving top-k over a candidate list per query (DESIGN.md 4.13), on a serve handle: query i ranks only the
 * items of its own list (item ids in any order, duplicates allowed), and row i of the result is bitwise what
 * bfl_serve_topk (with seen rows: bfl_seen_topk) returns for that query alone with its list set as the pool: the same
 * scores, item ids best first, ties to the earlier list position.  A query whose list is empty, or holds fewer than k
 * candidates once its seen items are left out, gets -1 / 0.0f padding; that is not an error.  The handle's pool is not
 * used.  k in [1, 4096].  Lists and seen rows are arguments of the call, so nothing of them stays on the handle.
 *  - cand_topk: HOST arrays.  cand_indptr[n] END offsets (row i holds the list of query i: cand_keys[cand_indptr[i - 1]
 *    .. cand_indptr[i]), from 0), keys in [0, n_items); seen rows (nullable) as bfl_seen_topk takes them.  Batches hold
 *    at most 2^24 list entries (bfl_cand_set_budget changes that; a longer row is a batch of its own) and the rows
 *    bfl_serve_topk would batch; each batch's lists are staged through two pinned buffers and uploaded while the
 *    previous batch runs.  Non-monotone offsets or a key out of range is BFL_ERR_ARG before any device work.
 *  - cand_topk_device: DEVICE arrays, stream-ordered on `stream`; query q reads row d_cand_row[q] of the candidate CSR
 *    (d_cand_row nullable: row q) and row d_seen_row[q] of the seen CSR (d_seen_indptr nullable: no seen rows;
 *    d_seen_row nullable: row q; rows non-decreasing).  Keys must be in [0, n_items).  The call synchronises `stream`
 *    once per internal batch to size its scratch.  d_out_val nullable.
 *  - cand_set_budget: list entries per batch of cand_topk (0: the default).
 * ===================================================================================== */
int bfl_cand_topk(bfl_serve_t* h, const int32_t* query_idx, int64_t n, int k, const int64_t* cand_indptr,
                  const int32_t* cand_keys, const int64_t* seen_indptr /* nullable */, const int32_t* seen_keys,
                  int32_t* out_idx, float* out_val /* nullable */);
int bfl_cand_topk_device(bfl_serve_t* h, const int32_t* d_query_idx, int64_t n, int k, const int64_t* d_cand_indptr,
                         const int32_t* d_cand_keys, const int32_t* d_cand_row /* nullable */,
                         const int64_t* d_seen_indptr /* nullable */, const int32_t* d_seen_keys,
                         const int32_t* d_seen_row /* nullable */, int32_t* d_out_idx,
                         float* d_out_val /* nullable */, void* stream);
int bfl_cand_set_budget(bfl_serve_t* h, int64_t list_entries);

/* =====================================================================================
 * Maximal Marginal Relevance re-ranking (DESIGN.md 4.15), on a serve handle: per row, k of its m candidates picked
 * greedily for relevance against similarity to the items already picked, the diversify option of ParALS / ParBPRMF
 * topk_recommendation.  Row i's candidates are d_cand_idx[i * m .. i * m + m) (item ids in [0, n_items), -1 pads;
 * duplicates are ordinary candidates) with their scores d_cand_val (what bfl_serve_topk_device, bfl_seen_topk_device
 * or bfl_cand_topk_device return at k = m).  Over the row's valid candidates:
 *  - rel_j = (s_j - s_min) / (s_max - s_min) in fp64, 1 when all scores are equal;
 *  - cos(a, b) of the item rows the handle holds (its ld and d, no bias): fp32 dot products in the fixed tiled order of
 *    bfl_eval_ild_device, the cosine in fp64, 0 when either row has zero norm;
 *  - step t = 0 .. k - 1 picks the unpicked candidate of the largest (1 - w) rel_j - w max_{p picked} cos(p, j) (the
 *    max term left out at t = 0), ties to the smaller position.
 * d_out_idx / d_out_val [n x k]: the picks in pick order with their scores bitwise as given (not sorted), -1 / 0.0f
 * once the valid candidates run out.  diversify = 0 returns the first k candidates of a best-first list.  A row's
 * output depends on that row alone.  1 <= k <= m <= 256, 0 <= diversify <= 1, n < 2^31; a bad argument is
 * BFL_ERR_ARG before any launch, a handle without items BFL_ERR_STATE.  DEVICE arrays, stream-ordered on `stream`;
 * nothing is uploaded and no scratch is allocated.
 * ===================================================================================== */
int bfl_mmr_rerank_device(bfl_serve_t* h, const int32_t* d_cand_idx, const float* d_cand_val, int64_t n, int m,
                          int k, float diversify, int32_t* d_out_idx, float* d_out_val, void* stream);

/* =====================================================================================
 * Per-category caps over ranked lists (DESIGN.md 4.18): the walk of ParALS / ParBPRMF topk_recommendation(categories,
 * category_cap) and buffalo_b200.parallel.cap_categories.  Row r of the candidates, d_cand_idx / d_cand_val
 * [r * m .. r * m + m) (item ids best first, -1 entries skipped, with their scores), continues the walk of state and
 * output row d_rows[r] (d_rows nullable: row r): in order, an item is accepted when its category d_categories[item] is
 * -1 or fewer than its cap items of that category are accepted already, until topk are accepted.  The cap of category
 * g is d_caps[g] (d_caps nullable: cap_all for every category); every category of a candidate must be in [-1, C) for
 * d_caps of C entries.  Accepted items go to d_out_idx / d_out_val [rows x topk] at the row's next free places with
 * their score bits; the caller fills those with -1 / 0.0f before the first call.  d_state [rows x (1 + 2 slots)] int32
 * holds per row the accepted count and an open-addressed table of `slots` (category + 1, count) pairs; the caller
 * zero-fills it before the first call.  slots: a power of two of at least 2 topk.  So calls over consecutive parts of
 * one ranking give what one call over the whole ranking gives, and a row's result depends on its own candidates alone.
 * One warp per row, no atomics.  Bad arguments are BFL_ERR_ARG before any launch.  DEVICE arrays, stream-ordered.
 * ===================================================================================== */
int bfl_category_walk_device(const int32_t* d_cand_idx, const float* d_cand_val, int64_t n, int m,
                             const int32_t* d_rows /* nullable */, const int32_t* d_categories,
                             const int32_t* d_caps /* nullable */, int cap_all, int topk, int slots, int32_t* d_state,
                             int32_t* d_out_idx, float* d_out_val, void* stream);

/* =====================================================================================
 * Inverted-file (IVF-Flat) index for batch serving (DESIGN.md 4.12).  build_device clusters n DEVICE rows (pitch ld,
 * first d columns, d <= 256) by spherical k-means into nlist lists (nlist in [1, min(n, 65536)], iters >= 1): nlist
 * distinct rows drawn with `seed` start it, each row goes to the centroid of the largest dot product (ties to the
 * smaller list), a centroid becomes the normalised sum of its members' unit rows (an empty list keeps its centroid).
 * The handle keeps the centroids, the lists (END offsets, row ids ascending) and list-major copies of the rows and of
 * the bias (d_bias nullable), so the caller's arrays may be freed after the call.  The same arguments and seed give a
 * bitwise equal index.
 *  - search_device: DEVICE queries [n x ldq] (ldq >= d) -> d_out_idx / d_out_val [n x k] (row ids best first, -1 /
 *    0.0f padding): per query the k best of the rows of the nprobe lists whose centroids score best (ties to the
 *    smaller list), each score bitwise that of bfl_serve_topk on the same rows and bias (use_bias), ties to the smaller
 *    row id.  nprobe = nlist returns bfl_serve_topk's result.  nprobe in [1, nlist], and at most 4096 unless it is
 *    nlist; k in [1, 4096].  The call synchronises `stream` first and returns when the results are written.
 *  - attach: binds the handle to the current device (BFL_ERR_CUDA without a Hopper GPU); build and search attach too.
 *  - set_batch_rows: queries per internal batch at most (0: chosen from the candidate scratch).
 *  - info / read: the index's shape; HOST copies of the centroids [nlist x ld], the END offsets [nlist] and the row
 *    ids [n] (each nullable).
 *  One call at a time per handle.  The handle owns one stream and a serve handle over the centroids and starts no
 *  thread; destroy releases all of it.  Argument errors are BFL_ERR_ARG, calls before a build BFL_ERR_STATE.
 * ===================================================================================== */
typedef struct bfl_ivf bfl_ivf_t;
bfl_ivf_t* bfl_ivf_create(void);
void bfl_ivf_destroy(bfl_ivf_t* h);
int bfl_ivf_attach(bfl_ivf_t* h);
int bfl_ivf_build_device(bfl_ivf_t* h, const float* d_rows, int64_t n, int ld, int d,
                         const float* d_bias /* nullable */, int nlist, int iters, uint64_t seed);
int bfl_ivf_search_device(bfl_ivf_t* h, const float* d_queries, int64_t n, int ldq, int nprobe, int k, int use_bias,
                          int32_t* d_out_idx, float* d_out_val, void* stream);
int bfl_ivf_set_batch_rows(bfl_ivf_t* h, int64_t rows);
int bfl_ivf_info(bfl_ivf_t* h, int64_t* n, int* nlist, int* ld, int* d);
int bfl_ivf_read(bfl_ivf_t* h, float* centroids /* nullable */, int64_t* offsets /* nullable */,
                 int32_t* ids /* nullable */);

/* =====================================================================================
 * Validation metrics on the device (DESIGN.md 4.8): the device path of Evaluable.get_validation_results
 * (buffalo/evaluate/base.py:44-148).  Device pointers, stream-ordered.  A "seen" CSR (END offsets, int32 keys, every
 * row non-decreasing) holds training rows; seen_row[q] names the row of query q.  The held-out CSR is indexed by user.
 *  - unsorted_rows: *d_count (device u64) = number of rows whose keys are not non-decreasing.
 *  - topk_masked: per query q, the k best items (score = queries[q] . items^T (+ item_bias), bitwise the scores of
 *    bfl_topk_device for the same arguments) among the items not in seen row seen_row[q]; score descending, then item
 *    ascending; -1 pads when fewer than k such items exist.  k <= 4096, n_items < 2^31.
 *  - ranking_terms: per query, from its ranked list (d_ranked [nq x k]) and held-out row of user d_users[q], the fp64
 *    terms (ndcg, ap / min(n_pos, k), accuracy, auc / (n_pos * n_neg), counted, no-negative) into d_terms [nq x 6];
 *    a query whose seen row is empty gets zeros.  d_gains / d_ideal: the host's 1 / log2(j + 2) and its prefix sums.
 *  - score_terms: per held-out triple, score = mode 0 (P[r] * Q[c]).sum(), 1 the same + Qb[c], 2 1 - ((P[r] - Q[c])^2).sum()
 *    in NumPy's float32 order (rows of `width` floats), err = score - val in fp64: d_terms [n x 2] = (err^2, |err|).
 *  - sum: column sums of d_terms [n x width] (width <= 8) into d_out[width], in a fixed order.
 * ===================================================================================== */
int bfl_eval_unsorted_rows_device(const int64_t* d_indptr, const int32_t* d_keys, int64_t rows,
                                  unsigned long long* d_count, void* stream);
int bfl_eval_topk_masked_device(const float* d_queries, int64_t nq, int ldq, const float* d_items, int64_t n_items,
                                int ldi, const float* d_item_bias /* nullable */, int d, int k,
                                const int64_t* d_seen_indptr, const int32_t* d_seen_keys, const int32_t* d_seen_row,
                                int32_t* d_out_idx, void* stream);
int bfl_eval_ranking_terms_device(const int32_t* d_ranked, int64_t nq, int k, const int32_t* d_users,
                                  const int64_t* d_seen_indptr, const int32_t* d_seen_row, const int64_t* d_gt_indptr,
                                  const int32_t* d_gt_keys, const double* d_gains, const double* d_ideal,
                                  int64_t num_items, double* d_terms, void* stream);
int bfl_eval_score_terms_device(const float* d_P, const float* d_Q, const float* d_Qb /* mode 1 */, int width, int mode,
                                const int32_t* d_rows, const int32_t* d_cols, const float* d_vals, int64_t n,
                                double* d_terms, void* stream);
int bfl_eval_sum_device(const double* d_terms, int64_t n, int width, double* d_out, void* stream);

/* =====================================================================================
 * Offline evaluation on held-out interactions (DESIGN.md 4.14): the device path of Evaluable.evaluate and
 * buffalo_b200.evaluate.evaluate_lists.  Device pointers, stream-ordered.  d_ranked [n x k] holds ranked item lists,
 * -1 for padding.  d_cutoffs [n_cut] holds the cutoffs ascending and distinct, each in [1, k].  d_terms holds one
 * [rows x 8] fp64 slab per cutoff, slab_stride doubles apart (>= 8 n); row q of a call writes row q of every slab.  Slab
 * columns: hit, recall, precision, ndcg, ap / min(|T|, K), reciprocal rank, ild, 1 if the ild counts.
 *  - cutoff_terms: per row q, its truth row d_truth_row[q] (d_truth_row nullable: row q) of the truth CSR (END
 *    offsets, every row ascending without duplicates); writes columns 0-5 and zeros in 6-7.  d_gains[i] = 1 / log2(i + 2)
 *    and d_ideal its prefix sums, at least as long as the largest cutoff.  A row with an empty truth row gets zeros.
 *  - ild: columns 6-7: over the valid entries among the first K, the mean of 1 - cos over all pairs of their rows of
 *    d_items [n_items x ld] (first d columns; cos = 0 when a row has zero norm), counted when there are at least two.
 *    kmax = the largest cutoff, at most 256 and at most k.
 *  - coverage_mark: d_first[item] = min(d_first[item], d_bucket[p]) for every entry at position p < kmax, where
 *    d_bucket[p] is the index of the smallest cutoff > p.  Start d_first at n_cut; calls on several batches accumulate.
 *  - coverage_count: d_count[c] (u64) = the number of items whose d_first is c, for c < n_cut (<= 4096).
 * ===================================================================================== */
int bfl_eval_cutoff_terms_device(const int32_t* d_ranked, int64_t n, int k, const int64_t* d_truth_indptr,
                                 const int32_t* d_truth_keys, const int32_t* d_truth_row /* nullable */,
                                 const int32_t* d_cutoffs, int n_cut, const double* d_gains, const double* d_ideal,
                                 double* d_terms, int64_t slab_stride, void* stream);
int bfl_eval_ild_device(const int32_t* d_ranked, int64_t n, int k, int kmax, const float* d_items, int ld, int d,
                        const int32_t* d_cutoffs, int n_cut, double* d_terms, int64_t slab_stride, void* stream);
int bfl_eval_coverage_mark_device(const int32_t* d_ranked, int64_t n, int k, const int32_t* d_bucket, int kmax,
                                  int32_t* d_first, void* stream);
int bfl_eval_coverage_count_device(const int32_t* d_first, int64_t n_items, int n_cut, unsigned long long* d_count,
                                   void* stream);

/* =====================================================================================
 * Ingest helpers (SURVEY.md 8(f-1), 8(f-4)).
 * CSR of one orientation from (major, minor, value) triples, the sort/compress stage of
 * MatrixMarket.create -> _sort_and_compressed_binarization (buffalo/data/mm.py:236-279,
 * buffalo/data/fileio.hpp:263-419): stable sort by (major, minor) (sort_minor = 0: by major only,
 * Stream's token order), indptr[num_major] = exclusive END offsets (buffalo/data/base.py:187-192).
 * Cumulative popularity table of BPRMF.prepare_sampling (buffalo/algo/bpr.py:99-111):
 * cum[i] = sum_{j<=i} count(j)^power.
 * ===================================================================================== */
int bfl_csr_from_triples_device(const int32_t* d_major, const int32_t* d_minor, const float* d_vals, int64_t nnz,
                                int32_t num_major, int32_t num_minor, int sort_minor, int64_t* d_indptr,
                                int32_t* d_key_out, float* d_val_out, void* stream);
int bfl_csr_from_triples_host(const int32_t* major, const int32_t* minor, const float* vals, int64_t nnz,
                              int32_t num_major, int32_t num_minor, int sort_minor, int64_t* indptr,
                              int32_t* key_out, float* val_out);
int bfl_popularity_table_device(const int32_t* d_keys, int64_t nnz, int32_t n_items, int power, int64_t* d_cum,
                                void* stream);
int bfl_popularity_table_host(const int32_t* keys, int64_t nnz, int32_t n_items, int power, int64_t* cum);

/* =====================================================================================
 * MatrixMarket text -> database on the device (SURVEY.md 8(f-1); DESIGN.md 4.6).  The caller parses the header
 * (banner, leading '%' lines, "U I nnz") and streams the rest of the file through the handle's two pinned staging
 * buffers; the triples stay on the device through the validation split and both CSR builds.
 *  - create: `nnz_hint` (the header's nnz) sizes the triple arrays; a file with more data lines than that reports
 *    nnz > nnz_hint from finish and cannot be split.  `block_bytes` is the size of each staging buffer,
 *    `header_lines` the number of lines before the first fed byte (for 1-based line numbers), `slow_cap` the number
 *    of value tokens the handle can leave to the host parser.
 *  - staging(slot): the pinned buffer of slot 0 or 1; waits until that buffer's previous upload has finished.
 *  - feed(slot, n, is_last): uploads n bytes of the slot and parses them, asynchronously.  The CALLER carries partial
 *    lines: a block that is not the last must end with '\n' (the bytes after the block's last '\n' start the next
 *    block).  Lines longer than BFL_MM_MAX_LINE bytes (line end excluded) are grammar rejections.
 *  - finish: waits for the parse; *nnz = data lines, *tokmask bit k set when some data line has k tokens,
 *    *reject_line / *range_line = smallest 1-based file line the grammar rejected / with an index outside
 *    [1, U] x [1, I] (-1: none), *n_slow = value tokens outside the exact fast path (compare with slow_cap).
 *  - slow_tokens: their data-line ordinals, byte offsets from the first fed byte and lengths (any order);
 *    patch_values writes the host-parsed values at those ordinals.
 *  - split(sample_idx, n, ...): strictly increasing data-line ordinals move to the host vali arrays, the others keep
 *    their order (n = 0 allowed, required before build).
 *  - build(orientation 0 = rowwise, 1 = colwise): one CSR (exclusive END offsets) into host arrays of num_rows
 *    resp. num_cols and nnz - n entries; each orientation once.
 *  - stats: summed device time of H2D, parse, patch, split, rowwise CSR, colwise CSR and D2H (stage_ms[7]) and the
 *    high-water mark of the device's default memory pool since create.
 * ===================================================================================== */
#define BFL_MM_MAX_LINE 1024
typedef struct bfl_mm_ingest bfl_mm_ingest_t;
bfl_mm_ingest_t* bfl_mm_ingest_create(int32_t num_rows, int32_t num_cols, int64_t nnz_hint, int64_t block_bytes,
                                      int64_t header_lines, int64_t slow_cap);
void bfl_mm_ingest_destroy(bfl_mm_ingest_t* h);
int bfl_mm_ingest_staging(bfl_mm_ingest_t* h, int slot, void** host_ptr);
int bfl_mm_ingest_feed(bfl_mm_ingest_t* h, int slot, int64_t n, int is_last);
int bfl_mm_ingest_finish(bfl_mm_ingest_t* h, int64_t* nnz, int32_t* tokmask, int64_t* reject_line, int64_t* range_line,
                         int64_t* n_slow);
int bfl_mm_ingest_slow_tokens(bfl_mm_ingest_t* h, int64_t n, int64_t* ordinal, int64_t* offset, int32_t* length);
int bfl_mm_ingest_patch_values(bfl_mm_ingest_t* h, const int64_t* ordinal, const float* val, int64_t n);
int bfl_mm_ingest_split(bfl_mm_ingest_t* h, const int64_t* sample_idx, int64_t n, int32_t* out_row, int32_t* out_col,
                        float* out_val);
int bfl_mm_ingest_build(bfl_mm_ingest_t* h, int orientation, int64_t* indptr, int32_t* key, float* val);
int bfl_mm_ingest_stats(bfl_mm_ingest_t* h, double* stage_ms, int64_t* peak_bytes);

/* =====================================================================================
 * Stream text -> database on the device (DESIGN.md 4.7).  One line per user of item tokens separated by whitespace;
 * the caller streams the whole file through the handle's two pinned staging buffers.  Tokens are interned in a device
 * hash table and numbered in first-appearance order (or by an iid list), the (user, item) pairs stay on the device
 * through the validation split and the CSR builds.
 *  - create: `block_bytes` per staging buffer; `ascii_ws` bit c set when byte c (< 64) separates tokens (must include
 *    '\n'); `uspace[n_uspace]` multi-byte whitespace code points, which decline the file; `hash_bits` < 64 truncates
 *    the token hash (tests: distinct tokens then share keys and the byte comparison must decline the file).
 *  - load_iid(names, offsets[n + 1], n): the UTF-8 item names, before the first block; a repeated name takes its last
 *    index, the table is frozen and a token it does not hold declines the file.
 *  - staging(slot) / feed(slot, n, is_last): as bfl_mm_ingest_*; every block but the last ends with '\n'.  Parsing is
 *    synchronous; after a decline the remaining blocks are skipped.
 *  - finish: *num_tokens, *num_lines ('\n' bytes), *num_items, *decline = reason bits (1 bare '\r', 2 invalid UTF-8,
 *    4 multi-byte whitespace, 8 token missing from the iid list, 16 hash collision, 32 device memory, 64 more than
 *    2^31 - 2 lines or items; 0: accepted) and *decline_line (smallest 1-based line with reason 1, 2, 4, 8 or 16; -1).
 *  - names: byte offset from the first fed byte and length of each item's first occurrence (no iid list).
 *  - split(num_users, method 0 none / 1 newest / 2 sample, newest_n, sample ordinals, as_matrix): holds out the last
 *    min(newest_n, len - 1) tokens of each session, or the given token ordinals; *n_vali = Counter(held) triples of
 *    all users, *n_train = distinct (user, item) pairs (as_matrix) or kept tokens; vali copies the triples out.
 *  - build(orientation): one CSR (END offsets, int32 key, float32 value) into host arrays of num_users resp. num_items
 *    and n_train entries; matrix: rowwise by (user, item) and colwise by (item, user) with counts as values; stream:
 *    rowwise only, in session order, value 1.
 *  - stats: summed device time of H2D, parse, intern, number, split, rowwise CSR, colwise CSR and D2H (stage_ms[8])
 *    and the high-water mark of the device's default memory pool since create.
 * ===================================================================================== */
typedef struct bfl_stream_ingest bfl_stream_ingest_t;
bfl_stream_ingest_t* bfl_stream_ingest_create(int64_t block_bytes, uint64_t ascii_ws, const int32_t* uspace, int32_t n_uspace,
                                              int32_t hash_bits);
void bfl_stream_ingest_destroy(bfl_stream_ingest_t* h);
int bfl_stream_ingest_staging(bfl_stream_ingest_t* h, int slot, void** host_ptr);
int bfl_stream_ingest_load_iid(bfl_stream_ingest_t* h, const char* names, const int64_t* offsets, int64_t n);
int bfl_stream_ingest_feed(bfl_stream_ingest_t* h, int slot, int64_t n, int is_last);
int bfl_stream_ingest_finish(bfl_stream_ingest_t* h, int64_t* num_tokens, int64_t* num_lines, int32_t* num_items,
                             int32_t* decline, int64_t* decline_line);
int bfl_stream_ingest_names(bfl_stream_ingest_t* h, int64_t* offset, int32_t* length);
int bfl_stream_ingest_split(bfl_stream_ingest_t* h, int32_t num_users, int method, int64_t newest_n, const int64_t* sample_idx,
                            int64_t n_sample, int as_matrix, int64_t* n_vali, int64_t* n_train);
int bfl_stream_ingest_vali(bfl_stream_ingest_t* h, int32_t* row, int32_t* col, float* val);
int bfl_stream_ingest_build(bfl_stream_ingest_t* h, int orientation, int64_t* indptr, int32_t* key, float* val);
int bfl_stream_ingest_stats(bfl_stream_ingest_t* h, double* stage_ms, int64_t* peak_bytes);

#ifdef __cplusplus
}
#endif
#endif /* BUFFALO_B200_H_ */
