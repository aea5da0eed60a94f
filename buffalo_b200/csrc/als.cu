// ALS backend: host-side state machine + C ABI (see include/buffalo_b200.h).
// Replaces als::CALS (lib/algo_impl/als/als.cc) / cuda_als::CuALS (lib/cuda/als/als.cu).
#include "als_fast.cuh"
#include "als_generic.cuh"
#include "bfl_common.cuh"
#include "explain.cuh"

using namespace bfl;

struct bfl_als : Holder {
    // options (als.cc:30-69)
    int num_cg_max_iters = 3;
    int optimizer_code = 2;  // 0 llt, 1 ldlt, 2 manual_cg, 8 ialspp
    int block_size = 32;
    bool adaptive_reg = false, compute_loss = true;
    float alpha = 8.f, reg_u = 0.1f, reg_i = 0.1f, eps = 1e-10f, cg_tolerance = 1e-10f;
    int kernel_mode = 0;  // 0 auto (d = 128: tensor-core kernel als_tc.cuh for rows above tc_min_nnz, tuned SIMT kernels
                          // otherwise), 1 force generic, 2 tuned SIMT kernels only (the round-1 path), 4 SIMT only with
                          // rows of 513..1536 nnz on the re-gathering class
    int tc_min_class = 2; // first row-length class (als_fast.cuh) solved by the tensor-core kernel (rows of <= 64 nnz stay on
                          // the SIMT classes 0, 1: an epilogue per row costs more than their whole SIMT solve; measured 400 vs 411 ms)
    int64_t sub_chunk_nnz = 16ll << 20;   // host-pointer path: entries per pipelined sub-chunk of one partial_update call
    // split-row chunk matrices and the training loss summed in a fixed order instead of with atomics: the same factors,
    // CSR, options and feed give bitwise the same P, Q and loss on every run (one GPU)
    bool deterministic = false;

    // CSR per axis: bound device CSR (device path), or just own_indptr (host-pointer path)
    DevBuf<int64_t> own_indptr[2];
    CsrBinding csr[2];
    DevBuf<int32_t> stage_keys;   // two halves: double-buffered sub-chunks of the host-pointer path
    DevBuf<float> stage_vals;
    cudaStream_t s_h2d = nullptr, s_d2h = nullptr;
    cudaEvent_t ev_h2d[2] = {nullptr, nullptr}, ev_comp[2] = {nullptr, nullptr};
    bool ph_set = false;
    bool indptr_uploaded[2] = {false, false};   // own_indptr[axis] holds the caller's offsets (host-pointer path)

    DevBuf<float> G;          // d x d
    int gram_axis = -1;       // axis whose full Gram G holds (the last precompute), -1 before one or after a partial one
    DevBuf<float> gram_part;  // partials of the two-stage Gram
    DevBuf<float> yui;        // generic ialspp scratch
    DevBuf<double> d_loss;    // 2 doubles
    DevBuf<double> loss_rows; // deterministic: (numerator, denominator) terms per row of the axis being updated
    DevBuf<double> loss_part; // deterministic: the loss tree's partials, one pair per kLossRows rows
    FastCache fast_cache;     // row-length bins of the tuned path, keyed by (indptr, row range)
    // tensor-core path (als_tc.cuh): max|Y| (noted by precompute, which reads the whole opposite factor anyway) and
    // max|v| of the launch -> power-of-two operand scale, all on the device
    DevBuf<unsigned int> tc_maxes;   // [0] bits of max|Y|, [1 + axis] bits of max|v| of that orientation's values
    DevBuf<float> tc_scales;         // [0] 2^e, [1] 2^-2e
    bool tc_on = false;
    const float* tc_vals_seen[2] = {nullptr, nullptr};   // resident CSR: max|v| is noted once per bound value array
    int64_t tc_vals_seen_n[2] = {0, 0};
    int n_peer[2] = {0, 0};   // fused multi-GPU exchange targets per axis
    float* peers[2][BFL_MAX_PEERS] = {};

    ~bfl_als() override {
        if (s_h2d) cudaStreamDestroy(s_h2d);
        if (s_d2h) cudaStreamDestroy(s_d2h);
        for (int i = 0; i < 2; ++i) {
            if (ev_h2d[i]) cudaEventDestroy(ev_h2d[i]);
            if (ev_comp[i]) cudaEventDestroy(ev_comp[i]);
        }
    }
    int apply_options(const JsonOpt& j) override;
};

int bfl_als::apply_options(const JsonOpt& j) {
    d = j.integer("d", 20);
    if (d <= 0 || d > 512) BFL_FAIL(BFL_ERR_OPTION, "d must be in [1, 512], got " + std::to_string(d));
    vdim = (d + 3) / 4 * 4;
    num_cg_max_iters = j.integer("num_cg_max_iters", 3);
    block_size = j.integer("block_size", 32);
    if (block_size <= 0) BFL_FAIL(BFL_ERR_OPTION, "block_size must be positive");
    adaptive_reg = j.flag("adaptive_reg", false);
    compute_loss = j.flag("compute_loss_on_training", true);
    alpha = (float)j.number("alpha", 8.0);
    reg_u = (float)j.number("reg_u", 0.1);
    reg_i = (float)j.number("reg_i", 0.1);
    eps = (float)j.number("eps", 1e-10);
    cg_tolerance = (float)j.number("cg_tolerance", 1e-10);
    kernel_mode = j.integer("_b200_kernel_mode", 0);
    // rows of classes >= 2 (> 64 nnz) on the tensor-core kernel: the fastest of the routings measured at C2 on an H100
    // (DESIGN.md 4.1)
    tc_min_class = std::max(0, std::min(7, j.integer("_b200_tc_min_class", 2)));
    sub_chunk_nnz = (int64_t)j.number("_b200_sub_chunk_nnz", (double)(16ll << 20));
    if (sub_chunk_nnz < 1) BFL_FAIL(BFL_ERR_OPTION, "_b200_sub_chunk_nnz must be positive");
    deterministic = j.flag("deterministic", false);
    // deterministic split rows: scratch budget of one batch of long rows (0: from the free device memory)
    const double det_mb = j.number("_b200_det_scratch_mb", 0.0);
    if (det_mb < 0) BFL_FAIL(BFL_ERR_OPTION, "_b200_det_scratch_mb must not be negative");
    fast_cache.det_budget = (size_t)(det_mb * (double)(1 << 20));
    std::string optimizer = j.string("optimizer", "manual_cg");
    if (d >= 128) optimizer = "ialspp";  // als.cc:46
    if (optimizer == "llt") optimizer_code = 0;
    else if (optimizer == "ldlt") optimizer_code = 1;
    else if (optimizer == "manual_cg") optimizer_code = 2;
    else if (optimizer == "ialspp") optimizer_code = 8;
    else
        BFL_FAIL(BFL_ERR_OPTION, "optimizer '" + optimizer +
                                     "' is not available on the H100 backend (supported: llt, ldlt, manual_cg, ialspp)");
    int rc = attach_device();
    if (rc != BFL_OK) return rc;
    if (!s_h2d) {
        BFL_CUDA(cudaStreamCreateWithFlags(&s_h2d, cudaStreamNonBlocking));
        BFL_CUDA(cudaStreamCreateWithFlags(&s_d2h, cudaStreamNonBlocking));
        for (int i = 0; i < 2; ++i) {
            BFL_CUDA(cudaEventCreateWithFlags(&ev_h2d[i], cudaEventDisableTiming));
            BFL_CUDA(cudaEventCreateWithFlags(&ev_comp[i], cudaEventDisableTiming));
        }
    }
    if (BFL_OK != G.reserve((size_t)d * d)) return BFL_ERR_CUDA;
    if (BFL_OK != d_loss.reserve(2)) return BFL_ERR_CUDA;
    tc_on = kernel_mode == 0 && tc::tc_split_applicable(optimizer_code, d, vdim, block_size);
    if (tc_on) {
        if (BFL_OK != tc_maxes.reserve(3) || BFL_OK != tc_scales.reserve(2)) return BFL_ERR_CUDA;
        BFL_CUDA(cudaMemsetAsync(tc_maxes.p, 0, 3 * sizeof(unsigned int), stream));
    }
    tc_vals_seen[0] = tc_vals_seen[1] = nullptr;
    opt_set = true;
    return BFL_OK;
}

namespace {

// max|Y| over the WHOLE opposite factor of `axis` (the tensor-core kernel's operand scale)
int note_factor_absmax(bfl_als* h, int axis, cudaStream_t st) {
    if (!h->tc_on) return BFL_OK;
    const float* F = axis == 0 ? h->dQ : h->dP;
    const int64_t rows = axis == 0 ? h->Q_rows : h->P_rows;
    return tc::tc_note_absmax(F, (size_t)rows * h->vdim, h->tc_maxes.p, h->num_sms, st);
}

int gram(bfl_als* h, const float* F, int64_t rows, cudaStream_t st) {
    const int D = h->d;
    const int nslab = (D + 127) / 128;
    int64_t ntiles = (rows + GRAM_TR - 1) / GRAM_TR;
    int gx = (int)std::min<int64_t>(std::max<int64_t>(ntiles, 1), (int64_t)h->num_sms * 2 / (nslab * nslab) + 1);
    if (BFL_OK != h->gram_part.reserve((size_t)gx * nslab * nslab * 128 * 128)) return BFL_ERR_CUDA;
    dim3 grid(gx, nslab * nslab);
    gram_partial_kernel<<<grid, GRAM_THREADS, 0, st>>>(F, rows, D, h->vdim, h->gram_part.p, nslab);
    BFL_LAUNCHED();
    gram_reduce_kernel<<<(D * D + 255) / 256, 256, 0, st>>>(h->gram_part.p, gx, nslab, D, h->G.p);
    BFL_LAUNCHED();
    return BFL_OK;
}

// det_loss: a.loss takes per-row terms (the kernels' DET instantiations)
template <int NC>
int launch_generic(bfl_als* h, const AlsArgs& a, int64_t nrows, bool det_loss, cudaStream_t st) {
    int grid = (int)std::min<int64_t>((nrows + GEN_WARPS - 1) / GEN_WARPS, (int64_t)h->num_sms * 8);
    if (grid < 1) grid = 1;
    if (h->optimizer_code == 8) {
        if (det_loss) als_ialspp_warp_kernel<NC, true><<<grid, GEN_WARPS * 32, 0, st>>>(a);
        else als_ialspp_warp_kernel<NC><<<grid, GEN_WARPS * 32, 0, st>>>(a);
    } else {
        if (det_loss) als_cg_warp_kernel<NC, true><<<grid, GEN_WARPS * 32, 0, st>>>(a);
        else als_cg_warp_kernel<NC><<<grid, GEN_WARPS * 32, 0, st>>>(a);
    }
    BFL_LAUNCHED();
    return BFL_OK;
}

// Solve rows [row_begin,row_end) of axis with keys/vals device buffers whose element 0 is global
// offset `shift`.  chunk_nnz = number of entries those rows span.  d_loss: the two sums, or (deterministic mode) the
// per-row terms indexed by absolute row.
int launch_row_solves(bfl_als* h, int axis, int64_t row_begin, int64_t row_end, const int32_t* keys, const float* vals,
                      int64_t shift, int64_t chunk_nnz, double* d_loss, cudaStream_t st) {
    AlsArgs a;
    a.X = axis == 0 ? h->dP : h->dQ;
    a.Y = axis == 0 ? h->dQ : h->dP;
    a.G = h->G.p;
    a.indptr = h->csr[axis].indptr;
    a.keys = keys;
    a.vals = vals;
    a.yui = nullptr;
    a.loss = d_loss;
    a.row_list = nullptr;
    a.shift = shift;
    a.row_begin = row_begin;
    a.row_end = row_end;
    a.Y_rows = axis == 0 ? h->Q_rows : h->P_rows;
    a.D = h->d;
    a.ld = h->vdim;
    a.block_size = h->block_size;
    a.max_iters = h->num_cg_max_iters;
    a.adaptive_reg = h->adaptive_reg;
    a.compute_loss = h->compute_loss;
    a.axis = axis;
    a.alpha = h->alpha;
    a.reg = axis == 0 ? h->reg_u : h->reg_i;
    a.eps = h->eps;
    a.tol = h->cg_tolerance;
    a.n_peer = h->n_peer[axis];
    for (int i = 0; i < BFL_MAX_PEERS; ++i) a.peerX[i] = i < a.n_peer ? h->peers[axis][i] : nullptr;
    a.tc_scales = nullptr;
    const bool det_loss = h->deterministic && a.loss && a.compute_loss;
    int64_t nrows = row_end - row_begin;
    if (h->tc_on) {
        // max|v| of this launch's values (a resident array is scanned once), then the operand scale -- device only
        if (vals != h->tc_vals_seen[axis] || chunk_nnz != h->tc_vals_seen_n[axis]) {
            int rc = tc::tc_note_absmax(vals, (size_t)std::max<int64_t>(chunk_nnz, 0), h->tc_maxes.p + 1 + axis, h->num_sms, st);
            if (rc != BFL_OK) return rc;
            h->tc_vals_seen[axis] = vals == h->csr[axis].vals ? vals : nullptr;   // staged host chunks: scanned every time
            h->tc_vals_seen_n[axis] = chunk_nnz;
        }
        int rc = tc::tc_update_scale(h->tc_maxes.p, h->tc_maxes.p + 1 + axis, h->alpha, h->tc_scales.p, st);
        if (rc != BFL_OK) return rc;
        a.tc_scales = h->tc_scales.p;
    }

    if (h->kernel_mode != 1 && fast_als_applicable(h->optimizer_code, h->d, h->vdim, h->block_size)) {
        const int32_t* left = nullptr;
        int64_t nleft = 0;
        // d = 128: classes tcmin..5 (65..1536 nnz by default) on the fused tensor-core kernel, classes 6, 7 (longer) in its split-row
        // mode; d = 256: classes 6, 7 (beyond 1536 nnz) in split-row mode
        int tcmin = FAST_NCLASS, splitmin = FAST_NCLASS;
        if (h->kernel_mode == 0 && tc::tc_applicable(h->optimizer_code, h->d, h->vdim, h->block_size)) {
            tcmin = h->tc_min_class;
            splitmin = 6;
        } else if (h->kernel_mode == 0 && tc::tc_split_applicable(h->optimizer_code, h->d, h->vdim, h->block_size)) {
            // d = 256: the re-gathering SIMT class (1537..12288 nnz) reads every gathered row 48 times (8 blocks x 6 passes);
            // the split-row mode reads it once and pays 2 x 256 KB of scratch traffic per row instead
            splitmin = 6;
        }
        int rc = fast_als_launch(a, h->fast_cache, h->num_sms, st, &left, &nleft, tcmin, splitmin, h->kernel_mode == 4 ? 1 : 0,
                                 h->deterministic);
        if (rc != BFL_OK || nleft == 0) return rc;
        // rows longer than the tuned kernels accept go through the generic kernel
        a.row_list = left;
        a.row_begin = 0;
        a.row_end = nleft;
        nrows = nleft;
    }

    if (h->optimizer_code == 0 || h->optimizer_code == 1) {
        const size_t smem = ((size_t)h->d * (h->d + 1) + 2 * h->d + (size_t)DIRECT_NB * h->d) * sizeof(float);
        if (smem > 220 * 1024) BFL_FAIL(BFL_ERR_OPTION, "llt/ldlt needs d <= 224 on this backend");
        int grid = (int)std::min<int64_t>(nrows, (int64_t)h->num_sms * 4);
        if (det_loss) {
            BFL_CUDA(cudaFuncSetAttribute(als_direct_cta_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            als_direct_cta_kernel<true><<<grid, DIRECT_THREADS, smem, st>>>(a);
        } else {
            BFL_CUDA(cudaFuncSetAttribute(als_direct_cta_kernel<>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            als_direct_cta_kernel<><<<grid, DIRECT_THREADS, smem, st>>>(a);
        }
        BFL_LAUNCHED();
        return BFL_OK;
    }
    if (h->optimizer_code == 8) {
        if (BFL_OK != h->yui.reserve((size_t)std::max<int64_t>(chunk_nnz, 1))) return BFL_ERR_CUDA;
        a.yui = h->yui.p;
    }
    const int nc = (h->d + 31) / 32;
    if (nc <= 1) return launch_generic<1>(h, a, nrows, det_loss, st);
    if (nc <= 2) return launch_generic<2>(h, a, nrows, det_loss, st);
    if (nc <= 4) return launch_generic<4>(h, a, nrows, det_loss, st);
    if (nc <= 8) return launch_generic<8>(h, a, nrows, det_loss, st);
    return launch_generic<16>(h, a, nrows, det_loss, st);
}

// launch_row_solves with the loss added into d_loss[0 .. 2).  Deterministic mode: every row of the range stores its
// terms (rows without entries keep the zeros written here) and a fixed tree over the range sums them, so the loss does
// not depend on which warp solved which rows.
int solve_rows(bfl_als* h, int axis, int64_t row_begin, int64_t row_end, const int32_t* keys, const float* vals,
               int64_t shift, int64_t chunk_nnz, double* d_loss, cudaStream_t st) {
    if (row_end <= row_begin) return BFL_OK;
    if (!(h->deterministic && h->compute_loss && d_loss))
        return launch_row_solves(h, axis, row_begin, row_end, keys, vals, shift, chunk_nnz, d_loss, st);
    const int64_t n = row_end - row_begin, nblk = (n + kLossRows - 1) / kLossRows;
    const int64_t max_rows = std::max(h->P_rows, h->Q_rows);
    if (BFL_OK != h->loss_rows.reserve(2 * (size_t)max_rows) ||
        BFL_OK != h->loss_part.reserve(2 * (size_t)((max_rows + kLossRows - 1) / kLossRows)))
        return BFL_ERR_CUDA;
    double* terms = h->loss_rows.p + 2 * row_begin;
    BFL_CUDA(cudaMemsetAsync(terms, 0, 2 * sizeof(double) * (size_t)n, st));
    int rc = launch_row_solves(h, axis, row_begin, row_end, keys, vals, shift, chunk_nnz, h->loss_rows.p, st);
    if (rc != BFL_OK) return rc;
    loss_tree_partial_kernel<2><<<(unsigned)nblk, 256, 0, st>>>(terms, n, h->loss_part.p);
    BFL_LAUNCHED();
    loss_tree_final_kernel<2><<<1, 256, 0, st>>>(h->loss_part.p, nblk, d_loss);
    BFL_LAUNCHED();
    return BFL_OK;
}

}  // namespace

extern "C" {

bfl_als_t* bfl_als_create(void) { return new (std::nothrow) bfl_als(); }

void bfl_als_destroy(bfl_als_t* h) { delete h; }

int bfl_als_init(bfl_als_t* h, const char* opt_path) { return init_holder(h, opt_path, true); }

int bfl_als_init_json(bfl_als_t* h, const char* json_text) { return init_holder(h, json_text, false); }

int bfl_als_get_vdim(bfl_als_t* h) { return h ? h->vdim : 0; }

int bfl_als_initialize_model(bfl_als_t* h, float* P, int32_t P_rows, float* Q, int32_t Q_rows) {
    if (!h || !h->opt_set) BFL_FAIL(BFL_ERR_STATE, "init() must succeed before initialize_model()");
    int rc = h->mirror_factors(P, P_rows, Q, Q_rows);
    if (rc != BFL_OK) return rc;
    BFL_CUDA(cudaMemcpyAsync(h->dP, P, sizeof(float) * (size_t)P_rows * h->vdim, cudaMemcpyHostToDevice, h->stream));
    BFL_CUDA(cudaMemcpyAsync(h->dQ, Q, sizeof(float) * (size_t)Q_rows * h->vdim, cudaMemcpyHostToDevice, h->stream));
    BFL_CUDA(cudaStreamSynchronize(h->stream));
    h->factors_ready = true;
    // a CSR bound earlier through bind_csr_device belongs to the previous model: drop the borrowed pointers
    for (int ax = 0; ax < 2; ++ax) {
        h->csr[ax] = CsrBinding();
        h->indptr_uploaded[ax] = false;
    }
    h->ph_set = false;
    h->fast_cache.clear();
    return BFL_OK;
}

int bfl_als_set_placeholder(bfl_als_t* h, const int64_t* lindptr, const int64_t* rindptr, size_t batch_size) {
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "initialize_model() must precede set_placeholder()");
    if (!lindptr || !rindptr) BFL_FAIL(BFL_ERR_ARG, "null indptr");
    if (BFL_OK != h->own_indptr[0].reserve((size_t)h->P_rows)) return BFL_ERR_CUDA;
    if (BFL_OK != h->own_indptr[1].reserve((size_t)h->Q_rows)) return BFL_ERR_CUDA;
    BFL_CUDA(cudaMemcpyAsync(h->own_indptr[0].p, lindptr, sizeof(int64_t) * h->P_rows, cudaMemcpyHostToDevice, h->stream));
    BFL_CUDA(cudaMemcpyAsync(h->own_indptr[1].p, rindptr, sizeof(int64_t) * h->Q_rows, cudaMemcpyHostToDevice, h->stream));
    h->csr[0].indptr = h->own_indptr[0].p;
    h->csr[1].indptr = h->own_indptr[1].p;
    h->fast_cache.clear();
    if (batch_size) {
        if (BFL_OK != h->stage_keys.reserve(batch_size)) return BFL_ERR_CUDA;
        if (BFL_OK != h->stage_vals.reserve(batch_size)) return BFL_ERR_CUDA;
    }
    BFL_CUDA(cudaStreamSynchronize(h->stream));
    h->ph_set = true;
    h->indptr_uploaded[0] = h->indptr_uploaded[1] = true;
    return BFL_OK;
}

int bfl_als_precompute(bfl_als_t* h, int axis) {
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "initialize_model() must precede precompute()");
    if (axis != 0 && axis != 1) BFL_FAIL(BFL_ERR_ARG, "axis must be 0 or 1");
    const float* F = axis == 0 ? h->dQ : h->dP;
    const int64_t rows = axis == 0 ? h->Q_rows : h->P_rows;
    h->gram_axis = -1;
    int rc = gram(h, F, rows, h->stream);
    if (rc != BFL_OK) return rc;
    h->gram_axis = axis;
    rc = note_factor_absmax(h, axis, h->stream);
    if (rc != BFL_OK) return rc;
    BFL_CUDA(cudaStreamSynchronize(h->stream));
    return BFL_OK;
}

int bfl_als_partial_update(bfl_als_t* h, int32_t start_x, int32_t next_x, const int64_t* indptr,
                           const int32_t* keys, const float* vals, int axis, double* loss_nume,
                           double* loss_deno) {
    if (loss_nume) *loss_nume = 0.0;
    if (loss_deno) *loss_deno = 0.0;
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "initialize_model() must precede partial_update()");
    if (!h->hostP) BFL_FAIL(BFL_ERR_STATE, "partial_update() is the host-pointer path; use bfl_als_update_device with bound device factors");
    if (axis != 0 && axis != 1) BFL_FAIL(BFL_ERR_ARG, "axis must be 0 or 1");
    if (next_x - start_x == 0) return BFL_OK;  // als.cc:115-118
    const int64_t rows = axis == 0 ? h->P_rows : h->Q_rows;
    if (start_x < 0 || next_x > rows || next_x < start_x || !indptr || !keys || !vals)
        BFL_FAIL(BFL_ERR_ARG, "bad chunk arguments");
    if (!h->indptr_uploaded[axis] || h->csr[axis].indptr != h->own_indptr[axis].p) {
        // the CPU holder needs no set_placeholder (als.py:156-158 only calls it for the accelerator);
        // upload this axis' end offsets on first use
        if (BFL_OK != h->own_indptr[axis].reserve((size_t)rows)) return BFL_ERR_CUDA;
        BFL_CUDA(cudaMemcpyAsync(h->own_indptr[axis].p, indptr, sizeof(int64_t) * rows, cudaMemcpyHostToDevice, h->stream));
        h->csr[axis].indptr = h->own_indptr[axis].p;
        h->indptr_uploaded[axis] = true;
        h->fast_cache.clear();
    }
    const int64_t beg = start_x == 0 ? 0 : indptr[start_x - 1];
    // The chunk is cut into row-aligned sub-chunks of <= SUB entries and software-pipelined over three streams:
    // H2D of sub-chunk k+1 (keys, vals) | row solves of sub-chunk k | D2H of the rows updated by sub-chunk k-1.
    // With pinned host buffers the PCIe traffic of the reference protocol (als.cu:361-364,403) overlaps the math.
    const int64_t SUB = h->sub_chunk_nnz;
    int64_t maxsub = 0;
    std::vector<int64_t> cut;  // row boundaries
    cut.push_back(start_x);
    {
        int64_t r = start_x;
        while (r < next_x) {
            const int64_t b0 = r == 0 ? 0 : indptr[r - 1];
            // largest r2 > r with indptr[r2-1] - b0 <= SUB (at least one row)
            int64_t lo = r + 1, hi = next_x;
            while (lo < hi) {
                const int64_t mid = (lo + hi + 1) >> 1;
                if (indptr[mid - 1] - b0 <= SUB) lo = mid; else hi = mid - 1;
            }
            maxsub = std::max(maxsub, indptr[lo - 1] - b0);
            cut.push_back(lo);
            r = lo;
        }
    }
    const int nsub = (int)cut.size() - 1;
    if (BFL_OK != h->stage_keys.reserve((size_t)std::max<int64_t>(2 * maxsub, 2))) return BFL_ERR_CUDA;
    if (BFL_OK != h->stage_vals.reserve((size_t)std::max<int64_t>(2 * maxsub, 2))) return BFL_ERR_CUDA;
    BFL_CUDA(cudaMemsetAsync(h->d_loss.p, 0, 2 * sizeof(double), h->stream));
    float* hostF = axis == 0 ? h->hostP : h->hostQ;
    float* devF = axis == 0 ? h->dP : h->dQ;
    for (int k = 0; k < nsub; ++k) {
        const int64_t r0 = cut[k], r1 = cut[k + 1];
        const int64_t b0 = r0 == 0 ? 0 : indptr[r0 - 1];
        const int64_t cnt = indptr[r1 - 1] - b0;
        const int slot = k & 1;
        int32_t* dk = h->stage_keys.p + (size_t)slot * maxsub;
        float* dv = h->stage_vals.p + (size_t)slot * maxsub;
        if (k >= 2) BFL_CUDA(cudaStreamWaitEvent(h->s_h2d, h->ev_comp[slot], 0));  // staging half is free again
        if (cnt > 0) {
            BFL_CUDA(cudaMemcpyAsync(dk, keys + (b0 - beg), sizeof(int32_t) * cnt, cudaMemcpyHostToDevice, h->s_h2d));
            BFL_CUDA(cudaMemcpyAsync(dv, vals + (b0 - beg), sizeof(float) * cnt, cudaMemcpyHostToDevice, h->s_h2d));
        }
        BFL_CUDA(cudaEventRecord(h->ev_h2d[slot], h->s_h2d));
        BFL_CUDA(cudaStreamWaitEvent(h->stream, h->ev_h2d[slot], 0));
        int rc = solve_rows(h, axis, r0, r1, dk, dv, b0, cnt, h->d_loss.p, h->stream);
        if (rc != BFL_OK) return rc;
        BFL_CUDA(cudaEventRecord(h->ev_comp[slot], h->stream));
        // copy the rows this sub-chunk updated back into the caller's matrix (als.cu:321-336,403)
        BFL_CUDA(cudaStreamWaitEvent(h->s_d2h, h->ev_comp[slot], 0));
        const size_t off = (size_t)r0 * h->vdim;
        BFL_CUDA(cudaMemcpyAsync(hostF + off, devF + off, sizeof(float) * (size_t)(r1 - r0) * h->vdim,
                                 cudaMemcpyDeviceToHost, h->s_d2h));
    }
    double hl[2] = {0.0, 0.0};
    BFL_CUDA(cudaMemcpyAsync(hl, h->d_loss.p, 2 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    BFL_CUDA(cudaStreamSynchronize(h->stream));
    BFL_CUDA(cudaStreamSynchronize(h->s_d2h));
    BFL_CUDA(cudaStreamSynchronize(h->s_h2d));
    if (loss_nume) *loss_nume = hl[0];
    if (loss_deno) *loss_deno = hl[1];
    return BFL_OK;
}

int bfl_als_bind_factors_device(bfl_als_t* h, float* dP, int64_t P_rows, float* dQ, int64_t Q_rows) {
    if (!h || !h->opt_set) BFL_FAIL(BFL_ERR_STATE, "init() must succeed before binding factors");
    int rc = h->borrow_factors(dP, P_rows, dQ, Q_rows);
    if (rc != BFL_OK) return rc;
    h->factors_ready = true;
    return BFL_OK;
}

int bfl_als_bind_csr_device(bfl_als_t* h, int axis, const int64_t* d_indptr, const int32_t* d_keys,
                            const float* d_vals, int64_t rows, int64_t nnz) {
    if (!h || !h->opt_set) BFL_FAIL(BFL_ERR_STATE, "init() must succeed before binding a CSR");
    if (axis != 0 && axis != 1) BFL_FAIL(BFL_ERR_ARG, "axis must be 0 or 1");
    int rc = h->csr[axis].bind(d_indptr, d_keys, d_vals, rows, nnz, true);
    if (rc != BFL_OK) return rc;
    h->fast_cache.clear();
    h->indptr_uploaded[axis] = false;
    h->tc_vals_seen[axis] = nullptr;
    return BFL_OK;
}

int bfl_als_precompute_device(bfl_als_t* h, int axis, void* stream) {
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "factors not bound");
    if (axis != 0 && axis != 1) BFL_FAIL(BFL_ERR_ARG, "axis must be 0 or 1");
    const float* F = axis == 0 ? h->dQ : h->dP;
    const int64_t rows = axis == 0 ? h->Q_rows : h->P_rows;
    h->gram_axis = -1;
    int rc = gram(h, F, rows, (cudaStream_t)stream);
    if (rc != BFL_OK) return rc;
    h->gram_axis = axis;
    return note_factor_absmax(h, axis, (cudaStream_t)stream);
}

int bfl_als_precompute_rows_device(bfl_als_t* h, int axis, int64_t row_begin, int64_t row_end, void* stream) {
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "factors not bound");
    if (axis != 0 && axis != 1) BFL_FAIL(BFL_ERR_ARG, "axis must be 0 or 1");
    const float* F = axis == 0 ? h->dQ : h->dP;
    const int64_t rows = axis == 0 ? h->Q_rows : h->P_rows;
    if (row_begin < 0 || row_end > rows || row_end < row_begin) BFL_FAIL(BFL_ERR_ARG, "bad row range");
    h->gram_axis = -1;
    // the operand scale needs max|Y| of the whole replica, not of the range (every rank gathers from all rows)
    int rc = note_factor_absmax(h, axis, (cudaStream_t)stream);
    if (rc != BFL_OK) return rc;
    if (row_end == row_begin) {
        BFL_CUDA(cudaMemsetAsync(h->G.p, 0, sizeof(float) * (size_t)h->d * h->d, (cudaStream_t)stream));
        return BFL_OK;
    }
    return gram(h, F + (size_t)row_begin * h->vdim, row_end - row_begin, (cudaStream_t)stream);
}

int bfl_als_update_device(bfl_als_t* h, int axis, int64_t row_begin, int64_t row_end, double* d_loss,
                          void* stream) {
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "factors not bound");
    if (axis != 0 && axis != 1) BFL_FAIL(BFL_ERR_ARG, "axis must be 0 or 1");
    const CsrBinding& c = h->csr[axis];
    if (!c.indptr || (!c.keys && c.nnz > 0)) BFL_FAIL(BFL_ERR_STATE, "no device CSR bound for this axis");
    int rc = c.check_range(row_begin, row_end);
    if (rc != BFL_OK) return rc;
    return solve_rows(h, axis, row_begin, row_end, c.keys, c.vals, 0, c.nnz, d_loss, (cudaStream_t)stream);
}

int bfl_als_set_peer_replicas(bfl_als_t* h, int axis, int n_peers, float* const* peer_ptrs) {
    if (!h || !h->opt_set) BFL_FAIL(BFL_ERR_STATE, "init() must succeed before set_peer_replicas()");
    if (axis != 0 && axis != 1) BFL_FAIL(BFL_ERR_ARG, "axis must be 0 or 1");
    if (n_peers < 0 || n_peers > BFL_MAX_PEERS || (n_peers > 0 && !peer_ptrs)) BFL_FAIL(BFL_ERR_ARG, "bad peer list");
    int cur = 0;
    BFL_CUDA(cudaGetDevice(&cur));
    for (int i = 0; i < n_peers; ++i) {
        if (!peer_ptrs[i] || ((uintptr_t)peer_ptrs[i] & 15)) BFL_FAIL(BFL_ERR_ARG, "peer pointers must be non-null, 16-byte aligned");
        // the replica lives on another GPU (mapped here through CUDA IPC): kernels of THIS device store into it,
        // which needs peer access from the current device to the owner
        cudaPointerAttributes attr;
        BFL_CUDA(cudaPointerGetAttributes(&attr, peer_ptrs[i]));
        if (getenv("BFL_DEBUG"))
            fprintf(stderr, "[bfl] peer %d axis %d ptr %p type %d device %d (current %d)\n", i, axis, (void*)peer_ptrs[i],
                    (int)attr.type, attr.device, cur);
        if (attr.type != cudaMemoryTypeDevice) BFL_FAIL(BFL_ERR_ARG, "peer replica is not device memory");
        if (attr.device != cur) {
            int can = 0;
            BFL_CUDA(cudaDeviceCanAccessPeer(&can, cur, attr.device));
            if (!can) BFL_FAIL(BFL_ERR_CUDA, "no peer access from device " + std::to_string(cur) + " to " + std::to_string(attr.device));
            cudaError_t e = cudaDeviceEnablePeerAccess(attr.device, 0);
            if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
            else if (e != cudaSuccess) BFL_FAIL(BFL_ERR_CUDA, std::string("cudaDeviceEnablePeerAccess: ") + cudaGetErrorString(e));
        }
        h->peers[axis][i] = peer_ptrs[i];
    }
    h->n_peer[axis] = n_peers;
    return BFL_OK;
}

int bfl_als_explain_device(bfl_als_t* h, const int64_t* d_indptr, const int32_t* d_keys, const float* d_vals, int64_t n,
                           const int32_t* d_targets, int k, int topm, float* d_scores, int32_t* d_out_keys,
                           float* d_out_contrib, void* stream) {
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "factors not bound");
    if (h->gram_axis != 0) BFL_FAIL(BFL_ERR_STATE, "explain needs the Gram of Q: bfl_als_precompute_device(axis 0) first");
    if (h->d > EXPLAIN_DMAX) BFL_FAIL(BFL_ERR_ARG, "explain supports d <= " + std::to_string(EXPLAIN_DMAX));
    if (k < 1 || k > EXPLAIN_KMAX) BFL_FAIL(BFL_ERR_ARG, "k must be in [1, " + std::to_string(EXPLAIN_KMAX) + "]");
    if (topm < 1 || topm > EXPLAIN_TOPM_MAX) BFL_FAIL(BFL_ERR_ARG, "topm must be in [1, " + std::to_string(EXPLAIN_TOPM_MAX) + "]");
    if (n < 0 || (n > 0 && (!d_indptr || !d_keys || !d_vals || !d_targets || !d_scores || !d_out_keys || !d_out_contrib)))
        BFL_FAIL(BFL_ERR_ARG, "bad explain arguments");
    ExplainArgs a;
    a.G = h->G.p;
    a.Q = h->dQ;
    a.Q_rows = h->Q_rows;
    a.D = h->d;
    a.ld = h->vdim;
    a.alpha = h->alpha;
    a.reg = h->reg_u;
    a.adaptive_reg = h->adaptive_reg;
    a.indptr = d_indptr;
    a.keys = d_keys;
    a.vals = d_vals;
    a.n = n;
    a.targets = d_targets;
    a.k = k;
    a.topm = topm;
    a.scores = d_scores;
    a.out_keys = d_out_keys;
    a.out_contrib = d_out_contrib;
    return explain_launch(a, h->num_sms, (cudaStream_t)stream);
}

int bfl_als_posterior_sample_device(bfl_als_t* h, const int64_t* d_indptr, const int32_t* d_keys, const float* d_vals,
                                    int64_t n, const float* d_mean, int ld, const int64_t* d_draw_keys, uint32_t seed,
                                    float scale, float* d_out, int64_t* d_failed, void* stream) {
    if (!h || !h->factors_ready) BFL_FAIL(BFL_ERR_STATE, "factors not bound");
    if (h->gram_axis != 0) BFL_FAIL(BFL_ERR_STATE, "posterior_sample needs the Gram of Q: bfl_als_precompute_device(axis 0) first");
    if (h->d > EXPLAIN_DMAX) BFL_FAIL(BFL_ERR_ARG, "posterior_sample supports d <= " + std::to_string(EXPLAIN_DMAX));
    if (ld < h->d) BFL_FAIL(BFL_ERR_ARG, "ld must be at least d");
    if (!(scale >= 0.f && scale <= 3.402823466e38f)) BFL_FAIL(BFL_ERR_ARG, "scale must be finite and >= 0");
    if (n < 0 || (n > 0 && (!d_indptr || !d_keys || !d_vals || !d_mean || !d_draw_keys || !d_out || !d_failed)))
        BFL_FAIL(BFL_ERR_ARG, "bad posterior_sample arguments");
    PosteriorArgs a;
    a.G = h->G.p;
    a.Q = h->dQ;
    a.D = h->d;
    a.ldq = h->vdim;
    a.alpha = h->alpha;
    a.reg = h->reg_u;
    a.adaptive_reg = h->adaptive_reg;
    a.indptr = d_indptr;
    a.keys = d_keys;
    a.vals = d_vals;
    a.n = n;
    a.ld = ld;
    a.mean = d_mean;
    a.draw_keys = d_draw_keys;
    a.seed = seed;
    a.scale = scale;
    a.out = d_out;
    a.failed = d_failed;
    return posterior_sample_launch(a, h->num_sms, (cudaStream_t)stream);
}

const float* bfl_als_gram_device(bfl_als_t* h) { return h ? h->G.p : nullptr; }
float* bfl_als_gram_device_mut(bfl_als_t* h) { return h ? h->G.p : nullptr; }

}  // extern "C"
