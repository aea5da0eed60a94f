// MatrixMarket text -> database on the device (SURVEY.md 8(f-1), DESIGN.md 4.6): the body of a coordinate MatrixMarket
// file is streamed through two pinned host buffers into a hand-written parser, and the (row, col, value) triples stay on
// the device through the validation split and both CSR builds (bfl_csr_from_triples_device).
//
// Parse of one block (a byte range that ends with '\n', or at the end of the file):
//   * a CTA stages a 4 KiB tile plus a halo of MM_MAXLINE bytes in shared memory with 16-byte loads and owns the lines
//     that START in its tile; line starts are found from per-thread 16-byte masks and a block scan;
//   * every line is parsed by one thread from shared memory: data / skip (blank or '%' comment) / grammar reject,
//     token count, row and col (1-based in the text, checked against [1, U] and [1, I]) and the value;
//   * pass 1 counts data lines and lines per tile, an int64 scan gives each tile its first ordinal and line number,
//     pass 2 parses again and writes the triples at their ordinals (file order).
// Values: a token of at most 15 digits whose decimal exponent (after folding in the fraction digits) lies in [-22, 22]
// is an exact integer times or divided by an exact power of ten, one correctly rounded double operation (Clinger's fast
// path), then __double2float_rn.  Every other value token is recorded as (ordinal, offset, length) and re-parsed on the
// host by the same reader the host path uses, then patched in.
#include <algorithm>
#include <vector>

#include "bfl_common.cuh"
#include "text_ingest.cuh"

using namespace bfl;

namespace {

constexpr int MM_THREADS = 256;
constexpr int MM_MAXLINE = BFL_MM_MAX_LINE;           // longest accepted line, its line end excluded
constexpr int MM_TILE = 4096;                           // bytes whose line starts one CTA owns (16 per thread)
constexpr int MM_HALO = MM_MAXLINE + 16;                // bytes staged past the tile: the longest line and its '\n'
constexpr int MM_SMEM = 16 + MM_TILE + MM_HALO;         // staged range [t0 - 16, t0 + MM_TILE + MM_HALO)
static_assert(MM_TILE == 16 * MM_THREADS, "one 16-byte line-start mask per thread");
static_assert(MM_SMEM % 16 == 0, "tile staging uses 16-byte vectors");

enum : int { L_NONE = 0, L_SKIP = 1, L_DATA = 2, L_REJECT = 3 };

struct MMState {
    long long ord_base;                  // data lines before the current block
    long long line_base;                 // lines before the current block (header excluded)
    unsigned long long reject_line;      // smallest 1-based file line the grammar rejected (ULLONG_MAX: none)
    unsigned long long range_line;       // smallest 1-based file line with an index outside [1, U] x [1, I]
    unsigned long long n_slow;           // value tokens left to the host parser
    unsigned int tokmask;                // bit k set: some data line has k tokens
};

__constant__ double c_p10[23] = {1e0,  1e1,  1e2,  1e3,  1e4,  1e5,  1e6,  1e7,  1e8,  1e9,  1e10, 1e11,
                                 1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22};

struct Line {
    int kind, ntok, slow;
    unsigned int row, col;               // 1-based as written, saturated at 2^31
    float val;
    int vbeg, vlen;                      // value token (tile coordinates) when slow
};

__device__ __forceinline__ bool is_ws(unsigned c) { return c == ' ' || c == '\t'; }
__device__ __forceinline__ bool is_digit(unsigned c) { return c - '0' < 10u; }
__device__ __forceinline__ bool is_tok(unsigned c) {
    return is_digit(c) || (c | 32u) - 'a' < 26u || c == '+' || c == '-' || c == '.';
}

// exact value of [+-] digits [. digits] [(e|E) [+-] digits] when Clinger's fast path applies; false -> slow token
__device__ bool fast_value(const unsigned char* s, int a, int b, float* out) {
    int i = a;
    bool neg = false;
    if (s[i] == '+' || s[i] == '-') neg = s[i++] == '-';
    unsigned long long m = 0;
    int nd = 0, nint = 0, nfrac = 0;
    for (; i < b && is_digit(s[i]); ++i, ++nint, ++nd)
        if (nd < 16) m = m * 10 + (s[i] - '0');
    if (nint == 0) return false;
    if (i < b && s[i] == '.') {
        for (++i; i < b && is_digit(s[i]); ++i, ++nfrac, ++nd)
            if (nd < 16) m = m * 10 + (s[i] - '0');
        if (nfrac == 0) return false;
    }
    int ex = 0;
    if (i < b && (s[i] | 32) == 'e') {
        ++i;
        bool eneg = false;
        if (i < b && (s[i] == '+' || s[i] == '-')) eneg = s[i++] == '-';
        int ne = 0;
        for (; i < b && is_digit(s[i]); ++i, ++ne) ex = min(ex * 10 + (s[i] - '0'), 100000);
        if (ne == 0) return false;
        if (eneg) ex = -ex;
    }
    if (i != b || nd > 15) return false;
    const int e10 = ex - nfrac;
    if (e10 < -22 || e10 > 22) return false;
    double v = (double)m;                                  // exact: m < 10^15 < 2^53
    v = e10 >= 0 ? __dmul_rn(v, c_p10[e10]) : __ddiv_rn(v, c_p10[-e10]);
    *out = __double2float_rn(neg ? -v : v);
    return true;
}

// 1-based index token: digits only, saturated; false when the token is not a plain unsigned integer
__device__ __forceinline__ bool parse_index(const unsigned char* s, int& p, int ce, unsigned int* out) {
    unsigned long long v = 0;
    const int b = p;
    for (; p < ce && is_digit(s[p]); ++p) v = min(v * 10 + (s[p] - '0'), 0x80000000ull);
    *out = (unsigned int)v;
    return p > b;
}

// characters allowed after '%': tab and printable bytes (any '\r' that is not part of the line's "\r\n" rejects)
__device__ __forceinline__ bool comment_ok(const unsigned char* s, int p, int ce) {
    for (; p < ce; ++p)
        if (s[p] < 0x20 && s[p] != '\t') return false;
    return true;
}

// Parse the line starting at tile position q.  s points at tile position 0 (s[-16..-1] are staged); avail = staged
// bytes from q = 0 that belong to the block.
__device__ Line parse_line(const unsigned char* s, int q, int avail, bool block_ends_file) {
    Line L;
    L.kind = L_REJECT;
    L.ntok = 0;
    L.slow = 0;
    L.row = L.col = 0;
    L.val = 1.0f;
    L.vbeg = L.vlen = 0;
    const int lim = min(avail, q + MM_MAXLINE + 1);
    int e = q;
    while (e < lim && s[e] != '\n') ++e;
    if (e == lim && !(lim == avail && block_ends_file)) return L;      // over-long, or a block cut inside a line
    int ce = e;
    if (e < avail && ce > q && s[ce - 1] == '\r') --ce;                // "\r\n" line end
    int p = q;
    if (p < ce && s[p] == '%') {
        if (comment_ok(s, p + 1, ce)) L.kind = L_SKIP;
        return L;
    }
    while (p < ce && is_ws(s[p])) ++p;
    if (p == ce) {
        L.kind = L_SKIP;                                                 // empty or whitespace-only
        return L;
    }
    // [ws] int ws int [ws real] [ws] [% ...]
    if (!parse_index(s, p, ce, &L.row) || p == ce || !is_ws(s[p])) return L;
    while (p < ce && is_ws(s[p])) ++p;
    if (!parse_index(s, p, ce, &L.col)) return L;
    if (p < ce && !is_ws(s[p]) && s[p] != '%') return L;
    while (p < ce && is_ws(s[p])) ++p;
    L.ntok = 2;
    if (p < ce && s[p] != '%') {
        const int a = p;
        while (p < ce && is_tok(s[p])) ++p;
        if (p < ce && !is_ws(s[p]) && s[p] != '%') return L;
        L.ntok = 3;
        if (!fast_value(s, a, p, &L.val)) {
            L.slow = 1;
            L.vbeg = a;
            L.vlen = p - a;
        }
        while (p < ce && is_ws(s[p])) ++p;
    }
    if (p < ce && (s[p] != '%' || !comment_ok(s, p + 1, ce))) return L;  // a fourth token or a bad comment
    L.kind = L_DATA;
    return L;
}

__device__ __forceinline__ int block_exclusive_scan_int(int v, int* total, int* wbuf) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(FULL, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) wbuf[w] = inc;
    __syncthreads();
    int before = 0, tot = 0;
#pragma unroll
    for (int i = 0; i < MM_THREADS / 32; ++i) {
        const int t = wbuf[i];
        before += i < w ? t : 0;
        tot += t;
    }
    __syncthreads();
    *total = tot;
    return before + inc - v;
}

struct TileSmem {
    alignas(16) unsigned char text[MM_SMEM];
    unsigned short starts[MM_TILE];
    int wbuf[MM_THREADS / 32];
};

// Stage the tile and list its line starts in order; returns the number of lines starting in the tile.
__device__ int stage_tile(TileSmem& sm, const unsigned char* __restrict__ text, long long n, long long t0) {
    const uint4* src = reinterpret_cast<const uint4*>(text + t0 - 16);
    uint4* dst = reinterpret_cast<uint4*>(sm.text);
    for (int k = threadIdx.x; k < MM_SMEM / 16; k += MM_THREADS) dst[k] = src[k];
    __syncthreads();
    const unsigned char* s = sm.text + 16;
    const int q0 = threadIdx.x * 16;
    unsigned mask = 0;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const long long g = t0 + q0 + j;
        if (g < n && (g == 0 || s[q0 + j - 1] == '\n')) mask |= 1u << j;
    }
    int nl;
    int off = block_exclusive_scan_int(__popc(mask), &nl, sm.wbuf);
    while (mask) {
        const int j = __ffs(mask) - 1;
        mask &= mask - 1;
        sm.starts[off++] = (unsigned short)(q0 + j);
    }
    __syncthreads();
    return nl;
}

// pass 1: counts[tile] = (lines << 32) | data lines
__global__ void __launch_bounds__(MM_THREADS) mm_count_kernel(const unsigned char* __restrict__ text, long long n, int is_last,
                                                              long long* __restrict__ counts) {
    __shared__ TileSmem sm;
    const long long t0 = (long long)blockIdx.x * MM_TILE;
    const int nl = stage_tile(sm, text, n, t0);
    const int avail = (int)(n - t0 < MM_TILE + MM_HALO ? n - t0 : MM_TILE + MM_HALO);
    const bool ends_file = is_last && t0 + avail == n;
    int data = 0;
    for (int i = threadIdx.x; i < nl; i += MM_THREADS)
        data += parse_line(sm.text + 16, sm.starts[i], avail, ends_file).kind == L_DATA;
    int tot;
    block_exclusive_scan_int(data, &tot, sm.wbuf);
    if (threadIdx.x == 0) counts[blockIdx.x] = ((long long)nl << 32) | (long long)tot;
}

struct WriteArgs {
    const unsigned char* text;
    long long n;
    int is_last;
    long long block_offset;              // offset of the block's first byte from the first fed byte
    long long header_lines;              // lines before the first fed byte
    const long long* incl;               // inclusive scan of mm_count_kernel's counts
    MMState* state;
    long long cap;                       // capacity of the triple arrays
    int32_t *row, *col;
    float* val;
    long long slow_cap;
    long long *slow_ord, *slow_pos;      // slow_pos = (offset << 11) | length
    int32_t num_rows, num_cols;
};

// pass 2: parse again and write the triples at their ordinals
__global__ void __launch_bounds__(MM_THREADS) mm_write_kernel(WriteArgs a) {
    __shared__ TileSmem sm;
    const long long t0 = (long long)blockIdx.x * MM_TILE;
    const int nl = stage_tile(sm, a.text, a.n, t0);
    const int avail = (int)(a.n - t0 < MM_TILE + MM_HALO ? a.n - t0 : MM_TILE + MM_HALO);
    const bool ends_file = a.is_last && t0 + avail == a.n;
    const long long before = blockIdx.x ? a.incl[blockIdx.x - 1] : 0;
    long long ord = a.state->ord_base + (before & 0xffffffffll);
    const long long line0 = a.header_lines + a.state->line_base + (before >> 32);
    unsigned tokmask = 0;
    for (int base = 0; base < nl; base += MM_THREADS) {
        const int i = base + threadIdx.x;
        Line L;
        L.kind = L_NONE;
        if (i < nl) L = parse_line(sm.text + 16, sm.starts[i], avail, ends_file);
        int tot;
        const long long o = ord + block_exclusive_scan_int(L.kind == L_DATA, &tot, sm.wbuf);
        ord += tot;
        const unsigned long long lineno = (unsigned long long)(line0 + i + 1);
        if (L.kind == L_REJECT) atomicMin(&a.state->reject_line, lineno);
        if (L.kind == L_DATA) {
            tokmask |= 1u << L.ntok;
            if (L.row < 1 || L.row > (unsigned)a.num_rows || L.col < 1 || L.col > (unsigned)a.num_cols) {
                atomicMin(&a.state->range_line, lineno);
            } else if (o < a.cap) {
                a.row[o] = (int32_t)L.row - 1;
                a.col[o] = (int32_t)L.col - 1;
                a.val[o] = L.val;
                if (L.slow) {
                    const unsigned long long k = atomicAdd(&a.state->n_slow, 1ull);
                    if ((long long)k < a.slow_cap) {
                        a.slow_ord[k] = o;
                        a.slow_pos[k] = ((a.block_offset + t0 + L.vbeg) << 11) | L.vlen;
                    }
                }
            }
        }
    }
    tokmask = __reduce_or_sync(FULL, tokmask);
    if ((threadIdx.x & 31) == 0 && tokmask) atomicOr(&a.state->tokmask, tokmask);
}

// the next block's ordinals and line numbers continue after this one's
__global__ void mm_advance_kernel(const long long* __restrict__ incl, long long tiles, MMState* state) {
    const long long tot = incl[tiles - 1];
    state->ord_base += tot & 0xffffffffll;
    state->line_base += tot >> 32;
}

__global__ void mm_patch_kernel(const long long* __restrict__ ord, const float* __restrict__ v, long long n, long long cap,
                                float* __restrict__ val) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        if (ord[i] >= 0 && ord[i] < cap) val[ord[i]] = v[i];
}

// vali arrays = entries at the sampled ordinals; the rest keep their order: entry i moves to i - #(samples < i)
__global__ void mm_gather_kernel(const long long* __restrict__ idx, long long ns, const int32_t* __restrict__ row,
                                 const int32_t* __restrict__ col, const float* __restrict__ val, int32_t* __restrict__ vrow,
                                 int32_t* __restrict__ vcol, float* __restrict__ vval) {
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < ns; j += (long long)gridDim.x * blockDim.x) {
        const long long i = idx[j];
        vrow[j] = row[i];
        vcol[j] = col[i];
        vval[j] = val[i];
    }
}
__global__ void mm_compact_kernel(const long long* __restrict__ idx, long long ns, long long n, const int32_t* __restrict__ row,
                                  const int32_t* __restrict__ col, const float* __restrict__ val, int32_t* __restrict__ orow,
                                  int32_t* __restrict__ ocol, float* __restrict__ oval) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        long long lo = 0, hi = ns;                        // lo = #(samples < i)
        while (lo < hi) {
            const long long mid = (lo + hi) >> 1;
            if (idx[mid] < i) lo = mid + 1;
            else hi = mid;
        }
        if (lo < ns && idx[lo] == i) continue;
        orow[i - lo] = row[i];
        ocol[i - lo] = col[i];
        oval[i - lo] = val[i];
    }
}

enum { ST_H2D = 0, ST_PARSE, ST_PATCH, ST_SPLIT, ST_CSR_ROW, ST_CSR_COL, ST_D2H, ST_COUNT };

}  // namespace

struct bfl_mm_ingest : TextIngest {
    int32_t num_rows = 0, num_cols = 0;
    long long cap = 0, buf_bytes = 0, header_lines = 0, slow_cap = 0;
    cudaStream_t copy = nullptr;                           // uploads of the staging buffers
    unsigned char* dev[2] = {nullptr, nullptr};            // device text buffers (16-byte front pad)
    cudaEvent_t parsed[2] = {nullptr, nullptr};
    bool parse_pending[2] = {false, false};
    long long nnz = -1;
    bool split_done = false;
    MMState* state = nullptr;
    long long* counts = nullptr;
    int32_t *row = nullptr, *col = nullptr;
    float* val = nullptr;
    long long *slow_ord = nullptr, *slow_pos = nullptr;

    ~bfl_mm_ingest() override {
        if (comp) cudaStreamSynchronize(comp);
        if (copy) cudaStreamSynchronize(copy);
        for (int i = 0; i < 2; ++i) {
            if (dev[i]) cudaFree(dev[i]);
            if (parsed[i]) cudaEventDestroy(parsed[i]);
        }
        for (void* p : {(void*)state, (void*)counts, (void*)row, (void*)col, (void*)val, (void*)slow_ord, (void*)slow_pos})
            if (p) cudaFree(p);
        if (copy) cudaStreamDestroy(copy);
    }
};

namespace {

void free_triples(bfl_mm_ingest* h) {
    if (h->row) cudaFreeAsync(h->row, h->comp);
    if (h->col) cudaFreeAsync(h->col, h->comp);
    if (h->val) cudaFreeAsync(h->val, h->comp);
    h->row = h->col = nullptr;
    h->val = nullptr;
}

}  // namespace

extern "C" {

bfl_mm_ingest_t* bfl_mm_ingest_create(int32_t num_rows, int32_t num_cols, int64_t nnz_hint, int64_t block_bytes,
                                      int64_t header_lines, int64_t slow_cap) {
    if (BFL_OK != require_device()) return nullptr;
    if (num_rows <= 0 || num_cols <= 0 || nnz_hint <= 0 || block_bytes < 16 || block_bytes > (1ll << 30) ||
        header_lines < 0 || slow_cap < 0) {
        set_error("bad MatrixMarket ingest arguments");
        return nullptr;
    }
    auto* h = new bfl_mm_ingest();
    h->num_rows = num_rows;
    h->num_cols = num_cols;
    h->cap = nnz_hint;
    h->header_lines = header_lines;
    h->slow_cap = std::max<int64_t>(slow_cap, 1);
    // the last tile of a block stages MM_SMEM bytes from 16 before its start
    h->buf_bytes = (block_bytes + MM_TILE - 1) / MM_TILE * MM_TILE + MM_SMEM;
    bool ok = setup(h, block_bytes, ST_COUNT) && cudaStreamCreateWithFlags(&h->copy, cudaStreamNonBlocking) == cudaSuccess;
    for (int i = 0; ok && i < 2; ++i)
        ok = cudaMallocAsync(&h->dev[i], (size_t)h->buf_bytes, h->comp) == cudaSuccess &&
             cudaMemsetAsync(h->dev[i], 0, (size_t)h->buf_bytes, h->comp) == cudaSuccess &&
             cudaEventCreateWithFlags(&h->parsed[i], cudaEventDisableTiming) == cudaSuccess;
    const long long tiles = (block_bytes + MM_TILE - 1) / MM_TILE;
    ok = ok && cudaMallocAsync(&h->state, sizeof(MMState), h->comp) == cudaSuccess &&
         cudaMallocAsync(&h->counts, sizeof(long long) * tiles, h->comp) == cudaSuccess &&
         cudaMallocAsync(&h->row, sizeof(int32_t) * h->cap, h->comp) == cudaSuccess &&
         cudaMallocAsync(&h->col, sizeof(int32_t) * h->cap, h->comp) == cudaSuccess &&
         cudaMallocAsync(&h->val, sizeof(float) * h->cap, h->comp) == cudaSuccess &&
         cudaMallocAsync(&h->slow_ord, sizeof(long long) * h->slow_cap, h->comp) == cudaSuccess &&
         cudaMallocAsync(&h->slow_pos, sizeof(long long) * h->slow_cap, h->comp) == cudaSuccess;
    if (ok) {
        MMState s0 = {0, 0, ~0ull, ~0ull, 0ull, 0u};
        ok = cudaMemcpyAsync(h->state, &s0, sizeof(s0), cudaMemcpyHostToDevice, h->comp) == cudaSuccess &&
             cudaStreamSynchronize(h->comp) == cudaSuccess;
    }
    return setup_done(h, ok, "MatrixMarket");
}

void bfl_mm_ingest_destroy(bfl_mm_ingest_t* h) { delete h; }

int bfl_mm_ingest_staging(bfl_mm_ingest_t* h, int slot, void** host_ptr) { return staging(h, slot, host_ptr); }

int bfl_mm_ingest_feed(bfl_mm_ingest_t* h, int slot, int64_t n, int is_last) {
    if (int rc = check_feed(h, slot, n, is_last)) return rc;
    if (n == 0) return BFL_OK;
    unsigned char* d = h->dev[slot] + 16;
    // the device buffer is free once the parse that last read it has finished
    if (h->parse_pending[slot]) BFL_CUDA(cudaStreamWaitEvent(h->copy, h->parsed[slot], 0));
    if (int rc = mark(h, ST_H2D, h->copy)) return rc;
    BFL_CUDA(cudaMemcpyAsync(d, h->host[slot], (size_t)n, cudaMemcpyHostToDevice, h->copy));
    if (int rc = mark(h, ST_H2D, h->copy)) return rc;
    BFL_CUDA(cudaEventRecord(h->copied[slot], h->copy));
    h->copy_pending[slot] = true;
    BFL_CUDA(cudaStreamWaitEvent(h->comp, h->copied[slot], 0));
    if (int rc = mark(h, ST_PARSE, h->comp)) return rc;
    const long long tiles = (n + MM_TILE - 1) / MM_TILE;
    mm_count_kernel<<<(unsigned)tiles, MM_THREADS, 0, h->comp>>>(d, n, is_last, h->counts);
    BFL_LAUNCHED();
    if (int rc = inclusive_scan_i64(h->counts, h->counts, tiles, h->comp)) return rc;
    WriteArgs a;
    a.text = d;
    a.n = n;
    a.is_last = is_last;
    a.block_offset = h->fed;
    a.header_lines = h->header_lines;
    a.incl = h->counts;
    a.state = h->state;
    a.cap = h->cap;
    a.row = h->row;
    a.col = h->col;
    a.val = h->val;
    a.slow_cap = h->slow_cap;
    a.slow_ord = h->slow_ord;
    a.slow_pos = h->slow_pos;
    a.num_rows = h->num_rows;
    a.num_cols = h->num_cols;
    mm_write_kernel<<<(unsigned)tiles, MM_THREADS, 0, h->comp>>>(a);
    BFL_LAUNCHED();
    mm_advance_kernel<<<1, 1, 0, h->comp>>>(h->counts, tiles, h->state);
    BFL_LAUNCHED();
    if (int rc = mark(h, ST_PARSE, h->comp)) return rc;
    BFL_CUDA(cudaEventRecord(h->parsed[slot], h->comp));
    h->parse_pending[slot] = true;
    h->fed += n;
    return BFL_OK;
}

int bfl_mm_ingest_finish(bfl_mm_ingest_t* h, int64_t* nnz, int32_t* tokmask, int64_t* reject_line, int64_t* range_line,
                         int64_t* n_slow) {
    if (!h || !nnz || !tokmask || !reject_line || !range_line || !n_slow) BFL_FAIL(BFL_ERR_ARG, "bad finish arguments");
    if (!h->last_fed) BFL_FAIL(BFL_ERR_STATE, "finish before the last block was fed");
    MMState s;
    BFL_CUDA(cudaStreamSynchronize(h->copy));
    BFL_CUDA(cudaMemcpyAsync(&s, h->state, sizeof(s), cudaMemcpyDeviceToHost, h->comp));
    BFL_CUDA(cudaStreamSynchronize(h->comp));
    for (int i = 0; i < 2; ++i) {                          // the text buffers are not needed any more
        BFL_CUDA(cudaFreeAsync(h->dev[i], h->comp));
        h->dev[i] = nullptr;
    }
    BFL_CUDA(cudaFreeAsync(h->counts, h->comp));
    h->counts = nullptr;
    h->nnz = s.ord_base;
    *nnz = s.ord_base;
    *tokmask = (int32_t)s.tokmask;
    *reject_line = s.reject_line == ~0ull ? -1 : (int64_t)s.reject_line;
    *range_line = s.range_line == ~0ull ? -1 : (int64_t)s.range_line;
    *n_slow = (int64_t)s.n_slow;
    return BFL_OK;
}

// slow value tokens: ordinal and byte offset from the first fed byte and length, in no particular order
int bfl_mm_ingest_slow_tokens(bfl_mm_ingest_t* h, int64_t n, int64_t* ordinal, int64_t* offset, int32_t* length) {
    if (!h || h->nnz < 0 || n < 0 || n > h->slow_cap || (n && (!ordinal || !offset || !length)))
        BFL_FAIL(BFL_ERR_ARG, "bad slow-token arguments");
    if (n == 0) return BFL_OK;
    std::vector<long long> pos((size_t)n);
    BFL_CUDA(cudaMemcpyAsync(ordinal, h->slow_ord, sizeof(long long) * n, cudaMemcpyDeviceToHost, h->comp));
    BFL_CUDA(cudaMemcpyAsync(pos.data(), h->slow_pos, sizeof(long long) * n, cudaMemcpyDeviceToHost, h->comp));
    BFL_CUDA(cudaStreamSynchronize(h->comp));
    for (long long i = 0; i < n; ++i) {
        offset[i] = pos[i] >> 11;
        length[i] = (int32_t)(pos[i] & 2047);
    }
    return BFL_OK;
}

int bfl_mm_ingest_patch_values(bfl_mm_ingest_t* h, const int64_t* ordinal, const float* val, int64_t n) {
    if (!h || h->nnz < 0 || h->split_done || n < 0 || (n && (!ordinal || !val))) BFL_FAIL(BFL_ERR_ARG, "bad patch arguments");
    if (n == 0) return BFL_OK;
    if (int rc = mark(h, ST_PATCH, h->comp)) return rc;
    long long* d_ord = nullptr;
    float* d_val = nullptr;
    BFL_CUDA(cudaMallocAsync(&d_ord, sizeof(long long) * n, h->comp));
    BFL_CUDA(cudaMallocAsync(&d_val, sizeof(float) * n, h->comp));
    BFL_CUDA(cudaMemcpyAsync(d_ord, ordinal, sizeof(long long) * n, cudaMemcpyHostToDevice, h->comp));
    BFL_CUDA(cudaMemcpyAsync(d_val, val, sizeof(float) * n, cudaMemcpyHostToDevice, h->comp));
    mm_patch_kernel<<<grid_for(n), 256, 0, h->comp>>>(d_ord, d_val, n, std::min(h->cap, h->nnz), h->val);
    BFL_LAUNCHED();
    BFL_CUDA(cudaFreeAsync(d_ord, h->comp));
    BFL_CUDA(cudaFreeAsync(d_val, h->comp));
    if (int rc = mark(h, ST_PATCH, h->comp)) return rc;
    BFL_CUDA(cudaStreamSynchronize(h->comp));              // the caller's host arrays may go away
    return BFL_OK;
}

int bfl_mm_ingest_split(bfl_mm_ingest_t* h, const int64_t* sample_idx, int64_t n, int32_t* out_row, int32_t* out_col,
                        float* out_val) {
    if (!h || h->nnz < 0 || h->split_done || n < 0 || (n && (!sample_idx || !out_row || !out_col || !out_val)))
        BFL_FAIL(BFL_ERR_ARG, "bad split arguments");
    if (h->nnz > h->cap) BFL_FAIL(BFL_ERR_STATE, "more data lines than the capacity given at create");
    for (int64_t j = 0; j < n; ++j)
        if (sample_idx[j] < 0 || sample_idx[j] >= h->nnz || (j && sample_idx[j] <= sample_idx[j - 1]))
            BFL_FAIL(BFL_ERR_ARG, "sample indexes must be strictly increasing data-line ordinals");
    const long long nt = h->nnz - n;
    h->split_done = true;
    if (n == 0) return BFL_OK;
    if (int rc = mark(h, ST_SPLIT, h->comp)) return rc;
    long long* d_idx = nullptr;
    int32_t *vr = nullptr, *vc = nullptr, *orow = nullptr, *ocol = nullptr;
    float *vv = nullptr, *oval = nullptr;
    BFL_CUDA(cudaMallocAsync(&d_idx, sizeof(long long) * n, h->comp));
    BFL_CUDA(cudaMallocAsync(&vr, sizeof(int32_t) * n, h->comp));
    BFL_CUDA(cudaMallocAsync(&vc, sizeof(int32_t) * n, h->comp));
    BFL_CUDA(cudaMallocAsync(&vv, sizeof(float) * n, h->comp));
    BFL_CUDA(cudaMemcpyAsync(d_idx, sample_idx, sizeof(long long) * n, cudaMemcpyHostToDevice, h->comp));
    mm_gather_kernel<<<grid_for(n), 256, 0, h->comp>>>(d_idx, n, h->row, h->col, h->val, vr, vc, vv);
    BFL_LAUNCHED();
    const size_t m = (size_t)std::max<long long>(nt, 1);
    BFL_CUDA(cudaMallocAsync(&orow, sizeof(int32_t) * m, h->comp));
    BFL_CUDA(cudaMallocAsync(&ocol, sizeof(int32_t) * m, h->comp));
    BFL_CUDA(cudaMallocAsync(&oval, sizeof(float) * m, h->comp));
    mm_compact_kernel<<<grid_for(h->nnz), 256, 0, h->comp>>>(d_idx, n, h->nnz, h->row, h->col, h->val, orow, ocol, oval);
    BFL_LAUNCHED();
    free_triples(h);
    h->row = orow;
    h->col = ocol;
    h->val = oval;
    if (int rc = mark(h, ST_SPLIT, h->comp)) return rc;
    BFL_CUDA(cudaMemcpyAsync(out_row, vr, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, h->comp));
    BFL_CUDA(cudaMemcpyAsync(out_col, vc, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, h->comp));
    BFL_CUDA(cudaMemcpyAsync(out_val, vv, sizeof(float) * n, cudaMemcpyDeviceToHost, h->comp));
    for (void* p : {(void*)d_idx, (void*)vr, (void*)vc, (void*)vv}) BFL_CUDA(cudaFreeAsync(p, h->comp));
    BFL_CUDA(cudaStreamSynchronize(h->comp));
    h->nnz = nt;
    return BFL_OK;
}

int bfl_mm_ingest_build(bfl_mm_ingest_t* h, int orientation, int64_t* indptr, int32_t* key, float* val) {
    if (!h || !h->split_done || orientation < 0 || orientation > 1 || h->built[orientation] || !indptr ||
        (h->nnz && (!key || !val)))
        BFL_FAIL(BFL_ERR_ARG, "bad build arguments (split first, each orientation once)");
    if (int rc = build_to_host(h, orientation, h->row, h->col, h->val, h->nnz, h->num_rows, h->num_cols, 1,
                               orientation ? ST_CSR_COL : ST_CSR_ROW, ST_D2H, indptr, key, val))
        return rc;
    if (h->built[0] && h->built[1]) free_triples(h);       // the sort's inputs are not needed any more
    return BFL_OK;
}

// stage_ms[7]: H2D, parse, patch, split, rowwise CSR, colwise CSR, D2H (summed device time of each stage);
// *peak_bytes: high-water mark of the device's default memory pool since create
int bfl_mm_ingest_stats(bfl_mm_ingest_t* h, double* stage_ms, int64_t* peak_bytes) {
    if (h) BFL_CUDA(cudaStreamSynchronize(h->copy));
    return stats(h, stage_ms, peak_bytes);
}

}  // extern "C"
