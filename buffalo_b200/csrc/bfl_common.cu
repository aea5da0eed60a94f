// Host-side plumbing shared by the ALS, SGD and pLSI backends: last-error slot, launch counter,
// device check, the holder core and the flat JSON option reader.
#include "bfl_common.cuh"

#include <cctype>
#include <fstream>
#include <sstream>

namespace bfl {

static thread_local std::string t_last_error;
std::atomic<long long> g_launches{0};

void set_error(const std::string& msg) { t_last_error = msg; }

int require_device() {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        cudaGetLastError();
        BFL_FAIL(BFL_ERR_CUDA, std::string("no CUDA device available (") +
                                   (e != cudaSuccess ? cudaGetErrorString(e) : "device count 0") +
                                   "); buffalo_b200 has no CPU fallback");
    }
    int dev = 0;
    BFL_CUDA(cudaGetDevice(&dev));
    int major = 0, minor = 0;
    BFL_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
    BFL_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
    if (major != 9 || minor != 0)   // sm_90a code (wgmma) runs on compute capability 9.0 only
        BFL_FAIL(BFL_ERR_CUDA, "buffalo_b200 kernels are compiled for sm_90a only; current device has compute capability " +
                                   std::to_string(major) + "." + std::to_string(minor));
    return BFL_OK;
}

// ---- holder core ----------------------------------------------------------------------
Holder::~Holder() {
    if (stream) cudaStreamDestroy(stream);
}

int Holder::attach_device() {
    if (BFL_OK != require_device()) return BFL_ERR_CUDA;
    int dev = 0;
    BFL_CUDA(cudaGetDevice(&dev));
    BFL_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
    if (!stream) BFL_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    return BFL_OK;
}

int Holder::borrow_factors(float* P, int64_t P_rows_, float* Q, int64_t Q_rows_) {
    if (!P || !Q || P_rows_ <= 0 || Q_rows_ <= 0) BFL_FAIL(BFL_ERR_ARG, "bad factor arguments");
    if (((uintptr_t)P | (uintptr_t)Q) & 15) BFL_FAIL(BFL_ERR_ARG, "device factor pointers must be 16-byte aligned");
    hostP = hostQ = nullptr;
    ownP.release();
    ownQ.release();
    dP = P;
    dQ = Q;
    P_rows = P_rows_;
    Q_rows = Q_rows_;
    return BFL_OK;
}

int Holder::mirror_factors(float* P, int64_t P_rows_, float* Q, int64_t Q_rows_) {
    if (!P || !Q || P_rows_ <= 0 || Q_rows_ <= 0) BFL_FAIL(BFL_ERR_ARG, "bad factor arguments");
    hostP = P;
    hostQ = Q;
    P_rows = P_rows_;
    Q_rows = Q_rows_;
    if (BFL_OK != ownP.reserve((size_t)P_rows * vdim)) return BFL_ERR_CUDA;
    if (BFL_OK != ownQ.reserve((size_t)Q_rows * vdim)) return BFL_ERR_CUDA;
    dP = ownP.p;
    dQ = ownQ.p;
    return BFL_OK;
}

int init_holder(Holder* h, const char* src, bool is_path) {
    if (!h || !src) BFL_FAIL(BFL_ERR_ARG, "null argument");
    JsonOpt j;
    std::string err;
    if (is_path ? !j.load(src, &err) : !j.parse(src, &err))
        BFL_FAIL(BFL_ERR_OPTION, is_path ? err : "Failed to parse: " + err);
    return h->apply_options(j);
}

int CsrBinding::bind(const int64_t* d_indptr, const int32_t* d_keys, const float* d_vals, int64_t n_rows,
                     int64_t n_nnz, bool with_vals) {
    if (!d_indptr || (n_nnz > 0 && (!d_keys || (with_vals && !d_vals))) || n_rows <= 0)
        BFL_FAIL(BFL_ERR_ARG, "bad CSR arguments");
    indptr = d_indptr;
    keys = d_keys;
    vals = d_vals;
    rows = n_rows;
    nnz = n_nnz;
    return BFL_OK;
}

int CsrBinding::check_range(int64_t row_begin, int64_t row_end) const {
    if (row_begin < 0 || row_end > rows || row_end < row_begin) BFL_FAIL(BFL_ERR_ARG, "bad row range");
    return BFL_OK;
}

int read_row_span(const int64_t* indptr, int64_t row_begin, int64_t row_end, cudaStream_t st, int64_t* begin,
                  int64_t* end) {
    int64_t ends[2] = {0, 0};
    if (row_begin > 0)
        BFL_CUDA(cudaMemcpyAsync(&ends[0], indptr + row_begin - 1, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    BFL_CUDA(cudaMemcpyAsync(&ends[1], indptr + row_end - 1, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    BFL_CUDA(cudaStreamSynchronize(st));
    *begin = ends[0];
    *end = ends[1];
    return BFL_OK;
}

// ---- JSON -----------------------------------------------------------------------------
namespace {
struct Cursor {
    const char* p;
    const char* end;
    std::string err;
    void ws() {
        while (p < end && std::isspace((unsigned char)*p)) ++p;
    }
    bool fail(const char* m) {
        if (err.empty()) err = m;
        return false;
    }
    bool str(std::string* out) {
        if (p >= end || *p != '"') return fail("expected string");
        ++p;
        std::string s;
        while (p < end && *p != '"') {
            if (*p == '\\') {
                ++p;
                if (p >= end) return fail("bad escape");
                switch (*p) {
                    case 'n': s += '\n'; break;
                    case 't': s += '\t'; break;
                    case 'r': s += '\r'; break;
                    case 'b': s += '\b'; break;
                    case 'f': s += '\f'; break;
                    case 'u':
                        if (end - p < 5) return fail("bad \\u escape");
                        s += '?';
                        p += 4;
                        break;
                    default: s += *p;
                }
                ++p;
            } else {
                s += *p++;
            }
        }
        if (p >= end) return fail("unterminated string");
        ++p;
        if (out) *out = s;
        return true;
    }
    bool skip_value() {
        ws();
        if (p >= end) return fail("unexpected end");
        if (*p == '"') return str(nullptr);
        if (*p == '{' || *p == '[') {
            char open = *p, close = (*p == '{') ? '}' : ']';
            ++p;
            ws();
            if (p < end && *p == close) {
                ++p;
                return true;
            }
            while (true) {
                ws();
                if (open == '{') {
                    if (!str(nullptr)) return false;
                    ws();
                    if (p >= end || *p != ':') return fail("expected ':'");
                    ++p;
                }
                if (!skip_value()) return false;
                ws();
                if (p < end && *p == ',') {
                    ++p;
                    continue;
                }
                if (p < end && *p == close) {
                    ++p;
                    return true;
                }
                return fail("expected ',' or close");
            }
        }
        // literal / number
        const char* s = p;
        while (p < end && *p != ',' && *p != '}' && *p != ']' && !std::isspace((unsigned char)*p)) ++p;
        return p > s ? true : fail("empty value");
    }
};
}  // namespace

bool JsonOpt::parse(const std::string& text, std::string* err) {
    Cursor c{text.data(), text.data() + text.size(), ""};
    c.ws();
    if (c.p >= c.end || *c.p != '{') {
        if (err) *err = "option JSON must be an object";
        return false;
    }
    ++c.p;
    c.ws();
    if (c.p < c.end && *c.p == '}') return true;
    while (true) {
        c.ws();
        std::string key;
        if (!c.str(&key)) break;
        c.ws();
        if (c.p >= c.end || *c.p != ':') {
            c.fail("expected ':'");
            break;
        }
        ++c.p;
        c.ws();
        if (c.p >= c.end) {
            c.fail("unexpected end");
            break;
        }
        if (*c.p == '"') {
            std::string v;
            if (!c.str(&v)) break;
            str[key] = v;
        } else if (*c.p == '{' || *c.p == '[') {
            if (!c.skip_value()) break;
        } else {
            const char* s = c.p;
            if (!c.skip_value()) break;
            std::string lit(s, c.p);
            if (lit == "true") boolean[key] = true;
            else if (lit == "false") boolean[key] = false;
            else if (lit == "null") {}
            else {
                char* e = nullptr;
                double v = std::strtod(lit.c_str(), &e);
                if (e == lit.c_str() || *e != '\0') {
                    if (lit == "NaN" || lit == "Infinity" || lit == "-Infinity") {
                        num[key] = lit == "NaN" ? NAN : (lit[0] == '-' ? -INFINITY : INFINITY);
                    } else {
                        c.fail("bad literal");
                        break;
                    }
                } else {
                    num[key] = v;
                }
            }
        }
        c.ws();
        if (c.p < c.end && *c.p == ',') {
            ++c.p;
            continue;
        }
        if (c.p < c.end && *c.p == '}') return true;
        c.fail("expected ',' or '}'");
        break;
    }
    if (err) *err = c.err.empty() ? "parse error" : c.err;
    return false;
}

bool JsonOpt::load(const char* path, std::string* err) {
    std::ifstream in(path);
    if (!in.is_open()) {
        if (err) *err = std::string("File not exists: ") + path;
        return false;
    }
    std::stringstream ss;
    ss << in.rdbuf();
    return parse(ss.str(), err);
}

}  // namespace bfl

extern "C" {
const char* bfl_last_error(void) { return bfl::t_last_error.c_str(); }
int bfl_abi_version(void) { return 1; }
int bfl_compiled_sm(void) { return 90; }
int bfl_require_device(void) { return bfl::require_device(); }
int64_t bfl_kernel_launch_count(void) { return (int64_t)bfl::g_launches.load(); }
void* bfl_ipc_open(const void* handle64) {
    if (!handle64) {
        bfl::set_error("null IPC handle");
        return nullptr;
    }
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, sizeof(h));
    void* base = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
        cudaGetLastError();
        bfl::set_error(std::string("cudaIpcOpenMemHandle: ") + cudaGetErrorString(e));
        return nullptr;
    }
    return base;
}
void* bfl_dev_alloc(size_t bytes) {
    if (bfl::require_device() != BFL_OK) return nullptr;
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e != cudaSuccess) {
        cudaGetLastError();
        bfl::set_error(std::string("cudaMalloc: ") + cudaGetErrorString(e));
        return nullptr;
    }
    return p;
}
int bfl_dev_free(void* p) {
    if (p) BFL_CUDA(cudaFree(p));
    return BFL_OK;
}
int bfl_ipc_export(void* dev_ptr, void* out_handle64) {
    if (!dev_ptr || !out_handle64) BFL_FAIL(BFL_ERR_ARG, "null argument");
    cudaIpcMemHandle_t h;
    BFL_CUDA(cudaIpcGetMemHandle(&h, dev_ptr));
    memcpy(out_handle64, &h, sizeof(h));
    return BFL_OK;
}
int bfl_ipc_close(void* base) {
    if (!base) return BFL_OK;
    BFL_CUDA(cudaIpcCloseMemHandle(base));
    return BFL_OK;
}
}
