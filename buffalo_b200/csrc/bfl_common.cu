// Host-side plumbing shared by the ALS and SGD backends: last-error slot, launch counter,
// device check, and the flat JSON option reader.
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
