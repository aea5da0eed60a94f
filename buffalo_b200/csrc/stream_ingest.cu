// Stream text -> database on the device (DESIGN.md 4.7): one line per user of whitespace-separated item tokens.  The
// text is streamed through two pinned host buffers; tokens are found byte-parallel, interned in a device hash table and
// numbered in first-appearance order, and the (user, item) pairs stay on the device through the validation split and
// the CSR builds (bfl_csr_from_triples_device).
//
// Parse of one block (a byte range that ends with '\n', or at the end of the file):
//   * each thread classifies 16 bytes plus 3 bytes of context on each side: separators (the ASCII whitespace set the
//     caller passes), '\n', a bare '\r', and the UTF-8 lead/continuation structure (strict: overlong forms,
//     surrogates and code points above U+10FFFF are invalid); multi-byte whitespace code points are reported, not
//     parsed;
//   * pass 1 counts token starts and '\n' per 4 KiB tile, an int64 scan gives each tile its first token ordinal and
//     line, pass 2 writes every token's line (the user), byte offset, length and a 64-bit hash of its bytes.
// Interning, in separate launches so that no thread ever waits for another: (a) claim a slot by CAS on the hash and
// atomicMin the first-occurrence ordinal into it, (b) the occurrence whose ordinal is the slot's minimum copies its
// bytes into a string pool and gets an entry, (c) every occurrence compares its bytes with its entry's and records the
// entry.  A mismatch is a hash collision between distinct tokens and declines the file.  The table grows (rehash) when
// its load passes 1/2 after a block, or when a claim finds no free slot.  With an iid list, the table is built from
// the names first (last index wins) and frozen; a token it does not hold declines the file.
#include <algorithm>
#include <climits>
#include <vector>

#include "bfl_common.cuh"
#include "text_ingest.cuh"

using namespace bfl;

namespace {

constexpr int ST_THREADS = 256;
constexpr int ST_TILE = 16 * ST_THREADS;                // bytes per CTA of the parse, 16 per thread
constexpr int ST_CTX = 3;                               // context bytes on each side (a UTF-8 sequence has <= 4 bytes)
constexpr int ST_WIN = 16 + 2 * ST_CTX;
constexpr int NO_BYTE = 0x100;                          // past the end of the block
constexpr int CT_ITEMS = 8;                             // compaction: contiguous items per thread
constexpr int CT_TILE = CT_ITEMS * ST_THREADS;
constexpr int MAX_USPACE = 32;
constexpr unsigned long long MAX_PROBES = 1024;         // an insert probing further reports overflow (table too full)

enum : unsigned { D_BARE_CR = 1, D_UTF8 = 2, D_USPACE = 4, D_IID_MISS = 8, D_COLLISION = 16, D_MEMORY = 32, D_LINES = 64 };

struct STState {
    unsigned long long decline_line;     // smallest 1-based line that carries a decline reason (ULLONG_MAX: none)
    unsigned int decline;                // D_* bits
    unsigned int overflow;               // a claim found no free slot
    unsigned long long n_entries;        // distinct tokens with a pool entry
    unsigned long long pool_used;        // bytes of the pool in use
};

struct Grammar {
    unsigned long long ascii_ws;         // bit c set: byte c < 64 separates tokens
    int n_uspace;
    int uspace[MAX_USPACE];              // multi-byte whitespace code points (declined)
};

struct Table {                           // open addressing, linear probing; key 0 = empty
    unsigned long long* key;
    long long* first;                    // smallest ordinal of the key (LLONG_MAX: none yet)
    int32_t* entry;                      // pool entry (-1: none yet)
    unsigned long long mask;
};

struct Entries {
    long long *off, *first, *foff;       // pool offset, first ordinal, offset of the first occurrence in the input
    int32_t* len;
};

__device__ __forceinline__ bool is_sep(int c, unsigned long long ws) { return c < 64 && ((ws >> c) & 1ull); }
__device__ __forceinline__ bool is_cont(int c) { return c < 0x100 && (c & 0xC0) == 0x80; }
__device__ __forceinline__ int lead_len(int c) {
    return c >= 0xC2 && c <= 0xDF ? 2 : c >= 0xE0 && c <= 0xEF ? 3 : c >= 0xF0 && c <= 0xF4 ? 4 : 0;
}

// D_UTF8, D_USPACE or 0 for the byte w[j]; w[j - 3 .. j + 3] are loaded
__device__ __forceinline__ unsigned utf8_check(const int* w, int j, const Grammar& g) {
    const int c = w[j];
    if (c < 0x80) return 0;
    if (is_cont(c)) {                    // owned by the lead k bytes back when that lead's sequence is longer than k
#pragma unroll
        for (int k = 1; k <= 3; ++k) {
            const int b = w[j - k];
            if (!is_cont(b)) return lead_len(b) > k ? 0u : D_UTF8;
        }
        return D_UTF8;
    }
    const int L = lead_len(c);
    if (!L) return D_UTF8;
    const int c1 = w[j + 1];
    if (!is_cont(c1) || (c == 0xE0 && c1 < 0xA0) || (c == 0xED && c1 > 0x9F) || (c == 0xF0 && c1 < 0x90) ||
        (c == 0xF4 && c1 > 0x8F))
        return D_UTF8;
    int cp = c & (0x7F >> L);
#pragma unroll
    for (int k = 1; k < 4; ++k) {
        if (k >= L) break;
        const int b = w[j + k];
        if (!is_cont(b)) return D_UTF8;
        cp = (cp << 6) | (b & 0x3F);
    }
    for (int k = 0; k < g.n_uspace; ++k)
        if (cp == g.uspace[k]) return D_USPACE;
    return 0;
}

// w[k] = byte g0 - 3 + k of the block; before the block is a line end, past its end NO_BYTE
__device__ __forceinline__ void load_window(const unsigned char* __restrict__ text, long long n, long long g0, int* w) {
#pragma unroll
    for (int k = 0; k < ST_CTX; ++k) {
        const long long g = g0 - ST_CTX + k;
        w[k] = g < 0 ? '\n' : text[g];
    }
    if (g0 + 16 <= n) {
        const uint4 v = *reinterpret_cast<const uint4*>(text + g0);
        const unsigned u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int k = 0; k < 16; ++k) w[ST_CTX + k] = (u[k >> 2] >> (8 * (k & 3))) & 255u;
    } else {
#pragma unroll
        for (int k = 0; k < 16; ++k) w[ST_CTX + k] = g0 + k < n ? text[g0 + k] : NO_BYTE;
    }
#pragma unroll
    for (int k = 0; k < ST_CTX; ++k) {
        const long long g = g0 + 16 + k;
        w[ST_CTX + 16 + k] = g < n ? text[g] : NO_BYTE;
    }
}

// bit j of *tok: a token starts at g0 + j; bit j of *nl: byte g0 + j is '\n'
__device__ __forceinline__ void masks(const int* w, unsigned long long ws, unsigned* tok, unsigned* nl) {
    unsigned t = 0, l = 0;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const int c = w[ST_CTX + j];
        if (c == NO_BYTE) continue;
        if (!is_sep(c, ws) && is_sep(w[ST_CTX + j - 1], ws)) t |= 1u << j;
        if (c == '\n') l |= 1u << j;
    }
    *tok = t;
    *nl = l;
}

__device__ __forceinline__ int block_exclusive_scan(int v, int* total, int* wbuf) {
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
    for (int i = 0; i < ST_THREADS / 32; ++i) {
        const int t = wbuf[i];
        before += i < w ? t : 0;
        tot += t;
    }
    __syncthreads();
    *total = tot;
    return before + inc - v;
}

__device__ __forceinline__ unsigned long long finish_hash(unsigned long long h, int bits) {
    h ^= h >> 33;                                          // fmix64
    h *= 0xff51afd7ed558ccdull;
    h ^= h >> 33;
    h *= 0xc4ceb9fe1a85ec53ull;
    h ^= h >> 33;
    if (bits < 64) return (h & ((1ull << bits) - 1)) + 1;  // truncated (tests): distinct tokens share keys
    return h ? h : 1;                                      // 0 marks an empty slot
}

__device__ __forceinline__ unsigned long long hash_bytes(const unsigned char* p, long long len, int bits) {
    unsigned long long h = 0xcbf29ce484222325ull;          // FNV-1a
    for (long long k = 0; k < len; ++k) h = (h ^ p[k]) * 0x100000001b3ull;
    return finish_hash(h, bits);
}

// pass 1: counts[tile] = (lines << 32) | tokens
__global__ void __launch_bounds__(ST_THREADS) st_count_kernel(const unsigned char* __restrict__ text, long long n,
                                                              unsigned long long ws, long long* __restrict__ counts) {
    __shared__ int wbuf[ST_THREADS / 32];
    const long long g0 = (long long)blockIdx.x * ST_TILE + threadIdx.x * 16;
    int w[ST_WIN];
    load_window(text, n, g0, w);
    unsigned tok, nl;
    masks(w, ws, &tok, &nl);
    int tot;
    block_exclusive_scan((__popc(nl) << 16) | __popc(tok), &tot, wbuf);
    if (threadIdx.x == 0) counts[blockIdx.x] = ((long long)(tot >> 16) << 32) | (long long)(tot & 0xffff);
}

struct WriteArgs {
    const unsigned char* text;
    long long n;
    long long tok_base, line_base;       // tokens and lines before the block
    const long long* incl;               // inclusive scan of st_count_kernel's counts
    Grammar g;
    int hash_bits;
    STState* state;
    int32_t* user;                       // [ordinal] line of the token
    long long* boff;                     // [block token] offset in the block
    int32_t* blen;
    unsigned long long* bhash;
};

// pass 2: check the grammar and write every token
__global__ void __launch_bounds__(ST_THREADS) st_write_kernel(WriteArgs a) {
    __shared__ int wbuf[ST_THREADS / 32];
    const long long g0 = (long long)blockIdx.x * ST_TILE + threadIdx.x * 16;
    int w[ST_WIN];
    load_window(a.text, a.n, g0, w);
    unsigned tok, nl;
    masks(w, a.g.ascii_ws, &tok, &nl);
    int tot;
    const int excl = block_exclusive_scan((__popc(nl) << 16) | __popc(tok), &tot, wbuf);
    const long long before = blockIdx.x ? a.incl[blockIdx.x - 1] : 0;
    const long long tok0 = (before & 0xffffffffll) + (excl & 0xffff);
    const long long line0 = a.line_base + (before >> 32) + (excl >> 16);
    unsigned bits = 0;
    unsigned long long bad_line = ~0ull;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const int c = w[ST_CTX + j];
        if (c == NO_BYTE) continue;
        unsigned b = utf8_check(w, ST_CTX + j, a.g);
        if (c == '\r' && w[ST_CTX + j + 1] != '\n') b |= D_BARE_CR;
        if (b) {
            bits |= b;
            bad_line = min(bad_line, (unsigned long long)(line0 + __popc(nl & ((1u << j) - 1u)) + 1));
        }
    }
    if (bits) {
        atomicOr(&a.state->decline, bits);
        atomicMin(&a.state->decline_line, bad_line);
    }
    int r = 0;
    while (tok) {
        const int j = __ffs(tok) - 1;
        tok &= tok - 1;
        const long long b = tok0 + r++;
        const long long s = g0 + j;
        long long e = s;
        unsigned long long h = 0xcbf29ce484222325ull;
        for (; e < a.n && !is_sep(a.text[e], a.g.ascii_ws); ++e) h = (h ^ a.text[e]) * 0x100000001b3ull;
        a.boff[b] = s;
        a.blen[b] = (int32_t)(e - s);
        a.bhash[b] = finish_hash(h, a.hash_bits);
        a.user[a.tok_base + b] = (int32_t)(line0 + __popc(nl & ((1u << j) - 1u)));
    }
}

// names (iid list): hash, offset and length of each
__global__ void st_name_kernel(const unsigned char* __restrict__ names, const long long* __restrict__ offs, long long n,
                               int bits, long long* __restrict__ boff, int32_t* __restrict__ blen,
                               unsigned long long* __restrict__ bhash) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        boff[i] = offs[i];
        blen[i] = (int32_t)(offs[i + 1] - offs[i]);
        bhash[i] = hash_bytes(names + offs[i], offs[i + 1] - offs[i], bits);
    }
}

// (a) claim: every occurrence finds or claims its key's slot; the slot keeps the smallest ordinal.  Occurrence i has
// ordinal ord_base + ord_step * i.  frozen: lookup only, a miss declines.  An insert gives up after MAX_PROBES slots
// and reports overflow; a key is always stored within MAX_PROBES of its home slot or by a rehash, so a later
// occurrence that gives up makes the table grow, never a duplicate key.
__global__ void st_claim_kernel(const unsigned long long* __restrict__ bhash, long long nb, long long ord_base, int ord_step,
                                Table t, int frozen, const int32_t* __restrict__ user, STState* st, int32_t* __restrict__ slot_of) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nb; i += (long long)gridDim.x * blockDim.x) {
        const unsigned long long h = bhash[i];
        const long long ord = ord_base + ord_step * i;
        unsigned long long pos = h & t.mask;
        long long found = -1;
        const unsigned long long limit = frozen ? t.mask + 1 : min(t.mask + 1, MAX_PROBES);
        for (unsigned long long probe = 0; probe < limit; ++probe, pos = (pos + 1) & t.mask) {
            unsigned long long k = t.key[pos];
            if (k == 0) {
                if (frozen) break;
                k = atomicCAS(&t.key[pos], 0ull, h);
                if (k == 0) k = h;
            }
            if (k == h) {
                found = (long long)pos;
                break;
            }
        }
        if (found < 0) {
            if (frozen) {
                atomicOr(&st->decline, (unsigned)D_IID_MISS);
                atomicMin(&st->decline_line, (unsigned long long)user[ord] + 1);
            } else {
                atomicOr(&st->overflow, 1u);
            }
        } else if (!frozen) {
            atomicMin(&t.first[found], ord);
        }
        slot_of[i] = (int32_t)found;
    }
}

// (b) the occurrence holding its slot's smallest ordinal copies its bytes into the pool and creates the entry
__global__ void st_pool_kernel(const unsigned char* __restrict__ text, const long long* __restrict__ boff,
                               const int32_t* __restrict__ blen, const int32_t* __restrict__ slot_of, long long nb,
                               long long ord_base, int ord_step, long long file_offset, Table t, Entries E,
                               unsigned char* __restrict__ pool, STState* st, unsigned char* __restrict__ is_first) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nb; i += (long long)gridDim.x * blockDim.x) {
        const int32_t pos = slot_of[i];
        const long long ord = ord_base + ord_step * i;
        if (pos < 0 || t.entry[pos] >= 0 || t.first[pos] != ord) continue;
        const int32_t len = blen[i];
        const long long e = (long long)atomicAdd(&st->n_entries, 1ull);
        const long long off = (long long)atomicAdd(&st->pool_used, (unsigned long long)len);
        const unsigned char* src = text + boff[i];
        for (int32_t k = 0; k < len; ++k) pool[off + k] = src[k];
        E.off[e] = off;
        E.len[e] = len;
        E.first[e] = ord;
        E.foff[e] = file_offset + boff[i];
        t.entry[pos] = (int32_t)e;
        if (is_first) is_first[ord] = 1;
    }
}

// (c) every occurrence compares its bytes with its entry's and records the entry
__global__ void st_verify_kernel(const unsigned char* __restrict__ text, const long long* __restrict__ boff,
                                 const int32_t* __restrict__ blen, const int32_t* __restrict__ slot_of, long long nb,
                                 long long ord_base, int ord_step, Table t, Entries E, const unsigned char* __restrict__ pool,
                                 const int32_t* __restrict__ user, STState* st, int32_t* __restrict__ item) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nb; i += (long long)gridDim.x * blockDim.x) {
        const int32_t pos = slot_of[i];
        if (pos < 0) continue;
        const long long ord = ord_base + ord_step * i;
        const int32_t e = t.entry[pos], len = blen[i];
        bool same = E.len[e] == len;
        const unsigned char *a = text + boff[i], *b = pool + E.off[e];
        for (int32_t k = 0; same && k < len; ++k) same = a[k] == b[k];
        if (!same) {
            atomicOr(&st->decline, (unsigned)D_COLLISION);
            if (user) atomicMin(&st->decline_line, (unsigned long long)user[ord] + 1);
        }
        if (item) item[ord] = e;
    }
}

__global__ void st_rehash_kernel(Table o, Table t) {
    for (unsigned long long s = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; s <= o.mask;
         s += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long k = o.key[s];
        if (!k) continue;
        unsigned long long pos = k & t.mask;                // keys are distinct and the new table has free slots
        while (atomicCAS(&t.key[pos], 0ull, k) != 0ull) pos = (pos + 1) & t.mask;
        t.first[pos] = o.first[s];
        t.entry[pos] = o.entry[s];
    }
}

__global__ void st_table_init_kernel(Table t) {
    for (unsigned long long s = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; s <= t.mask;
         s += (unsigned long long)gridDim.x * blockDim.x) {
        t.key[s] = 0;
        t.first[s] = LLONG_MAX;
        t.entry[s] = -1;
    }
}

// ---- order-keeping compaction: Op::keep(i), Op::write(i, out) over [0, n) -------------------------------------
template <class Op>
__global__ void __launch_bounds__(ST_THREADS) ct_count_kernel(Op op, long long n, long long* __restrict__ counts) {
    __shared__ int wbuf[ST_THREADS / 32];
    const long long b = (long long)blockIdx.x * CT_TILE + threadIdx.x * CT_ITEMS;
    int c = 0;
    for (int j = 0; j < CT_ITEMS; ++j) c += b + j < n && op.keep(b + j);
    int tot;
    block_exclusive_scan(c, &tot, wbuf);
    if (threadIdx.x == 0) counts[blockIdx.x] = tot;
}
template <class Op>
__global__ void __launch_bounds__(ST_THREADS) ct_write_kernel(Op op, long long n, const long long* __restrict__ incl) {
    __shared__ int wbuf[ST_THREADS / 32];
    const long long b = (long long)blockIdx.x * CT_TILE + threadIdx.x * CT_ITEMS;
    int c = 0;
    for (int j = 0; j < CT_ITEMS; ++j) c += b + j < n && op.keep(b + j);
    int tot;
    long long o = (blockIdx.x ? incl[blockIdx.x - 1] : 0) + block_exclusive_scan(c, &tot, wbuf);
    for (int j = 0; j < CT_ITEMS; ++j)
        if (b + j < n && op.keep(b + j)) op.write(b + j, o++);
}

struct FlagPos {                         // positions of the set flags
    const unsigned char* flag;
    long long* pos;
    __device__ bool keep(long long i) const { return flag[i] != 0; }
    __device__ void write(long long i, long long o) const { pos[o] = i; }
};
struct KeptPairs {                       // (user, item) of the clear flags
    const unsigned char* flag;
    const int32_t *user, *item;
    int32_t *ou, *oi;
    __device__ bool keep(long long i) const { return flag[i] == 0; }
    __device__ void write(long long i, long long o) const {
        ou[o] = user[i];
        oi[o] = item[i];
    }
};
struct RunStarts {                       // first position of each run of equal (user, item) in sorted pairs
    const int32_t *user, *item;
    long long* pos;
    __device__ bool keep(long long i) const { return i == 0 || user[i] != user[i - 1] || item[i] != item[i - 1]; }
    __device__ void write(long long i, long long o) const { pos[o] = i; }
};

// start[v] = first position of key v in the non-decreasing key[0..n), start[nseg] = n
__global__ void seg_start_kernel(const int32_t* __restrict__ key, long long n, int32_t nseg, long long* __restrict__ start) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += (long long)gridDim.x * blockDim.x) {
        const long long lo = i ? (long long)key[i - 1] + 1 : 0, hi = i < n ? (long long)key[i] : nseg;
        for (long long v = lo; v <= hi; ++v) start[v] = i;
    }
}

__global__ void mark_newest_kernel(const long long* __restrict__ start, int32_t nu, long long n, unsigned char* __restrict__ flag) {
    for (long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x; u < nu; u += (long long)gridDim.x * blockDim.x) {
        const long long s = start[u], e = start[u + 1];
        if (e == s) continue;
        const long long hold = max(0ll, min(n, e - s - 1));
        for (long long i = e - hold; i < e; ++i) flag[i] = 1;
    }
}
__global__ void mark_sample_kernel(const long long* __restrict__ idx, long long n, unsigned char* __restrict__ flag) {
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (long long)gridDim.x * blockDim.x)
        flag[idx[j]] = 1;
}
__global__ void gather_pairs_kernel(const long long* __restrict__ pos, long long n, const int32_t* __restrict__ user,
                                    const int32_t* __restrict__ item, int32_t* __restrict__ ou, int32_t* __restrict__ oi) {
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (long long)gridDim.x * blockDim.x) {
        ou[j] = user[pos[j]];
        oi[j] = item[pos[j]];
    }
}

// held (user, item) -> Counter(held).items() per user: distinct items in order of first occurrence, with counts
__global__ void vali_count_kernel(const long long* __restrict__ start, int32_t nu, const int32_t* __restrict__ item,
                                  long long* __restrict__ cnt) {
    for (long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x; u < nu; u += (long long)gridDim.x * blockDim.x) {
        const long long s = start[u], e = start[u + 1];
        long long c = 0;
        for (long long i = s; i < e; ++i) {
            bool seen = false;
            for (long long k = s; k < i && !seen; ++k) seen = item[k] == item[i];
            c += !seen;
        }
        cnt[u] = c;
    }
}
__global__ void vali_write_kernel(const long long* __restrict__ start, int32_t nu, const int32_t* __restrict__ item,
                                  const long long* __restrict__ incl, int32_t* __restrict__ vr, int32_t* __restrict__ vc,
                                  float* __restrict__ vv) {
    for (long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x; u < nu; u += (long long)gridDim.x * blockDim.x) {
        const long long s = start[u], e = start[u + 1];
        long long o = u ? incl[u - 1] : 0;
        for (long long i = s; i < e; ++i) {
            bool seen = false;
            for (long long k = s; k < i && !seen; ++k) seen = item[k] == item[i];
            if (seen) continue;
            long long c = 0;
            for (long long k = i; k < e; ++k) c += item[k] == item[i];
            vr[o] = (int32_t)u;
            vc[o] = item[i];
            vv[o] = (float)c;
            ++o;
        }
    }
}

// runs of equal (user, item) -> one entry with the run length as value
__global__ void collapse_kernel(const long long* __restrict__ pos, long long m, long long n, const int32_t* __restrict__ user,
                                const int32_t* __restrict__ item, int32_t* __restrict__ ou, int32_t* __restrict__ oi,
                                float* __restrict__ ov) {
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < m; j += (long long)gridDim.x * blockDim.x) {
        const long long p = pos[j];
        ou[j] = user[p];
        oi[j] = item[p];
        ov[j] = (float)((j + 1 < m ? pos[j + 1] : n) - p);
    }
}

__global__ void fill_kernel(float* __restrict__ v, long long n, float x) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) v[i] = x;
}

// item id of each entry: its rank in first-appearance order (pos = ordinals of the first occurrences, ascending)
__global__ void rank_entries_kernel(const long long* __restrict__ pos, long long m, const int32_t* __restrict__ entry_of,
                                    Entries E, int32_t* __restrict__ e_item, long long* __restrict__ name_off,
                                    int32_t* __restrict__ name_len) {
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < m; j += (long long)gridDim.x * blockDim.x) {
        const int32_t e = entry_of[pos[j]];
        e_item[e] = (int32_t)j;
        name_off[j] = E.foff[e];
        name_len[j] = E.len[e];
    }
}
// iid: the entry of a name holds ordinal (count - 1 - largest index of that name)
__global__ void iid_entries_kernel(Entries E, long long m, long long count, int32_t* __restrict__ e_item) {
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < m; e += (long long)gridDim.x * blockDim.x)
        e_item[e] = (int32_t)(count - 1 - E.first[e]);
}
__global__ void remap_kernel(int32_t* __restrict__ item, long long n, const int32_t* __restrict__ e_item) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        item[i] = e_item[item[i]];
}

enum { ST_H2D = 0, ST_PARSE, ST_INTERN, ST_NUMBER, ST_SPLIT, ST_CSR_ROW, ST_CSR_COL, ST_D2H, ST_COUNT };

}  // namespace

struct bfl_stream_ingest : TextIngest {
    long long buf_bytes = 0, tmp_cap = 0;
    int hash_bits = 64;
    Grammar g{};
    unsigned char* dev = nullptr;                          // device text buffer (16-byte front pad)
    STState* state = nullptr;
    long long* counts = nullptr;
    // per block token
    long long* boff = nullptr;
    int32_t *blen = nullptr, *slot_of = nullptr;
    unsigned long long* bhash = nullptr;
    // per token (ordinal)
    long long tok_cap = 0, tokens = 0, lines = 0;
    bool open_line = false;                                // the input does not end with '\n'
    int32_t *user = nullptr, *item = nullptr;
    unsigned char* flag = nullptr;                         // first occurrence, then held for validation
    // interning
    Table t{};
    Entries E{};
    long long e_cap = 0, pool_cap = 0, n_entries = 0, pool_used = 0;
    unsigned char* pool = nullptr;
    long long iid_count = -1;                              // >= 0: frozen table of that many names
    unsigned decline = 0;
    long long decline_line = -1;
    bool finished = false, split_done = false, as_matrix = false;
    int32_t num_items = 0, num_users = 0;
    std::vector<long long> name_off;
    std::vector<int32_t> name_len;
    // validation and training entries
    long long n_vali = 0, n_train = 0;
    int32_t *vr = nullptr, *vc = nullptr, *tu = nullptr, *ti = nullptr;
    float *vv = nullptr, *tv = nullptr;

    ~bfl_stream_ingest() override {
        if (comp) cudaStreamSynchronize(comp);
        for (void* p : {(void*)dev, (void*)state, (void*)counts, (void*)boff, (void*)blen, (void*)slot_of, (void*)bhash,
                        (void*)user, (void*)item, (void*)flag, (void*)t.key, (void*)t.first, (void*)t.entry, (void*)E.off,
                        (void*)E.first, (void*)E.foff, (void*)E.len, (void*)pool, (void*)vr, (void*)vc, (void*)vv, (void*)tu,
                        (void*)ti, (void*)tv})
            if (p) cudaFree(p);
    }
};

namespace {

template <class T>
void dfree(bfl_stream_ingest* h, T*& p) {
    if (p) cudaFreeAsync(p, h->comp);
    p = nullptr;
}

// grows p to hold at least `need` elements, keeping the first `keep`; false when the device is out of memory
template <class T>
bool grow(bfl_stream_ingest* h, T*& p, long long& cap, long long need, long long keep, bool set_cap = true) {
    if (need <= cap) return true;
    const long long nc = std::max(need, cap * 2);
    T* q = nullptr;
    if (cudaMallocAsync(&q, sizeof(T) * (size_t)nc, h->comp) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    if (keep && cudaMemcpyAsync(q, p, sizeof(T) * (size_t)keep, cudaMemcpyDeviceToDevice, h->comp) != cudaSuccess) return false;
    dfree(h, p);
    p = q;
    if (set_cap) cap = nc;
    return true;
}

int read_state(bfl_stream_ingest* h, STState* s) {
    BFL_CUDA(cudaMemcpyAsync(s, h->state, sizeof(STState), cudaMemcpyDeviceToHost, h->comp));
    BFL_CUDA(cudaStreamSynchronize(h->comp));
    return BFL_OK;
}

int alloc_table(bfl_stream_ingest* h, Table* t, unsigned long long slots) {
    BFL_CUDA(cudaMallocAsync(&t->key, sizeof(unsigned long long) * slots, h->comp));
    BFL_CUDA(cudaMallocAsync(&t->first, sizeof(long long) * slots, h->comp));
    BFL_CUDA(cudaMallocAsync(&t->entry, sizeof(int32_t) * slots, h->comp));
    t->mask = slots - 1;
    st_table_init_kernel<<<grid_for((long long)slots), 256, 0, h->comp>>>(*t);
    BFL_LAUNCHED();
    return BFL_OK;
}

void free_table(bfl_stream_ingest* h, Table* t) {
    dfree(h, t->key);
    dfree(h, t->first);
    dfree(h, t->entry);
}

int rehash(bfl_stream_ingest* h, unsigned long long slots) {
    Table nt{};
    if (int rc = alloc_table(h, &nt, slots)) return rc;
    st_rehash_kernel<<<grid_for((long long)(h->t.mask + 1)), 256, 0, h->comp>>>(h->t, nt);
    BFL_LAUNCHED();
    free_table(h, &h->t);
    h->t = nt;
    return BFL_OK;
}

// entries and pool room for nb more occurrences of `bytes` bytes in all
bool reserve_entries(bfl_stream_ingest* h, long long nb, long long bytes) {
    const long long keep = h->n_entries, cap = h->e_cap;
    long long c = cap;
    bool ok = grow(h, h->E.off, c, keep + nb, keep, false) && grow(h, h->E.first, c, keep + nb, keep, false) &&
              grow(h, h->E.foff, c, keep + nb, keep, false) && grow(h, h->E.len, c, keep + nb, keep, false);
    if (ok && keep + nb > cap) h->e_cap = std::max(keep + nb, cap * 2);
    return ok && grow(h, h->pool, h->pool_cap, h->pool_used + bytes + 1, h->pool_used);
}

// claim -> (grow on overflow) -> pool -> verify for nb occurrences of text
int intern(bfl_stream_ingest* h, const unsigned char* text, long long nb, long long ord_base, int ord_step, long long file_offset,
           bool frozen, const int32_t* user, int32_t* item, unsigned char* is_first) {
    if (nb == 0) return BFL_OK;
    const int grid = grid_for(nb);
    for (;;) {
        st_claim_kernel<<<grid, 256, 0, h->comp>>>(h->bhash, nb, ord_base, ord_step, h->t, frozen, user, h->state, h->slot_of);
        BFL_LAUNCHED();
        STState s;
        if (int rc = read_state(h, &s)) return rc;
        if (!s.overflow) break;
        const unsigned zero = 0;
        BFL_CUDA(cudaMemcpyAsync(&h->state->overflow, &zero, sizeof(zero), cudaMemcpyHostToDevice, h->comp));
        unsigned long long slots = 4 * (h->t.mask + 1);  // room for every occurrence of the block at load 1/2
        while ((long long)slots < 2 * (h->n_entries + nb)) slots *= 2;
        if (int rc = rehash(h, slots)) return rc;
    }
    if (!frozen) {
        st_pool_kernel<<<grid, 256, 0, h->comp>>>(text, h->boff, h->blen, h->slot_of, nb, ord_base, ord_step, file_offset, h->t,
                                                  h->E, h->pool, h->state, is_first);
        BFL_LAUNCHED();
    }
    st_verify_kernel<<<grid, 256, 0, h->comp>>>(text, h->boff, h->blen, h->slot_of, nb, ord_base, ord_step, h->t, h->E, h->pool,
                                                user, h->state, item);
    BFL_LAUNCHED();
    STState s;
    if (int rc = read_state(h, &s)) return rc;
    h->n_entries = (long long)s.n_entries;
    h->pool_used = (long long)s.pool_used;
    if (2 * h->n_entries > (long long)(h->t.mask + 1)) {   // keep the load at or below 1/2 between blocks
        unsigned long long slots = h->t.mask + 1;
        while (2 * h->n_entries > (long long)slots / 2) slots *= 2;
        if (int rc = rehash(h, slots)) return rc;
    }
    return BFL_OK;
}

bool reserve_block_temps(bfl_stream_ingest* h, long long nb) {
    long long c = h->tmp_cap;
    return grow(h, h->boff, c, nb, 0, false) && grow(h, h->blen, c, nb, 0, false) && grow(h, h->bhash, c, nb, 0, false) &&
           grow(h, h->slot_of, h->tmp_cap, nb, 0);
}

template <class Op>
int compact(bfl_stream_ingest* h, Op op, long long n, long long* kept) {
    *kept = 0;
    if (n == 0) return BFL_OK;
    const long long tiles = (n + CT_TILE - 1) / CT_TILE;
    long long* counts = nullptr;
    BFL_CUDA(cudaMallocAsync(&counts, sizeof(long long) * tiles, h->comp));
    ct_count_kernel<Op><<<(unsigned)tiles, ST_THREADS, 0, h->comp>>>(op, n, counts);
    BFL_LAUNCHED();
    if (int rc = inclusive_scan_i64(counts, counts, tiles, h->comp)) return rc;
    ct_write_kernel<Op><<<(unsigned)tiles, ST_THREADS, 0, h->comp>>>(op, n, counts);
    BFL_LAUNCHED();
    BFL_CUDA(cudaMemcpyAsync(kept, counts + tiles - 1, sizeof(long long), cudaMemcpyDeviceToHost, h->comp));
    BFL_CUDA(cudaFreeAsync(counts, h->comp));
    BFL_CUDA(cudaStreamSynchronize(h->comp));
    return BFL_OK;
}

}  // namespace

extern "C" {

bfl_stream_ingest_t* bfl_stream_ingest_create(int64_t block_bytes, uint64_t ascii_ws, const int32_t* uspace, int32_t n_uspace,
                                              int32_t hash_bits) {
    if (BFL_OK != require_device()) return nullptr;
    if (block_bytes < 16 || block_bytes > (1ll << 30) || n_uspace < 0 || n_uspace > MAX_USPACE || (n_uspace && !uspace) ||
        hash_bits < 1 || hash_bits > 64 || !((ascii_ws >> '\n') & 1)) {
        set_error("bad Stream ingest arguments");
        return nullptr;
    }
    auto* h = new bfl_stream_ingest();
    h->hash_bits = hash_bits;
    h->g.ascii_ws = ascii_ws;
    h->g.n_uspace = n_uspace;
    for (int i = 0; i < n_uspace; ++i) h->g.uspace[i] = uspace[i];
    h->buf_bytes = (block_bytes + ST_TILE - 1) / ST_TILE * ST_TILE + 16;
    const long long tiles = (block_bytes + ST_TILE - 1) / ST_TILE;
    bool ok = setup(h, block_bytes, ST_COUNT) && cudaMallocAsync(&h->dev, (size_t)h->buf_bytes, h->comp) == cudaSuccess &&
              cudaMemsetAsync(h->dev, 0, (size_t)h->buf_bytes, h->comp) == cudaSuccess &&
              cudaMallocAsync(&h->state, sizeof(STState), h->comp) == cudaSuccess &&
              cudaMallocAsync(&h->counts, sizeof(long long) * tiles, h->comp) == cudaSuccess &&
              alloc_table(h, &h->t, 1 << 16) == BFL_OK;
    if (ok) {
        STState s0 = {~0ull, 0u, 0u, 0ull, 0ull};
        ok = cudaMemcpyAsync(h->state, &s0, sizeof(s0), cudaMemcpyHostToDevice, h->comp) == cudaSuccess &&
             cudaStreamSynchronize(h->comp) == cudaSuccess;
    }
    return setup_done(h, ok, "Stream");
}

void bfl_stream_ingest_destroy(bfl_stream_ingest_t* h) { delete h; }

int bfl_stream_ingest_staging(bfl_stream_ingest_t* h, int slot, void** host_ptr) { return staging(h, slot, host_ptr); }

int bfl_stream_ingest_load_iid(bfl_stream_ingest_t* h, const char* names, const int64_t* offsets, int64_t n) {
    if (!h || n <= 0 || !offsets || (offsets[n] && !names) || offsets[0] != 0) BFL_FAIL(BFL_ERR_ARG, "bad iid arguments");
    if (h->fed || h->iid_count >= 0) BFL_FAIL(BFL_ERR_STATE, "load the iid list once, before the first block");
    for (int64_t i = 0; i < n; ++i)
        if (offsets[i + 1] < offsets[i]) BFL_FAIL(BFL_ERR_ARG, "iid offsets must not decrease");
    const long long bytes = offsets[n];
    unsigned long long slots = 1 << 16;
    while ((long long)slots < 2 * n) slots *= 2;
    free_table(h, &h->t);
    if (int rc = alloc_table(h, &h->t, slots)) return rc;
    if (!reserve_block_temps(h, n) || !reserve_entries(h, n, bytes)) BFL_FAIL(BFL_ERR_CUDA, "out of device memory for the iid list");
    unsigned char* d_names = nullptr;
    long long* d_offs = nullptr;
    BFL_CUDA(cudaMallocAsync(&d_names, (size_t)std::max<long long>(bytes, 1), h->comp));
    BFL_CUDA(cudaMallocAsync(&d_offs, sizeof(long long) * (n + 1), h->comp));
    if (bytes) BFL_CUDA(cudaMemcpyAsync(d_names, names, (size_t)bytes, cudaMemcpyHostToDevice, h->comp));
    BFL_CUDA(cudaMemcpyAsync(d_offs, offsets, sizeof(long long) * (n + 1), cudaMemcpyHostToDevice, h->comp));
    if (int rc = mark(h, ST_INTERN, h->comp)) return rc;
    st_name_kernel<<<grid_for(n), 256, 0, h->comp>>>(d_names, d_offs, n, h->hash_bits, h->boff, h->blen, h->bhash);
    BFL_LAUNCHED();
    // name i gets ordinal n - 1 - i: the slot's minimum is the name's LAST index (a dict comprehension keeps the last)
    if (int rc = intern(h, d_names, n, n - 1, -1, 0, false, nullptr, nullptr, nullptr)) return rc;
    if (int rc = mark(h, ST_INTERN, h->comp)) return rc;
    BFL_CUDA(cudaFreeAsync(d_names, h->comp));
    BFL_CUDA(cudaFreeAsync(d_offs, h->comp));
    h->iid_count = n;
    return BFL_OK;
}

int bfl_stream_ingest_feed(bfl_stream_ingest_t* h, int slot, int64_t n, int is_last) {
    if (int rc = check_feed(h, slot, n, is_last)) return rc;
    if (n) h->open_line = h->host[slot][n - 1] != '\n';
    if (n == 0 || h->decline) return BFL_OK;
    unsigned char* d = h->dev + 16;
    if (int rc = mark(h, ST_H2D, h->comp)) return rc;
    BFL_CUDA(cudaMemcpyAsync(d, h->host[slot], (size_t)n, cudaMemcpyHostToDevice, h->comp));
    if (int rc = mark(h, ST_H2D, h->comp)) return rc;
    if (int rc = mark(h, ST_PARSE, h->comp)) return rc;
    const long long tiles = (n + ST_TILE - 1) / ST_TILE;
    st_count_kernel<<<(unsigned)tiles, ST_THREADS, 0, h->comp>>>(d, n, h->g.ascii_ws, h->counts);
    BFL_LAUNCHED();
    if (int rc = inclusive_scan_i64(h->counts, h->counts, tiles, h->comp)) return rc;
    long long tot = 0;
    BFL_CUDA(cudaMemcpyAsync(&tot, h->counts + tiles - 1, sizeof(long long), cudaMemcpyDeviceToHost, h->comp));
    BFL_CUDA(cudaStreamSynchronize(h->comp));
    const long long nb = tot & 0xffffffffll, nl = tot >> 32;
    const long long keep = h->tokens;
    long long c1 = h->tok_cap, c2 = h->tok_cap;
    const bool frozen = h->iid_count >= 0;
    if (!reserve_block_temps(h, nb) || !grow(h, h->user, c1, keep + nb, keep) || !grow(h, h->item, c2, keep + nb, keep) ||
        !grow(h, h->flag, h->tok_cap, keep + nb, keep) || (!frozen && !reserve_entries(h, nb, n))) {
        h->decline |= D_MEMORY;
        return BFL_OK;
    }
    if (!frozen && keep + nb > keep) BFL_CUDA(cudaMemsetAsync(h->flag + keep, 0, (size_t)nb, h->comp));
    WriteArgs a;
    a.text = d;
    a.n = n;
    a.tok_base = h->tokens;
    a.line_base = h->lines;
    a.incl = h->counts;
    a.g = h->g;
    a.hash_bits = h->hash_bits;
    a.state = h->state;
    a.user = h->user;
    a.boff = h->boff;
    a.blen = h->blen;
    a.bhash = h->bhash;
    st_write_kernel<<<(unsigned)tiles, ST_THREADS, 0, h->comp>>>(a);
    BFL_LAUNCHED();
    if (int rc = mark(h, ST_PARSE, h->comp)) return rc;
    if (int rc = mark(h, ST_INTERN, h->comp)) return rc;
    if (int rc = intern(h, d, nb, h->tokens, 1, h->fed, frozen, h->user, h->item, frozen ? nullptr : h->flag)) return rc;
    if (int rc = mark(h, ST_INTERN, h->comp)) return rc;
    STState s;
    if (int rc = read_state(h, &s)) return rc;
    h->decline |= s.decline;
    h->tokens += nb;
    h->lines += nl;
    h->fed += n;
    return BFL_OK;
}

// *num_lines: '\n' bytes fed (the caller adds a last line without one); *decline: D_* bits (0: the device built the
// table), *decline_line: smallest 1-based line with a grammar, iid or collision reason (-1: none)
int bfl_stream_ingest_finish(bfl_stream_ingest_t* h, int64_t* num_tokens, int64_t* num_lines, int32_t* num_items,
                             int32_t* decline, int64_t* decline_line) {
    if (!h || !num_tokens || !num_lines || !num_items || !decline || !decline_line) BFL_FAIL(BFL_ERR_ARG, "bad finish arguments");
    if (!h->last_fed || h->finished) BFL_FAIL(BFL_ERR_STATE, "finish once, after the last block was fed");
    STState s;
    if (int rc = read_state(h, &s)) return rc;
    h->finished = true;
    h->decline |= s.decline;
    if (h->lines >= INT32_MAX - 1 || h->n_entries >= INT32_MAX) h->decline |= D_LINES;   // int32 user and item ids
    for (void** p : {(void**)&h->dev, (void**)&h->counts, (void**)&h->boff, (void**)&h->blen, (void**)&h->slot_of, (void**)&h->bhash}) {
        if (*p) BFL_CUDA(cudaFreeAsync(*p, h->comp));
        *p = nullptr;
    }
    *num_tokens = h->tokens;
    *num_lines = h->lines;
    *decline = (int32_t)h->decline;
    *decline_line = s.decline_line == ~0ull ? -1 : (int64_t)s.decline_line;
    *num_items = 0;
    if (h->decline) return BFL_OK;
    if (int rc = mark(h, ST_NUMBER, h->comp)) return rc;
    const long long m = h->n_entries;
    int32_t* e_item = nullptr;
    BFL_CUDA(cudaMallocAsync(&e_item, sizeof(int32_t) * std::max<long long>(m, 1), h->comp));
    if (h->iid_count >= 0) {
        iid_entries_kernel<<<grid_for(m), 256, 0, h->comp>>>(h->E, m, h->iid_count, e_item);
        BFL_LAUNCHED();
        h->num_items = (int32_t)h->iid_count;
    } else {
        long long* pos = nullptr;
        long long* noff = nullptr;
        int32_t* nlen = nullptr;
        BFL_CUDA(cudaMallocAsync(&pos, sizeof(long long) * std::max<long long>(m, 1), h->comp));
        BFL_CUDA(cudaMallocAsync(&noff, sizeof(long long) * std::max<long long>(m, 1), h->comp));
        BFL_CUDA(cudaMallocAsync(&nlen, sizeof(int32_t) * std::max<long long>(m, 1), h->comp));
        long long nf = 0;
        if (int rc = compact(h, FlagPos{h->flag, pos}, h->tokens, &nf)) return rc;
        if (nf != m) BFL_FAIL(BFL_ERR_STATE, "first occurrences and pool entries disagree");
        if (m) {
            rank_entries_kernel<<<grid_for(m), 256, 0, h->comp>>>(pos, m, h->item, h->E, e_item, noff, nlen);
            BFL_LAUNCHED();
        }
        h->name_off.resize((size_t)m);
        h->name_len.resize((size_t)m);
        if (m) {
            BFL_CUDA(cudaMemcpyAsync(h->name_off.data(), noff, sizeof(long long) * m, cudaMemcpyDeviceToHost, h->comp));
            BFL_CUDA(cudaMemcpyAsync(h->name_len.data(), nlen, sizeof(int32_t) * m, cudaMemcpyDeviceToHost, h->comp));
        }
        for (void* p : {(void*)pos, (void*)noff, (void*)nlen}) BFL_CUDA(cudaFreeAsync(p, h->comp));
        h->num_items = (int32_t)m;
    }
    if (h->tokens) {
        remap_kernel<<<grid_for(h->tokens), 256, 0, h->comp>>>(h->item, h->tokens, e_item);
        BFL_LAUNCHED();
    }
    BFL_CUDA(cudaFreeAsync(e_item, h->comp));
    free_table(h, &h->t);
    for (void** p : {(void**)&h->E.off, (void**)&h->E.first, (void**)&h->E.foff, (void**)&h->E.len, (void**)&h->pool}) {
        if (*p) BFL_CUDA(cudaFreeAsync(*p, h->comp));
        *p = nullptr;
    }
    if (int rc = mark(h, ST_NUMBER, h->comp)) return rc;
    BFL_CUDA(cudaStreamSynchronize(h->comp));
    *num_items = h->num_items;
    return BFL_OK;
}

// byte offset from the first fed byte and length of each item's first occurrence, by item id (no iid list)
int bfl_stream_ingest_names(bfl_stream_ingest_t* h, int64_t* offset, int32_t* length) {
    if (!h || !h->finished || h->decline || h->iid_count >= 0 || (h->num_items && (!offset || !length)))
        BFL_FAIL(BFL_ERR_ARG, "bad names arguments (finish without a decline and without an iid list first)");
    std::copy(h->name_off.begin(), h->name_off.end(), offset);
    std::copy(h->name_len.begin(), h->name_len.end(), length);
    return BFL_OK;
}

// method 0: none, 1: newest (hold the last min(newest_n, len - 1) tokens of each session), 2: sample (hold the token
// ordinals in sample_idx).  as_matrix: the training entries are the distinct (user, item) pairs with counts, else the
// kept tokens in order with value 1.  *n_vali = validation triples (Counter(held) per user), *n_train = training entries.
int bfl_stream_ingest_split(bfl_stream_ingest_t* h, int32_t num_users, int method, int64_t newest_n, const int64_t* sample_idx,
                            int64_t n_sample, int as_matrix, int64_t* n_vali, int64_t* n_train) {
    if (!h || !h->finished || h->decline || h->split_done || num_users <= 0 || method < 0 || method > 2 || n_sample < 0 ||
        (n_sample && !sample_idx) || !n_vali || !n_train)
        BFL_FAIL(BFL_ERR_ARG, "bad split arguments");
    if (h->lines + h->open_line > num_users) BFL_FAIL(BFL_ERR_ARG, "fewer users than lines");
    const long long T = h->tokens;
    for (int64_t j = 0; j < n_sample; ++j)
        if (sample_idx[j] < 0 || sample_idx[j] >= T) BFL_FAIL(BFL_ERR_ARG, "sample ordinals must lie in [0, tokens)");
    h->split_done = true;
    h->num_users = num_users;
    h->as_matrix = as_matrix != 0;
    cudaStream_t st = h->comp;
    if (int rc = mark(h, ST_SPLIT, h->comp)) return rc;
    long long *ustart = nullptr, *hpos = nullptr, *hstart = nullptr, *vcnt = nullptr;
    int32_t *hu = nullptr, *hi = nullptr;
    const size_t T1 = (size_t)std::max<long long>(T, 1);
    BFL_CUDA(cudaMallocAsync(&ustart, sizeof(long long) * ((size_t)num_users + 1), st));
    seg_start_kernel<<<grid_for(T + 1), 256, 0, st>>>(h->user, T, num_users, ustart);
    BFL_LAUNCHED();
    if (!h->flag) BFL_CUDA(cudaMallocAsync(&h->flag, T1, st));
    BFL_CUDA(cudaMemsetAsync(h->flag, 0, T1, st));
    if (method == 1) {
        mark_newest_kernel<<<grid_for(num_users), 256, 0, st>>>(ustart, num_users, newest_n, h->flag);
        BFL_LAUNCHED();
    } else if (method == 2 && n_sample) {
        long long* d_idx = nullptr;
        BFL_CUDA(cudaMallocAsync(&d_idx, sizeof(long long) * n_sample, st));
        BFL_CUDA(cudaMemcpyAsync(d_idx, sample_idx, sizeof(long long) * n_sample, cudaMemcpyHostToDevice, st));
        mark_sample_kernel<<<grid_for(n_sample), 256, 0, st>>>(d_idx, n_sample, h->flag);
        BFL_LAUNCHED();
        BFL_CUDA(cudaFreeAsync(d_idx, st));
    }
    BFL_CUDA(cudaFreeAsync(ustart, st));
    // held tokens -> validation triples
    long long nh = 0;
    BFL_CUDA(cudaMallocAsync(&hpos, sizeof(long long) * T1, st));
    if (int rc = compact(h, FlagPos{h->flag, hpos}, T, &nh)) return rc;
    const size_t nh1 = (size_t)std::max<long long>(nh, 1);
    BFL_CUDA(cudaMallocAsync(&hu, sizeof(int32_t) * nh1, st));
    BFL_CUDA(cudaMallocAsync(&hi, sizeof(int32_t) * nh1, st));
    if (nh) {
        gather_pairs_kernel<<<grid_for(nh), 256, 0, st>>>(hpos, nh, h->user, h->item, hu, hi);
        BFL_LAUNCHED();
    }
    BFL_CUDA(cudaFreeAsync(hpos, st));
    BFL_CUDA(cudaMallocAsync(&hstart, sizeof(long long) * ((size_t)num_users + 1), st));
    BFL_CUDA(cudaMallocAsync(&vcnt, sizeof(long long) * (size_t)num_users, st));
    seg_start_kernel<<<grid_for(nh + 1), 256, 0, st>>>(hu, nh, num_users, hstart);
    BFL_LAUNCHED();
    vali_count_kernel<<<grid_for(num_users), 256, 0, st>>>(hstart, num_users, hi, vcnt);
    BFL_LAUNCHED();
    if (int rc = inclusive_scan_i64(vcnt, vcnt, num_users, st)) return rc;
    long long nv = 0;
    BFL_CUDA(cudaMemcpyAsync(&nv, vcnt + num_users - 1, sizeof(long long), cudaMemcpyDeviceToHost, st));
    BFL_CUDA(cudaStreamSynchronize(st));
    const size_t nv1 = (size_t)std::max<long long>(nv, 1);
    BFL_CUDA(cudaMallocAsync(&h->vr, sizeof(int32_t) * nv1, st));
    BFL_CUDA(cudaMallocAsync(&h->vc, sizeof(int32_t) * nv1, st));
    BFL_CUDA(cudaMallocAsync(&h->vv, sizeof(float) * nv1, st));
    vali_write_kernel<<<grid_for(num_users), 256, 0, st>>>(hstart, num_users, hi, vcnt, h->vr, h->vc, h->vv);
    BFL_LAUNCHED();
    for (void* p : {(void*)hu, (void*)hi, (void*)hstart, (void*)vcnt}) BFL_CUDA(cudaFreeAsync(p, st));
    h->n_vali = nv;
    // kept tokens in order
    const long long nk = T - nh;
    const size_t nk1 = (size_t)std::max<long long>(nk, 1);
    int32_t *ku = nullptr, *ki = nullptr;
    BFL_CUDA(cudaMallocAsync(&ku, sizeof(int32_t) * nk1, st));
    BFL_CUDA(cudaMallocAsync(&ki, sizeof(int32_t) * nk1, st));
    long long got = 0;
    if (int rc = compact(h, KeptPairs{h->flag, h->user, h->item, ku, ki}, T, &got)) return rc;
    for (void** p : {(void**)&h->user, (void**)&h->item, (void**)&h->flag}) {
        BFL_CUDA(cudaFreeAsync(*p, st));
        *p = nullptr;
    }
    float* ones = nullptr;
    BFL_CUDA(cudaMallocAsync(&ones, sizeof(float) * nk1, st));
    fill_kernel<<<grid_for(nk), 256, 0, st>>>(ones, nk, 1.0f);
    BFL_LAUNCHED();
    if (!h->as_matrix) {
        h->tu = ku;
        h->ti = ki;
        h->tv = ones;
        h->n_train = nk;
    } else {
        // Counter(kept) per user: sort the pairs by (user, item) (users are already in order), count equal runs
        int64_t* ind = nullptr;
        int32_t* skey = nullptr;
        float* sval = nullptr;
        long long* rpos = nullptr;
        BFL_CUDA(cudaMallocAsync(&ind, sizeof(int64_t) * (size_t)num_users, st));
        BFL_CUDA(cudaMallocAsync(&skey, sizeof(int32_t) * nk1, st));
        BFL_CUDA(cudaMallocAsync(&sval, sizeof(float) * nk1, st));
        int rc = bfl_csr_from_triples_device(ku, ki, ones, nk, num_users, std::max(h->num_items, 1), 1, ind, skey, sval, st);
        if (rc != BFL_OK) return rc;
        for (void* p : {(void*)ind, (void*)sval, (void*)ki, (void*)ones}) BFL_CUDA(cudaFreeAsync(p, st));
        BFL_CUDA(cudaMallocAsync(&rpos, sizeof(long long) * nk1, st));
        long long m = 0;
        if ((rc = compact(h, RunStarts{ku, skey, rpos}, nk, &m))) return rc;
        const size_t m1 = (size_t)std::max<long long>(m, 1);
        BFL_CUDA(cudaMallocAsync(&h->tu, sizeof(int32_t) * m1, st));
        BFL_CUDA(cudaMallocAsync(&h->ti, sizeof(int32_t) * m1, st));
        BFL_CUDA(cudaMallocAsync(&h->tv, sizeof(float) * m1, st));
        if (m) {
            collapse_kernel<<<grid_for(m), 256, 0, st>>>(rpos, m, nk, ku, skey, h->tu, h->ti, h->tv);
            BFL_LAUNCHED();
        }
        for (void* p : {(void*)rpos, (void*)ku, (void*)skey}) BFL_CUDA(cudaFreeAsync(p, st));
        h->n_train = m;
    }
    if (int rc = mark(h, ST_SPLIT, h->comp)) return rc;
    BFL_CUDA(cudaStreamSynchronize(st));
    *n_vali = h->n_vali;
    *n_train = h->n_train;
    return BFL_OK;
}

int bfl_stream_ingest_vali(bfl_stream_ingest_t* h, int32_t* row, int32_t* col, float* val) {
    if (!h || !h->split_done || (h->n_vali && (!row || !col || !val))) BFL_FAIL(BFL_ERR_ARG, "bad vali arguments (split first)");
    if (h->n_vali == 0) return BFL_OK;
    BFL_CUDA(cudaMemcpyAsync(row, h->vr, sizeof(int32_t) * h->n_vali, cudaMemcpyDeviceToHost, h->comp));
    BFL_CUDA(cudaMemcpyAsync(col, h->vc, sizeof(int32_t) * h->n_vali, cudaMemcpyDeviceToHost, h->comp));
    BFL_CUDA(cudaMemcpyAsync(val, h->vv, sizeof(float) * h->n_vali, cudaMemcpyDeviceToHost, h->comp));
    BFL_CUDA(cudaStreamSynchronize(h->comp));
    return BFL_OK;
}

// orientation 0: rowwise (matrix: sorted by (user, item); stream: session order), 1: colwise (matrix only), into host
// arrays of num_users resp. num_items END offsets and n_train entries
int bfl_stream_ingest_build(bfl_stream_ingest_t* h, int orientation, int64_t* indptr, int32_t* key, float* val) {
    if (!h || !h->split_done || orientation < 0 || orientation > 1 || (orientation && !h->as_matrix) || h->built[orientation] ||
        !indptr || (h->n_train && (!key || !val)))
        BFL_FAIL(BFL_ERR_ARG, "bad build arguments (split first, each orientation once, colwise in matrix mode)");
    return build_to_host(h, orientation, h->tu, h->ti, h->tv, h->n_train, h->num_users, h->num_items, h->as_matrix ? 1 : 0,
                         orientation ? ST_CSR_COL : ST_CSR_ROW, ST_D2H, indptr, key, val);
}

// stage_ms[8]: H2D, parse, intern, number, split, rowwise CSR, colwise CSR, D2H (summed device time of each stage);
// *peak_bytes: high-water mark of the device's default memory pool since create
int bfl_stream_ingest_stats(bfl_stream_ingest_t* h, double* stage_ms, int64_t* peak_bytes) {
    return stats(h, stage_ms, peak_bytes);
}

}  // extern "C"
