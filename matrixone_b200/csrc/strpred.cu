// strpred.cu -- string predicates of the Go elementwise engine over varlena operands (CHAR, VARCHAR, BINARY, VARBINARY, BLOB, TEXT, DATALINK):
//   comparisons   func_compare.go:224-226,353-360,744-748,871-875,1125-1129,1252-1256: = / != are bytes.Equal, < <= > >= bytes.Compare
//   LIKE          opBuiltInRegexp.likeFn, func_builtin_regexp.go:51-69: a const pattern that optimizeRuleForLike (:91-280) takes is
//                 matched by its byte-level rule ("tier A"); any other pattern by regularMatchForLikeOp (:618-672), ^(?s:...)$ over runes
//                 ("tier B"), which a wildcard-only glob matcher decides exactly: `_` is one rune, `%` any run of runes.
// funcIds and argument layout: include/mo_b200.h (MO_XCALL_GO_COMPARE over the varlena types, MO_XCALL_GO_LIKE); the operand protocol:
// goengine.cuh.
//
// Every launch is one grid-stride row kernel: one thread per row, so the 24-byte cells and the bool result are read and written by
// consecutive lanes.  A warp owns 32 consecutive rows, i.e. one half word of the result null bitmap, which its ballot writes whole: rnulls
// | n1 | n2 (a const NULL operand: every row) with no second pass.  Cells of NULL and skipped rows are never read.  A non-inline cell outside
// its area is recorded as the lowest such row per operand in a small status record, which the call reads back -- its one synchronise.
#include "goengine.cuh"
#include "keytable.cuh"
#include <algorithm>
#include <cstdio>
#include <string>
#include <vector>

using namespace mob;

namespace {

constexpr int kCtasPerSm = 16;
constexpr uint32_t kSmemAux = 16384;   // a const pattern's literals / tokens up to this size are copied to shared memory, longer ones stay in global
static_assert(kSmemAux == kInSmemBytes, "an IN table is an aux block: one shared-memory budget for both IN paths");
enum { LIKE_EXACT = 0, LIKE_PREFIX, LIKE_SUFFIX, LIKE_CHAIN };
constexpr int32_t kAny1 = -1, kAnySeq = -2;   // tier-B tokens; a literal rune is its code point (>= 0)
constexpr int32_t kRuneError = 0xFFFD;

// ~(lowest row whose cell points outside its area) per operand, 0 = none
struct Status { unsigned long long bad_inv[2]; };

// bytes.Compare
__device__ __forceinline__ int str_cmp(const Str &x, const Str &y) {
    const uint32_t m = x.len < y.len ? x.len : y.len;
    for (uint32_t j = 0; j < m; j++) {
        const uint32_t a = x.at(j), b = y.at(j);
        if (a != b) return a < b ? -1 : 1;
    }
    return x.len == y.len ? 0 : (x.len < y.len ? -1 : 1);
}

__device__ __forceinline__ bool match_at(const Str &v, uint32_t pos, const uint8_t *lit, uint32_t L) {
    for (uint32_t j = 0; j < L; j++) if (v.at(pos + j) != lit[j]) return false;
    return true;
}
// bytes.Index(v[from:], lit) + from, or -1
__device__ __forceinline__ int64_t find_from(const Str &v, uint32_t from, const uint8_t *lit, uint32_t L) {
    if (L == 0) return from;
    const uint32_t c0 = lit[0];
    for (uint32_t pos = from; pos + L <= v.len; pos++)
        if (v.at(pos) == c0 && match_at(v, pos + 1, lit + 1, L - 1)) return pos;
    return -1;
}

// utf8.DecodeRune of b[i:] (i < n; b(j) is byte j): an invalid, overlong, surrogate or truncated sequence is (RuneError, 1).  One rule for
// the kernels (b = a value) and for the host's tokeniser of const patterns (b = the pattern's bytes).
template <class B>
__host__ __device__ __forceinline__ int32_t decode_utf8(const B &b, uint32_t i, uint32_t n, uint32_t &size) {
    const uint32_t b0 = b(i);
    n -= i;
    size = 1;
    if (b0 < 0x80) return (int32_t)b0;
    if (b0 < 0xC2 || b0 > 0xF4) return kRuneError;
    const uint32_t sz = b0 < 0xE0 ? 2 : (b0 < 0xF0 ? 3 : 4);
    if (n < sz) return kRuneError;
    const uint32_t lo = b0 == 0xE0 ? 0xA0 : (b0 == 0xF0 ? 0x90 : 0x80), hi = b0 == 0xED ? 0x9F : (b0 == 0xF4 ? 0x8F : 0xBF);
    const uint32_t b1 = b(i + 1);
    if (b1 < lo || b1 > hi) return kRuneError;
    if (sz == 2) { size = 2; return (int32_t)(((b0 & 0x1F) << 6) | (b1 & 0x3F)); }
    const uint32_t b2 = b(i + 2);
    if (b2 < 0x80 || b2 > 0xBF) return kRuneError;
    if (sz == 3) { size = 3; return (int32_t)(((b0 & 0x0F) << 12) | ((b1 & 0x3F) << 6) | (b2 & 0x3F)); }
    const uint32_t b3 = b(i + 3);
    if (b3 < 0x80 || b3 > 0xBF) return kRuneError;
    size = 4;
    return (int32_t)(((b0 & 0x07) << 18) | ((b1 & 0x3F) << 12) | ((b2 & 0x3F) << 6) | (b3 & 0x3F));
}
struct StrBytes { const Str &v; __device__ __forceinline__ uint32_t operator()(uint32_t j) const { return v.at(j); } };
__device__ __forceinline__ int32_t decode_rune(const Str &v, uint32_t i, uint32_t &size) { return decode_utf8(StrBytes{v}, i, v.len, size); }

// tier-B pattern sources: tok(pi, next) -> the token at pi and the position after it
struct TokensPat {          // a const pattern, tokenised on the host
    const int32_t *t; uint32_t n;
    __device__ __forceinline__ uint32_t end() const { return n; }
    __device__ __forceinline__ int32_t tok(uint32_t pi, uint32_t &next) const { next = pi + 1; return t[pi]; }
};
struct BytesPat {           // a column pattern, tokenised as the matcher walks it (the replace() loop of regularMatchForLikeOp)
    const Str &s;
    __device__ __forceinline__ uint32_t end() const { return s.len; }
    __device__ __forceinline__ int32_t tok(uint32_t pi, uint32_t &next) const {
        uint32_t sz;
        const int32_t r = decode_rune(s, pi, sz);
        if (r == '\\') {
            if (pi + sz < s.len) { uint32_t sz2; const int32_t r2 = decode_rune(s, pi + sz, sz2); next = pi + sz + sz2; return r2; }
            next = pi + sz; return '\\';               // a trailing lone backslash is a literal backslash
        }
        next = pi + sz;
        return r == '_' ? kAny1 : (r == '%' ? kAnySeq : r);
    }
};

// two pointers over subject runes and pattern tokens, backtracking to the last `%`: exact for literals, any-one and any-run tokens
template <class P>
__device__ __forceinline__ bool glob_match(const Str &v, const P &pat) {
    const uint32_t pend = pat.end();
    uint32_t si = 0, pi = 0, star_pi = 0, star_si = 0;
    bool star = false;
    while (si < v.len) {
        if (pi < pend) {
            uint32_t pn;
            const int32_t t = pat.tok(pi, pn);
            if (t == kAnySeq) { star = true; star_pi = pn; star_si = si; pi = pn; continue; }
            uint32_t sz;
            const int32_t r = decode_rune(v, si, sz);
            if (t == kAny1 || t == r) { si += sz; pi = pn; continue; }
        }
        if (!star) return false;
        uint32_t sz;
        decode_rune(v, star_si, sz);
        star_si += sz; si = star_si; pi = star_pi;
    }
    while (pi < pend) { uint32_t pn; if (pat.tok(pi, pn) != kAnySeq) return false; pi = pn; }
    return true;
}

// ---- the per-row predicates: value of row i; bad1 / bad2 set when that operand's cell is bad (the row is then not written)
struct CmpPred {
    int op;
    __device__ __forceinline__ bool operator()(const Operand &a, const Operand &b, uint64_t i, const uint8_t *, bool &bad1, bool &bad2) const {
        Str x, y;
        bad1 = !load_str(a, i, x); bad2 = !load_str(b, i, y);
        if (bad1 || bad2) return false;
        if (op == CMP_EQ || op == CMP_NE) {
            const bool eq = x.len == y.len && str_cmp(x, y) == 0;
            return op == CMP_EQ ? eq : !eq;
        }
        return cmp_op(str_cmp(x, y), 0, op);
    }
};
// tier A: aux = u32 segment lengths [nseg] + their bytes.  EXACT: len == s + L + e and v[s, s + L) == lit ; PREFIX: v[s, s + L) == lit ;
// SUFFIX: v[len - e - L, len - e) == lit (both need len >= s + L + e) ; CHAIN: ordered bytes.Index of every segment
struct LikeAPred {
    int mode; uint32_t s, e, nseg;
    __device__ __forceinline__ bool operator()(const Operand &a, const Operand &, uint64_t i, const uint8_t *aux, bool &bad1, bool &bad2) const {
        Str v;
        bad2 = false; bad1 = !load_str(a, i, v);
        if (bad1) return false;
        const uint32_t *seg = reinterpret_cast<const uint32_t *>(aux);
        const uint8_t *lit = aux + 4 * nseg;
        if (mode == LIKE_CHAIN) {
            uint32_t pos = 0;
            for (uint32_t k = 0; k < nseg; k++) {
                const uint32_t L = seg[k];
                const int64_t at = find_from(v, pos, lit, L);
                if (at < 0) return false;
                pos = (uint32_t)at + L; lit += L;
            }
            return true;
        }
        const uint32_t L = seg[0];
        if (mode == LIKE_EXACT) return v.len == s + L + e && match_at(v, s, lit, L);
        if (v.len < s + L + e) return false;
        return match_at(v, mode == LIKE_PREFIX ? s : v.len - e - L, lit, L);
    }
};
struct LikeBConstPred {      // aux = int32 tokens [ntok]
    uint32_t ntok;
    __device__ __forceinline__ bool operator()(const Operand &a, const Operand &, uint64_t i, const uint8_t *aux, bool &bad1, bool &bad2) const {
        Str v;
        bad2 = false; bad1 = !load_str(a, i, v);
        if (bad1) return false;
        return glob_match(v, TokensPat{reinterpret_cast<const int32_t *>(aux), ntok});
    }
};
struct LikeBColPred {
    __device__ __forceinline__ bool operator()(const Operand &a, const Operand &b, uint64_t i, const uint8_t *, bool &bad1, bool &bad2) const {
        Str v, p;
        bad1 = !load_str(a, i, v); bad2 = !load_str(b, i, p);
        if (bad1 || bad2) return false;
        return glob_match(v, BytesPat{p});
    }
};

// rows [0, n): skipped when the result null bit is set on entry, NULL when an operand is (all_null: every row), else r[i] = pred.
// The loop runs to a multiple of 64 so that every word of the bitmap is written whole (bits past n cleared).
template <class P>
__global__ void __launch_bounds__(kThreads)
str_row_kernel(uint8_t *__restrict__ r, uint32_t *__restrict__ rn32, uint64_t n, Operand a, Operand b, P pred, const uint8_t *aux, uint32_t aux_len,
               int all_null, Status *st) {
    extern __shared__ __align__(16) uint8_t sm_aux[];
    const uint8_t *ax = aux;
    if (aux_len && aux_len <= kSmemAux) {
        for (uint32_t k = threadIdx.x; k < aux_len; k += kThreads) sm_aux[k] = aux[k];
        __syncthreads();
        ax = sm_aux;
    }
    const uint64_t n64 = (n + 63) & ~63ull;
    for (uint64_t i = blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < n64; i += (uint64_t)gridDim.x * kThreads) {
        const bool in = i < n;
        bool isnull = false;
        if (in) {
            const bool skip = (rn32[i >> 5] >> (i & 31)) & 1u;
            isnull = skip || all_null || bm_test(a.nulls, a.cst ? 0 : i) || bm_test(b.nulls, b.cst ? 0 : i);
            if (!isnull) {
                bool bad1, bad2;
                const bool v = pred(a, b, i, ax, bad1, bad2);
                if (bad1) atomicMax(&st->bad_inv[0], ~(unsigned long long)(a.cst ? 0 : i));
                if (bad2) atomicMax(&st->bad_inv[1], ~(unsigned long long)(b.cst ? 0 : i));
                if (!bad1 && !bad2) r[i] = v ? 1 : 0;
            }
        }
        const unsigned m = __ballot_sync(0xffffffffu, isnull);
        if ((threadIdx.x & 31) == 0) rn32[i >> 5] = m;
    }
}

// the status record, zeroed on the stream
Status *arm_status(ThreadCtx &t, Stager &st, const char *what) {
    Status *dst = (Status *)st.tmp(sizeof(Status));
    if (st.failed) return nullptr;
    if (cudaMemsetAsync(dst, 0, sizeof(Status), t.stream) != cudaSuccess) { set_error("%s: memset failed", what); return nullptr; }
    return dst;
}

// enqueues the row kernel over the device aux block, reads back the status record dst and names the lowest bad cell
template <class P>
int run_rows(ThreadCtx &t, Stager &st, uint8_t *r, uint64_t *rn, uint64_t len, const Operand &a, const Operand &b, const P &pred,
             const uint8_t *aux, uint32_t aux_len, int all_null, const char *what, Status *dst) {
    const size_t smem = aux_len && aux_len <= kSmemAux ? aux_len : 0;
    cudaEventRecord(t.kev0, t.stream);
    str_row_kernel<P><<<grid_rows(len, kCtasPerSm), kThreads, smem, t.stream>>>(r, reinterpret_cast<uint32_t *>(rn), len, a, b, pred, aux, aux_len, all_null, dst);
    cudaEventRecord(t.kev1, t.stream);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    if (cudaError_t e = cudaGetLastError()) { set_error("%s: kernel launch failed: %s", what, cudaGetErrorString(e)); return MO_RC_INTERNAL_ERROR; }
    Status hs;
    if (int rc = read_back(t, &hs, dst, sizeof hs)) return rc;
    for (int k = 0; k < 2; k++) {
        if (!hs.bad_inv[k]) continue;
        int rc = st.finish();
        if (rc) return rc;
        set_error("%s: operand %d row %llu: varlena cell outside its area", what, k + 1, (unsigned long long)~hs.bad_inv[k]);
        return MO_RC_INVALID_ARGUMENT;
    }
    return st.complete();
}
// the same with a host aux block (a const pattern), uploaded first
template <class P>
int run_rows(ThreadCtx &t, Stager &st, uint8_t *r, uint64_t *rn, uint64_t len, const Operand &a, const Operand &b, const P &pred,
             const std::vector<uint8_t> &aux_host, int all_null, const char *what) {
    uint8_t *aux = nullptr;
    const uint32_t aux_len = (uint32_t)aux_host.size();
    if (aux_len) {
        aux = (uint8_t *)st.tmp(aux_len);
        if (st.failed) return MO_RC_INTERNAL_ERROR;
        // pageable source: the runtime copies it into its own staging before this returns, so the vector may go out of scope
        if (cudaMemcpyAsync(aux, aux_host.data(), aux_len, cudaMemcpyHostToDevice, t.stream) != cudaSuccess) {
            set_error("%s: pattern upload failed", what); return MO_RC_INTERNAL_ERROR;
        }
    }
    Status *dst = arm_status(t, st, what);
    if (!dst) return MO_RC_INTERNAL_ERROR;
    return run_rows(t, st, r, rn, len, a, b, pred, aux, aux_len, all_null, what, dst);
}

// ---- IN / NOT IN (opOperatorStrIn): Go's map[string]bool of the list as kt_insert_str words (an XXH3 tag and the list index of the value)
// in mask + 1 slots, which the row kernel takes as its aux block -- in shared memory up to kSmemAux (== kInSmemBytes) bytes
__device__ __forceinline__ uint64_t str_hash_of(const Operand &c, uint64_t row, const Str &s) {
    const uint8_t *p = s.inl ? (const uint8_t *)c.data + 24 * (c.cst ? 0 : row) + 1 : s.p;
    return xxh3::hash_bytes(p, s.len, 0).lo;
}
__device__ __forceinline__ bool str_eq(const Str &x, const Str &y) { return x.len == y.len && str_cmp(x, y) == 0; }

// list element j (not NULL) into the set; a bad cell is recorded as operand 2's
__global__ void __launch_bounds__(kThreads) in_str_build_kernel(uint64_t *slots, uint64_t mask, Operand l, uint64_t m, Status *st) {
    for (uint64_t j = blockIdx.x * (uint64_t)kThreads + threadIdx.x; j < m; j += (uint64_t)gridDim.x * kThreads) {
        Str v;
        if (bm_test(l.nulls, j)) continue;
        if (!load_str(l, j, v)) { atomicMax(&st->bad_inv[1], ~(unsigned long long)j); continue; }
        const uint64_t h = str_hash_of(l, j, v);
        kt_insert_str(slots, mask, h, str_word(h, j), [&](uint32_t r) { Str w; return load_str(l, r, w) && str_eq(v, w); });
    }
}
// b = the list (its nulls are the build's, not the row kernel's); aux = the slots, none for the empty set
struct InPred {
    uint64_t mask; int negate;
    __device__ __forceinline__ bool operator()(const Operand &a, const Operand &b, uint64_t i, const uint8_t *aux, bool &bad1, bool &bad2) const {
        Str x;
        uint32_t row;
        bad2 = false; bad1 = !load_str(a, i, x);
        if (bad1 || !aux) return negate;
        const bool found = kt_find_str(reinterpret_cast<const uint64_t *>(aux), mask, str_hash_of(a, i, x),
                                       [&](uint32_t r) { Str y; return load_str(b, r, y) && str_eq(x, y); }, row);
        return found != (negate != 0);
    }
};

// ---- LIKE, host side
// the const pattern's value, read from the caller's memory.  rc != 0: a bad cell (error set).  *is_null: the const NULL pattern.
int read_const_pattern(ThreadCtx &t, const mo_xcall_args_t &a, std::string &pat, bool &is_null) {
    if (int rc = const_null(t, (const uint64_t *)a.pnulls, is_null)) return rc;
    if (is_null) return MO_RC_SUCCESS;
    uint8_t cell[MO_VARLENA_SZ];
    if (int rc = read_const(t, cell, a.pdata, MO_VARLENA_SZ)) return rc;
    uint32_t w[3];
    memcpy(w, cell, sizeof w);
    const VarlenaCell v = varlena_cell(w[0], w[1], w[2], a.parea, a.areaSz);
    if (!v.ok) { set_error("go like: operand 2 row 0: varlena cell outside its area"); return MO_RC_INVALID_ARGUMENT; }
    if (v.inl) { pat.assign((const char *)cell + 1, v.len); return MO_RC_SUCCESS; }
    pat.resize(v.len);
    return read_const(t, &pat[0], a.parea + v.off, v.len);
}

// functionUtil.RemoveEscapeChar: `\x` -> x; a trailing lone backslash is kept
std::string remove_escape(const std::string &s) {
    std::string o;
    for (size_t i = 0; i < s.size(); i++) {
        if (s[i] == '\\' && i + 1 < s.size()) i++;
        o.push_back(s[i]);
    }
    return o;
}

// optimizeRuleForLike restated: true and (mode, s, e, segments) when the rule takes the pattern
bool classify_like(const std::string &pat, int &mode, uint32_t &s, uint32_t &e, std::vector<std::string> &segs) {
    const size_t n = pat.size();
    s = e = 0;
    segs.clear();
    auto one = [&](int m, uint32_t s_, uint32_t e_, std::string lit) { mode = m; s = s_; e = e_; segs.push_back(std::move(lit)); return true; };
    if (n == 0) return one(LIKE_EXACT, 0, 0, "");                                  // rule 1
    if (n == 1) {
        if (pat[0] == '%') return one(LIKE_PREFIX, 0, 0, "");                      // 2.1
        if (pat[0] == '_') return one(LIKE_EXACT, 1, 0, "");                       // 2.2: one byte
        return one(LIKE_EXACT, 0, 0, pat);                                         // 2.3
    }
    const char c0 = pat[0];
    char c1 = pat[n - 1];
    const std::string mid = pat.substr(1, n - 2);
    auto wild = [](char c) { return c == '%' || c == '_'; };
    if (mid.find_first_of("_%") == std::string::npos) {
        if (n > 2 && pat[n - 2] == '\\') c1 = '\\';                                // the last byte is escaped: a literal
        if (!wild(c0) && !wild(c1)) return one(LIKE_EXACT, 0, 0, remove_escape(pat));                  // 4.1
        if (c0 == '_' && !wild(c1)) return one(LIKE_EXACT, 1, 0, remove_escape(pat.substr(1)));        // 4.2
        if (c0 == '%' && !wild(c1)) return one(LIKE_SUFFIX, 0, 0, remove_escape(pat.substr(1)));       // 4.3
        if (c1 == '_' && !wild(c0)) return one(LIKE_EXACT, 0, 1, remove_escape(pat.substr(0, n - 1))); // 4.4
        if (c1 == '%' && !wild(c0)) return one(LIKE_PREFIX, 0, 0, remove_escape(pat.substr(0, n - 1)));// 4.5
        if (c0 == '%' && c1 == '%') { mode = LIKE_CHAIN; segs.push_back(remove_escape(mid)); return true; }  // 4.6
        if (c0 == '%' && c1 == '_') return one(LIKE_SUFFIX, 0, 1, remove_escape(mid));                 // 4.7
        if (c0 == '_' && c1 == '%') return one(LIKE_PREFIX, 1, 0, remove_escape(mid));                 // 4.8
        return false;                                                              // _lit_: no rule
    }
    if (c0 == '%' && c1 == '%' && mid.find('_') == std::string::npos && pat.find("\\%") == std::string::npos) {
        mode = LIKE_CHAIN;                                                         // %a%b%...%: ordered bytes.Index, escapes kept as bytes
        size_t from = 1;
        for (size_t k = 1; k < n; k++) if (pat[k] == '%') { segs.push_back(pat.substr(from, k - from)); from = k + 1; }
        return true;
    }
    return false;
}

struct HostBytes { const uint8_t *p; __host__ __device__ uint32_t operator()(uint32_t j) const { return p[j]; } };
int32_t host_decode(const std::string &p, size_t i, size_t &size) {
    uint32_t sz;
    const int32_t r = decode_utf8(HostBytes{(const uint8_t *)p.data()}, (uint32_t)i, (uint32_t)p.size(), sz);
    size = sz;
    return r;
}

// the tokens of regularMatchForLikeOp's replace(): `\x` the literal rune x, a trailing `\` a literal backslash, `_` any one rune, `%` any run
std::vector<int32_t> tokenize(const std::string &p) {
    std::vector<int32_t> out;
    size_t i = 0;
    while (i < p.size()) {
        size_t sz;
        const int32_t r = host_decode(p, i, sz);
        i += sz;
        if (r == '\\') {
            if (i < p.size()) { out.push_back(host_decode(p, i, sz)); i += sz; }
            else out.push_back('\\');
        } else out.push_back(r == '_' ? kAny1 : (r == '%' ? kAnySeq : r));
    }
    return out;
}

}  // namespace

namespace mob {

// MO_XCALL_GO_COMPARE(op, T) for the varlena types (goelem.cu routes them here)
int go_str_compare(ThreadCtx &t, int op, mo_xcall_args_t *args, uint64_t len) {
    const char *what = "go compare";
    Stager st(t);
    uint8_t *r; uint64_t *rn;
    Operand a, b;
    if (int rc = stage_result(st, args[0], 1, len, true, true, what, r, rn)) return rc;
    if (int rc = stage_operand(st, args[1], MO_VARLENA_SZ, len, what, 1, a)) return rc;
    if (int rc = stage_operand(st, args[2], MO_VARLENA_SZ, len, what, 2, b)) return rc;
    return run_rows(t, st, r, rn, len, a, b, CmpPred{op}, std::vector<uint8_t>(), 0, what);
}

// MO_XCALL_GO_IN(T) / MO_XCALL_GO_NOT_IN(T) for the varlena types (goelem.cu routes them here).  Launches: the build (nvalues > 0), then
// the row kernel; one read-back of the status record.
int go_str_in(ThreadCtx &t, int negate, mo_xcall_args_t *args, uint64_t len) {
    const char *what = negate ? "go not in" : "go in";
    Stager st(t);
    uint8_t *r; uint64_t *rn;
    Operand a, l;
    uint64_t m, mask;
    if (int rc = stage_result(st, args[0], 1, len, true, true, what, r, rn)) return rc;
    if (int rc = stage_operand(st, args[1], MO_VARLENA_SZ, len, what, 1, a)) return rc;
    if (int rc = stage_in_list(t, st, args, MO_VARLENA_SZ, what, l, m, mask)) return rc;
    Status *dst = arm_status(t, st, what);
    if (!dst) return MO_RC_INTERNAL_ERROR;
    uint64_t *slots = nullptr;
    const uint64_t bytes = m ? (mask + 1) * 8 : 0;
    if (m) {
        slots = (uint64_t *)st.tmp(bytes);
        if (st.failed) return MO_RC_INTERNAL_ERROR;
        MOB_CUDA_TRY(cudaMemsetAsync(slots, 0xff, bytes, t.stream));
        in_str_build_kernel<<<grid_rows(m, kCtasPerSm), kThreads, 0, t.stream>>>(slots, mask, l, m, dst);
        MOB_LAUNCH_CHECK();
    }
    Operand lb = l;
    lb.nulls = nullptr;
    return run_rows(t, st, r, rn, len, a, lb, InPred{mask, negate}, (const uint8_t *)slots, (uint32_t)std::min<uint64_t>(bytes, 0xffffffffu), 0,
                    what, dst);
}

// MO_XCALL_GO_LIKE: args [0] bool result (+pnulls in/out) ; [1] the string ; [2] the pattern
int xcall_go_like(mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (len == 0) return MO_RC_SUCCESS;
    const char *what = "go like";
    Stager st(t);
    uint8_t *r; uint64_t *rn;
    Operand a, b;
    if (int rc = stage_result(st, args[0], 1, len, true, true, what, r, rn)) return rc;
    if (int rc = stage_operand(st, args[1], MO_VARLENA_SZ, len, what, 1, a)) return rc;
    if (!is_const(args[2], MO_VARLENA_SZ, len)) {
        if (int rc = stage_operand(st, args[2], MO_VARLENA_SZ, len, what, 2, b)) return rc;
        return run_rows(t, st, r, rn, len, a, b, LikeBColPred{}, std::vector<uint8_t>(), 0, what);
    }
    // a const pattern is read on the host, from the caller's memory
    std::string pat;
    bool pat_null = false;
    if (!args[2].pdata) { set_error("go like: operand 2 has no cells"); return MO_RC_INVALID_ARGUMENT; }
    if (int rc = read_const_pattern(t, args[2], pat, pat_null)) return rc;
    if (pat_null) return run_rows(t, st, r, rn, len, a, b, LikeBColPred{}, std::vector<uint8_t>(), 1, what);   // every row NULL
    int mode;
    uint32_t s, e;
    std::vector<std::string> segs;
    std::vector<uint8_t> aux;
    if (classify_like(pat, mode, s, e, segs)) {
        for (const std::string &g : segs) { const uint32_t L = (uint32_t)g.size(); aux.insert(aux.end(), (const uint8_t *)&L, (const uint8_t *)&L + 4); }
        for (const std::string &g : segs) aux.insert(aux.end(), g.begin(), g.end());
        return run_rows(t, st, r, rn, len, a, b, LikeAPred{mode, s, e, (uint32_t)segs.size()}, aux, 0, what);
    }
    const std::vector<int32_t> tok = tokenize(pat);
    aux.resize(4 * tok.size());
    if (!tok.empty()) memcpy(aux.data(), tok.data(), aux.size());
    return run_rows(t, st, r, rn, len, a, b, LikeBConstPred{(uint32_t)tok.size()}, aux, 0, what);
}

}  // namespace mob
