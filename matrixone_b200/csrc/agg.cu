// agg.cu -- single-column aggregates without group-by (the reference's H0 path: Group.buildOneBatch ->
// agg.BulkFill, pkg/sql/colexec/group/exec2.go:305-315) : SUM / AVG / COUNT / MIN / MAX over a fixed-width
// column + nulls bitmap.  Semantics: pkg/sql/colexec/aggexec/sumavg2.go:133-199,254-353, count2.go:120-146,
// minmax2.go:49-80.
//
// HBM-bound streaming reduction: every thread issues 4 independent 128-bit L1-bypassing loads per iteration
// (grid = SMs x CTAS_PER_SM persistent CTAs, grid-stride), the nulls word for 64 rows is a warp-broadcast
// load, partials are combined by warp shuffles -> shared memory -> one per-CTA record; the last CTA to finish
// (atomicInc ticket) folds the per-CTA records in index order, so results are run-to-run deterministic.
//
// Algorithmic bytes: sizeof(T) per row (+ 1/8 byte per row with a nulls bitmap).
#include "common.cuh"
#include <cstring>
#include <cmath>

using namespace mob;

namespace {

constexpr int kThreads = 256;
constexpr int kCtasPerSm = 4;
constexpr int kUnroll = 8;   // 8 x 128-bit loads in flight per thread: 128 KB per SM at 1024 threads

enum Kind { K_SUM_SIGNED = 0, K_SUM_UNSIGNED = 1, K_SUM_FLOAT = 2, K_MIN = 3, K_MAX = 4 };

// Per-CTA / final record.  Meaning of the words depends on Kind:
//  SUM_SIGNED  : w0 = two's-complement (wrapping) sum ; w2 = max |v| : if max|v| * (non-null rows) fits int64 no prefix can overflow (w3 unused)
//  SUM_UNSIGNED: w0,w1 = sum (lo,hi)
//  SUM_FLOAT   : d = sum (double)
//  MIN / MAX   : w0 = value bits (zero-extended), w1 = smallest row index of a non-null row (floats: NaN rule), w2 = the row of w0
//                (the first row that reaches the extreme, so -0.0 and 0.0 tie as the serial loop ties them)
//  all         : cnt = non-null rows
struct Rec { uint64_t w0, w1, w2, w3; double d; uint64_t cnt; uint64_t pad0, pad1; };
// signed SUM: can a prefix of the serial sum leave int64?  Not if every |v| <= INT64_MAX / rows (then even the sum of all magnitudes fits).
__device__ __forceinline__ bool sum_check_needed(const Rec &r) { return r.cnt != 0 && r.w2 > (uint64_t)INT64_MAX / r.cnt; }

__device__ __forceinline__ void add128(uint64_t &lo, uint64_t &hi, uint64_t x) { lo += x; hi += (lo < x); }
__device__ __forceinline__ void add128p(uint64_t &lo, uint64_t &hi, uint64_t lo2, uint64_t hi2) {
    lo += lo2; hi += hi2 + (lo < lo2);
}

template <typename T> struct Bits { };
template <typename T> __device__ __forceinline__ uint64_t to_bits(T v) { uint64_t r = 0; memcpy(&r, &v, sizeof(T)); return r; }
template <typename T> __device__ __forceinline__ T from_bits(uint64_t b) { T v; memcpy(&v, &b, sizeof(T)); return v; }

template <typename T, int KIND>
struct Acc {
    uint64_t w0 = 0, w1 = 0, w2 = 0, w3 = 0, cnt = 0;
    double d = 0.0;
    T mm;
    bool has = false;
    uint64_t first = ~0ull;
    uint64_t at = ~0ull;   // MIN / MAX: the row the kept value came from

    __device__ __forceinline__ void add(T v, uint64_t row) {
        cnt++;
        if (KIND == K_SUM_SIGNED) {
            const int64_t x = (int64_t)v;
            w0 += (uint64_t)x;
            const uint64_t m = x < 0 ? (0ull - (uint64_t)x) : (uint64_t)x;   // one compare + select instead of a 128-bit running sum of magnitudes
            w2 = m > w2 ? m : w2;
        } else if (KIND == K_SUM_UNSIGNED) {
            add128(w0, w1, (uint64_t)v);
        } else if (KIND == K_SUM_FLOAT) {
            d = d + (double)v;  // sums[g] += float64(val), sumavg2.go:153
        } else {
            // a thread sees its rows in rising order, so the strict compare keeps the first row of a tie (-0.0 before 0.0)
            if (!has) { has = true; mm = v; first = row; at = row; }
            else if (KIND == K_MIN ? (v < mm) : (v > mm)) { mm = v; at = row; }       // strict compare, minmax2.go:73
            else if (mm != mm && !(v != v)) { /* running value NaN but not the global first row: Go would never hold it */ mm = v; at = row; }
        }
    }
    __device__ __forceinline__ void merge(const Rec &r) {
        if (r.cnt == 0) return;
        if (KIND == K_SUM_SIGNED) { w0 += r.w0; w2 = r.w2 > w2 ? r.w2 : w2; }
        else if (KIND == K_SUM_UNSIGNED) { add128p(w0, w1, r.w0, r.w1); }
        else if (KIND == K_SUM_FLOAT) { d = d + r.d; }
        else {
            T v = from_bits<T>(r.w0);
            if (!has) { has = true; mm = v; first = r.w1; at = r.w2; }
            else {
                if (r.w1 < first) first = r.w1;
                // an equal value from an earlier row wins: the serial loop keeps the first row that reaches the extreme
                if ((KIND == K_MIN ? (v < mm) : (v > mm)) || (v == mm && r.w2 < at)) { mm = v; at = r.w2; }
                else if (mm != mm && !(v != v)) { mm = v; at = r.w2; }
            }
        }
        cnt += r.cnt;
    }
    __device__ __forceinline__ Rec rec() const {
        Rec r; r.w0 = w0; r.w1 = w1; r.w2 = w2; r.w3 = w3; r.d = d; r.cnt = cnt; r.pad0 = r.pad1 = 0;
        if (KIND == K_MIN || KIND == K_MAX) { r.w0 = has ? to_bits<T>(mm) : 0; r.w1 = first; r.w2 = at; }
        return r;
    }
};

__device__ __forceinline__ Rec shfl_rec(const Rec &r, int o) {
    Rec q;
    q.w0 = __shfl_xor_sync(0xffffffffu, r.w0, o); q.w1 = __shfl_xor_sync(0xffffffffu, r.w1, o);
    q.w2 = __shfl_xor_sync(0xffffffffu, r.w2, o); q.w3 = __shfl_xor_sync(0xffffffffu, r.w3, o);
    q.d = __shfl_xor_sync(0xffffffffu, r.d, o); q.cnt = __shfl_xor_sync(0xffffffffu, r.cnt, o);
    q.pad0 = q.pad1 = 0;
    return q;
}

// Combine two records in a FIXED order (a then b): used by every tree level so the association is data independent.
template <typename T, int KIND>
__device__ __forceinline__ Rec combine(const Rec &a, const Rec &b) {
    Acc<T, KIND> x;
    x.merge(a); x.merge(b);
    return x.rec();
}

template <typename T, int KIND>
__device__ Rec block_reduce(Rec r) {
    __shared__ Rec sm[kThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        Rec q = shfl_rec(r, o);
        // lower lane first keeps (a,b) order identical on both partners for the commutative-but-not-associative fp add
        r = (lane & o) ? combine<T, KIND>(q, r) : combine<T, KIND>(r, q);
    }
    if (lane == 0) sm[warp] = r;
    __syncthreads();
    if (warp == 0) {
        Rec z; z.w0 = z.w1 = z.w2 = z.w3 = 0; z.d = 0; z.cnt = 0; z.pad0 = z.pad1 = 0;
        r = lane < kThreads / 32 ? sm[lane] : z;
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) {
            Rec q = shfl_rec(r, o);
            r = (lane & o) ? combine<T, KIND>(q, r) : combine<T, KIND>(r, q);
        }
    }
    __syncthreads();
    return r;  // valid in warp 0
}

struct Seg { __int128 total, maxp, minp; };
enum Cls { C_SIGNED = 0, C_UNSIGNED = 1, C_FLOAT = 2, C_MINMAX = 3, C_COUNT = 4 };
// the result / partial state in device memory (the caller's, or staged for a host result): the last CTA writes it itself (no second
// launch); rc, when set, receives the state's rc word for the synchronous form to return
struct AggStateOut { uint64_t *res; uint64_t res_words; uint64_t *rnulls; int64_t *rc; int op; int cls; };

__device__ __forceinline__ void write_agg_state(const Rec &rec, const AggStateOut &so, int32_t ov) {
    uint64_t bits = 0, cnt = rec.cnt; int64_t rc = MO_RC_SUCCESS; const bool isnull = cnt == 0 && so.cls != C_COUNT;
    double dsum = 0.0;
    if (so.cls == C_SIGNED) { bits = rec.w0; dsum = (double)(int64_t)rec.w0; if (ov) rc = MO_RC_OUT_OF_RANGE; }
    else if (so.cls == C_UNSIGNED) { bits = rec.w0; dsum = (double)rec.w0; if (rec.w1) rc = MO_RC_OUT_OF_RANGE; }
    else if (so.cls == C_FLOAT) { dsum = rec.d; memcpy(&bits, &dsum, 8); }
    else bits = rec.w0;
    // a 1-word result of AVG is the final value; a 3-word result is the partial STATE (sum in the SUM return type, count, rc) and AVG divides at the merge
    if (so.op == MO_AGG_AVG && so.res_words < 3 && !isnull) { double avg = dsum / (double)cnt; memcpy(&bits, &avg, 8); }
    so.res[0] = bits;
    if (so.res_words >= 2) so.res[1] = cnt;
    if (so.res_words >= 3) so.res[2] = (uint64_t)rc;
    if (so.rnulls) so.rnulls[0] = isnull ? 1ull : 0ull;
    if (so.rc) *so.rc = rc;
}

// col must be 16-byte aligned for the vector path (vec = true); rows are [0, n).
template <typename T, int KIND>
__global__ void __launch_bounds__(kThreads, kCtasPerSm)
agg_kernel(const T *__restrict__ col, const uint64_t *__restrict__ nulls, uint64_t n, bool vec,
           Rec *__restrict__ partials, Rec *__restrict__ out, unsigned *ticket, AggStateOut so) {
    constexpr int V = 16 / sizeof(T);  // rows per 128-bit load
    Acc<T, KIND> acc;
    const uint64_t tid = blockIdx.x * (uint64_t)kThreads + threadIdx.x;
    const uint64_t nthreads = (uint64_t)gridDim.x * kThreads;
    uint64_t done = 0;
    if (vec) {
        const uint64_t nvec = n / V;
        const int4 *p = reinterpret_cast<const int4 *>(col);
        uint64_t v = tid;
        for (; v + (kUnroll - 1) * nthreads < nvec; v += kUnroll * nthreads) {
            int4 x[kUnroll];
#pragma unroll
            for (int k = 0; k < kUnroll; k++) x[k] = ld_stream16(p + v + k * nthreads);
#pragma unroll
            for (int k = 0; k < kUnroll; k++) {
                const uint64_t row0 = (v + k * nthreads) * V;
                uint32_t nb = nulls ? (uint32_t)((__ldg(nulls + (row0 >> 6)) >> (row0 & 63)) & ((1u << V) - 1u)) : 0u;
                if (V == 16 && nulls) nb = (uint32_t)((__ldg(nulls + (row0 >> 6)) >> (row0 & 63)) & 0xffffu);
                T e[V];
                memcpy(e, &x[k], 16);
#pragma unroll
                for (int j = 0; j < V; j++)
                    if (!((nb >> j) & 1u)) acc.add(e[j], row0 + j);
            }
        }
        for (; v < nvec; v += nthreads) {
            int4 x = ld_stream16(p + v);
            const uint64_t row0 = v * V;
            uint32_t nb = nulls ? (uint32_t)((__ldg(nulls + (row0 >> 6)) >> (row0 & 63)) & (V == 16 ? 0xffffu : ((1u << V) - 1u))) : 0u;
            T e[V];
            memcpy(e, &x, 16);
#pragma unroll
            for (int j = 0; j < V; j++)
                if (!((nb >> j) & 1u)) acc.add(e[j], row0 + j);
        }
        done = nvec * V;
    }
    // scalar tail (and the whole column when it is not 16-byte aligned)
    for (uint64_t i = done + tid; i < n; i += nthreads)
        if (!bm_test(nulls, i)) acc.add(col[i], i);

    Rec r = block_reduce<T, KIND>(acc.rec());
    __shared__ bool last;
    if (threadIdx.x == 0) {
        partials[blockIdx.x] = r;
        __threadfence();
        unsigned t = atomicInc(ticket, gridDim.x - 1);  // wraps to 0 after the last CTA: reusable without a memset
        last = (t == gridDim.x - 1);
    }
    __syncthreads();
    if (last) {
        __threadfence();
        Acc<T, KIND> f;
        for (unsigned b = threadIdx.x; b < gridDim.x; b += kThreads) f.merge(partials[b]);  // fixed index order per thread
        Rec fr = block_reduce<T, KIND>(f.rec());
        if (threadIdx.x == 0) {
            if ((KIND == K_MIN || KIND == K_MAX) && fr.cnt) {
                // Go rule (minmax2.go:69-75): the first non-null value initialises; a NaN there is never replaced
                T fv = col[fr.w1];
                if (fv != fv) fr.w0 = to_bits<T>(fv);
            }
            *out = fr;
        }
        if (so.res) {
            // signed SUM whose magnitudes do not fit int64 (pathological): the exact serial-order prefix check, done by this CTA alone --
            // thread k summarises rows [k * seg, (k + 1) * seg) as (total, max prefix, min prefix), thread 0 folds the 256 summaries in order
            __shared__ Seg sseg[KIND == K_SUM_SIGNED ? kThreads : 1];
            __shared__ Rec sfr;
            __shared__ int32_t sov;
            if (threadIdx.x == 0) { sfr = fr; sov = 0; }
            __syncthreads();
            if (KIND == K_SUM_SIGNED && sum_check_needed(sfr)) {
                const uint64_t seg = (n + kThreads - 1) / kThreads;
                const uint64_t r0 = (uint64_t)threadIdx.x * seg, r1 = r0 + seg < n ? r0 + seg : n;
                __int128 tot = 0, mx = 0, mn = 0;
                for (uint64_t i = r0; i < r1; i++) {
                    if (bm_test(nulls, i)) continue;
                    tot += (__int128)(int64_t)col[i];
                    if (tot > mx) mx = tot;
                    if (tot < mn) mn = tot;
                }
                sseg[threadIdx.x].total = tot; sseg[threadIdx.x].maxp = mx; sseg[threadIdx.x].minp = mn;
                __syncthreads();
                if (threadIdx.x == 0) {
                    __int128 run = 0;
                    const __int128 hi = (__int128)INT64_MAX, lo = (__int128)INT64_MIN;
                    for (int k = 0; k < kThreads; k++) {
                        if (run + sseg[k].maxp > hi || run + sseg[k].minp < lo) { sov = 1; break; }
                        run += sseg[k].total;
                    }
                }
                __syncthreads();
            }
            if (threadIdx.x == 0) write_agg_state(sfr, so, sov);
        }
    }
}

template <typename T, int KIND>
int launch_agg(ThreadCtx &t, const void *dcol, const uint64_t *dnulls, uint64_t n, const AggStateOut &so) {
    int grid = num_sms() * kCtasPerSm;
    uint64_t work = (n + (16 / sizeof(T)) * kThreads - 1) / ((16 / sizeof(T)) * kThreads);
    if ((uint64_t)grid > work) grid = work ? (int)work : 1;
    Rec *partials = (Rec *)arena_alloc(t, sizeof(Rec) * (size_t)(grid + 1));
    if (!partials) return MO_RC_INTERNAL_ERROR;
    Rec *out = partials + grid;
    bool vec = (((uintptr_t)dcol) & 15) == 0;
    cudaEventRecord(t.kev0, t.stream);
    agg_kernel<T, KIND><<<grid, kThreads, 0, t.stream>>>((const T *)dcol, dnulls, n, vec, partials, out, t.ctrl, so);
    cudaEventRecord(t.kev1, t.stream);
    MOB_LAUNCH_CHECK();
    return MO_RC_SUCCESS;
}

template <typename T>
int launch_agg_typed(ThreadCtx &t, const void *dcol, const uint64_t *dnulls, uint64_t n, const AggStateOut &so) {
    if (so.op == MO_AGG_MIN) return launch_agg<T, K_MIN>(t, dcol, dnulls, n, so);
    if (so.op == MO_AGG_MAX) return launch_agg<T, K_MAX>(t, dcol, dnulls, n, so);
    if (so.cls == C_FLOAT) return launch_agg<T, K_SUM_FLOAT>(t, dcol, dnulls, n, so);
    if (so.cls == C_UNSIGNED) return launch_agg<T, K_SUM_UNSIGNED>(t, dcol, dnulls, n, so);
    return launch_agg<T, K_SUM_SIGNED>(t, dcol, dnulls, n, so);
}

__global__ void popcount_kernel(const uint64_t *p, uint64_t nbits, unsigned long long *out) {
    // count set bits among the first nbits (last word masked, cgo/bitmap.h:110-131)
    uint64_t nw = (nbits + 63) >> 6;
    unsigned long long c = 0;
    for (uint64_t w = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; w < nw; w += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t v = p[w];
        if (w == nw - 1 && (nbits & 63)) v &= ((1ull << (nbits & 63)) - 1ull);
        c += __popcll(v);
    }
    c = warp_sum(c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, c);
}

// *dout = set bits among the first nbits of dp (nbits > 0), in stream order
int launch_popcount(ThreadCtx &t, const uint64_t *dp, uint64_t nbits, unsigned long long *dout) {
    MOB_CUDA_TRY(cudaMemsetAsync(dout, 0, 8, t.stream));
    uint64_t nw = (nbits + 63) >> 6;
    int grid = (int)((nw + 255) / 256);
    if (grid > num_sms() * 8) grid = num_sms() * 8;
    popcount_kernel<<<grid, 256, 0, t.stream>>>(dp, nbits, dout);
    MOB_LAUNCH_CHECK();
    return MO_RC_SUCCESS;
}

// COUNT, or an empty column: the state without a column scan (COUNT subtracts the null count popcount_kernel left in *nullcount)
__global__ void agg_state_kernel(uint64_t len, const unsigned long long *nullcount, AggStateOut so) {
    Rec r{};
    if (so.cls == C_COUNT) r.w0 = r.cnt = len - (nullcount ? *nullcount : 0ull);
    write_agg_state(r, so, 0);
}

// ---- MergeGroup for H0 aggregates: fold `n` partial states (value bits, non-null count, rc) in order (BatchMerge, sumavg2.go:205-248,
// count2.go, minmax2.go:90-110).  1 thread: n is the number of pipelines / GPUs.
template <typename T>
__device__ bool mm_less(uint64_t a, uint64_t b) { return from_bits<T>(a) < from_bits<T>(b); }

__global__ void agg_merge_kernel(const uint64_t *parts, uint64_t n, int op, int T, int cls, uint64_t *res, uint64_t res_words, uint64_t *rnulls, int64_t *rc_out) {
    uint64_t bits = 0, cnt = 0; int64_t rc = MO_RC_SUCCESS; bool has = false;
    double dsum = 0.0;
    for (uint64_t i = 0; i < n; i++) {
        const uint64_t b = parts[3 * i], c = parts[3 * i + 1]; const int64_t prc = (int64_t)parts[3 * i + 2];
        if (prc && !rc) rc = prc;
        if (op == MO_AGG_COUNT) { bits += b; cnt += c; continue; }
        if (c == 0) continue;   // a NULL partial is skipped
        if (!has) { has = true; bits = b; cnt = c; memcpy(&dsum, &b, 8); continue; }
        cnt += c;
        if (cls == C_FLOAT) { double x; memcpy(&x, &b, 8); dsum = dsum + x; memcpy(&bits, &dsum, 8); }
        else if (cls == C_SIGNED) {
            const int64_t v1 = (int64_t)bits, v2 = (int64_t)b, sum = (int64_t)(bits + b);
            if (((v1 > 0 && v2 > 0 && sum <= 0) || (v1 < 0 && v2 < 0 && sum >= 0)) && !rc) rc = MO_RC_OUT_OF_RANGE;   // int64OfCheck
            bits = (uint64_t)sum;
        } else if (cls == C_UNSIGNED) {
            const uint64_t sum = bits + b;
            if ((sum < bits || sum < b) && !rc) rc = MO_RC_OUT_OF_RANGE;                                                   // uint64OfCheck
            bits = sum;
        } else {   // MIN / MAX: strict compare, the earlier partial wins ties (minmax2.go:97-104)
            bool repl = false;
#define MMCASE(TT) repl = op == MO_AGG_MIN ? mm_less<TT>(b, bits) : mm_less<TT>(bits, b)
            switch (T) {
            case MO_T_BOOL: case MO_T_UINT8: MMCASE(uint8_t); break;
            case MO_T_INT8: MMCASE(int8_t); break;
            case MO_T_INT16: MMCASE(int16_t); break;
            case MO_T_UINT16: MMCASE(uint16_t); break;
            case MO_T_INT32: case MO_T_DATE: MMCASE(int32_t); break;
            case MO_T_UINT32: MMCASE(uint32_t); break;
            case MO_T_UINT64: MMCASE(uint64_t); break;
            case MO_T_FLOAT32: MMCASE(float); break;
            case MO_T_FLOAT64: MMCASE(double); break;
            default: MMCASE(int64_t); break;
            }
#undef MMCASE
            if (repl) bits = b;
        }
    }
    const bool isnull = op != MO_AGG_COUNT && !has;
    if (op == MO_AGG_AVG && has && res_words < 3) {   // float64(sum) / float64(cnt), sumavg2.go:331
        if (cls == C_SIGNED) dsum = (double)(int64_t)bits; else if (cls == C_UNSIGNED) dsum = (double)bits; else memcpy(&dsum, &bits, 8);
        double avg = dsum / (double)cnt; memcpy(&bits, &avg, 8);
    }
    res[0] = bits;
    if (res_words >= 2) res[1] = cnt;
    if (res_words >= 3) res[2] = (uint64_t)rc;
    if (rnulls) rnulls[0] = isnull ? 1ull : 0ull;
    if (rc_out) *rc_out = rc;
}

}  // namespace

namespace mob {

// MO_XCALL_AGG_MERGE(op, T): args[0] = result (as MO_XCALL_AGG), args[1] = len partial states of 24 bytes each
int xcall_agg_merge(int op, int T, mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (!type_size(T) || op < 0 || op > MO_AGG_AVG) { set_error("agg merge: bad op/type"); return MO_RC_INVALID_ARGUMENT; }
    if (!args[0].pdata || args[0].dataSz < 8 || args[1].dataSz < 24 * len) { set_error("agg merge: result needs 8 bytes, partial states 24 bytes each"); return MO_RC_INVALID_ARGUMENT; }
    const bool is_signed = T >= MO_T_INT8 && T <= MO_T_INT64, is_unsigned = T >= MO_T_UINT8 && T <= MO_T_UINT64;
    const int cls = op == MO_AGG_COUNT ? C_COUNT : (op == MO_AGG_MIN || op == MO_AGG_MAX) ? C_MINMAX : is_signed ? C_SIGNED : is_unsigned ? C_UNSIGNED : C_FLOAT;
    Stager st(t);
    const uint64_t *dparts = (const uint64_t *)st.in(args[1].pdata, 24 * len);
    uint64_t *dres = (uint64_t *)st.out(args[0].pdata, args[0].dataSz >= 24 ? 24 : args[0].dataSz >= 16 ? 16 : 8);
    uint64_t *dn = (uint64_t *)st.out(args[0].pnulls, args[0].pnulls ? 8 : 0);
    // the asynchronous form leaves errors in the merged state's rc word; the synchronous form copies the rc back with the results
    const bool async = st.resident();
    int64_t hrc = 0;
    int64_t *drc = async ? nullptr : (int64_t *)st.out(&hrc, 8);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    agg_merge_kernel<<<1, 1, 0, t.stream>>>(dparts, len, op, T, cls, dres, args[0].dataSz / 8, dn, drc);
    MOB_LAUNCH_CHECK();
    const int rc = st.complete();
    if (rc || async) return rc;
    if (hrc) set_error("data out of range: merged SUM overflows its 64-bit state");
    return (int)hrc;
}

int bitmap_count_device(ThreadCtx &t, const uint64_t *dp, uint64_t nbits, uint64_t *count) {
    if (nbits == 0 || !dp) { *count = 0; return MO_RC_SUCCESS; }
    unsigned long long *dout = (unsigned long long *)arena_alloc(t, 8);
    if (!dout) return MO_RC_INTERNAL_ERROR;
    int rc = launch_popcount(t, dp, nbits, dout);
    return rc ? rc : read_back(t, count, dout, 8);
}

// XCall family MO_XCALL_AGG(op, T): args[0] = result, args[1] = column.  See include/mo_b200.h.
// When the column, the result and their nulls words live in device memory the call only enqueues work on the calling thread's stream: no read-back, no
// synchronisation.  This is what lets a multi-GPU caller hand the partial state straight to NCCL (MergeGroup seam, mergeGroup.go:132-247)
// and merge on the device.  Otherwise the same kernels write staged buffers, and the call returns the state's rc.
int xcall_agg(int op, int T, mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    const int sz = type_size(T);
    if (!sz || T == MO_T_BOOL && op != MO_AGG_COUNT && op != MO_AGG_MIN && op != MO_AGG_MAX) { set_error("agg: unsupported type %d", T); return MO_RC_INVALID_ARGUMENT; }
    if (!args[0].pdata || args[0].dataSz < 8) { set_error("agg: result vector must hold 8 bytes"); return MO_RC_INVALID_ARGUMENT; }
    if (args[1].dataSz < (uint64_t)sz * len) { set_error("agg: column shorter than len"); return MO_RC_INVALID_ARGUMENT; }
    if (op < 0 || op > MO_AGG_AVG) { set_error("agg: unknown op %d", op); return MO_RC_INVALID_ARGUMENT; }
    const bool is_signed = T >= MO_T_INT8 && T <= MO_T_INT64, is_unsigned = T >= MO_T_UINT8 && T <= MO_T_UINT64;
    const int cls = op == MO_AGG_COUNT ? C_COUNT : (op == MO_AGG_MIN || op == MO_AGG_MAX) ? C_MINMAX : is_signed ? C_SIGNED : is_unsigned ? C_UNSIGNED : C_FLOAT;
    if (cls == C_FLOAT && T != MO_T_FLOAT32 && T != MO_T_FLOAT64) { set_error("sum: unsupported type %d", T); return MO_RC_INVALID_ARGUMENT; }
    Stager st(t);
    const void *dcol = st.in(args[1].pdata, (size_t)sz * len);
    const uint64_t *dnulls = (const uint64_t *)st.in(args[1].pnulls, args[1].pnulls ? ((len + 63) / 64) * 8 : 0);
    // 1 word: the value; 2: + non-null rows; 3: + rc (the partial state MO_XCALL_AGG_MERGE folds)
    const uint64_t words = args[0].dataSz >= 24 ? 3 : args[0].dataSz / 8;
    // the synchronous form stages the host results and the rc word as one block: one copy back, as for an 8192-row call it is most of the cost
    const bool hres = !st.device(args[0].pdata), hnulls = !st.device(args[0].pnulls);
    const bool async = st.resident();
    struct { uint64_t words[3], nulls; int64_t rc; } h{};
    uint64_t *dh = async ? nullptr : (uint64_t *)st.out(&h, sizeof h);
    const AggStateOut so{hres ? dh : (uint64_t *)args[0].pdata, words, hnulls ? dh + 3 : args[0].pnulls, async ? nullptr : (int64_t *)dh + 4, op, cls};
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    int rc = MO_RC_SUCCESS;
    if (op == MO_AGG_COUNT || len == 0) {
        unsigned long long *dcount = nullptr;
        if (op == MO_AGG_COUNT && dnulls && len) {
            dcount = (unsigned long long *)st.tmp(8);
            if (st.failed) return MO_RC_INTERNAL_ERROR;
            rc = launch_popcount(t, dnulls, len, dcount);
            if (rc) return rc;
        }
        agg_state_kernel<<<1, 1, 0, t.stream>>>(len, dcount, so);
        MOB_LAUNCH_CHECK();
    } else {
        switch (T) {
        case MO_T_BOOL: case MO_T_UINT8: rc = launch_agg_typed<uint8_t>(t, dcol, dnulls, len, so); break;
        case MO_T_INT8: rc = launch_agg_typed<int8_t>(t, dcol, dnulls, len, so); break;
        case MO_T_INT16: rc = launch_agg_typed<int16_t>(t, dcol, dnulls, len, so); break;
        case MO_T_UINT16: rc = launch_agg_typed<uint16_t>(t, dcol, dnulls, len, so); break;
        case MO_T_INT32: case MO_T_DATE: rc = launch_agg_typed<int32_t>(t, dcol, dnulls, len, so); break;
        case MO_T_UINT32: rc = launch_agg_typed<uint32_t>(t, dcol, dnulls, len, so); break;
        case MO_T_INT64: case MO_T_TIME: case MO_T_DATETIME: case MO_T_TIMESTAMP: rc = launch_agg_typed<int64_t>(t, dcol, dnulls, len, so); break;
        case MO_T_UINT64: rc = launch_agg_typed<uint64_t>(t, dcol, dnulls, len, so); break;
        case MO_T_FLOAT32: rc = launch_agg_typed<float>(t, dcol, dnulls, len, so); break;
        case MO_T_FLOAT64: rc = launch_agg_typed<double>(t, dcol, dnulls, len, so); break;
        default: set_error("agg: unsupported type %d", T); return MO_RC_INVALID_ARGUMENT;
        }
        if (rc) return rc;
    }
    rc = st.complete();
    if (rc || async) return rc;   // the asynchronous form leaves errors in the state's rc word
    if (hres) memcpy(args[0].pdata, h.words, 8 * words);
    if (hnulls) memcpy(args[0].pnulls, &h.nulls, 8);
    return (int)h.rc;
}

}  // namespace mob
