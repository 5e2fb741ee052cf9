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
//  MIN / MAX   : w0 = value bits (zero-extended), w1 = smallest row index of a non-null row (floats: NaN rule)
//  all         : cnt = non-null rows
struct Rec { uint64_t w0, w1, w2, w3; double d; uint64_t cnt; uint64_t pad0, pad1; };
// signed SUM: can a prefix of the serial sum leave int64?  Not if every |v| <= INT64_MAX / rows (then even the sum of all magnitudes fits).
__host__ __device__ __forceinline__ bool sum_check_needed(const Rec &r) { return r.cnt != 0 && r.w2 > (uint64_t)INT64_MAX / r.cnt; }

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
            if (!has) { has = true; mm = v; first = row; }
            else if (KIND == K_MIN ? (v < mm) : (v > mm)) mm = v;       // strict compare, minmax2.go:73
            else if (mm != mm && !(v != v)) { /* running value NaN but not the global first row: Go would never hold it */ mm = v; }
        }
    }
    __device__ __forceinline__ void merge(const Rec &r) {
        if (r.cnt == 0) return;
        if (KIND == K_SUM_SIGNED) { w0 += r.w0; w2 = r.w2 > w2 ? r.w2 : w2; }
        else if (KIND == K_SUM_UNSIGNED) { add128p(w0, w1, r.w0, r.w1); }
        else if (KIND == K_SUM_FLOAT) { d = d + r.d; }
        else {
            T v = from_bits<T>(r.w0);
            if (!has) { has = true; mm = v; first = r.w1; }
            else {
                if (r.w1 < first) first = r.w1;
                if (KIND == K_MIN ? (v < mm) : (v > mm)) mm = v;
                else if (mm != mm && !(v != v)) mm = v;
            }
        }
        cnt += r.cnt;
    }
    __device__ __forceinline__ Rec rec() const {
        Rec r; r.w0 = w0; r.w1 = w1; r.w2 = w2; r.w3 = w3; r.d = d; r.cnt = cnt; r.pad0 = r.pad1 = 0;
        if (KIND == K_MIN || KIND == K_MAX) { r.w0 = has ? to_bits<T>(mm) : 0; r.w1 = first; }
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
// asynchronous form: the last CTA writes the caller's device-resident result / partial state itself (no second launch)
struct AggStateOut { uint64_t *res; uint64_t res_words; uint64_t *rnulls; int op; int cls; };

__device__ __forceinline__ void write_agg_state(const Rec &rec, const AggStateOut &so, int32_t ov) {
    uint64_t bits = 0, cnt = rec.cnt; int64_t rc = MO_RC_SUCCESS; const bool isnull = cnt == 0;
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

// ---- exact serial-order overflow check for SUM over signed ints (slow path, rare) ---------------------------------
// Go errors at the first row whose running sum leaves int64 (int64OfCheck, sumavg2.go:89-94).  Each thread summarises a
// contiguous segment as (total, max prefix, min prefix) in 128-bit; segments are then folded in row order.

// `gate` (async path): the aggregate record of the same call; when its magnitude sum fits int64 no prefix can overflow and the
// whole grid returns at once
__device__ __forceinline__ bool prefix_check_needed(const Rec *gate) { return !gate || sum_check_needed(*gate); }

template <typename T>
__global__ void prefix_seg_kernel(const T *__restrict__ col, const uint64_t *__restrict__ nulls, uint64_t n, uint64_t seg_rows, uint64_t nseg,
                                  Seg *segs, const Rec *gate) {
    if (!prefix_check_needed(gate)) return;
    uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (s >= nseg) return;   // the grid is rounded up to whole CTAs: surplus threads own no segment
    uint64_t r0 = s * seg_rows, r1 = r0 + seg_rows;
    if (r1 > n) r1 = n;
    __int128 tot = 0, mx = 0, mn = 0;
    for (uint64_t i = r0; i < r1; i++) {
        if (bm_test(nulls, i)) continue;
        tot += (__int128)(int64_t)col[i];
        if (tot > mx) mx = tot;
        if (tot < mn) mn = tot;
    }
    segs[s].total = tot; segs[s].maxp = mx; segs[s].minp = mn;
}
__global__ void prefix_fold_kernel(const Seg *segs, uint64_t nseg, int32_t *overflow, const Rec *gate) {
    if (!prefix_check_needed(gate)) { *overflow = 0; return; }
    __int128 run = 0; int32_t ov = 0;
    const __int128 hi = (__int128)INT64_MAX, lo = (__int128)INT64_MIN;
    for (uint64_t s = 0; s < nseg; s++) {
        if (run + segs[s].maxp > hi || run + segs[s].minp < lo) { ov = 1; break; }
        run += segs[s].total;
    }
    *overflow = ov;
}

template <typename T, int KIND>
int launch_agg(ThreadCtx &t, const void *dcol, const uint64_t *dnulls, uint64_t n, Rec *hrec, Rec **drec = nullptr, AggStateOut so = AggStateOut{nullptr, 0, nullptr, 0, 0}) {
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
    if (drec) { *drec = out; return MO_RC_SUCCESS; }   // async: the record stays on the device
    return read_back(t, hrec, out, sizeof(Rec));
}

template <typename T>
int signed_prefix_overflow(ThreadCtx &t, const void *dcol, const uint64_t *dnulls, uint64_t n, int32_t *ov, const Rec *gate = nullptr,
                           int32_t **dov_out = nullptr) {
    const uint64_t nseg_target = (uint64_t)num_sms() * 256;
    uint64_t seg_rows = (n + nseg_target - 1) / nseg_target;
    if (seg_rows < 64) seg_rows = 64;
    uint64_t nseg = (n + seg_rows - 1) / seg_rows;
    Seg *segs = (Seg *)arena_alloc(t, sizeof(Seg) * nseg + 16);
    if (!segs) return MO_RC_INTERNAL_ERROR;
    int32_t *dov = (int32_t *)(segs + nseg);
    prefix_seg_kernel<T><<<(unsigned)((nseg + 255) / 256), 256, 0, t.stream>>>((const T *)dcol, dnulls, n, seg_rows, nseg, segs, gate);
    MOB_LAUNCH_CHECK();
    prefix_fold_kernel<<<1, 1, 0, t.stream>>>(segs, nseg, dov, gate);
    MOB_LAUNCH_CHECK();
    if (dov_out) { *dov_out = dov; return MO_RC_SUCCESS; }   // async: the flag stays on the device
    return read_back(t, ov, dov, 4);
}

template <typename T>
int run_sum_signed(ThreadCtx &t, const void *dcol, const uint64_t *dnulls, uint64_t n, int64_t *sum, uint64_t *cnt) {
    Rec r;
    int rc = launch_agg<T, K_SUM_SIGNED>(t, dcol, dnulls, n, &r);
    if (rc) return rc;
    *cnt = r.cnt;
    // |every prefix| <= sum of |v|: if that fits int64 nothing can overflow and the wrapping sum is the exact sum
    *sum = (int64_t)r.w0;
    if (!sum_check_needed(r)) return MO_RC_SUCCESS;
    // otherwise decide with the exact serial-order prefix check; when it passes, the total fits and the wrapping sum is exact
    int32_t ov = 0;
    rc = signed_prefix_overflow<T>(t, dcol, dnulls, n, &ov);
    if (rc) return rc;
    return ov ? MO_RC_OUT_OF_RANGE : MO_RC_SUCCESS;
}

template <typename T>
int run_sum_unsigned(ThreadCtx &t, const void *dcol, const uint64_t *dnulls, uint64_t n, uint64_t *sum, uint64_t *cnt) {
    Rec r;
    int rc = launch_agg<T, K_SUM_UNSIGNED>(t, dcol, dnulls, n, &r);
    if (rc) return rc;
    *cnt = r.cnt; *sum = r.w0;
    return r.w1 ? MO_RC_OUT_OF_RANGE : MO_RC_SUCCESS;  // prefixes are monotone: overflow iff the exact total exceeds 2^64-1
}

template <typename T>
int run_sum_float(ThreadCtx &t, const void *dcol, const uint64_t *dnulls, uint64_t n, double *sum, uint64_t *cnt) {
    Rec r;
    int rc = launch_agg<T, K_SUM_FLOAT>(t, dcol, dnulls, n, &r);
    if (rc) return rc;
    *cnt = r.cnt; *sum = r.d;
    return MO_RC_SUCCESS;
}

template <typename T, int KIND>
int run_minmax(ThreadCtx &t, const void *dcol, const uint64_t *dnulls, uint64_t n, uint64_t *bits, uint64_t *cnt) {
    Rec r;
    int rc = launch_agg<T, KIND>(t, dcol, dnulls, n, &r);
    if (rc) return rc;
    *cnt = r.cnt; *bits = r.w0;
    return MO_RC_SUCCESS;
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

// ---- device-resident results (the asynchronous form) ----------------------------------------------------------------------------
// When the column AND the result vector live in device memory the call only enqueues work on the calling thread's stream: no host
// read-back, no synchronisation.  A 1-thread kernel turns the aggregate record into the caller's result words.  This is what lets a
// multi-GPU caller hand the partial state straight to NCCL (MergeGroup seam, mergeGroup.go:132-247) and merge on the device.
__global__ void agg_state_kernel(const Rec *rec, int op, int cls, uint64_t len, const unsigned long long *nullcount, const Seg *segs, uint64_t nseg,
                                 uint64_t *res, uint64_t res_words, uint64_t *rnulls) {
    uint64_t bits = 0, cnt = 0; int64_t rc = MO_RC_SUCCESS; bool isnull = false;
    // signed SUM whose magnitudes do not fit int64: fold the serial-order segment summaries (prefix_seg_kernel ran behind the same gate)
    int32_t ov = 0;
    if (cls == C_SIGNED && segs && prefix_check_needed(rec)) {
        __int128 run = 0;
        const __int128 hi = (__int128)INT64_MAX, lo = (__int128)INT64_MIN;
        for (uint64_t s = 0; s < nseg; s++) {
            if (run + segs[s].maxp > hi || run + segs[s].minp < lo) { ov = 1; break; }
            run += segs[s].total;
        }
    }
    const int32_t *ovflag = &ov;
    if (cls == C_COUNT) { cnt = len - (nullcount ? *nullcount : 0ull); bits = cnt; }
    else {
        cnt = rec->cnt; isnull = cnt == 0;
        double dsum = 0.0;
        if (cls == C_SIGNED) {
            bits = rec->w0; dsum = (double)(int64_t)rec->w0;
            if (sum_check_needed(*rec) && ovflag && *ovflag) rc = MO_RC_OUT_OF_RANGE;
        } else if (cls == C_UNSIGNED) { bits = rec->w0; dsum = (double)rec->w0; if (rec->w1) rc = MO_RC_OUT_OF_RANGE; }
        else if (cls == C_FLOAT) { dsum = rec->d; memcpy(&bits, &dsum, 8); }
        else bits = rec->w0;
        // a 1-word result of AVG is the final value; a 3-word result is the partial STATE (sum in the SUM return type, count, rc) and AVG divides at the merge
        if (op == MO_AGG_AVG && res_words < 3 && !isnull) { double avg = dsum / (double)cnt; memcpy(&bits, &avg, 8); }
    }
    res[0] = bits;
    if (res_words >= 2) res[1] = cnt;
    if (res_words >= 3) res[2] = (uint64_t)rc;
    if (rnulls) rnulls[0] = isnull ? 1ull : 0ull;
}

template <typename T>
static int agg_async_typed(ThreadCtx &t, int op, int cls, const void *dcol, const uint64_t *dnulls, uint64_t n, Rec **drec, AggStateOut so) {
    // ONE launch: the last CTA of the aggregate kernel writes the caller's result / state (and, for a signed SUM whose magnitudes do not fit
    // int64, runs the exact serial-order check itself)
    if (op == MO_AGG_MIN) return launch_agg<T, K_MIN>(t, dcol, dnulls, n, nullptr, drec, so);
    if (op == MO_AGG_MAX) return launch_agg<T, K_MAX>(t, dcol, dnulls, n, nullptr, drec, so);
    if (cls == C_FLOAT) return launch_agg<T, K_SUM_FLOAT>(t, dcol, dnulls, n, nullptr, drec, so);
    if (cls == C_UNSIGNED) return launch_agg<T, K_SUM_UNSIGNED>(t, dcol, dnulls, n, nullptr, drec, so);
    return launch_agg<T, K_SUM_SIGNED>(t, dcol, dnulls, n, nullptr, drec, so);
}

static int xcall_agg_async(ThreadCtx &t, int op, int T, mo_xcall_args_t *args, uint64_t len) {
    const void *dcol = args[1].pdata;
    const uint64_t *dnulls = args[1].pnulls;
    const bool is_signed = T >= MO_T_INT8 && T <= MO_T_INT64, is_unsigned = T >= MO_T_UINT8 && T <= MO_T_UINT64;
    const bool is_float = T == MO_T_FLOAT32 || T == MO_T_FLOAT64;
    Rec *drec = nullptr; unsigned long long *dcount = nullptr;
    bool state_written = false;
    int cls, rc = MO_RC_SUCCESS;
    Rec *zero = (Rec *)arena_alloc(t, sizeof(Rec));
    if (!zero) return MO_RC_INTERNAL_ERROR;
    if (op == MO_AGG_COUNT) {
        cls = C_COUNT;
        if (dnulls && len) {
            dcount = (unsigned long long *)arena_alloc(t, 8);
            if (!dcount) return MO_RC_INTERNAL_ERROR;
            MOB_CUDA_TRY(cudaMemsetAsync(dcount, 0, 8, t.stream));
            uint64_t nw = (len + 63) >> 6;
            int grid = (int)((nw + 255) / 256);
            if (grid > num_sms() * 8) grid = num_sms() * 8;
            popcount_kernel<<<grid, 256, 0, t.stream>>>(dnulls, len, dcount);
            MOB_LAUNCH_CHECK();
        }
    } else if (op == MO_AGG_MIN || op == MO_AGG_MAX || op == MO_AGG_SUM || op == MO_AGG_AVG) {
        const bool mm = op == MO_AGG_MIN || op == MO_AGG_MAX;
        cls = mm ? C_MINMAX : is_signed ? C_SIGNED : is_unsigned ? C_UNSIGNED : C_FLOAT;
        if (!mm && !is_signed && !is_unsigned && !is_float) { set_error("sum: unsupported type %d", T); return MO_RC_INVALID_ARGUMENT; }
        const AggStateOut so{(uint64_t *)args[0].pdata, args[0].dataSz / 8, args[0].pnulls, op, cls};
        state_written = len != 0;
        if (len == 0) { MOB_CUDA_TRY(cudaMemsetAsync(zero, 0, sizeof(Rec), t.stream)); drec = zero; }
        else switch (T) {
        case MO_T_BOOL: case MO_T_UINT8: rc = agg_async_typed<uint8_t>(t, op, cls, dcol, dnulls, len, &drec, so); break;
        case MO_T_INT8: rc = agg_async_typed<int8_t>(t, op, cls, dcol, dnulls, len, &drec, so); break;
        case MO_T_INT16: rc = agg_async_typed<int16_t>(t, op, cls, dcol, dnulls, len, &drec, so); break;
        case MO_T_UINT16: rc = agg_async_typed<uint16_t>(t, op, cls, dcol, dnulls, len, &drec, so); break;
        case MO_T_INT32: case MO_T_DATE: rc = agg_async_typed<int32_t>(t, op, cls, dcol, dnulls, len, &drec, so); break;
        case MO_T_UINT32: rc = agg_async_typed<uint32_t>(t, op, cls, dcol, dnulls, len, &drec, so); break;
        case MO_T_INT64: case MO_T_TIME: case MO_T_DATETIME: case MO_T_TIMESTAMP: rc = agg_async_typed<int64_t>(t, op, cls, dcol, dnulls, len, &drec, so); break;
        case MO_T_UINT64: rc = agg_async_typed<uint64_t>(t, op, cls, dcol, dnulls, len, &drec, so); break;
        case MO_T_FLOAT32: rc = agg_async_typed<float>(t, op, cls, dcol, dnulls, len, &drec, so); break;
        case MO_T_FLOAT64: rc = agg_async_typed<double>(t, op, cls, dcol, dnulls, len, &drec, so); break;
        default: set_error("agg: unsupported type %d", T); return MO_RC_INVALID_ARGUMENT;
        }
        if (rc) return rc;
    } else { set_error("agg: unknown op %d", op); return MO_RC_INVALID_ARGUMENT; }
    if (!state_written) {   // COUNT, or an empty column
        agg_state_kernel<<<1, 1, 0, t.stream>>>(drec, op, cls, len, dcount, nullptr, 0, (uint64_t *)args[0].pdata, args[0].dataSz / 8, args[0].pnulls);
        MOB_LAUNCH_CHECK();
    }
    arena_reset(t);   // stream order protects the scratch: the next call's kernels queue behind these
    return MO_RC_SUCCESS;
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
    const bool async = is_device_ptr(args[0].pdata) && (len == 0 || is_device_ptr(args[1].pdata));
    Stager st(t);
    const uint64_t *dparts = (const uint64_t *)st.in(args[1].pdata, 24 * len);
    uint64_t *dres = (uint64_t *)st.out(args[0].pdata, args[0].dataSz >= 24 ? 24 : args[0].dataSz >= 16 ? 16 : 8);
    uint64_t *dn = (uint64_t *)st.out(args[0].pnulls, args[0].pnulls ? 8 : 0);
    if (st.failed) { st.finish(); return MO_RC_INTERNAL_ERROR; }
    int64_t *drc = async ? nullptr : (int64_t *)st.tmp(8);
    if (st.failed) { st.finish(); return MO_RC_INTERNAL_ERROR; }
    agg_merge_kernel<<<1, 1, 0, t.stream>>>(dparts, len, op, T, cls, dres, args[0].dataSz / 8, dn, drc);
    MOB_LAUNCH_CHECK();
    if (async) { st.release_async(); return MO_RC_SUCCESS; }   // the merged state's rc word carries errors
    int rc = MO_RC_SUCCESS;
    int64_t hrc = 0;
    int r2 = read_back(t, &hrc, drc, 8);
    if (r2) rc = r2; else if (hrc) { rc = (int)hrc; set_error("data out of range: merged SUM overflows its 64-bit state"); }
    int frc = st.finish();
    return rc ? rc : frc;
}

int bitmap_count_device(ThreadCtx &t, const uint64_t *dp, uint64_t nbits, uint64_t *count) {
    if (nbits == 0 || !dp) { *count = 0; return MO_RC_SUCCESS; }
    unsigned long long *dout = (unsigned long long *)arena_alloc(t, 8);
    if (!dout) return MO_RC_INTERNAL_ERROR;
    MOB_CUDA_TRY(cudaMemsetAsync(dout, 0, 8, t.stream));
    uint64_t nw = (nbits + 63) >> 6;
    int grid = (int)((nw + 255) / 256);
    if (grid > num_sms() * 8) grid = num_sms() * 8;
    popcount_kernel<<<grid, 256, 0, t.stream>>>(dp, nbits, dout);
    MOB_LAUNCH_CHECK();
    return read_back(t, count, dout, 8);
}

// XCall family MO_XCALL_AGG(op, T): args[0] = result, args[1] = column.  See include/mo_b200.h.
int xcall_agg(int op, int T, mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    const int sz = type_size(T);
    if (!sz || T == MO_T_BOOL && op != MO_AGG_COUNT && op != MO_AGG_MIN && op != MO_AGG_MAX) { set_error("agg: unsupported type %d", T); return MO_RC_INVALID_ARGUMENT; }
    if (!args[0].pdata || args[0].dataSz < 8) { set_error("agg: result vector must hold 8 bytes"); return MO_RC_INVALID_ARGUMENT; }
    if (args[1].dataSz < (uint64_t)sz * len) { set_error("agg: column shorter than len"); return MO_RC_INVALID_ARGUMENT; }
    if (is_device_ptr(args[0].pdata) && (len == 0 || is_device_ptr(args[1].pdata)) && (!args[0].pnulls || is_device_ptr(args[0].pnulls)) &&
        (!args[1].pnulls || is_device_ptr(args[1].pnulls)))
        return xcall_agg_async(t, op, T, args, len);
    Stager st(t);
    const void *dcol = st.in(args[1].pdata, (size_t)sz * len);
    const uint64_t *dnulls = (const uint64_t *)st.in(args[1].pnulls, args[1].pnulls ? ((len + 63) / 64) * 8 : 0);
    if (st.failed) { st.finish(); return MO_RC_INTERNAL_ERROR; }

    uint64_t bits = 0, cnt = 0; int rc = MO_RC_SUCCESS; bool isnull = false;
    const bool is_signed = T >= MO_T_INT8 && T <= MO_T_INT64, is_unsigned = T >= MO_T_UINT8 && T <= MO_T_UINT64;
    const bool is_float = T == MO_T_FLOAT32 || T == MO_T_FLOAT64;
    if (len == 0) { isnull = (op != MO_AGG_COUNT); }
    else if (op == MO_AGG_COUNT) {
        uint64_t nn = 0;
        rc = bitmap_count_device(t, dnulls, dnulls ? len : 0, &nn);
        bits = len - nn;
    } else if (op == MO_AGG_SUM || op == MO_AGG_AVG) {
        double dsum = 0; int64_t isum = 0; uint64_t usum = 0;
        if (is_signed) {
            switch (sz) {
            case 1: rc = run_sum_signed<int8_t>(t, dcol, dnulls, len, &isum, &cnt); break;
            case 2: rc = run_sum_signed<int16_t>(t, dcol, dnulls, len, &isum, &cnt); break;
            case 4: rc = run_sum_signed<int32_t>(t, dcol, dnulls, len, &isum, &cnt); break;
            default: rc = run_sum_signed<int64_t>(t, dcol, dnulls, len, &isum, &cnt); break;
            }
            memcpy(&bits, &isum, 8); dsum = (double)isum;
        } else if (is_unsigned) {
            switch (sz) {
            case 1: rc = run_sum_unsigned<uint8_t>(t, dcol, dnulls, len, &usum, &cnt); break;
            case 2: rc = run_sum_unsigned<uint16_t>(t, dcol, dnulls, len, &usum, &cnt); break;
            case 4: rc = run_sum_unsigned<uint32_t>(t, dcol, dnulls, len, &usum, &cnt); break;
            default: rc = run_sum_unsigned<uint64_t>(t, dcol, dnulls, len, &usum, &cnt); break;
            }
            bits = usum; dsum = (double)usum;
        } else if (is_float) {
            if (sz == 4) rc = run_sum_float<float>(t, dcol, dnulls, len, &dsum, &cnt);
            else rc = run_sum_float<double>(t, dcol, dnulls, len, &dsum, &cnt);
            memcpy(&bits, &dsum, 8);
        } else { set_error("sum: unsupported type %d", T); rc = MO_RC_INVALID_ARGUMENT; }
        isnull = cnt == 0;
        if (op == MO_AGG_AVG && args[0].dataSz >= 24) { /* partial STATE: the raw sum, the merge divides */ }
        else if (op == MO_AGG_AVG && !isnull) { double avg = dsum / (double)cnt; memcpy(&bits, &avg, 8); }  // sumavg2.go:331
    } else if (op == MO_AGG_MIN || op == MO_AGG_MAX) {
#define MM(TT) (op == MO_AGG_MIN ? run_minmax<TT, K_MIN>(t, dcol, dnulls, len, &bits, &cnt) : run_minmax<TT, K_MAX>(t, dcol, dnulls, len, &bits, &cnt))
        switch (T) {
        case MO_T_BOOL: case MO_T_UINT8: rc = MM(uint8_t); break;
        case MO_T_INT8: rc = MM(int8_t); break;
        case MO_T_INT16: rc = MM(int16_t); break;
        case MO_T_UINT16: rc = MM(uint16_t); break;
        case MO_T_INT32: case MO_T_DATE: rc = MM(int32_t); break;
        case MO_T_UINT32: rc = MM(uint32_t); break;
        case MO_T_INT64: case MO_T_TIME: case MO_T_DATETIME: case MO_T_TIMESTAMP: rc = MM(int64_t); break;
        case MO_T_UINT64: rc = MM(uint64_t); break;
        case MO_T_FLOAT32: rc = MM(float); break;
        case MO_T_FLOAT64: rc = MM(double); break;
        default: rc = MO_RC_INVALID_ARGUMENT;
        }
#undef MM
        isnull = cnt == 0;
    } else { set_error("agg: unknown op %d", op); rc = MO_RC_INVALID_ARGUMENT; }

    // write the result (host memory directly; device memory through the stream)
    if (rc == MO_RC_SUCCESS || rc == MO_RC_OUT_OF_RANGE) {
        uint64_t nullword = isnull ? 1ull : 0ull;
        if (op == MO_AGG_COUNT) cnt = bits;
        uint64_t words[3] = {bits, cnt, (uint64_t)(int64_t)rc};
        const size_t wb = args[0].dataSz >= 24 ? 24 : args[0].dataSz >= 16 ? 16 : 8;   // 8: value; 16: + non-null rows; 24: + rc (partial state)
        if (is_device_ptr(args[0].pdata)) cudaMemcpyAsync(args[0].pdata, words, wb, cudaMemcpyHostToDevice, t.stream);
        else memcpy(args[0].pdata, words, wb);
        if (args[0].pnulls) {
            if (is_device_ptr(args[0].pnulls)) cudaMemcpyAsync(args[0].pnulls, &nullword, 8, cudaMemcpyHostToDevice, t.stream);
            else memcpy(args[0].pnulls, &nullword, 8);
        }
    }
    int frc = st.finish();
    return rc ? rc : frc;
}

}  // namespace mob
