// tpch.cu -- fused scan -> filter -> project -> aggregate kernels for the two OLAP shapes BASELINE.json names.
//
// The reference runs these as an operator chain that materialises a vector per expression node and compacts every
// column after each conjunct (table_scan -> filter -> projection -> group: pkg/sql/colexec/filter/filter.go:87-153,
// pkg/sql/colexec/group/exec2.go:296-367, aggexec/sumavg2.go:133-199).  Here each shape is ONE pass over the
// columns, no byte is read twice, nothing is written but a few hundred bytes of partials.  Q1 reads every byte (~98 % of its
// rows pass).  Q6 reads shipdate whole and each later column only in the DRAM blocks where a row is still alive after the earlier
// conjuncts, like the reference's conjunct-by-conjunct filter: on TPC-H data 13 B/row at 64-byte blocks instead of 28 (DESIGN 5.1).
//
//   Q6  SUM(price*disc) WHERE date in [lo,hi) AND disc BETWEEN a AND b AND qty < c     28 B/row algorithmic (q6.sql:50-61)
//   Q1  filter date <= cutoff, group by (returnflag, linestatus), 8 aggregates          38 B/row packed keys,
//                                                                                        84 B/row varlena keys (q1.sql:1-21)
//
// Mapping: a "pair" is two consecutive rows.  Lane l of a warp owns pair (w*32 + l), so one warp instruction reads
// 64 consecutive rows: 256 B of the int32 column (LDG.64/lane) and 512 B of each float64 column (LDG.128/lane) --
// whole 32-byte sectors, nothing fetched twice.  kUnroll pairs are in flight per thread; grid = SMs x CTAs/SM
// persistent CTAs, grid-stride.  Products are rounded exactly as the reference's separate multiply / add nodes do
// (__dmul_rn/__dadd_rn, no FMA contraction), so only the summation ORDER differs from the serial Go loop.
// Reduction: registers -> warp shuffles -> shared memory -> per-CTA record; the last CTA (atomicInc ticket) folds
// the records in CTA-index order => bitwise run-to-run deterministic for a fixed grid.
//
// Q1 has one kernel per input class, chosen from the input (launch_q1):
//   q1_tma_kernel<4>  packed keys, shipdate and key columns 16-byte aligned, n >= 64 tiles of 1024 rows: one producer warp per
//                     CTA streams whole tiles into shared memory with cp.async.bulk, 16 consumer warps reduce them
//   q1_kernel<4>      everything else (varlena keys, unaligned columns, fewer rows): the pair mapping above, loads into registers
// A pass keeps at most 4 groups per CTA; when it sees more it reports overflow and q1_kernel<8> runs the input again.
#include "common.cuh"
#include <algorithm>
#include <cstring>
#include <atomic>

using namespace mob;

namespace {

constexpr int kThreads = 256;

// =========================================================================================================
// Q6
// =========================================================================================================
typedef unsigned __int128 u128;

// device result (the caller's, or staged for a host result): sum at res[0], qualifying rows at res[1] when res_words >= 2, nulls word
// bit 0 = "no row qualified" -- the layout MO_XCALL_Q6_MERGE consumes
struct Q6DevOut { double *res; uint64_t res_words; uint64_t *rnulls; };

// Value domains of the Q6 scan.  The pair mapping, the conjunct-order loads and the reduction below are shared; a domain supplies the
// column type, the SUM node over one row and the sum's reduction.
//   Q6F64  float64 columns: product and every addition rounded as the reference's separate nodes (__dmul_rn / __dadd_rn)
//   Q6Dec  Decimal64 columns of one scale s <= 4 (int64 unscaled): the exact d64Mul product (Decimal128 at scale 2s, never rounded) summed
//          modulo 2^128, and the OR of the product magnitudes, whose bit length bounds every running sum (q6_dec_rare)
struct Q6F64 {
    typedef double V; typedef double2 V2; typedef double Sum; typedef mo_q6_params_t Params;
    static __device__ __forceinline__ V2 load2_if(bool p, const V *a) { return ld_stream16_f64_if(p, a); }
    static __device__ __forceinline__ Sum zero() { return 0.0; }
    static __device__ __forceinline__ Sum plus(Sum a, Sum b) { return __dadd_rn(a, b); }
    static __device__ __forceinline__ Sum warp_sum(Sum s) { return warp_sum_f64(s); }
    // s starts at +0.0 and can never become -0.0 under round-to-nearest, so s + 0.0 == s
    static __device__ __forceinline__ void add(bool ok, V di, V pr, Sum &s) {
        double prod = __dmul_rn(pr, di);         // projection node l_extendedprice * l_discount
        s = __dadd_rn(s, ok ? prod : 0.0);       // SUM node
    }
    static __device__ __forceinline__ Sum &odd(Sum &, Sum &s1) { return s1; }
    static __device__ __forceinline__ void write(Q6DevOut o, Sum f, unsigned long long fc) {
        if (!o.res) return;
        o.res[0] = f;
        if (o.res_words >= 2) reinterpret_cast<long long *>(o.res)[1] = (long long)fc;
        if (o.rnulls) o.rnulls[0] = fc ? 0ull : 1ull;
    }
};
// mag: OR over the rows of (high word of |product|) | (low word != 0), so |product| < 2^(64 + bit length of mag) -- a bound on every
// product that costs one 64-bit register
struct DecSum { u128 s; uint64_t mag; };
struct Q6Dec {
    typedef int64_t V; typedef longlong2 V2; typedef DecSum Sum; typedef mo_q6_dec_params_t Params;
    static __device__ __forceinline__ V2 load2_if(bool p, const V *a) { return ld_stream16_s64_if(p, a); }
    static __device__ __forceinline__ Sum zero() { return DecSum{0, 0}; }
    static __device__ __forceinline__ Sum plus(Sum a, Sum b) { return DecSum{a.s + b.s, a.mag | b.mag}; }
    static __device__ __forceinline__ Sum warp_sum(Sum v) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const uint64_t sl = __shfl_xor_sync(0xffffffffu, (uint64_t)v.s, o), sh = __shfl_xor_sync(0xffffffffu, (uint64_t)(v.s >> 64), o);
            v.s += ((u128)sh << 64) | sl;
            v.mag |= __shfl_xor_sync(0xffffffffu, v.mag, o);
        }
        return v;
    }
    // d64Mul (arith_decimal_fast.go): |pr| * |di| < 2^126, so the 128-bit product is exact; the sign is applied after
    static __device__ __forceinline__ void add(bool ok, V di, V pr, Sum &s) {
        const uint64_t ap = pr < 0 ? 0ull - (uint64_t)pr : (uint64_t)pr, ad = di < 0 ? 0ull - (uint64_t)di : (uint64_t)di;
        const uint64_t lo = ap * ad, hi = __umul64hi(ap, ad);
        const u128 m = ((u128)hi << 64) | lo;
        const u128 v = (pr < 0) != (di < 0) ? (u128)0 - m : m;
        s.s += ok ? v : (u128)0;
        s.mag |= ok ? (hi | (uint64_t)(lo != 0)) : 0ull;
    }
    static __device__ __forceinline__ void write(Q6DevOut, Sum, unsigned long long) {}   // q6_dec_fold_kernel writes the result
    // integer addition is associative: the odd rows share the even rows' accumulator (the float64 domain keeps two for its fixed order)
    static __device__ __forceinline__ Sum &odd(Sum &s0, Sum &) { return s0; }
};

template <class D> struct Q6Rec { typename D::Sum sum; unsigned long long cnt; };

// SUM node over one row: the projection l_extendedprice * l_discount is added where the row passed all three conjuncts, 0 elsewhere
template <class D>
__device__ __forceinline__ void q6_add(bool ok, typename D::V di, typename D::V pr, typename D::Sum &s, unsigned &cnt) {
    D::add(ok, di, pr, s);
    cnt += ok;
}
template <class D>
__device__ __forceinline__ void q6_row(const typename D::Params &P, int32_t d, typename D::V di, typename D::V q, typename D::V pr,
                                       typename D::Sum &s, unsigned &cnt) {
    q6_add<D>((d >= P.date_lo) & (d < P.date_hi) & (di >= P.disc_lo) & (di <= P.disc_hi) & (q < P.qty_hi), di, pr, s, cnt);
}

// deterministic reduction of the per-thread state: warp shuffles, shared memory, per-CTA record; the last CTA folds the records in
// CTA-index order
template <class D>
__device__ __forceinline__ void q6_finish(typename D::Sum s0, typename D::Sum s1, unsigned cnt, Q6Rec<D> *__restrict__ partials,
                                          Q6Rec<D> *__restrict__ out, unsigned *ticket, Q6DevOut dres) {
    typedef typename D::Sum Sum;
    Sum s = D::plus(s0, s1);
    unsigned long long c64 = cnt;
    s = D::warp_sum(s);
    c64 = warp_sum(c64);
    __shared__ Sum ss[kThreads / 32];
    __shared__ unsigned long long sc[kThreads / 32];
    __shared__ bool last;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { ss[warp] = s; sc[warp] = c64; }
    __syncthreads();
    if (threadIdx.x == 0) {
        Sum t = D::zero(); unsigned long long tc = 0;
#pragma unroll
        for (int w = 0; w < kThreads / 32; w++) { t = D::plus(t, ss[w]); tc += sc[w]; }
        partials[blockIdx.x].sum = t; partials[blockIdx.x].cnt = tc;
        __threadfence();
        unsigned tk = atomicInc(ticket, gridDim.x - 1);
        last = (tk == gridDim.x - 1);
    }
    __syncthreads();
    if (last) {
        __threadfence();
        Sum t = D::zero(); unsigned long long tc = 0;
        for (unsigned bIdx = threadIdx.x; bIdx < gridDim.x; bIdx += kThreads) { t = D::plus(t, partials[bIdx].sum); tc += partials[bIdx].cnt; }
        t = D::warp_sum(t); tc = warp_sum(tc);
        __syncthreads();
        if (lane == 0) { ss[warp] = t; sc[warp] = tc; }
        __syncthreads();
        if (threadIdx.x == 0) {
            Sum f = D::zero(); unsigned long long fc = 0;
#pragma unroll
            for (int w = 0; w < kThreads / 32; w++) { f = D::plus(f, ss[w]); fc += sc[w]; }
            out->sum = f; out->cnt = fc;
            D::write(dres, f, fc);
        }
    }
}

// Dense scan: all four columns of every pair.  Selected by q6_variant = 1: the arm the selective kernel is timed and tested against.
template <class D, int UNROLL, int CTAS>
__global__ void __launch_bounds__(kThreads, CTAS)
q6_kernel(const int32_t *__restrict__ sd, const typename D::V *__restrict__ disc, const typename D::V *__restrict__ qty,
          const typename D::V *__restrict__ price, uint64_t n, typename D::Params P, Q6Rec<D> *__restrict__ partials,
          Q6Rec<D> *__restrict__ out, unsigned *ticket, Q6DevOut dres) {
    typedef typename D::V V;
    const uint64_t npairs = n >> 1;
    const uint64_t tid = blockIdx.x * (uint64_t)kThreads + threadIdx.x;
    const uint64_t nthreads = (uint64_t)gridDim.x * kThreads;
    typename D::Sum s0 = D::zero(), s1 = D::zero();
    unsigned cnt = 0;  // a thread sees < 2^32 rows

    uint64_t p = tid;
    for (; p + (UNROLL - 1) * nthreads < npairs; p += UNROLL * nthreads) {
        int2 d[UNROLL]; int4 a[UNROLL], b[UNROLL], c[UNROLL];
#pragma unroll
        for (int k = 0; k < UNROLL; k++) {
            const uint64_t q = p + k * nthreads;
            d[k] = ld_stream8(sd + 2 * q);
            a[k] = ld_stream16(disc + 2 * q);
            b[k] = ld_stream16(qty + 2 * q);
            c[k] = ld_stream16(price + 2 * q);
        }
#pragma unroll
        for (int k = 0; k < UNROLL; k++) {
            V di[2], qq[2], pr[2];
            memcpy(di, &a[k], 16); memcpy(qq, &b[k], 16); memcpy(pr, &c[k], 16);
            q6_row<D>(P, d[k].x, di[0], qq[0], pr[0], s0, cnt);
            q6_row<D>(P, d[k].y, di[1], qq[1], pr[1], D::odd(s0, s1), cnt);
        }
    }
    for (; p < npairs; p += nthreads) {
        int2 d = ld_stream8(sd + 2 * p);
        int4 a = ld_stream16(disc + 2 * p), b = ld_stream16(qty + 2 * p), c = ld_stream16(price + 2 * p);
        V di[2], qq[2], pr[2];
        memcpy(di, &a, 16); memcpy(qq, &b, 16); memcpy(pr, &c, 16);
        q6_row<D>(P, d.x, di[0], qq[0], pr[0], s0, cnt);
        q6_row<D>(P, d.y, di[1], qq[1], pr[1], D::odd(s0, s1), cnt);
    }
    if ((n & 1) && tid == 0) q6_row<D>(P, sd[n - 1], disc[n - 1], qty[n - 1], price[n - 1], s0, cnt);  // odd tail row
    q6_finish<D>(s0, s1, cnt, partials, out, ticket, dres);
}

// Selective scan (the default): the columns are read in dependent rounds, in the reference's conjunct order (filter.go:87-153).
// shipdate is read for every pair; a lane then reads its 16 B of discount only if a row of its pair is inside the date range, its
// quantity only if a row also passed the discount test, and its price only if a row passed all three.  DRAM moves a block only if
// one of its rows is still alive (DESIGN 5.1 has the byte model).  The next batch's shipdate is in flight while the current batch's
// rounds run, so a batch costs three round trips.  Merging the quantity and price rounds measured slower for Q6: it reads more.
// Same grid, pair -> thread mapping, per-thread order and s0 / s1 split as q6_kernel, and a row whose columns were not read adds +0.0
// exactly as a failing row does there: the result is bit-identical to the dense kernel's.
template <class D, int UNROLL>
__global__ void __launch_bounds__(kThreads, 4)
q6_selective_kernel(const int32_t *__restrict__ sd, const typename D::V *__restrict__ disc, const typename D::V *__restrict__ qty,
                    const typename D::V *__restrict__ price, uint64_t n, typename D::Params P, Q6Rec<D> *__restrict__ partials,
                    Q6Rec<D> *__restrict__ out, unsigned *ticket, Q6DevOut dres) {
    typedef typename D::V V;
    const uint64_t npairs = n >> 1;
    const uint64_t tid = blockIdx.x * (uint64_t)kThreads + threadIdx.x;
    const uint64_t nthreads = (uint64_t)gridDim.x * kThreads;
    const int lane = threadIdx.x & 31;
    typename D::Sum s0 = D::zero(), s1 = D::zero();
    unsigned cnt = 0;  // a thread sees < 2^32 rows

    // The batched loop runs while the warp's LAST lane has a whole batch, so its trip count is warp-uniform; what is left goes to the
    // per-thread loop below, and every thread still visits its pairs in ascending order.
    const uint64_t span = (uint64_t)(31 - lane) + (UNROLL - 1) * nthreads;
    uint64_t p = tid;
    bool more = p + span < npairs;
    int2 dn[UNROLL];
    if (more) {
#pragma unroll
        for (int k = 0; k < UNROLL; k++) dn[k] = ld_stream8(sd + 2 * (p + k * nthreads));
    }
    while (more) {
        int2 d[UNROLL];
#pragma unroll
        for (int k = 0; k < UNROLL; k++) d[k] = dn[k];
        const uint64_t pn = p + UNROLL * nthreads;
        more = pn + span < npairs;
        if (more) {
#pragma unroll
            for (int k = 0; k < UNROLL; k++) dn[k] = ld_stream8(sd + 2 * (pn + k * nthreads));
        }
        bool m0[UNROLL], m1[UNROLL];   // row still alive
        typename D::V2 a[UNROLL], b[UNROLL], c[UNROLL];
#pragma unroll
        for (int k = 0; k < UNROLL; k++) {
            m0[k] = (d[k].x >= P.date_lo) & (d[k].x < P.date_hi);
            m1[k] = (d[k].y >= P.date_lo) & (d[k].y < P.date_hi);
            a[k] = D::load2_if(m0[k] | m1[k], disc + 2 * (p + k * nthreads));
        }
#pragma unroll
        for (int k = 0; k < UNROLL; k++) {
            m0[k] = m0[k] & (a[k].x >= P.disc_lo) & (a[k].x <= P.disc_hi);
            m1[k] = m1[k] & (a[k].y >= P.disc_lo) & (a[k].y <= P.disc_hi);
            b[k] = D::load2_if(m0[k] | m1[k], qty + 2 * (p + k * nthreads));
        }
#pragma unroll
        for (int k = 0; k < UNROLL; k++) {
            m0[k] = m0[k] & (b[k].x < P.qty_hi);
            m1[k] = m1[k] & (b[k].y < P.qty_hi);
            c[k] = D::load2_if(m0[k] | m1[k], price + 2 * (p + k * nthreads));
        }
#pragma unroll
        for (int k = 0; k < UNROLL; k++) {   // a dead row's unread columns are 0; it adds 0 like any failing row
            q6_add<D>(m0[k], a[k].x, c[k].x, s0, cnt);
            q6_add<D>(m1[k], a[k].y, c[k].y, D::odd(s0, s1), cnt);
        }
        p = pn;
    }
    for (; p < npairs; p += nthreads) {
        int2 d = ld_stream8(sd + 2 * p);
        int4 a = ld_stream16(disc + 2 * p), b = ld_stream16(qty + 2 * p), c = ld_stream16(price + 2 * p);
        V di[2], qq[2], pr[2];
        memcpy(di, &a, 16); memcpy(qq, &b, 16); memcpy(pr, &c, 16);
        q6_row<D>(P, d.x, di[0], qq[0], pr[0], s0, cnt);
        q6_row<D>(P, d.y, di[1], qq[1], pr[1], D::odd(s0, s1), cnt);
    }
    if ((n & 1) && tid == 0) q6_row<D>(P, sd[n - 1], disc[n - 1], qty[n - 1], price[n - 1], s0, cnt);  // odd tail row
    q6_finish<D>(s0, s1, cnt, partials, out, ticket, dres);
}

// =========================================================================================================
// Q1
// =========================================================================================================
constexpr int kQ1Vals = 5;  // sum_qty, sum_price, sum_disc_price, sum_charge, sum_disc
struct Q1Slot { unsigned long long first_row; unsigned long long cnt; double v[kQ1Vals]; unsigned key; unsigned used; };
struct Q1Rec { Q1Slot slot[MO_Q1_MAX_GROUPS]; unsigned overflow; unsigned pad; };
constexpr unsigned kEmptyKey = 0xffffffffu;
constexpr int kQ1MaxGrid = 1024;  // upper bound on the grid (the last-CTA fold keeps a [grid][8] byte map in shared memory)

// Shared state of one CTA: key -> slot dictionary (slots handed out first-come) + overflow flag
struct Q1Shared {
    unsigned dict[MO_Q1_MAX_GROUPS];
    unsigned overflow;
};

// Per-thread aggregation state (registers).  Control flow of every method is WARP-UNIFORM: all 32 lanes call row() together
// and the dictionary slow path is taken by the whole warp (ballot + one elected lane doing the CAS).  A first version let
// lanes diverge inside the insert loop; some warps then never reconverged and ran ~8x slower to the end of the kernel.
template <int G>
struct Q1Thread {
    double acc[G][kQ1Vals];
    unsigned cnt[G];
    unsigned long long first[G];
    unsigned dk[G];  // register copy of the dictionary
    Q1Shared *S;
    int32_t cutoff;
    int lane;

    __device__ __forceinline__ void init(Q1Shared *s, int32_t cut) {
        S = s; cutoff = cut; lane = threadIdx.x & 31;
#pragma unroll
        for (int g = 0; g < G; g++) {
            cnt[g] = 0; first[g] = ~0ull; dk[g] = kEmptyKey;
#pragma unroll
            for (int j = 0; j < kQ1Vals; j++) acc[g][j] = 0.0;
        }
    }

    __device__ __forceinline__ int find_slot(unsigned key, bool valid) {
        int slot = -1;
#pragma unroll
        for (int g = 0; g < G; g++) if (dk[g] == key) slot = g;
        bool settled = !valid || slot >= 0;   // a lane is settled once its key has been looked up in the shared dictionary
        unsigned miss = __ballot_sync(0xffffffffu, !settled);
        while (miss) {
            const int leader = __ffs(miss) - 1;
            const unsigned lkey = __shfl_sync(0xffffffffu, key, leader);
            // Claim or find lkey in the shared dictionary.  EVERY lane issues the same idempotent CAS sequence (same address,
            // same value): an elected-lane `if (lane == leader) { loop }` left the warp split in two groups for the rest of
            // the kernel (ncu: 16.0 active threads per instruction, profiles/r01_ncu_summary.md), doubling the issue cost.
            bool ok = false;
#pragma unroll
            for (int g = 0; g < G; g++) {
                const unsigned prev = ok ? lkey : atomicCAS(&S->dict[g], kEmptyKey, lkey);
                ok = ok || prev == kEmptyKey || prev == lkey;
            }
            if (!ok) S->overflow = 1;
            __syncwarp();
#pragma unroll
            for (int g = 0; g < G; g++) dk[g] = ((volatile unsigned *)S->dict)[g];
            slot = -1;
#pragma unroll
            for (int g = 0; g < G; g++) if (dk[g] == key) slot = g;
            if (key == lkey || slot >= 0) settled = true;   // lkey lanes are settled either way (slot found, or dictionary full)
            miss = __ballot_sync(0xffffffffu, !settled);
        }
        return slot;
    }

    // `inb` = the row exists; the shipdate filter is folded into `valid`.
    // Group dispatch without branches: acc[g][j] = fma(v_j, ind_g, acc[g][j]) with ind_g = 1.0 for the row's slot and 0.0 for the
    // others.  fma(v, 1.0, a) == RN(v + a) (bit-identical to the reference's add) and fma(v, 0.0, a) == a for finite v, so all 32
    // lanes stay active.  Rows holding Inf/NaN would poison the other groups through 0 * Inf, so a warp that sees one takes the
    // exact predicated path.
    __device__ __forceinline__ void row(uint64_t r, bool inb, int32_t d, double q, double pr, double di, double tx, unsigned key) {
        const bool valid = inb && d <= cutoff;        // l_shipdate <= cutoff
        const int slot = find_slot(key, valid);
        const double t1 = __dsub_rn(1.0, di);         // 1 - l_discount
        const double t2 = __dmul_rn(pr, t1);          // l_extendedprice * (1 - l_discount)
        const double t3 = __dadd_rn(1.0, tx);         // 1 + l_tax
        const double t4 = __dmul_rn(t2, t3);          // ... * (1 + l_tax)
        const bool finite = (fabs(t4) + fabs(q)) < INFINITY;   // false for any Inf/NaN among q, pr, di, tx (and on overflow)
        if (__any_sync(0xffffffffu, valid && !finite)) {
#pragma unroll
            for (int g = 0; g < G; g++) {   // selects, not branches: lanes must not diverge here either
                const bool m = valid && slot == g;
                acc[g][0] = m ? __dadd_rn(acc[g][0], q) : acc[g][0];
                acc[g][1] = m ? __dadd_rn(acc[g][1], pr) : acc[g][1];
                acc[g][2] = m ? __dadd_rn(acc[g][2], t2) : acc[g][2];
                acc[g][3] = m ? __dadd_rn(acc[g][3], t4) : acc[g][3];
                acc[g][4] = m ? __dadd_rn(acc[g][4], di) : acc[g][4];
                if (m && cnt[g] == 0) first[g] = r;
                cnt[g] += m;
            }
            return;
        }
#pragma unroll
        for (int g = 0; g < G; g++) {
            const bool m = valid && slot == g;
            const double ind = __hiloint2double(m ? 0x3ff00000 : 0, 0);   // 1.0 or 0.0
            acc[g][0] = __fma_rn(q, ind, acc[g][0]);
            acc[g][1] = __fma_rn(pr, ind, acc[g][1]);
            acc[g][2] = __fma_rn(t2, ind, acc[g][2]);
            acc[g][3] = __fma_rn(t4, ind, acc[g][3]);
            acc[g][4] = __fma_rn(di, ind, acc[g][4]);
            if (m && cnt[g] == 0) first[g] = r;       // a thread visits its rows in increasing order
            cnt[g] += m;
        }
    }
};

// key of one row: packed uint8 columns (KEYMODE 0) or MatrixOne varlena cells (KEYMODE 1: 24 B, inline: bs[0]=len,
// bs[1..]=bytes; cgo/xcall.h:33-61); an empty string keys as 0
template <int KEYMODE>
__device__ __forceinline__ unsigned q1_key_scalar(const uint8_t *rf, const uint8_t *ls, uint64_t r) {
    if (KEYMODE == 0) return rf[r] | ((unsigned)ls[r] << 8);
    return (rf[24 * r] ? rf[24 * r + 1] : 0u) | ((ls[24 * r] ? (unsigned)ls[24 * r + 1] : 0u) << 8);
}

// CTA reduction + last-CTA fold, shared by both kernels.  kT = threads per CTA.
template <int G, int kT>
__device__ void q1_epilogue(Q1Thread<G> &T, Q1Shared &S, Q1Rec *__restrict__ partials, Q1Rec *__restrict__ out, unsigned *ticket) {
    __syncthreads();  // dictionary final
    // Register slots are indexed by the CTA dictionary, identical for every thread of the CTA.
    constexpr int kW = kT / 32;
    __shared__ double sv[kW][G][kQ1Vals];
    __shared__ unsigned long long scnt[kW][G], sfirst[kW][G];
    __shared__ bool last;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int g = 0; g < G; g++) {
        unsigned long long c64 = T.cnt[g], f = T.first[g];
        c64 = warp_sum(c64);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { unsigned long long of = __shfl_xor_sync(0xffffffffu, f, o); f = of < f ? of : f; }
#pragma unroll
        for (int j = 0; j < kQ1Vals; j++) {
            double v = warp_sum_f64(T.acc[g][j]);
            if (lane == 0) sv[warp][g][j] = v;
        }
        if (lane == 0) { scnt[warp][g] = c64; sfirst[warp][g] = f; }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        Q1Rec &R = partials[blockIdx.x];
        for (int g = 0; g < G; g++) {
            Q1Slot s; s.cnt = 0; s.first_row = ~0ull; s.key = S.dict[g]; s.used = S.dict[g] != kEmptyKey;
            for (int j = 0; j < kQ1Vals; j++) s.v[j] = 0.0;
            for (int w = 0; w < kW; w++) {
                s.cnt += scnt[w][g];
                if (sfirst[w][g] < s.first_row) s.first_row = sfirst[w][g];
                for (int j = 0; j < kQ1Vals; j++) s.v[j] = __dadd_rn(s.v[j], sv[w][g][j]);
            }
            R.slot[g] = s;
        }
        for (int g = G; g < MO_Q1_MAX_GROUPS; g++) { Q1Slot z; memset(&z, 0, sizeof z); z.key = kEmptyKey; R.slot[g] = z; }
        R.overflow = S.overflow; R.pad = 0;
        __threadfence();
        unsigned tk = atomicInc(ticket, gridDim.x - 1);
        last = (tk == gridDim.x - 1);
    }
    __syncthreads();
    if (last) {
        // Fold the CTA records (MergeGroup: re-hash partial keys + BatchMerge, mergeGroup.go:132-247) with the whole CTA:
        //  1. one thread per CTA record maps its local slots to final slots (shared dictionary, atomicCAS);
        //  2. one thread per (final slot, value) sums that value over the CTA records IN CTA-INDEX ORDER, so the result
        //     is bitwise deterministic although the dictionary slot order is not (the host sorts groups by first_row).
        __threadfence();
        __shared__ unsigned fdict[MO_Q1_MAX_GROUPS];
        __shared__ unsigned char inv[kQ1MaxGrid][MO_Q1_MAX_GROUPS];   // [cta][final slot] -> local slot or 0xff
        __shared__ unsigned f_overflow;
        if (threadIdx.x < MO_Q1_MAX_GROUPS) fdict[threadIdx.x] = kEmptyKey;
        if (threadIdx.x == 0) f_overflow = 0;
        for (unsigned i = threadIdx.x; i < gridDim.x * MO_Q1_MAX_GROUPS; i += kT) inv[i / MO_Q1_MAX_GROUPS][i % MO_Q1_MAX_GROUPS] = 0xff;
        __syncthreads();
        for (unsigned bIdx = threadIdx.x; bIdx < gridDim.x; bIdx += kT) {
            const Q1Rec &R = partials[bIdx];
            if (R.overflow) f_overflow = 1;
#pragma unroll
            for (int g = 0; g < G; g++) {
                if (!R.slot[g].used || R.slot[g].cnt == 0) continue;
                const unsigned key = R.slot[g].key;
                int dst = -1;
                for (int x = 0; x < MO_Q1_MAX_GROUPS; x++) {
                    const unsigned prev = atomicCAS(&fdict[x], kEmptyKey, key);
                    if (prev == kEmptyKey || prev == key) { dst = x; break; }
                }
                if (dst < 0) f_overflow = 1; else inv[bIdx][dst] = (unsigned char)g;
            }
        }
        __syncthreads();
        if (threadIdx.x < MO_Q1_MAX_GROUPS * 8) {
            const int sl = threadIdx.x >> 3, j = threadIdx.x & 7;
            Q1Slot &D = out->slot[sl];
            if (j < kQ1Vals) {
                double a = 0.0;
                for (unsigned bIdx = 0; bIdx < gridDim.x; bIdx++) { const unsigned g = inv[bIdx][sl]; if (g != 0xff) a = __dadd_rn(a, partials[bIdx].slot[g].v[j]); }
                D.v[j] = a;
            } else if (j == 5) {
                unsigned long long c = 0;
                for (unsigned bIdx = 0; bIdx < gridDim.x; bIdx++) { const unsigned g = inv[bIdx][sl]; if (g != 0xff) c += partials[bIdx].slot[g].cnt; }
                D.cnt = c;
            } else if (j == 6) {
                unsigned long long f = ~0ull;
                for (unsigned bIdx = 0; bIdx < gridDim.x; bIdx++) { const unsigned g = inv[bIdx][sl]; if (g != 0xff) { const unsigned long long r = partials[bIdx].slot[g].first_row; f = r < f ? r : f; } }
                D.first_row = f;
            } else {
                D.key = fdict[sl]; D.used = fdict[sl] != kEmptyKey;
                if (sl == 0) { out->overflow = f_overflow; out->pad = 0; }
            }
        }
        __syncthreads();
    }
}

// ---- register kernel: direct loads into registers (pairs of rows, UNROLL pairs in flight per thread) ---------------------
template <int G, int UNROLL, int CTAS, int KEYMODE>
__global__ void __launch_bounds__(kThreads, CTAS)
q1_kernel(const int32_t *__restrict__ sd, const double *__restrict__ qty, const double *__restrict__ price,
          const double *__restrict__ disc, const double *__restrict__ tax, const uint8_t *__restrict__ rf,
          const uint8_t *__restrict__ ls, uint64_t n, int32_t cutoff, Q1Rec *__restrict__ partials,
          Q1Rec *__restrict__ out, unsigned *ticket, const Q1Rec *gate) {
    // the 8-slot retry is enqueued behind the 4-slot pass and runs only if that pass overflowed its dictionary
    if (gate && !gate->overflow) return;
    __shared__ Q1Shared S;
    S.dict[threadIdx.x & (MO_Q1_MAX_GROUPS - 1)] = kEmptyKey;   // all threads write (same values): no lane-dependent branch
    S.overflow = 0;
    __syncthreads();
    Q1Thread<G> T;
    T.init(&S, cutoff);
    const int lane = threadIdx.x & 31;

    auto load_keys = [&](uint64_t pair, unsigned &k0, unsigned &k1) {
        if (KEYMODE == 0) {
            unsigned short a = __ldg(reinterpret_cast<const unsigned short *>(rf) + pair);
            unsigned short b = __ldg(reinterpret_cast<const unsigned short *>(ls) + pair);
            k0 = (a & 0xffu) | ((b & 0xffu) << 8);
            k1 = (a >> 8) | ((b >> 8) << 8);
        } else {
            const uint64_t r0 = 2 * pair;   // head 8 bytes of each 24-byte cell hold len + first chars
            uint2 a0 = __ldg(reinterpret_cast<const uint2 *>(rf + 24 * r0)), a1 = __ldg(reinterpret_cast<const uint2 *>(rf + 24 * (r0 + 1)));
            uint2 b0 = __ldg(reinterpret_cast<const uint2 *>(ls + 24 * r0)), b1 = __ldg(reinterpret_cast<const uint2 *>(ls + 24 * (r0 + 1)));
            auto ch = [](uint2 h) -> unsigned { return (h.x & 0xffu) ? ((h.x >> 8) & 0xffu) : 0u; };
            k0 = ch(a0) | (ch(b0) << 8);
            k1 = ch(a1) | (ch(b1) << 8);
        }
    };

    const uint64_t npairs = n >> 1;
    const uint64_t tid = blockIdx.x * (uint64_t)kThreads + threadIdx.x;
    const uint64_t nthreads = (uint64_t)gridDim.x * kThreads;
    const uint64_t wbase = tid - lane;   // first pair of this warp: loop bounds depend on it only => uniform per warp
    uint64_t pw = wbase;
    for (; pw + 31 + (UNROLL - 1) * nthreads < npairs; pw += UNROLL * nthreads) {   // all 32 lanes x UNROLL pairs in range
        int2 d[UNROLL]; int4 a[UNROLL], b[UNROLL], c[UNROLL], e[UNROLL]; unsigned k0[UNROLL], k1[UNROLL];
#pragma unroll
        for (int k = 0; k < UNROLL; k++) {
            const uint64_t q = pw + lane + k * nthreads;
            d[k] = ld_stream8(sd + 2 * q);
            a[k] = ld_stream16(qty + 2 * q);
            b[k] = ld_stream16(price + 2 * q);
            c[k] = ld_stream16(disc + 2 * q);
            e[k] = ld_stream16(tax + 2 * q);
            load_keys(q, k0[k], k1[k]);
        }
#pragma unroll
        for (int k = 0; k < UNROLL; k++) {
            const uint64_t q = pw + lane + k * nthreads;
            double qq[2], pr[2], di[2], tx[2];
            memcpy(qq, &a[k], 16); memcpy(pr, &b[k], 16); memcpy(di, &c[k], 16); memcpy(tx, &e[k], 16);
            T.row(2 * q, true, d[k].x, qq[0], pr[0], di[0], tx[0], k0[k]);
            T.row(2 * q + 1, true, d[k].y, qq[1], pr[1], di[1], tx[1], k1[k]);
        }
    }
    for (; pw < npairs; pw += nthreads) {   // ragged end: same code, lanes past the end carry inb = false
        const uint64_t q = pw + lane;
        const bool inb = q < npairs;
        int2 d = make_int2(0, 0); int4 a = make_int4(0, 0, 0, 0), b = a, c = a, e = a; unsigned k0 = 0, k1 = 0;
        if (inb) {
            d = ld_stream8(sd + 2 * q);
            a = ld_stream16(qty + 2 * q); b = ld_stream16(price + 2 * q); c = ld_stream16(disc + 2 * q); e = ld_stream16(tax + 2 * q);
            load_keys(q, k0, k1);
        }
        double qq[2], pr[2], di[2], tx[2];
        memcpy(qq, &a, 16); memcpy(pr, &b, 16); memcpy(di, &c, 16); memcpy(tx, &e, 16);
        T.row(2 * q, inb, d.x, qq[0], pr[0], di[0], tx[0], k0);
        T.row(2 * q + 1, inb, d.y, qq[1], pr[1], di[1], tx[1], k1);
    }
    if (tid < 32) {   // odd tail row: handled by warp 0 of CTA 0, lane 0 carries it
        const bool has = (n & 1) && lane == 0;
        const uint64_t r = n - 1;
        unsigned key = 0; int32_t dd = 0; double v0 = 0, v1 = 0, v2 = 0, v3 = 0;
        if (has) { key = q1_key_scalar<KEYMODE>(rf, ls, r); dd = sd[r]; v0 = qty[r]; v1 = price[r]; v2 = disc[r]; v3 = tax[r]; }
        T.row(r, has, dd, v0, v1, v2, v3, key);
    }
    q1_epilogue<G, kThreads>(T, S, partials, out, ticket);
}

// ---- TMA kernel: CTA-wide bulk-copy pipeline (packed keys) ---------------------------------------------------------------------------
// ONE producer warp streams 1024-row tiles -- 7 bulk copies of 1-8 KB per tile, 4 tiles (156 KB) in flight per SM -- and the 16 consumer
// warps share each tile: full[stage] (transaction count) / empty[stage] (one arrival per consumer warp) mbarriers, no CTA barrier in the
// steady state.  Two staged designs lost to it (DESIGN 5.1): per-lane 16-byte cp.async (LDGSTS) into per-warp rings is not merged into
// sector requests the way LDG.128 is, so every 32-byte sector crossed the L2 -> SM crossbar twice; per-warp rings filled with one
// cp.async.bulk per 64-row column slice fixed that but drowned the TMA unit in tiny copies (7 per 64 rows).
constexpr int kCtaTileRows = 1024, kCtaStages = 4, kCtaConsumers = 16;
constexpr int kCtaTileBytes = kCtaTileRows * 38;   // 4096 shipdate + 4 x 8192 + 2 x 1024
constexpr int kCtaThreads = (kCtaConsumers + 1) * 32;

__device__ __forceinline__ void q1_mbar_init(unsigned long long *bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(count));
}
__device__ __forceinline__ void q1_mbar_expect_tx(unsigned long long *bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void q1_mbar_wait(unsigned long long *bar, unsigned parity) {
    asm volatile(
        "{\n.reg .pred p;\nQ1_WAIT:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra Q1_DONE;\nbra Q1_WAIT;\nQ1_DONE:\n}"
        ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void q1_bulk_copy(void *smem, const void *gmem, unsigned bytes, unsigned long long *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"((unsigned)__cvta_generic_to_shared(smem)), "l"(gmem), "r"(bytes), "r"((unsigned)__cvta_generic_to_shared(bar)) : "memory");
}

__device__ __forceinline__ void q1_mbar_arrive(unsigned long long *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"((unsigned)__cvta_generic_to_shared(bar)) : "memory");
}

template <int G>
__global__ void __launch_bounds__(kCtaThreads, 1)
q1_tma_kernel(const int32_t *__restrict__ sd, const double *__restrict__ qty, const double *__restrict__ price,
              const double *__restrict__ disc, const double *__restrict__ tax, const uint8_t *__restrict__ rf,
              const uint8_t *__restrict__ ls, uint64_t n, int32_t cutoff, Q1Rec *__restrict__ partials,
              Q1Rec *__restrict__ out, unsigned *ticket) {
    extern __shared__ __align__(16) unsigned char ring[];   // [stage][kCtaTileBytes], then full[] and empty[] mbarriers
    __shared__ Q1Shared S;
    S.dict[threadIdx.x & (MO_Q1_MAX_GROUPS - 1)] = kEmptyKey;
    S.overflow = 0;
    unsigned long long *full = reinterpret_cast<unsigned long long *>(ring + (size_t)kCtaStages * kCtaTileBytes);
    unsigned long long *empty = full + kCtaStages;
    if (threadIdx.x == 0) {
#pragma unroll
        for (int s = 0; s < kCtaStages; s++) { q1_mbar_init(&full[s], 1); q1_mbar_init(&empty[s], kCtaConsumers); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    Q1Thread<G> T;
    T.init(&S, cutoff);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t ntiles = n / kCtaTileRows;
    // tiles of this CTA: blockIdx.x, blockIdx.x + gridDim.x, ...
    const uint64_t mine = ntiles > blockIdx.x ? (ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

    if (warp == kCtaConsumers) {
        // ---------------- producer warp: lane 0 issues, the others idle (they rejoin at the epilogue barrier)
        if (lane == 0) {
            for (uint64_t k = 0; k < mine; k++) {
                const int stage = (int)(k % kCtaStages);
                if (k >= kCtaStages) q1_mbar_wait(&empty[stage], (unsigned)(((k / kCtaStages) - 1) & 1));   // every consumer warp released the slot
                unsigned char *s = ring + (size_t)stage * kCtaTileBytes;
                const uint64_t r0 = (blockIdx.x + k * gridDim.x) * (uint64_t)kCtaTileRows;
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                q1_mbar_expect_tx(&full[stage], kCtaTileBytes);
                q1_bulk_copy(s, sd + r0, 4096, &full[stage]);
                q1_bulk_copy(s + 4096, qty + r0, 8192, &full[stage]);
                q1_bulk_copy(s + 12288, price + r0, 8192, &full[stage]);
                q1_bulk_copy(s + 20480, disc + r0, 8192, &full[stage]);
                q1_bulk_copy(s + 28672, tax + r0, 8192, &full[stage]);
                q1_bulk_copy(s + 36864, rf + r0, 1024, &full[stage]);
                q1_bulk_copy(s + 37888, ls + r0, 1024, &full[stage]);
            }
        }
    } else {
        // ---------------- consumer warps: thread t owns rows t and t + 512 of every tile
        for (uint64_t k = 0; k < mine; k++) {
            const int stage = (int)(k % kCtaStages);
            q1_mbar_wait(&full[stage], (unsigned)((k / kCtaStages) & 1));
            const unsigned char *s = ring + (size_t)stage * kCtaTileBytes;
            const uint64_t r0 = (blockIdx.x + k * gridDim.x) * (uint64_t)kCtaTileRows;
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int rl = threadIdx.x + 512 * h;
                const int32_t d = *reinterpret_cast<const int32_t *>(s + rl * 4);
                const double q = *reinterpret_cast<const double *>(s + 4096 + rl * 8);
                const double pr = *reinterpret_cast<const double *>(s + 12288 + rl * 8);
                const double di = *reinterpret_cast<const double *>(s + 20480 + rl * 8);
                const double tx = *reinterpret_cast<const double *>(s + 28672 + rl * 8);
                const unsigned key = (unsigned)s[36864 + rl] | ((unsigned)s[37888 + rl] << 8);
                T.row(r0 + rl, true, d, q, pr, di, tx, key);
            }
            __syncwarp();
            if (lane == 0) q1_mbar_arrive(&empty[stage]);
        }
        // rows past the last full tile (< 1024): warp 0 of CTA 0, direct loads
        if (blockIdx.x == 0 && warp == 0) {
            for (uint64_t r = ntiles * kCtaTileRows + lane; r - lane < n; r += 32) {
                const bool has = r < n;
                unsigned key = 0; int32_t dd = 0; double v0 = 0, v1 = 0, v2 = 0, v3 = 0;
                if (has) { key = q1_key_scalar<0>(rf, ls, r); dd = sd[r]; v0 = qty[r]; v1 = price[r]; v2 = disc[r]; v3 = tax[r]; }
                T.row(r, has, dd, v0, v1, v2, v3, key);
            }
        }
    }
    q1_epilogue<G, kCtaThreads>(T, S, partials, out, ticket);
}

__device__ void q1_finalize(const Q1Rec &F, mo_q1_result_t *res, int64_t row_base) {
    memset(res, 0, sizeof *res);
    int order[MO_Q1_MAX_GROUPS], ng = 0;
    for (int g = 0; g < MO_Q1_MAX_GROUPS; g++) if (F.slot[g].used && F.slot[g].cnt) order[ng++] = g;
    for (int i = 1; i < ng; i++)  // first-seen (row) order == the reference's group-id order
        for (int j = i; j > 0 && F.slot[order[j]].first_row < F.slot[order[j - 1]].first_row; j--) { int t = order[j]; order[j] = order[j - 1]; order[j - 1] = t; }
    res->ngroups = ng;
    for (int i = 0; i < ng; i++) {
        const Q1Slot &s = F.slot[order[i]];
        mo_q1_group_t &o = res->groups[i];
        o.returnflag = (uint8_t)(s.key & 0xff); o.linestatus = (uint8_t)((s.key >> 8) & 0xff);
        o.first_row = (int64_t)s.first_row + row_base;
        o.sum_qty = s.v[0]; o.sum_base_price = s.v[1]; o.sum_disc_price = s.v[2]; o.sum_charge = s.v[3]; o.sum_disc = s.v[4];
        o.count_order = (int64_t)s.cnt;
        const double c = (double)s.cnt;   // avg = float64(sum)/float64(cnt), sumavg2.go:331
        o.avg_qty = s.v[0] / c; o.avg_price = s.v[1] / c; o.avg_disc = s.v[4] / c;
    }
}

// pick the pass that did not overflow, order the groups, write the device result.  ngroups = -1 reports "more than MO_Q1_MAX_GROUPS
// distinct keys" (the synchronous form returns MO_RC_INVALID_ARGUMENT for that).
__global__ void q1_finalize_kernel(const Q1Rec *narrow, const Q1Rec *wide, mo_q1_result_t *res, int64_t row_base) {
    const Q1Rec *F = (narrow && !narrow->overflow) ? narrow : wide;
    if (!F || F->overflow) { memset(res, 0, sizeof *res); res->ngroups = -1; return; }
    q1_finalize(*F, res, row_base);
}

// MergeGroup on the device (mergeGroup.go:132-247): re-hash the partial group keys of `nparts` results and BatchMerge them IN ORDER
// (rank order => deterministic); groups come back in global first-seen row order.  One thread: <= 8 groups x nparts.
__global__ void q1_merge_kernel(const mo_q1_result_t *parts, uint64_t nparts, mo_q1_result_t *res) {
    mo_q1_result_t R; memset(&R, 0, sizeof R);
    bool bad = false;
    for (uint64_t p = 0; p < nparts && !bad; p++) {
        const mo_q1_result_t &P = parts[p];
        if (P.ngroups < 0 || P.ngroups > MO_Q1_MAX_GROUPS) { bad = true; break; }
        for (int64_t g = 0; g < P.ngroups; g++) {
            const mo_q1_group_t &s = P.groups[g];
            int dst = -1;
            for (int64_t x = 0; x < R.ngroups; x++) if (R.groups[x].returnflag == s.returnflag && R.groups[x].linestatus == s.linestatus) { dst = (int)x; break; }
            if (dst < 0) {
                if (R.ngroups == MO_Q1_MAX_GROUPS) { bad = true; break; }
                R.groups[R.ngroups++] = s;
                continue;
            }
            mo_q1_group_t &D = R.groups[dst];
            D.sum_qty = __dadd_rn(D.sum_qty, s.sum_qty); D.sum_base_price = __dadd_rn(D.sum_base_price, s.sum_base_price);
            D.sum_disc_price = __dadd_rn(D.sum_disc_price, s.sum_disc_price); D.sum_charge = __dadd_rn(D.sum_charge, s.sum_charge);
            D.sum_disc = __dadd_rn(D.sum_disc, s.sum_disc);
            D.count_order += s.count_order;
            if (s.first_row < D.first_row) D.first_row = s.first_row;
        }
    }
    if (bad) { memset(res, 0, sizeof *res); res->ngroups = -1; return; }
    for (int64_t i = 1; i < R.ngroups; i++)
        for (int64_t j = i; j > 0 && R.groups[j].first_row < R.groups[j - 1].first_row; j--) { mo_q1_group_t tmp = R.groups[j]; R.groups[j] = R.groups[j - 1]; R.groups[j - 1] = tmp; }
    for (int64_t i = 0; i < R.ngroups; i++) {
        mo_q1_group_t &o = R.groups[i];
        const double c = (double)o.count_order;
        o.avg_qty = o.sum_qty / c; o.avg_price = o.sum_base_price / c; o.avg_disc = o.sum_disc / c;
    }
    *res = R;
}

// MergeGroup for the Q6 shape: (sum, count) partials added in order; an empty partial is NULL and skipped (sumavg2.go:222-236)
__global__ void q6_merge_kernel(const double *parts, uint64_t nparts, Q6DevOut o) {
    double total = 0.0; long long cnt = 0; bool any = false;
    for (uint64_t p = 0; p < nparts; p++) {
        const double s = parts[2 * p]; const long long c = reinterpret_cast<const long long *>(parts)[2 * p + 1];
        if (c == 0) continue;
        total = any ? __dadd_rn(total, s) : s; any = true; cnt += c;
    }
    o.res[0] = total;
    if (o.res_words >= 2) reinterpret_cast<long long *>(o.res)[1] = cnt;
    if (o.rnulls) o.rnulls[0] = any ? 0ull : 1ull;
}

// ---- Q6 over Decimal64 ------------------------------------------------------------------------------------------------------------------
// Running state of one MO_XCALL_Q6_DEC_FILTER_SUM call across its chunks (device scratch, zeroed before the first chunk)
struct Q6DecRun { u128 sum; unsigned long long mag, cnt, err1; };   // err1 = failing row + 1, 0 = none

// bit length of the largest |product| a DecSum.mag admits
__device__ __forceinline__ int dec_mag_bits(uint64_t mag) { return mag ? 128 - __clzll((long long)mag) : 0; }
// z = x + y; true when the checked Add128 fails (decimal.go Add128: equal signs in, the other sign out)
__device__ __forceinline__ bool add128_overflows(u128 x, u128 y, u128 &z) {
    z = x + y;
    const bool sx = (x >> 127) != 0, sy = (y >> 127) != 0, sz = (z >> 127) != 0;
    return sx == sy && sz != sx;
}
__device__ __forceinline__ u128 dec128_get(mo_dec128_t v) { return ((u128)v.hi << 64) | v.lo; }
__device__ __forceinline__ mo_dec128_t dec128_put(u128 x) { return mo_dec128_t{(uint64_t)x, (uint64_t)(x >> 64)}; }

// row r of a chunk passes the three conjuncts: its d64Mul product in v
__device__ __forceinline__ bool q6_dec_row(const mo_q6_dec_params_t &P, const int32_t *sd, const int64_t *disc, const int64_t *qty,
                                           const int64_t *price, uint64_t r, u128 &v) {
    if (!(sd[r] >= P.date_lo && sd[r] < P.date_hi && disc[r] >= P.disc_lo && disc[r] <= P.disc_hi && qty[r] < P.qty_hi)) return false;
    DecSum s = Q6Dec::zero();
    Q6Dec::add(true, disc[r], price[r], s);
    v = s.s;
    return true;
}

// Every running sum of the call is below 2^dec_mag_bits(bound) times the call's row count 2^lg_rows.  While that stays under 2^127 no
// prefix can overflow (on TPC-H data by more than 30 bits) and the chunk is only folded into the running state.  Otherwise -- the rare
// path -- the three q6_dec_walk kernels find the first row of the chunk where the row-order running sum, continued from the exact sum of
// the earlier chunks as the reference's SUM runs it, leaves int128.
__device__ __forceinline__ bool q6_dec_rare(const Q6DecRun *run, const Q6Rec<Q6Dec> *chunk, int lg_rows) {
    return !run->err1 && dec_mag_bits(run->mag | chunk->sum.mag) + lg_rows > 127;
}
// 192-bit two's complement: an int128 prefix plus fewer than 2^63 products below 2^126 stays inside it
struct W192 { u128 lo; int64_t hi; };
__device__ __forceinline__ void w192_add(W192 &w, u128 v) {      // w += v, v a sign-extended int128
    const u128 z = w.lo + v;
    w.hi += (int64_t)(z < w.lo) - (int64_t)(v >> 127);
    w.lo = z;
}
__device__ __forceinline__ bool w192_in_i128(const W192 &w) { return w.hi == -(int64_t)(w.lo >> 127); }

constexpr int kWalkCtas = 128, kWalkSegs = kWalkCtas * kThreads;   // contiguous row segments of the rare-path walk, one per thread
__device__ __forceinline__ void walk_segment(uint64_t m, uint64_t &r, uint64_t &end) {
    const uint64_t t = blockIdx.x * (uint64_t)kThreads + threadIdx.x, per = (m + kWalkSegs - 1) / kWalkSegs;
    r = t * per < m ? t * per : m;
    end = r + per < m ? r + per : m;
}
// walk 1: the exact sum of each segment's qualifying products
__global__ void __launch_bounds__(kThreads)
q6_dec_walk_sums(const int32_t *sd, const int64_t *disc, const int64_t *qty, const int64_t *price, uint64_t m, mo_q6_dec_params_t P,
                 const Q6Rec<Q6Dec> *chunk, const Q6DecRun *run, int lg_rows, W192 *seg) {
    if (!q6_dec_rare(run, chunk, lg_rows)) return;
    uint64_t r, end;
    walk_segment(m, r, end);
    W192 w{0, 0};
    u128 v;
    for (; r < end; r++) if (q6_dec_row(P, sd, disc, qty, price, r, v)) w192_add(w, v);
    seg[blockIdx.x * kThreads + threadIdx.x] = w;
}
// walk 2 (one thread): exclusive prefix of the segment sums, from the running sum of the earlier chunks
__global__ void q6_dec_walk_scan(W192 *seg, const Q6Rec<Q6Dec> *chunk, const Q6DecRun *run, int lg_rows) {
    if (!q6_dec_rare(run, chunk, lg_rows)) return;
    W192 acc{run->sum, -(int64_t)(run->sum >> 127)};
    for (int t = 0; t < kWalkSegs; t++) {
        const W192 s = seg[t];
        seg[t] = acc;
        const u128 lo = acc.lo + s.lo;
        acc.hi += s.hi + (int64_t)(lo < acc.lo);
        acc.lo = lo;
    }
}
// walk 3: each segment continues the running sum from its prefix in row order; the lowest row where it leaves int128 fails the call.  A
// segment whose prefix is already outside int128 holds no first failure: an earlier segment's walk finds it.
__global__ void __launch_bounds__(kThreads)
q6_dec_walk_find(const int32_t *sd, const int64_t *disc, const int64_t *qty, const int64_t *price, uint64_t m, uint64_t r0,
                 mo_q6_dec_params_t P, const W192 *seg, const Q6Rec<Q6Dec> *chunk, const Q6DecRun *run, int lg_rows,
                 unsigned long long *fail_row) {
    if (!q6_dec_rare(run, chunk, lg_rows)) return;
    uint64_t r, end;
    walk_segment(m, r, end);
    W192 w = seg[blockIdx.x * kThreads + threadIdx.x];
    if (!w192_in_i128(w)) return;
    u128 v;
    for (; r < end; r++) {
        if (!q6_dec_row(P, sd, disc, qty, price, r, v)) continue;
        w192_add(w, v);
        if (!w192_in_i128(w)) { atomicMin(fail_row, (unsigned long long)(P.row_base + (int64_t)(r0 + r))); return; }
    }
}

// After the scan of one chunk (rows [r0, r0 + m) of the call) and its rare-path walk: the chunk's sum (modulo 2^128: exact whenever no
// prefix overflowed) and the walk's failing row join the running state; after the last chunk (res != NULL) the caller-layout result is written.
__global__ void q6_dec_fold_kernel(mo_q6_dec_params_t P, const Q6Rec<Q6Dec> *chunk, const unsigned long long *fail_row, Q6DecRun *run,
                                   mo_q6_dec_result_t *res, uint64_t *rnulls) {
    Q6DecRun R = *run;
    if (chunk) {
        R.mag |= chunk->sum.mag;
        if (!R.err1 && *fail_row != ~0ull) R.err1 = *fail_row + 1;
        R.sum += chunk->sum.s;
        R.cnt += chunk->cnt;
    }
    *run = R;
    if (!res) return;
    res->revenue = dec128_put(R.sum);
    res->count = (int64_t)R.cnt;
    res->err_row = R.err1 ? (int64_t)R.err1 - 1 : -1;
    res->rc = R.err1 ? MO_RC_INVALID_ARGUMENT : MO_RC_SUCCESS;
    res->scale = 2 * P.scale;
    if (rnulls) rnulls[0] = R.cnt ? 0ull : 1ull;
}

// MergeGroup of Q6_DEC partials in order: empty partials skipped; a failing partial fails the merge with the lowest err_row among the failing
// partials; otherwise the sum is checked as BatchMerge's Add128 (sum_decimal_fast.go), and an overflow there or a partial of another scale
// fails the merge with err_row = -1
__global__ void q6_dec_merge_kernel(const mo_q6_dec_result_t *parts, uint64_t nparts, mo_q6_dec_result_t *res, uint64_t *rnulls) {
    u128 sum = 0; long long cnt = 0, perr = -1; int prc = MO_RC_SUCCESS, scale = -1; bool bad = false;
    for (uint64_t p = 0; p < nparts; p++) {
        const mo_q6_dec_result_t &P = parts[p];
        if (P.rc != MO_RC_SUCCESS) {
            if (prc == MO_RC_SUCCESS) prc = P.rc;
            if (P.err_row >= 0 && (perr < 0 || P.err_row < perr)) perr = P.err_row;
        }
        if (P.count == 0) continue;
        if (scale < 0) scale = P.scale;
        bad = add128_overflows(sum, dec128_get(P.revenue), sum) || P.scale != scale || bad;
        cnt += P.count;
    }
    res->revenue = dec128_put(sum);
    res->count = cnt;
    res->rc = prc != MO_RC_SUCCESS ? prc : (bad ? MO_RC_INVALID_ARGUMENT : MO_RC_SUCCESS);
    res->err_row = prc != MO_RC_SUCCESS ? perr : -1;
    res->scale = scale >= 0 ? scale : (nparts ? parts[0].scale : 0);
    if (rnulls) rnulls[0] = cnt ? 0ull : 1ull;
}

// kernel choice (MoB200_SetTuning): 0 = chosen from the input; 1 = the reference arm (dense q6_kernel, register q1_kernel)
int g_q6_variant = 0, g_q1_variant = 0;

}  // namespace

namespace mob {

int g_plan_specialise = 1;
int xcall_plan(mo_xcall_args_t *args, uint64_t len);

int tuning_set(const char *name, int value) {
    int search_answer;
    if (search_tuning(name, value, &search_answer)) return search_answer;
    if (!strcmp(name, "q6_variant")) { if (value != 0 && value != 1) return -1; g_q6_variant = value; return 0; }
    if (!strcmp(name, "plan_specialise")) { g_plan_specialise = value; return 0; }
    if (!strcmp(name, "q1_variant")) { if (value != 0 && value != 1) return -1; g_q1_variant = value; return 0; }
    if (!strcmp(name, "strkey_hash_bits")) { if (value < 0 || value > 63) return -1; g_strkey_hash_bits = value; return 0; }
    return -1;
}

// chunk of rows processed per launch when inputs are staged from the host (bounds device scratch)
static const uint64_t kHostChunkRows = 32ull << 20;

static bool aligned_to(const void *p, uintptr_t a) { return (((uintptr_t)p) & (a - 1)) == 0; }

// The Q6 scan of one chunk in domain D; the whole-chunk record lands in *rec (arena memory, valid until the caller rewinds the arena)
template <class D>
static int launch_q6(ThreadCtx &t, const int32_t *sd, const typename D::V *disc, const typename D::V *qty, const typename D::V *price,
                     uint64_t n, const typename D::Params &P, Q6DevOut dres, Q6Rec<D> **rec = nullptr) {
    if (!aligned_to(sd, 8) || !aligned_to(disc, 16) || !aligned_to(qty, 16) || !aligned_to(price, 16)) {
        set_error("q6: columns must be 16-byte aligned (int32 column 8-byte)"); return MO_RC_INVALID_ARGUMENT;
    }
    const int variant = g_q6_variant;
    int grid = num_sms() * 4;
    uint64_t work = (n / 2 + kThreads - 1) / kThreads;
    if ((uint64_t)grid > work) grid = work ? (int)work : 1;
    Q6Rec<D> *partials = (Q6Rec<D> *)arena_alloc(t, sizeof(Q6Rec<D>) * (size_t)(grid + 1));
    if (!partials) return MO_RC_INTERNAL_ERROR;
    Q6Rec<D> *out = partials + grid;
    if (rec) *rec = out;
    cudaEventRecord(t.kev0, t.stream);
    switch (variant) {
    case 1: q6_kernel<D, 4, 4><<<grid, kThreads, 0, t.stream>>>(sd, disc, qty, price, n, P, partials, out, t.ctrl, dres); break;
    default: q6_selective_kernel<D, 3><<<grid, kThreads, 0, t.stream>>>(sd, disc, qty, price, n, P, partials, out, t.ctrl, dres); break;
    }
    cudaEventRecord(t.kev1, t.stream);
    MOB_LAUNCH_CHECK();
    return MO_RC_SUCCESS;
}

// Chunks of a scan: device columns are one chunk; host columns are staged kHostChunkRows rows at a time inside the caller's Stager, each
// chunk's scratch handed back before the next chunk is staged (its copies queue behind the previous kernel on the same stream).
static uint64_t scan_chunks(bool dev, uint64_t len) { return dev ? (len ? 1 : 0) : (len + kHostChunkRows - 1) / kHostChunkRows; }

// columns [0, ncols) all host or all device; false (error set) otherwise
static bool same_residency(const char *what, const uint8_t *const *cols, int ncols, bool *dev) {
    *dev = is_device_ptr(cols[0]);
    for (int i = 1; i < ncols; i++) if (is_device_ptr(cols[i]) != *dev) { set_error("%s: columns must all be host or all device", what); return false; }
    return true;
}

// The Q6 scan of host or device columns {shipdate, discount, quantity, price} into a caller-layout device result.  Partial results of
// several chunks are merged in chunk order exactly like per-pipeline partials in MergeGroup (BatchMerge, sumavg2.go:222-236); with no
// rows the merge of zero partials writes the empty (NULL) result.
int q6_run(ThreadCtx &t, Stager &st, const uint8_t *const cols[4], uint64_t len, const mo_q6_params_t &P, double *res, uint64_t res_words,
           uint64_t *rnulls) {
    bool dev;
    if (!same_residency("q6", cols, 4, &dev)) return MO_RC_INVALID_ARGUMENT;
    const Q6DevOut dres{res, res_words, rnulls};
    const uint64_t nchunks = scan_chunks(dev, len);
    double *parts = nchunks == 1 ? nullptr : (double *)st.tmp(16 * nchunks);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    for (uint64_t i = 0; i < nchunks; i++) {
        const uint64_t r0 = i * kHostChunkRows, m = nchunks == 1 ? len : std::min(kHostChunkRows, len - r0);
        const ArenaMark mark = arena_mark(t);
        const void *c[4] = {st.in(cols[0] + 4 * r0, 4 * m), st.in(cols[1] + 8 * r0, 8 * m), st.in(cols[2] + 8 * r0, 8 * m), st.in(cols[3] + 8 * r0, 8 * m)};
        if (st.failed) return MO_RC_INTERNAL_ERROR;
        const int rc = launch_q6<Q6F64>(t, (const int32_t *)c[0], (const double *)c[1], (const double *)c[2], (const double *)c[3], m, P,
                                        nchunks == 1 ? dres : Q6DevOut{parts + 2 * i, 2, nullptr});
        if (rc) return rc;
        arena_rewind(t, mark);
    }
    if (nchunks != 1) {
        q6_merge_kernel<<<1, 1, 0, t.stream>>>(parts, nchunks, dres);
        MOB_LAUNCH_CHECK();
    }
    return MO_RC_SUCCESS;
}

int xcall_q6(mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (!args[0].pdata || args[0].dataSz < 8) { set_error("q6: result must hold 8 bytes"); return MO_RC_INVALID_ARGUMENT; }
    if (args[1].dataSz < 4 * len || args[2].dataSz < 8 * len || args[3].dataSz < 8 * len || args[4].dataSz < 8 * len) {
        set_error("q6: column shorter than len"); return MO_RC_INVALID_ARGUMENT;
    }
    mo_q6_params_t P;
    if (int rc = read_param(t, args[5], &P, sizeof P, sizeof P, "q6: params")) return rc;
    bool nullable = false;
    for (int i = 1; i <= 4; i++) nullable = nullable || args[i].pnulls != nullptr;
    if (nullable) {
        // nullable inputs: the same query through the generic fused operator (plan.cu), which carries a nulls bitmap on every column --
        // a NULL predicate operand rejects the row, a NULL product is skipped by SUM.  The specialised kernel above is the no-nulls fast path.
        mo_plan_t Q; memset(&Q, 0, sizeof Q);
        Q.ncols = 4; Q.col_type[0] = MO_T_DATE; Q.col_type[1] = Q.col_type[2] = Q.col_type[3] = MO_T_FLOAT64;
        Q.npreds = 4;
        Q.pred[0] = mo_plan_pred_t{0, 3, (double)P.date_lo, 0.0}; Q.pred[1] = mo_plan_pred_t{0, 4, (double)P.date_hi, 0.0};
        Q.pred[2] = mo_plan_pred_t{1, 6, P.disc_lo, P.disc_hi};    Q.pred[3] = mo_plan_pred_t{2, 4, P.qty_hi, 0.0};
        Q.ninstr = 1; Q.instr[0] = mo_plan_instr_t{MO_PLAN_OP_MUL, 3, 1, 0, 0.0};      // l_extendedprice * l_discount
        Q.naggs = 1; Q.agg[0] = mo_plan_agg_t{MO_AGG_SUM, 4};
        struct { mo_plan_result_header_t h; mo_plan_group_t g; mo_plan_agg_value_t a; } R;
        memset(&R, 0, sizeof R);
        mo_xcall_args_t pa[6]; memset(pa, 0, sizeof pa);
        pa[0].pdata = (uint8_t *)&R; pa[0].dataSz = sizeof R;
        pa[1].pdata = (uint8_t *)&Q; pa[1].dataSz = sizeof Q;
        pa[2] = args[1]; pa[3] = args[2]; pa[4] = args[3]; pa[5] = args[4];
        int rc = xcall_plan(pa, len);
        if (rc) return rc;
        // sum in word 0, qualifying rows in word 1 when the buffer holds 16 bytes, nulls word bit 0 = "no row qualified"
        const bool any = R.h.ngroups > 0 && R.a.count > 0;
        const double sum = any ? R.a.value : 0.0;
        const int64_t rows = R.h.ngroups > 0 ? R.g.rows : 0;
        unsigned char w[16];
        memcpy(w, &sum, 8); memcpy(w + 8, &rows, 8);
        rc = write_param(t, args[0].pdata, w, args[0].dataSz >= 16 ? 16 : 8);
        if (rc || !args[0].pnulls) return rc;
        const uint64_t nullword = any ? 0ull : 1ull;
        return write_param(t, args[0].pnulls, &nullword, 8);
    }

    // resident columns AND a device result and nulls word: enqueue only (no read-back, no synchronisation); the result is ordered on the
    // calling thread's stream, ready for NCCL + MO_XCALL_Q6_MERGE or a later MoB200_Download
    Stager st(t);
    double *dres = (double *)st.out(args[0].pdata, args[0].dataSz >= 16 ? 16 : 8);
    uint64_t *dn = (uint64_t *)st.out(args[0].pnulls, args[0].pnulls ? 8 : 0);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    const uint8_t *cols[4] = {args[1].pdata, args[2].pdata, args[3].pdata, args[4].pdata};
    const int rc = q6_run(t, st, cols, len, P, dres, args[0].dataSz / 8, dn);
    if (rc) return rc;
    return st.complete();
}

// The Q6 scan of Decimal64 columns (host or device) into a device mo_q6_dec_result_t.  Chunks as q6_run; while a chunk's columns are still
// staged, the rare-path walk kernels (which return at once while the magnitude bound holds) check it and q6_dec_fold_kernel folds it into
// the call's running state in chunk order.
static int q6_dec_run(ThreadCtx &t, Stager &st, const uint8_t *const cols[4], uint64_t len, const mo_q6_dec_params_t &P,
                      mo_q6_dec_result_t *res, uint64_t *rnulls) {
    bool dev;
    if (!same_residency("q6 dec", cols, 4, &dev)) return MO_RC_INVALID_ARGUMENT;
    const uint64_t nchunks = scan_chunks(dev, len);
    Q6DecRun *run = (Q6DecRun *)st.tmp(sizeof(Q6DecRun));
    unsigned long long *fail_row = (unsigned long long *)st.tmp(8);
    W192 *seg = (W192 *)st.tmp(sizeof(W192) * kWalkSegs);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    MOB_CUDA_TRY(cudaMemsetAsync(run, 0, sizeof(Q6DecRun), t.stream));
    MOB_CUDA_TRY(cudaMemsetAsync(fail_row, 0xff, 8, t.stream));
    int lg_rows = 0;
    while (lg_rows < 64 && (1ull << lg_rows) < len) lg_rows++;
    if (nchunks == 0) {
        q6_dec_fold_kernel<<<1, 1, 0, t.stream>>>(P, nullptr, fail_row, run, res, rnulls);
        MOB_LAUNCH_CHECK();
    }
    for (uint64_t i = 0; i < nchunks; i++) {
        const uint64_t r0 = i * kHostChunkRows, m = nchunks == 1 ? len : std::min(kHostChunkRows, len - r0);
        const ArenaMark mark = arena_mark(t);
        const void *c[4] = {st.in(cols[0] + 4 * r0, 4 * m), st.in(cols[1] + 8 * r0, 8 * m), st.in(cols[2] + 8 * r0, 8 * m), st.in(cols[3] + 8 * r0, 8 * m)};
        if (st.failed) return MO_RC_INTERNAL_ERROR;
        const int32_t *sd = (const int32_t *)c[0];
        const int64_t *disc = (const int64_t *)c[1], *qty = (const int64_t *)c[2], *price = (const int64_t *)c[3];
        Q6Rec<Q6Dec> *rec = nullptr;
        const int rc = launch_q6<Q6Dec>(t, sd, disc, qty, price, m, P, Q6DevOut{nullptr, 0, nullptr}, &rec);
        if (rc) return rc;
        q6_dec_walk_sums<<<kWalkCtas, kThreads, 0, t.stream>>>(sd, disc, qty, price, m, P, rec, run, lg_rows, seg);
        q6_dec_walk_scan<<<1, 1, 0, t.stream>>>(seg, rec, run, lg_rows);
        q6_dec_walk_find<<<kWalkCtas, kThreads, 0, t.stream>>>(sd, disc, qty, price, m, r0, P, seg, rec, run, lg_rows, fail_row);
        const bool last = i + 1 == nchunks;
        q6_dec_fold_kernel<<<1, 1, 0, t.stream>>>(P, rec, fail_row, run, last ? res : nullptr, last ? rnulls : nullptr);
        MOB_LAUNCH_CHECK();
        arena_rewind(t, mark);
    }
    return MO_RC_SUCCESS;
}

// rc / err_row of a Q6_DEC result that the synchronous form returns
static int q6_dec_status(ThreadCtx &t, const void *res, const char *what) {
    mo_q6_dec_result_t R;
    if (is_device_ptr(res)) { const int rc = read_back(t, &R, res, sizeof R); if (rc) return rc; }
    else memcpy(&R, res, sizeof R);
    if (R.rc == MO_RC_SUCCESS) return MO_RC_SUCCESS;
    if (R.err_row >= 0) set_error("%s: invalid input: Decimal128 Add overflow at row %lld", what, (long long)R.err_row);
    else set_error("%s: invalid input: Decimal128 Add overflow or partials of different scales", what);
    return R.rc;
}

// MO_XCALL_Q6_DEC_FILTER_SUM: see include/mo_b200.h
int xcall_q6_dec(mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (!args[0].pdata || args[0].dataSz < sizeof(mo_q6_dec_result_t)) { set_error("q6 dec: result must hold a mo_q6_dec_result_t"); return MO_RC_INVALID_ARGUMENT; }
    if (args[1].dataSz < 4 * len || args[2].dataSz < 8 * len || args[3].dataSz < 8 * len || args[4].dataSz < 8 * len) {
        set_error("q6 dec: column shorter than len"); return MO_RC_INVALID_ARGUMENT;
    }
    for (int i = 1; i <= 4; i++)
        if (args[i].pnulls) { set_error("q6 dec: the DECIMAL(15,2) lineitem columns are NOT NULL; column %d has a nulls bitmap", i); return MO_RC_INVALID_ARGUMENT; }
    mo_q6_dec_params_t P;
    if (int rc = read_param(t, args[5], &P, sizeof P, sizeof P, "q6 dec: params")) return rc;
    if (P.scale < 0 || P.scale > 4) { set_error("q6 dec: scale %d outside 0..4", (int)P.scale); return MO_RC_INVALID_ARGUMENT; }
    Stager st(t);
    mo_q6_dec_result_t *dres = (mo_q6_dec_result_t *)st.out(args[0].pdata, sizeof(mo_q6_dec_result_t));
    uint64_t *dn = (uint64_t *)st.out(args[0].pnulls, args[0].pnulls ? 8 : 0);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    const uint8_t *cols[4] = {args[1].pdata, args[2].pdata, args[3].pdata, args[4].pdata};
    int rc = q6_dec_run(t, st, cols, len, P, dres, dn);
    if (rc) return rc;
    const bool async = st.resident();
    rc = st.complete();
    if (rc || async) return rc;
    return q6_dec_status(t, args[0].pdata, "q6 dec");
}

// MO_XCALL_Q6_DEC_MERGE: args[0] = result as MO_XCALL_Q6_DEC_FILTER_SUM ; args[1] = len partial mo_q6_dec_result_t
int xcall_q6_dec_merge(mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (!args[0].pdata || args[0].dataSz < sizeof(mo_q6_dec_result_t) || args[1].dataSz < sizeof(mo_q6_dec_result_t) * len) {
        set_error("q6 dec merge: result and partials are mo_q6_dec_result_t"); return MO_RC_INVALID_ARGUMENT;
    }
    Stager st(t);
    const mo_q6_dec_result_t *dparts = (const mo_q6_dec_result_t *)st.in(args[1].pdata, sizeof(mo_q6_dec_result_t) * len);
    mo_q6_dec_result_t *dres = (mo_q6_dec_result_t *)st.out(args[0].pdata, sizeof(mo_q6_dec_result_t));
    uint64_t *dn = (uint64_t *)st.out(args[0].pnulls, args[0].pnulls ? 8 : 0);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    q6_dec_merge_kernel<<<1, 1, 0, t.stream>>>(dparts, len, dres, dn);
    MOB_LAUNCH_CHECK();
    const bool async = st.resident();
    const int rc = st.complete();
    if (rc || async) return rc;
    return q6_dec_status(t, args[0].pdata, "q6 dec merge");
}

// device addresses of the Q1 input columns; the key columns hold packed uint8 values or 24-byte varlena cells
struct Q1Cols { const int32_t *sd; const double *qty, *price, *disc, *tax; const uint8_t *rf, *ls; };

// the 4-slot pass, the 8-slot pass that runs only if the 4-slot pass overflowed its dictionary, and q1_finalize_kernel, which writes the
// caller-layout result of the pass that did not overflow (ngroups = -1 when both did)
static int launch_q1(ThreadCtx &t, const Q1Cols &c, bool varlena, uint64_t n, int32_t cutoff, mo_q1_result_t *dres, int64_t row_base) {
    if (!aligned_to(c.sd, 8) || !aligned_to(c.qty, 16) || !aligned_to(c.price, 16) || !aligned_to(c.disc, 16) || !aligned_to(c.tax, 16) ||
        !aligned_to(c.rf, varlena ? 8 : 2) || !aligned_to(c.ls, varlena ? 8 : 2)) {
        set_error("q1: columns must be 16-byte aligned (int32 column 8-byte, key columns 2/8-byte)"); return MO_RC_INVALID_ARGUMENT;
    }
    // The TMA kernel bulk-copies 1024-row tiles of every column, so it needs packed keys and 16-byte aligned sources.  Below 64 tiles
    // the register kernel serves: there the rows past the last whole tile (up to 1023, taken by one warp) cost the TMA kernel more than
    // the register kernel's whole pass (DESIGN 5.1).  q1_variant = 1 forces the register kernel, the arm the TMA kernel is tested against.
    const bool tma = !varlena && aligned_to(c.sd, 16) && aligned_to(c.rf, 16) && aligned_to(c.ls, 16) && n >= (uint64_t)kCtaTileRows * 64 &&
                     g_q1_variant != 1;
    // TMA kernel: one CTA per SM, each taking whole tiles; register kernel: two CTAs per SM, each thread at least one pair
    auto grid_of = [&](bool use_tma) {
        const uint64_t work = use_tma ? n / kCtaTileRows : (n / 2 + kThreads - 1) / kThreads;
        int grid = num_sms() * (use_tma ? 1 : 2);
        if ((uint64_t)grid > work) grid = work ? (int)work : 1;
        return grid > kQ1MaxGrid ? kQ1MaxGrid : grid;
    };
    int grid = grid_of(tma);
    Q1Rec *partials = (Q1Rec *)arena_alloc(t, sizeof(Q1Rec) * (size_t)(grid + 1));
    if (!partials) return MO_RC_INTERNAL_ERROR;
    Q1Rec *narrow = partials + grid;
    cudaEventRecord(t.kev0, t.stream);
    if (tma) {
        const size_t smem = (size_t)kCtaStages * kCtaTileBytes + 2 * kCtaStages * 8;
        static bool tattr = false;
        if (!tattr) {
            cudaError_t e = cudaFuncSetAttribute(q1_tma_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess) { set_error("q1: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e)); return MO_RC_INTERNAL_ERROR; }
            tattr = true;
        }
        q1_tma_kernel<4><<<grid, kCtaThreads, smem, t.stream>>>(c.sd, c.qty, c.price, c.disc, c.tax, c.rf, c.ls, n, cutoff, partials, narrow, t.ctrl);
    } else if (varlena) {
        q1_kernel<4, 2, 2, 1><<<grid, kThreads, 0, t.stream>>>(c.sd, c.qty, c.price, c.disc, c.tax, c.rf, c.ls, n, cutoff, partials, narrow, t.ctrl, nullptr);
    } else {
        q1_kernel<4, 2, 2, 0><<<grid, kThreads, 0, t.stream>>>(c.sd, c.qty, c.price, c.disc, c.tax, c.rf, c.ls, n, cutoff, partials, narrow, t.ctrl, nullptr);
    }
    cudaEventRecord(t.kev1, t.stream);
    MOB_LAUNCH_CHECK();
    grid = grid_of(false);
    partials = (Q1Rec *)arena_alloc(t, sizeof(Q1Rec) * (size_t)(grid + 1));
    if (!partials) return MO_RC_INTERNAL_ERROR;
    Q1Rec *wide = partials + grid;
    if (varlena) q1_kernel<8, 2, 2, 1><<<grid, kThreads, 0, t.stream>>>(c.sd, c.qty, c.price, c.disc, c.tax, c.rf, c.ls, n, cutoff, partials, wide, t.ctrl, narrow);
    else q1_kernel<8, 2, 2, 0><<<grid, kThreads, 0, t.stream>>>(c.sd, c.qty, c.price, c.disc, c.tax, c.rf, c.ls, n, cutoff, partials, wide, t.ctrl, narrow);
    MOB_LAUNCH_CHECK();
    q1_finalize_kernel<<<1, 1, 0, t.stream>>>(narrow, wide, dres, row_base);
    MOB_LAUNCH_CHECK();
    return MO_RC_SUCCESS;
}

// The Q1 scan of host or device columns {shipdate, quantity, extendedprice, discount, tax, returnflag, linestatus} into a device
// mo_q1_result_t (first_row offset by row_base).  Chunks as q6_run; their results are merged in chunk order by q1_merge_kernel.
int q1_run(ThreadCtx &t, Stager &st, const uint8_t *const cols[7], bool varlena, uint64_t len, int32_t cutoff, int64_t row_base,
           mo_q1_result_t *res) {
    bool dev;
    if (!same_residency("q1", cols, 7, &dev)) return MO_RC_INVALID_ARGUMENT;
    const uint64_t ksz = varlena ? 24 : 1;
    const uint64_t nchunks = scan_chunks(dev, len);
    mo_q1_result_t *parts = nchunks == 1 ? nullptr : (mo_q1_result_t *)st.tmp(sizeof(mo_q1_result_t) * nchunks);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    for (uint64_t i = 0; i < nchunks; i++) {
        const uint64_t r0 = i * kHostChunkRows, m = nchunks == 1 ? len : std::min(kHostChunkRows, len - r0);
        const ArenaMark mark = arena_mark(t);
        const Q1Cols d{(const int32_t *)st.in(cols[0] + 4 * r0, 4 * m), (const double *)st.in(cols[1] + 8 * r0, 8 * m),
                       (const double *)st.in(cols[2] + 8 * r0, 8 * m), (const double *)st.in(cols[3] + 8 * r0, 8 * m),
                       (const double *)st.in(cols[4] + 8 * r0, 8 * m), (const uint8_t *)st.in(cols[5] + ksz * r0, ksz * m),
                       (const uint8_t *)st.in(cols[6] + ksz * r0, ksz * m)};
        if (st.failed) return MO_RC_INTERNAL_ERROR;
        const int rc = launch_q1(t, d, varlena, m, cutoff, nchunks == 1 ? res : parts + i, row_base + (int64_t)r0);
        if (rc) return rc;
        arena_rewind(t, mark);
    }
    if (nchunks != 1) {
        q1_merge_kernel<<<1, 1, 0, t.stream>>>(parts, nchunks, res);
        MOB_LAUNCH_CHECK();
    }
    return MO_RC_SUCCESS;
}

int xcall_q1(mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (!args[0].pdata || args[0].dataSz < sizeof(mo_q1_result_t)) { set_error("q1: result buffer too small"); return MO_RC_INVALID_ARGUMENT; }
    if (args[1].dataSz < 4 * len) { set_error("q1: shipdate shorter than len"); return MO_RC_INVALID_ARGUMENT; }
    for (int i = 2; i <= 5; i++) if (args[i].dataSz < 8 * len) { set_error("q1: column %d shorter than len", i); return MO_RC_INVALID_ARGUMENT; }
    bool q1_nullable = false;
    for (int i = 1; i <= 7; i++) q1_nullable = q1_nullable || args[i].pnulls != nullptr;
    bool varlena;
    if (args[6].dataSz == len && args[7].dataSz == len) varlena = false;
    else if (args[6].dataSz == 24 * len && args[7].dataSz == 24 * len) varlena = true;
    else { set_error("q1: key columns must be packed uint8 (len bytes) or varlena cells (24*len bytes)"); return MO_RC_INVALID_ARGUMENT; }
    mo_q1_params_t P{0, 0, 0};   // an int32 cutoff alone, or the whole block: row_base makes first_row values global row numbers
    if (int rc = read_param(t, args[8], &P, 4, sizeof P, "q1: cutoff param")) return rc;
    const bool dev = is_device_ptr(args[1].pdata);
    for (int i = 2; i <= 7; i++) if (is_device_ptr(args[i].pdata) != dev) { set_error("q1: columns must all be host or all device"); return MO_RC_INVALID_ARGUMENT; }
    if (q1_nullable) {
        // nullable inputs: the generic fused operator (plan.cu).  NULL shipdate rejects the row; NULL values are skipped by their aggregates;
        // a NULL key is its own group (has_null_keys; its key byte reads 0 here).  Packed uint8 keys only.
        if (varlena) { set_error("q1: nullable columns need packed uint8 key columns"); return MO_RC_INVALID_ARGUMENT; }
        mo_plan_t Q; memset(&Q, 0, sizeof Q);
        Q.ncols = 7; Q.col_type[0] = MO_T_DATE; for (int c = 1; c <= 4; c++) Q.col_type[c] = MO_T_FLOAT64; Q.col_type[5] = Q.col_type[6] = MO_T_UINT8;
        Q.row_base = P.row_base; Q.has_null_keys = (args[6].pnulls || args[7].pnulls) ? 1 : 0;
        Q.npreds = 1; Q.pred[0] = mo_plan_pred_t{0, 5, (double)P.cutoff, 0.0};
        Q.ninstr = 5;
        Q.instr[0] = mo_plan_instr_t{MO_PLAN_OP_CONST, 0, 0, 0, 1.0};        // slot 7: 1
        Q.instr[1] = mo_plan_instr_t{MO_PLAN_OP_SUB, 7, 3, 0, 0.0};          // slot 8: 1 - l_discount
        Q.instr[2] = mo_plan_instr_t{MO_PLAN_OP_MUL, 2, 8, 0, 0.0};          // slot 9: l_extendedprice * (1 - l_discount)
        Q.instr[3] = mo_plan_instr_t{MO_PLAN_OP_ADD, 7, 4, 0, 0.0};          // slot 10: 1 + l_tax
        Q.instr[4] = mo_plan_instr_t{MO_PLAN_OP_MUL, 9, 10, 0, 0.0};         // slot 11: ... * (1 + l_tax)
        Q.nkeys = 2; Q.key_col[0] = 5; Q.key_col[1] = 6;
        Q.naggs = 6;
        Q.agg[0] = mo_plan_agg_t{MO_AGG_SUM, 1}; Q.agg[1] = mo_plan_agg_t{MO_AGG_SUM, 2}; Q.agg[2] = mo_plan_agg_t{MO_AGG_SUM, 9}; Q.agg[3] = mo_plan_agg_t{MO_AGG_SUM, 11};
        Q.agg[4] = mo_plan_agg_t{MO_AGG_SUM, 3}; Q.agg[5] = mo_plan_agg_t{MO_AGG_COUNT, -1};
        struct Rec { mo_plan_group_t g; mo_plan_agg_value_t a[6]; };
        struct { mo_plan_result_header_t h; Rec r[MO_Q1_MAX_GROUPS]; } R;
        memset(&R, 0, sizeof R);
        mo_xcall_args_t pa[9]; memset(pa, 0, sizeof pa);
        pa[0].pdata = (uint8_t *)&R; pa[0].dataSz = sizeof R;
        pa[1].pdata = (uint8_t *)&Q; pa[1].dataSz = sizeof Q;
        for (int c = 0; c < 7; c++) pa[2 + c] = args[1 + c];
        int rc = xcall_plan(pa, len);
        if (rc) { if (rc == MO_RC_INVALID_ARGUMENT) set_error("q1: more than %d distinct group keys", MO_Q1_MAX_GROUPS); return rc; }
        mo_q1_result_t res; memset(&res, 0, sizeof res);
        res.ngroups = R.h.ngroups;
        for (int64_t g = 0; g < R.h.ngroups; g++) {
            const Rec &r = R.r[g]; mo_q1_group_t &o = res.groups[g];
            const int shift = Q.has_null_keys ? 8 : 0;   // has_null mode: marker byte, then the value byte
            const bool n0 = Q.has_null_keys && (r.g.key & 0xff) != 0;
            o.returnflag = n0 ? 0 : (uint8_t)((r.g.key >> shift) & 0xff);
            const int off1 = Q.has_null_keys ? (n0 ? 1 : 2) : 1;
            const bool n1 = Q.has_null_keys && ((r.g.key >> (8 * off1)) & 0xff) != 0;
            o.linestatus = n1 ? 0 : (uint8_t)((r.g.key >> (8 * (off1 + (Q.has_null_keys ? 1 : 0)))) & 0xff);
            o.first_row = r.g.first_row;
            o.sum_qty = r.a[0].value; o.sum_base_price = r.a[1].value; o.sum_disc_price = r.a[2].value; o.sum_charge = r.a[3].value; o.sum_disc = r.a[4].value;
            o.avg_qty = r.a[0].count ? r.a[0].value / (double)r.a[0].count : 0.0;
            o.avg_price = r.a[1].count ? r.a[1].value / (double)r.a[1].count : 0.0;
            o.avg_disc = r.a[4].count ? r.a[4].value / (double)r.a[4].count : 0.0;
            o.count_order = r.a[5].count;
        }
        return write_param(t, args[0].pdata, &res, sizeof res);
    }

    const uint8_t *cols[7] = {args[1].pdata, args[2].pdata, args[3].pdata, args[4].pdata, args[5].pdata, args[6].pdata, args[7].pdata};
    Stager st(t);
    mo_q1_result_t *dres = (mo_q1_result_t *)st.out(args[0].pdata, sizeof(mo_q1_result_t));
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    int rc = q1_run(t, st, cols, varlena, len, P.cutoff, P.row_base, dres);
    if (rc) return rc;
    const bool async = st.resident();   // resident columns AND a device result: enqueue only (see xcall_q6)
    rc = st.complete();
    if (rc || async) return rc;   // more than MO_Q1_MAX_GROUPS keys: ngroups = -1 in the result
    int64_t ngroups;
    if (is_device_ptr(args[0].pdata)) { rc = read_back(t, &ngroups, args[0].pdata, 8); if (rc) return rc; }
    else ngroups = ((const mo_q1_result_t *)args[0].pdata)->ngroups;
    if (ngroups < 0) {
        set_error("q1: more than %d distinct group keys; the fused small-cardinality kernel does not apply", MO_Q1_MAX_GROUPS);
        return MO_RC_INVALID_ARGUMENT;
    }
    return MO_RC_SUCCESS;
}

// MO_XCALL_Q6_MERGE: args[0] = result as MO_XCALL_Q6_FILTER_SUM ; args[1] = len partial results of 16 bytes (sum f64, count i64)
int xcall_q6_merge(mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (!args[0].pdata || args[0].dataSz < 8 || args[1].dataSz < 16 * len) { set_error("q6 merge: result needs 8 bytes, partials 16 bytes each"); return MO_RC_INVALID_ARGUMENT; }
    Stager st(t);
    const double *dparts = (const double *)st.in(args[1].pdata, 16 * len);
    double *dres = (double *)st.out(args[0].pdata, args[0].dataSz >= 16 ? 16 : 8);
    uint64_t *dn = (uint64_t *)st.out(args[0].pnulls, args[0].pnulls ? 8 : 0);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    q6_merge_kernel<<<1, 1, 0, t.stream>>>(dparts, len, Q6DevOut{dres, args[0].dataSz / 8, dn});
    MOB_LAUNCH_CHECK();
    return st.complete();
}

// MO_XCALL_Q1_MERGE: args[0] = mo_q1_result_t ; args[1] = len partial mo_q1_result_t (first_row already global: row_base param)
int xcall_q1_merge(mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (!args[0].pdata || args[0].dataSz < sizeof(mo_q1_result_t) || args[1].dataSz < sizeof(mo_q1_result_t) * len) { set_error("q1 merge: buffers too small"); return MO_RC_INVALID_ARGUMENT; }
    Stager st(t);
    const mo_q1_result_t *dparts = (const mo_q1_result_t *)st.in(args[1].pdata, sizeof(mo_q1_result_t) * len);
    mo_q1_result_t *dres = (mo_q1_result_t *)st.out(args[0].pdata, sizeof(mo_q1_result_t));
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    q1_merge_kernel<<<1, 1, 0, t.stream>>>(dparts, len, dres);
    MOB_LAUNCH_CHECK();
    const bool async = st.resident();
    const int rc = st.complete();
    if (rc || async) return rc;
    if (!is_device_ptr(args[0].pdata) && ((mo_q1_result_t *)args[0].pdata)->ngroups < 0) { set_error("q1 merge: more than %d distinct group keys", MO_Q1_MAX_GROUPS); return MO_RC_INVALID_ARGUMENT; }
    return MO_RC_SUCCESS;
}

}  // namespace mob
