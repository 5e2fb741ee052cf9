// plan.cu -- the generic fused scan -> filter -> project -> (hash) group -> aggregate operator: ONE pass over the columns for any
// plan of the shape the colexec pipeline runs per block (table_scan -> filter -> projection -> group, SURVEY.md section 8 rows
// a12-a19):
//
//   N conjunctive predicates   compare / BETWEEN of a column with constants          (filter.go:87-153, func_compare.go, operator_between.go)
//   an expression program      + - * / over columns and constants, SSA form          (evalExpression.go:575-640: one node per instruction)
//   group-by                   <= 8 key bytes packed like fillKeys                   (group/exec2.go:296-367, inthashmap.go:92-183)
//   K aggregates               SUM / AVG / COUNT / COUNT(*) / MIN / MAX              (aggexec/{sumavg2,count2,minmax2}.go)
//
// with a nulls bitmap on every input column.  tpch.cu holds the two hand-specialised instances of this operator (Q6, Q1); this file
// is the operator itself: a small warp-uniform interpreter.  Every thread owns one row per iteration; column values and instruction
// results live in a shared-memory register file vreg[slot][thread] (conflict-free: slot-major), so operand selection is one LDS
// instead of a chain of selects; null-ness of every slot is one bit of a per-thread mask.  Groups are found in a per-CTA shared
// memory hash table (first-come slots), whose partial states are folded into a global table when the CTA retires; rows whose CTA
// table is full go to the global table directly.
//
// Arithmetic is float64 (the reference's type for TPC-H style expressions over float columns): integer columns enter expressions
// converted to float64 (exact below 2^53); each instruction rounds once like the reference's separate nodes (no FMA contraction).
// Group sums are accumulated with atomics: the association order is not fixed (results agree with the serial loop to ~1e-13).
#include "common.cuh"
#include "keytable.cuh"
#include <cmath>
#include <cstring>
#include <algorithm>

using namespace mob;

namespace {

constexpr int kThreads = 128;
constexpr int kCtaSlots = 32;           // per-CTA group table (shared atomics)
constexpr int kPriv = 4;               // groups whose state every thread keeps PRIVATELY in shared memory (no atomics, no shuffles)

struct PlanCols { const uint8_t *data[MO_PLAN_MAX_COLS]; const uint64_t *nulls[MO_PLAN_MAX_COLS]; };

// global group table / result staging (device arena)
struct PlanGlobal {
    uint64_t *key; unsigned long long *first_row; unsigned long long *rows;   // [cap]
    double *acc; unsigned long long *cnt;                                      // [cap][naggs]
    uint64_t mask;                                                             // cap - 1: a keytable.cuh table of cap + 1 slots
    unsigned *overflow;
};

__device__ __forceinline__ double agg_identity(int kind) {
    if (kind == MO_AGG_MIN) return __longlong_as_double((long long)~0ull);   // ordered-key domain: all ones
    if (kind == MO_AGG_MAX) return __longlong_as_double(0ll);
    return 0.0;
}
// accumulate v into *a (shared or global)
__device__ __forceinline__ void agg_apply(int kind, double *a, double v) {
    if (kind == MO_AGG_MIN) { if (v == v) atomicMin(reinterpret_cast<unsigned long long *>(a), flt_key(v)); }
    else if (kind == MO_AGG_MAX) { if (v == v) atomicMax(reinterpret_cast<unsigned long long *>(a), flt_key(v)); }
    else if (kind == MO_AGG_SUM || kind == MO_AGG_AVG) atomicAdd(a, v);
}
// fold a partial state p into *a
__device__ __forceinline__ void agg_fold(int kind, double *a, double p) {
    if (kind == MO_AGG_MIN) atomicMin(reinterpret_cast<unsigned long long *>(a), (unsigned long long)__double_as_longlong(p));
    else if (kind == MO_AGG_MAX) atomicMax(reinterpret_cast<unsigned long long *>(a), (unsigned long long)__double_as_longlong(p));
    else if (kind == MO_AGG_SUM || kind == MO_AGG_AVG) atomicAdd(a, p);
}


__device__ __forceinline__ bool global_find(PlanGlobal &G, uint64_t key, uint64_t &slot) {
    if (kt_insert(G.key, G.mask, key, slot)) return true;
    *G.overflow = 1;
    return false;
}

__global__ void plan_init_kernel(PlanGlobal G, int naggs, const mo_plan_t *P) {
    const uint64_t cap1 = G.mask + 2;
    for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s < cap1; s += (uint64_t)gridDim.x * blockDim.x) {
        G.key[s] = kEmptyKey; G.first_row[s] = ~0ull; G.rows[s] = 0;
        for (int a = 0; a < naggs; a++) { G.acc[s * naggs + a] = agg_identity(P->agg[a].kind); G.cnt[s * naggs + a] = 0; }
    }
}

// ---- the interpreter: VECTORISED, like the reference's own execution model (one operator over a batch at a time) --------------------------
// A CTA works on tiles of kThreads x R rows; thread t owns rows t, t + kThreads, ... of the tile.  Every operator of the plan -- column load,
// predicate, expression node, key column, aggregate -- is decoded ONCE per tile: the switch on type / opcode sits OUTSIDE the loop over the
// thread's R rows (explicitly: the compiler does not unswitch it), so the inner loops are straight-line code over a shared-memory register
// file vreg[slot][r][thread] (thread-minor: conflict-free).  Every slot has a DOMAIN fixed by the host when the plan is decoded: integer
// columns that only feed integer predicates or group keys stay raw int64 (compared as integers, never converted); columns that feed an
// expression or an aggregate are converted to float64 once, when they are loaded.  Column loads are issued kGroup columns at a time before
// anything consumes them (kGroup x R loads in flight per thread).
constexpr int R = 4;
constexpr int kGroup = 4;      // columns whose loads are issued together

struct PlanAux {                       // host-prepared decode of the descriptor
    int sz[MO_PLAN_MAX_COLS];          // element width in bytes
    int ext[MO_PLAN_MAX_COLS];         // after the load: 0 nothing (zero-extended), 1 / 2 / 3 sign-extend from 8 / 16 / 32 bits
    int tof[MO_PLAN_MAX_COLS];         // then: 0 keep, 1 int64 -> float64, 2 uint64 -> float64, 3 float32 bits -> float64
    int pred_mode[MO_PLAN_MAX_PREDS];  // 0 float64 slot vs P.pred lo / hi, 1 raw int64 vs ilo / ihi, 2 raw uint64 vs ilo / ihi (unsigned),
                                       // 3 never true, 4 true unless the operand is NULL
    int pred_slot[MO_PLAN_MAX_PREDS];  // PHYSICAL slot the predicate reads
    long long ilo[MO_PLAN_MAX_PREDS], ihi[MO_PLAN_MAX_PREDS];
    int raw_phys[MO_PLAN_MAX_COLS];    // -1, or a physical slot keeping the column's raw integer for predicates when its own slot turns float64
    unsigned key_nulls;                // null bits of the nullable key columns (has_null_keys == 0: a row with a NULL key joins no group)
    int key_mode[MO_PLAN_MAX_KEYS];    // 0 raw integer slot, 1 float64 slot holding an integer (exact: < 8-byte types), 2 reload the 8 bytes from the column,
                                       // 3 float64 slot holding a float32 (key = its float32 bits), 4 float64 bits
    int key_shift[MO_PLAN_MAX_KEYS];   // bit offset of the column inside the packed key when has_null_keys == 0
    int need_cnt;                      // some aggregate input can be NULL (nullable column or a division): per-aggregate counts are kept
    int phys[MO_PLAN_MAX_COLS + MO_PLAN_MAX_INSTR];   // value slot -> PHYSICAL slot of the shared-memory register file (slots are reused once dead)
    int nphys;
};

#define PLAN_FORJ _Pragma("unroll") for (int j = 0; j < R; j++)
#define PLAN_SLOT(s, j) my[((s) * R + (j)) * kThreads]

__device__ __forceinline__ uint64_t plan_key_bits(int mode, unsigned long long slotv, const uint8_t *col, uint64_t r) {
    switch (mode) {
    case 1: return (uint64_t)(long long)__longlong_as_double((long long)slotv);
    case 2: return reinterpret_cast<const unsigned long long *>(col)[r];
    case 3: return (uint64_t)__float_as_uint((float)__longlong_as_double((long long)slotv));
    default: return slotv;
    }
}

__global__ void __launch_bounds__(kThreads, 4)
plan_kernel(const mo_plan_t *__restrict__ Pg, const PlanAux *__restrict__ Ag, PlanCols C, uint64_t n, PlanGlobal G) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ mo_plan_t P;
    __shared__ PlanAux X;
    for (int i = threadIdx.x; i < (int)(sizeof(mo_plan_t) / 4); i += kThreads) reinterpret_cast<uint32_t *>(&P)[i] = reinterpret_cast<const uint32_t *>(Pg)[i];
    for (int i = threadIdx.x; i < (int)(sizeof(PlanAux) / 4); i += kThreads) reinterpret_cast<uint32_t *>(&X)[i] = reinterpret_cast<const uint32_t *>(Ag)[i];
    __syncthreads();
    const int nslots = X.nphys, naggs = P.naggs;
    unsigned long long *vreg = reinterpret_cast<unsigned long long *>(smem_raw);                      // [(physical slot * R + j) * kThreads + tid]
    uint64_t *tkey = reinterpret_cast<uint64_t *>(vreg + (size_t)nslots * R * kThreads);              // [kCtaSlots]
    unsigned long long *tfirst = reinterpret_cast<unsigned long long *>(tkey + kCtaSlots);
    unsigned long long *trows = tfirst + kCtaSlots;
    double *tacc = reinterpret_cast<double *>(trows + kCtaSlots);                                     // [kCtaSlots][naggs]
    unsigned long long *tcnt = reinterpret_cast<unsigned long long *>(tacc + (size_t)kCtaSlots * naggs);
    for (int s = threadIdx.x; s < kCtaSlots; s += kThreads) {
        tkey[s] = kEmptyKey; tfirst[s] = ~0ull; trows[s] = 0;
        for (int a = 0; a < naggs; a++) { tacc[s * naggs + a] = agg_identity(P.agg[a].kind); tcnt[s * naggs + a] = 0; }
    }
    // The first kPriv distinct keys a CTA meets (a first-come dictionary, as in the Q1 kernel) get PRIVATE per-thread state in shared memory,
    // thread-minor so every access is conflict-free: a row then costs naggs x (LDS, op, STS) on its own copy -- no atomics, no shuffles.  Plans
    // with few groups (or none) live entirely here; further keys go to the shared CTA table, then to the global one.
    __shared__ unsigned long long pdict[kPriv];
    double *pacc0 = reinterpret_cast<double *>(tcnt + (size_t)kCtaSlots * naggs);                     // [(g * naggs + a) * kThreads + tid]
    unsigned *pcnt0 = reinterpret_cast<unsigned *>(pacc0 + (size_t)kPriv * naggs * kThreads);
    unsigned *prows0 = pcnt0 + (X.need_cnt ? (size_t)kPriv * naggs * kThreads : 0);                   // [g * kThreads + tid]  (the per-aggregate counts exist only when an input can be NULL)
    unsigned long long *pfirst0 = reinterpret_cast<unsigned long long *>(prows0 + (size_t)kPriv * kThreads);
    double *pacc = pacc0 + threadIdx.x; unsigned *pcnt = pcnt0 + threadIdx.x, *prows = prows0 + threadIdx.x; unsigned long long *pfirst = pfirst0 + threadIdx.x;
    if (threadIdx.x < kPriv) pdict[threadIdx.x] = kEmptyKey;
    for (int g = 0; g < kPriv; g++) {
        for (int a = 0; a < naggs; a++) { pacc[(g * naggs + a) * kThreads] = agg_identity(P.agg[a].kind); if (X.need_cnt) pcnt[(g * naggs + a) * kThreads] = 0u; }
        prows[g * kThreads] = 0u; pfirst[g * kThreads] = ~0ull;
    }
    unsigned long long dk[kPriv];
#pragma unroll
    for (int g = 0; g < kPriv; g++) dk[g] = kEmptyKey;
    bool dict_full = false;
    __syncthreads();
    unsigned long long *my = vreg + threadIdx.x;
    const uint64_t tile_rows = (uint64_t)kThreads * R;
    for (uint64_t base = blockIdx.x * tile_rows; base < n; base += (uint64_t)gridDim.x * tile_rows) {
        const uint64_t r0 = base + threadIdx.x;
        unsigned nb[R];
        bool ok[R];
        PLAN_FORJ { nb[j] = 0; ok[j] = r0 + (uint64_t)j * kThreads < n; }
        // ---- table scan
        for (int c0 = 0; c0 < P.ncols; c0 += kGroup) {
            unsigned long long raw[kGroup][R], nw[kGroup][R];
#pragma unroll
            for (int g = 0; g < kGroup; g++) {
                const int c = c0 + g;
                if (c < P.ncols) {
                    const uint8_t *d = C.data[c]; const uint64_t *nu = C.nulls[c];
                    const int sz = X.sz[c];
                    if (sz == 8) { PLAN_FORJ raw[g][j] = ok[j] ? __ldg(reinterpret_cast<const unsigned long long *>(d) + r0 + (uint64_t)j * kThreads) : 0ull; }
                    else if (sz == 4) { PLAN_FORJ raw[g][j] = ok[j] ? (unsigned long long)__ldg(reinterpret_cast<const unsigned *>(d) + r0 + (uint64_t)j * kThreads) : 0ull; }
                    else if (sz == 2) { PLAN_FORJ raw[g][j] = ok[j] ? (unsigned long long)__ldg(reinterpret_cast<const unsigned short *>(d) + r0 + (uint64_t)j * kThreads) : 0ull; }
                    else { PLAN_FORJ raw[g][j] = ok[j] ? (unsigned long long)__ldg(d + r0 + (uint64_t)j * kThreads) : 0ull; }
                    if (nu) { PLAN_FORJ nw[g][j] = ok[j] ? __ldg(reinterpret_cast<const unsigned long long *>(nu) + ((r0 + (uint64_t)j * kThreads) >> 6)) : 0ull; }
                    else { PLAN_FORJ nw[g][j] = 0ull; }
                }
            }
#pragma unroll
            for (int g = 0; g < kGroup; g++) {
                const int c = c0 + g;
                if (c < P.ncols) {
                    const int ext = X.ext[c], tof = X.tof[c];
                    if (ext == 3) { PLAN_FORJ raw[g][j] = (unsigned long long)(long long)(int32_t)raw[g][j]; }
                    else if (ext == 2) { PLAN_FORJ raw[g][j] = (unsigned long long)(long long)(int16_t)raw[g][j]; }
                    else if (ext == 1) { PLAN_FORJ raw[g][j] = (unsigned long long)(long long)(int8_t)raw[g][j]; }
                    const int rp = X.raw_phys[c];
                    if (rp >= 0) { PLAN_FORJ PLAN_SLOT(rp, j) = raw[g][j]; }
                    if (tof == 1) { PLAN_FORJ raw[g][j] = (unsigned long long)__double_as_longlong((double)(long long)raw[g][j]); }
                    else if (tof == 2) { PLAN_FORJ raw[g][j] = (unsigned long long)__double_as_longlong((double)raw[g][j]); }
                    else if (tof == 3) { PLAN_FORJ raw[g][j] = (unsigned long long)__double_as_longlong((double)__uint_as_float((unsigned)raw[g][j])); }
                    const int pc = X.phys[c];
                    PLAN_FORJ { PLAN_SLOT(pc, j) = raw[g][j]; nb[j] |= (unsigned)((nw[g][j] >> ((r0 + (uint64_t)j * kThreads) & 63)) & 1ull) << c; }
                }
            }
        }
        // ---- filter: conjunction; a NULL operand makes the conjunct not-true (filter.go:125-141 keeps rows with !null && true)
        for (int q = 0; q < P.npreds; q++) {
            const int c = P.pred[q].col, op = P.pred[q].op, pc = X.pred_slot[q], mode = X.pred_mode[q];
#define PLAN_PRED(XT, LOADX, EXPR) PLAN_FORJ { const XT x = LOADX; ok[j] = ok[j] && (EXPR) && !((nb[j] >> c) & 1u); }
#define PLAN_PRED_SWITCH(XT, LOADX)                                       \
            switch (op) {                                                 \
            case 0: PLAN_PRED(XT, LOADX, x == lo) break;                  \
            case 1: PLAN_PRED(XT, LOADX, x != lo) break;                  \
            case 2: PLAN_PRED(XT, LOADX, x > lo) break;                   \
            case 3: PLAN_PRED(XT, LOADX, x >= lo) break;                  \
            case 4: PLAN_PRED(XT, LOADX, x < lo) break;                   \
            case 5: PLAN_PRED(XT, LOADX, x <= lo) break;                  \
            default: PLAN_PRED(XT, LOADX, x >= lo && x <= hi) break;      /* BETWEEN, inclusive (operator_between.go:138-199) */ \
            }
            if (mode == 1) {
                const long long lo = X.ilo[q], hi = X.ihi[q];
                PLAN_PRED_SWITCH(long long, (long long)PLAN_SLOT(pc, j))
            } else if (mode == 2) {
                const unsigned long long lo = (unsigned long long)X.ilo[q], hi = (unsigned long long)X.ihi[q];
                PLAN_PRED_SWITCH(unsigned long long, PLAN_SLOT(pc, j))
            } else if (mode == 0) {
                const double lo = P.pred[q].lo, hi = P.pred[q].hi;
                PLAN_PRED_SWITCH(double, __longlong_as_double((long long)PLAN_SLOT(pc, j)))
            } else {
                const bool t = mode == 4;
                PLAN_FORJ ok[j] = ok[j] && t && !((nb[j] >> c) & 1u);
            }
        }
        if (!P.has_null_keys && X.key_nulls) { const unsigned kn = X.key_nulls; PLAN_FORJ ok[j] = ok[j] && !(nb[j] & kn); }   // fillKeys: zValues[i] = 0
        if (!(ok[0] | ok[1] | ok[2] | ok[3])) continue;
        // ---- group keys (fillKeys): one column at a time.  BEFORE the projection: keys only read column slots, which the expression nodes may reuse
        uint64_t keys[R];
        PLAN_FORJ keys[j] = 0;
        if (!P.has_null_keys) {
            for (int k = 0; k < P.nkeys; k++) {
                const int c = P.key_col[k], mode = X.key_mode[k], sh = X.key_shift[k];
                const uint64_t mask = X.sz[c] < 8 ? (1ull << (8 * X.sz[c])) - 1ull : ~0ull;
                const int pc = X.phys[c];
                PLAN_FORJ if (ok[j]) keys[j] |= (plan_key_bits(mode, PLAN_SLOT(pc, j), C.data[c], r0 + (uint64_t)j * kThreads) & mask) << sh;
            }
        } else {   // has_null mode: a marker byte per column, a NULL contributes the marker only -> the byte offset depends on the row
            PLAN_FORJ {
                if (ok[j]) {
                    int off = 0; uint64_t key = 0;
                    for (int k = 0; k < P.nkeys; k++) {
                        const int c = P.key_col[k], sz = X.sz[c];
                        if ((nb[j] >> c) & 1u) { key |= 1ull << (8 * off); off += 1; continue; }
                        off += 1;
                        uint64_t raw = plan_key_bits(X.key_mode[k], PLAN_SLOT(X.phys[c], j), C.data[c], r0 + (uint64_t)j * kThreads);
                        if (sz < 8) raw &= (1ull << (8 * sz)) - 1ull;
                        if (off < 8) key |= raw << (8 * off);
                        off += sz;
                    }
                    keys[j] = key;
                }
            }
        }
        // ---- projection: SSA program over float64 slots, one rounding per node (the reference evaluates one expression node at a time too)
        for (int i = 0; i < P.ninstr; i++) {
            const int dst = P.ncols + i, op = P.instr[i].op, sa = P.instr[i].a, sb = P.instr[i].b;
            const int pd = X.phys[dst], pa = op != MO_PLAN_OP_CONST ? X.phys[sa] : 0, pb = op >= MO_PLAN_OP_ADD ? X.phys[sb] : 0;   // null bits are per VALUE slot, storage per physical slot
#define PLAN_A __longlong_as_double((long long)PLAN_SLOT(pa, j))
#define PLAN_B __longlong_as_double((long long)PLAN_SLOT(pb, j))
#define PLAN_BIN(EXPR) PLAN_FORJ { const double a = PLAN_A, b = PLAN_B; PLAN_SLOT(pd, j) = (unsigned long long)__double_as_longlong(EXPR); \
                                   nb[j] |= (((nb[j] >> sa) | (nb[j] >> sb)) & 1u) << dst; }
            switch (op) {
            case MO_PLAN_OP_CONST: { const unsigned long long imm = (unsigned long long)__double_as_longlong(P.instr[i].imm); PLAN_FORJ PLAN_SLOT(pd, j) = imm; } break;
            case MO_PLAN_OP_COL: PLAN_FORJ { PLAN_SLOT(pd, j) = PLAN_SLOT(pa, j); nb[j] |= ((nb[j] >> sa) & 1u) << dst; } break;
            case MO_PLAN_OP_ADD: PLAN_BIN(__dadd_rn(a, b)) break;
            case MO_PLAN_OP_SUB: PLAN_BIN(__dsub_rn(a, b)) break;
            case MO_PLAN_OP_MUL: PLAN_BIN(__dmul_rn(a, b)) break;
            default:             // x / 0 -> NULL (SELECT behaviour)
                PLAN_FORJ { const double a = PLAN_A, b = PLAN_B; const bool z = b == 0.0;
                            PLAN_SLOT(pd, j) = (unsigned long long)__double_as_longlong(z ? 0.0 : __ddiv_rn(a, b));
                            nb[j] |= ((((nb[j] >> sa) | (nb[j] >> sb)) & 1u) | (z ? 1u : 0u)) << dst; }
                break;
            }
        }
        // ---- private-dictionary lookup per row (the dictionary state is sequential)
        int ps[R];
        PLAN_FORJ {
            ps[j] = -1;
            if (ok[j]) {
                const uint64_t key = keys[j];
                const bool sentinel = key == kEmptyKey;    // the all-ones key is also the empty-entry marker: it never gets private state
                int p = -1;
#pragma unroll
                for (int g = 0; g < kPriv; g++) if (dk[g] == key && !sentinel) p = g;
                if (p < 0 && !dict_full && !sentinel) {
                    bool okc = false;
#pragma unroll
                    for (int g = 0; g < kPriv; g++) {
                        const unsigned long long prev = okc ? key : atomicCAS(&pdict[g], (unsigned long long)kEmptyKey, (unsigned long long)key);
                        okc = okc || prev == kEmptyKey || prev == key;
                    }
                    bool full = true;
#pragma unroll
                    for (int g = 0; g < kPriv; g++) { dk[g] = ((volatile unsigned long long *)pdict)[g]; full = full && dk[g] != kEmptyKey; if (dk[g] == key) p = g; }
                    dict_full = full;
                }
                ps[j] = p;
                if (p >= 0) {
                    prows[p * kThreads] += 1u;
                    if (pfirst[p * kThreads] == ~0ull) pfirst[p * kThreads] = (uint64_t)P.row_base + r0 + (uint64_t)j * kThreads;   // a thread meets its rows in increasing order
                }
            }
        }
        // ---- the aggregates, COLUMN AT A TIME over the thread's rows that live in private state
        for (int a = 0; a < naggs; a++) {
            const int vs = P.agg[a].value, kind = P.agg[a].kind;
            const int ab = a * kThreads, gstride = naggs * kThreads, pv = vs >= 0 ? X.phys[vs] : 0;
            if (vs < 0) { if (X.need_cnt) { PLAN_FORJ if (ps[j] >= 0) pcnt[ps[j] * gstride + ab] += 1u; } continue; }          // COUNT(*)
            if (X.need_cnt) { PLAN_FORJ if (ps[j] >= 0 && !((nb[j] >> vs) & 1u)) pcnt[ps[j] * gstride + ab] += 1u; }
            if (kind == MO_AGG_SUM || kind == MO_AGG_AVG) {
                PLAN_FORJ if (ps[j] >= 0 && !((nb[j] >> vs) & 1u)) { const int ix = ps[j] * gstride + ab; pacc[ix] = __dadd_rn(pacc[ix], __longlong_as_double((long long)PLAN_SLOT(pv, j))); }
            } else if (kind == MO_AGG_MIN) {
                PLAN_FORJ if (ps[j] >= 0 && !((nb[j] >> vs) & 1u)) {
                    const double v = __longlong_as_double((long long)PLAN_SLOT(pv, j)); const int ix = ps[j] * gstride + ab;
                    if (v == v) { const unsigned long long kv = flt_key(v); if (kv < (unsigned long long)__double_as_longlong(pacc[ix])) pacc[ix] = __longlong_as_double((long long)kv); }
                }
            } else if (kind == MO_AGG_MAX) {
                PLAN_FORJ if (ps[j] >= 0 && !((nb[j] >> vs) & 1u)) {
                    const double v = __longlong_as_double((long long)PLAN_SLOT(pv, j)); const int ix = ps[j] * gstride + ab;
                    if (v == v) { const unsigned long long kv = flt_key(v); if (kv > (unsigned long long)__double_as_longlong(pacc[ix])) pacc[ix] = __longlong_as_double((long long)kv); }
                }
            }
        }
        // ---- rows whose key is not in the private dictionary: shared CTA table, then the global table
        PLAN_FORJ {
            if (ok[j] && ps[j] < 0) {
                const unsigned nullbits = nb[j];
                const uint64_t key = keys[j];
                const uint64_t grow = (uint64_t)P.row_base + r0 + (uint64_t)j * kThreads;
                int slot = -1;
                if (key != kEmptyKey) {   // the CTA table has no all-ones key slot: that key goes to the global table
                    unsigned s;
                    if (kt_insert(tkey, (unsigned)(kCtaSlots - 1), key, s)) slot = (int)s;
                }
                unsigned long long *first_p = slot >= 0 ? &tfirst[slot] : nullptr, *rows_p = slot >= 0 ? &trows[slot] : nullptr;
                double *acc_p = slot >= 0 ? &tacc[slot * naggs] : nullptr; unsigned long long *cnt_p = slot >= 0 ? &tcnt[slot * naggs] : nullptr;
                bool have = true;
                if (slot < 0) {
                    uint64_t gs;
                    if (!global_find(G, key, gs)) have = false;
                    else { first_p = &G.first_row[gs]; rows_p = &G.rows[gs]; acc_p = &G.acc[gs * naggs]; cnt_p = &G.cnt[gs * naggs]; }
                }
                if (have) {
                    first_row_min(first_p, grow);
                    atomicAdd(rows_p, 1ull);
                    for (int a = 0; a < naggs; a++) {
                        const int vs = P.agg[a].value;
                        if (vs < 0) { atomicAdd(&cnt_p[a], 1ull); continue; }            // COUNT(*)
                        if ((nullbits >> vs) & 1u) continue;                             // aggregates skip NULLs
                        agg_apply(P.agg[a].kind, &acc_p[a], __longlong_as_double((long long)PLAN_SLOT(X.phys[vs], j)));
                        atomicAdd(&cnt_p[a], 1ull);
                    }
                }
            }
        }
    }
    // ---- retire: the CTA first folds its threads' private states (one thread per (group, aggregate), a fixed order), then touches the global
    // table once per (group, aggregate) instead of once per thread
    __syncthreads();
    for (int ga = threadIdx.x; ga < kPriv * naggs; ga += kThreads) {
        const int g = ga / naggs, a = ga % naggs, kind = P.agg[a].kind;
        const unsigned long long pk = pdict[g];
        if (pk == kEmptyKey) continue;
        double acc = agg_identity(kind); unsigned long long cnt = 0;
        for (int t = 0; t < kThreads; t++) {
            const int ix = ga * kThreads + t;
            const unsigned long long c = X.need_cnt ? pcnt0[ix] : prows0[g * kThreads + t];   // without per-aggregate counts every row of the group fed every aggregate
            if (c == 0) continue;
            cnt += c;
            const double v = pacc0[ix];
            if (kind == MO_AGG_SUM || kind == MO_AGG_AVG) acc = __dadd_rn(acc, v);
            else if (kind == MO_AGG_MIN) { if ((unsigned long long)__double_as_longlong(v) < (unsigned long long)__double_as_longlong(acc)) acc = v; }
            else if (kind == MO_AGG_MAX) { if ((unsigned long long)__double_as_longlong(v) > (unsigned long long)__double_as_longlong(acc)) acc = v; }
        }
        if (cnt == 0) continue;
        uint64_t gs;
        if (!global_find(G, pk, gs)) continue;
        agg_fold(kind, &G.acc[gs * naggs + a], acc);
        atomicAdd(&G.cnt[gs * naggs + a], cnt);
    }
    for (int g = threadIdx.x; g < kPriv; g += kThreads) {
        const unsigned long long pk = pdict[g];
        if (pk == kEmptyKey) continue;
        unsigned long long rows = 0, first = ~0ull;
        for (int t = 0; t < kThreads; t++) { rows += prows0[g * kThreads + t]; const unsigned long long f = pfirst0[g * kThreads + t]; if (f < first) first = f; }
        if (rows == 0) continue;
        uint64_t gs;
        if (!global_find(G, pk, gs)) continue;
        atomicMin(&G.first_row[gs], first);
        atomicAdd(&G.rows[gs], rows);
    }
    // ---- and the shared CTA table
    for (int s = threadIdx.x; s < kCtaSlots; s += kThreads) {
        if (tkey[s] == kEmptyKey || trows[s] == 0) continue;
        uint64_t gs;
        if (!global_find(G, tkey[s], gs)) continue;
        atomicMin(&G.first_row[gs], tfirst[s]);
        atomicAdd(&G.rows[gs], trows[s]);
        for (int a = 0; a < naggs; a++) {
            if (tcnt[s * naggs + a] == 0) continue;
            agg_fold(P.agg[a].kind, &G.acc[gs * naggs + a], tacc[s * naggs + a]);
            atomicAdd(&G.cnt[gs * naggs + a], tcnt[s * naggs + a]);
        }
    }
}

// collect the used slots, order them by first row (= the reference's group-id order) and write the result records
__global__ void plan_collect_kernel(PlanGlobal G, uint32_t *used, unsigned long long *nused) {
    for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s <= G.mask + 1; s += (uint64_t)gridDim.x * blockDim.x)
        if (G.rows[s] != 0) { const unsigned long long i = atomicAdd(nused, 1ull); used[i] = (uint32_t)s; }
}
__global__ void plan_emit_kernel(PlanGlobal G, const mo_plan_t *P, const uint32_t *used, const unsigned long long *nused, uint8_t *res, uint64_t res_cap_groups,
                                 int sort_limit) {
    const unsigned long long ng = *nused;
    const int naggs = P->naggs;
    const size_t rec = sizeof(mo_plan_group_t) + sizeof(mo_plan_agg_value_t) * (size_t)naggs;
    mo_plan_result_header_t *H = reinterpret_cast<mo_plan_result_header_t *>(res);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        H->ngroups = (int64_t)ng; H->sorted = ng <= (unsigned long long)sort_limit ? 1 : 0; H->overflow = (*G.overflow || ng > res_cap_groups) ? 1 : 0; H->reserved = 0;
    }
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < ng; i += (unsigned long long)gridDim.x * blockDim.x) {
        const uint32_t s = used[i];
        unsigned long long pos = i;
        if (ng <= (unsigned long long)sort_limit) {   // rank by first row: the reference numbers groups in first-seen order
            pos = 0;
            const unsigned long long f = G.first_row[s];
            for (unsigned long long j = 0; j < ng; j++) { const unsigned long long fj = G.first_row[used[j]]; pos += (fj < f || (fj == f && j < i)) ? 1 : 0; }
        }
        if (pos >= res_cap_groups) continue;
        mo_plan_group_t *g = reinterpret_cast<mo_plan_group_t *>(res + sizeof(mo_plan_result_header_t) + rec * pos);
        g->key = G.key[s]; g->first_row = (int64_t)G.first_row[s]; g->rows = (int64_t)G.rows[s];
        mo_plan_agg_value_t *av = reinterpret_cast<mo_plan_agg_value_t *>(g + 1);
        for (int a = 0; a < naggs; a++) {
            const int kind = P->agg[a].kind;
            const unsigned long long c = G.cnt[(size_t)s * naggs + a];
            double v = G.acc[(size_t)s * naggs + a];
            if (kind == MO_AGG_MIN || kind == MO_AGG_MAX) v = c ? flt_unkey((unsigned long long)__double_as_longlong(v)) : 0.0;
            else if (kind == MO_AGG_AVG) v = c ? v / (double)c : 0.0;          // float64(sum) / float64(cnt), sumavg2.go:331
            else if (kind == MO_AGG_COUNT) v = (double)c;
            av[a].value = v; av[a].count = (int64_t)c;                          // count == 0: the aggregate is NULL (COUNT: 0)
        }
    }
}

// ---- recognised shapes: the two hand-specialised instances of this operator (tpch.cu) ---------------------------------------------------
// A descriptor that IS the Q6 shape  SUM(c3 * c1) WHERE c0 >= lo AND c0 < hi AND c1 BETWEEN a AND b AND c2 < q  over (DATE, f64, f64, f64)
// or the Q1 shape (q1.sql: filter c0 <= cutoff, keys (c5, c6) uint8, the eight aggregates in select-list order) over non-nullable resident or
// host columns runs the specialised kernel, which streams at the HBM roofline; the result is rewritten in this operator's record format.
struct Q6Out { double sum; long long rows; };
__global__ void plan_from_q6_kernel(const Q6Out *q, uint8_t *res) {
    mo_plan_result_header_t *H = reinterpret_cast<mo_plan_result_header_t *>(res);
    H->ngroups = q->rows ? 1 : 0; H->sorted = 1; H->overflow = 0; H->reserved = 0;
    if (q->rows) {
        mo_plan_group_t *g = reinterpret_cast<mo_plan_group_t *>(res + sizeof(mo_plan_result_header_t));
        g->key = 0; g->first_row = -1; g->rows = q->rows;     // the specialised kernel does not track the first qualifying row
        mo_plan_agg_value_t *a = reinterpret_cast<mo_plan_agg_value_t *>(g + 1);
        a->value = q->sum; a->count = q->rows;
    }
}
__global__ void plan_from_q1_kernel(const mo_q1_result_t *q, uint8_t *res, uint64_t res_groups, int *fallback) {
    mo_plan_result_header_t *H = reinterpret_cast<mo_plan_result_header_t *>(res);
    if (q->ngroups < 0 || (uint64_t)q->ngroups > res_groups) { *fallback = 1; return; }   // more than 8 groups: the generic path answers
    *fallback = 0;
    H->ngroups = q->ngroups; H->sorted = 1; H->overflow = 0; H->reserved = 0;
    const size_t rec = sizeof(mo_plan_group_t) + 8 * sizeof(mo_plan_agg_value_t);
    for (int64_t i = 0; i < q->ngroups; i++) {
        const mo_q1_group_t &s = q->groups[i];
        mo_plan_group_t *g = reinterpret_cast<mo_plan_group_t *>(res + sizeof(mo_plan_result_header_t) + rec * i);
        g->key = (uint64_t)s.returnflag | ((uint64_t)s.linestatus << 8); g->first_row = s.first_row; g->rows = s.count_order;
        mo_plan_agg_value_t *a = reinterpret_cast<mo_plan_agg_value_t *>(g + 1);
        const double v[8] = {s.sum_qty, s.sum_base_price, s.sum_disc_price, s.sum_charge, s.avg_qty, s.avg_price, s.avg_disc, (double)s.count_order};
        for (int k = 0; k < 8; k++) { a[k].value = v[k]; a[k].count = s.count_order; }
    }
}

static bool is_q6_shape(const mo_plan_t &P) {
    if (P.ncols != 4 || P.npreds != 4 || P.ninstr != 1 || P.nkeys != 0 || P.naggs != 1) return false;
    if ((P.col_type[0] != MO_T_DATE && P.col_type[0] != MO_T_INT32) || P.col_type[1] != MO_T_FLOAT64 || P.col_type[2] != MO_T_FLOAT64 || P.col_type[3] != MO_T_FLOAT64) return false;
    const mo_plan_pred_t *q = P.pred;
    if (q[0].col != 0 || q[0].op != 3 || q[1].col != 0 || q[1].op != 4 || q[2].col != 1 || q[2].op != 6 || q[3].col != 2 || q[3].op != 4) return false;
    if (q[0].lo != (double)(int32_t)q[0].lo || q[1].lo != (double)(int32_t)q[1].lo) return false;
    const mo_plan_instr_t &m = P.instr[0];
    if (m.op != MO_PLAN_OP_MUL || !((m.a == 3 && m.b == 1) || (m.a == 1 && m.b == 3))) return false;
    return P.agg[0].kind == MO_AGG_SUM && P.agg[0].value == 4;
}
static bool is_q1_shape(const mo_plan_t &P) {
    if (P.ncols != 7 || P.npreds != 1 || P.ninstr != 5 || P.nkeys != 2 || P.naggs != 8 || P.has_null_keys) return false;
    if (P.col_type[0] != MO_T_DATE && P.col_type[0] != MO_T_INT32) return false;
    for (int c = 1; c <= 4; c++) if (P.col_type[c] != MO_T_FLOAT64) return false;
    if (P.col_type[5] != MO_T_UINT8 || P.col_type[6] != MO_T_UINT8 || P.key_col[0] != 5 || P.key_col[1] != 6) return false;
    if (P.pred[0].col != 0 || P.pred[0].op != 5 || P.pred[0].lo != (double)(int32_t)P.pred[0].lo) return false;
    const mo_plan_instr_t *in = P.instr;
    if (in[0].op != MO_PLAN_OP_CONST || in[0].imm != 1.0) return false;
    if (in[1].op != MO_PLAN_OP_SUB || in[1].a != 7 || in[1].b != 3) return false;
    if (in[2].op != MO_PLAN_OP_MUL || in[2].a != 2 || in[2].b != 8) return false;
    if (in[3].op != MO_PLAN_OP_ADD || in[3].a != 7 || in[3].b != 4) return false;
    if (in[4].op != MO_PLAN_OP_MUL || in[4].a != 9 || in[4].b != 10) return false;
    const int kind[8] = {MO_AGG_SUM, MO_AGG_SUM, MO_AGG_SUM, MO_AGG_SUM, MO_AGG_AVG, MO_AGG_AVG, MO_AGG_AVG, MO_AGG_COUNT};
    const int val[8] = {1, 2, 9, 11, 1, 2, 3, -1};
    for (int a = 0; a < 8; a++) if (P.agg[a].kind != kind[a] || P.agg[a].value != val[a]) return false;
    return true;
}

}  // namespace

namespace mob {

int q6_run(ThreadCtx &t, Stager &st, const uint8_t *const cols[4], uint64_t len, const mo_q6_params_t &P, double *res, uint64_t res_words,
           uint64_t *rnulls);
int q1_run(ThreadCtx &t, Stager &st, const uint8_t *const cols[7], bool varlena, uint64_t len, int32_t cutoff, int64_t row_base,
           mo_q1_result_t *res);
extern int g_plan_specialise;   // MoB200_SetTuning("plan_specialise", 0) forces the interpreter (tests, profiling)

// Runs the specialised kernel when the descriptor is the Q6 or Q1 shape over non-nullable columns and sets *answered; otherwise (and when
// the Q1 scan finds more groups than the result can take) the interpreter must run.
static int plan_try_specialised(ThreadCtx &t, const mo_plan_t &P, mo_xcall_args_t *args, uint64_t len, uint64_t res_groups, bool *answered) {
    *answered = false;
    if (!g_plan_specialise || len == 0) return MO_RC_SUCCESS;
    for (int c = 0; c < P.ncols; c++) if (args[2 + c].pnulls) return MO_RC_SUCCESS;
    const bool q6 = is_q6_shape(P), q1 = !q6 && is_q1_shape(P);
    if (!q6 && !q1) return MO_RC_SUCCESS;
    Stager st(t);
    const uint8_t *cols[7];
    for (int c = 0; c < P.ncols; c++) { cols[c] = args[2 + c].pdata; st.device(cols[c]); }   // residency decides the Q1 fallback below
    // the kernels below write the header and the groups they found: the rest of a host result is uploaded first so that the copy-back keeps it
    const uint64_t ngroups_max = q6 ? 1 : std::min<uint64_t>(res_groups, MO_Q1_MAX_GROUPS);
    uint8_t *dres = (uint8_t *)st.out(args[0].pdata, sizeof(mo_plan_result_header_t) + (sizeof(mo_plan_group_t) + sizeof(mo_plan_agg_value_t) * P.naggs) * ngroups_max, true);
    void *dq = st.tmp(q6 ? sizeof(Q6Out) : sizeof(mo_q1_result_t));
    int *dflag = (int *)st.tmp(4);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    if (q6) {
        const mo_q6_params_t Q{(int32_t)P.pred[0].lo, (int32_t)P.pred[1].lo, P.pred[2].lo, P.pred[2].hi, P.pred[3].lo};
        const int rc = q6_run(t, st, cols, len, Q, (double *)dq, 2, nullptr);
        if (rc) return rc;
        plan_from_q6_kernel<<<1, 1, 0, t.stream>>>((const Q6Out *)dq, dres);
        MOB_LAUNCH_CHECK();
    } else {
        int rc = q1_run(t, st, cols, false, len, (int32_t)P.pred[0].lo, P.row_base, (mo_q1_result_t *)dq);
        if (rc == MO_RC_INVALID_ARGUMENT && !st.resident()) return st.finish();   // host columns with device ones, or unaligned: the interpreter takes them
        if (rc) return rc;
        plan_from_q1_kernel<<<1, 1, 0, t.stream>>>((const mo_q1_result_t *)dq, dres, res_groups, dflag);
        MOB_LAUNCH_CHECK();
        // more than the result's groups cannot be known without this read-back
        int fallback = 0;
        rc = read_back(t, &fallback, dflag, 4);
        if (rc) return rc;
        if (fallback) return st.finish();
    }
    *answered = true;
    return st.complete();
}

// MO_XCALL_PLAN: args [0] result buffer ; [1] mo_plan_t ; [2 .. 2 + ncols) the columns (+pnulls).  len = rows.  See include/mo_b200.h.
int xcall_plan(mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    mo_plan_t P;
    if (int rc = read_param(t, args[1], &P, sizeof P, sizeof P, "plan: mo_plan_t descriptor")) return rc;
    if (P.ncols < 1 || P.ncols > MO_PLAN_MAX_COLS || P.npreds < 0 || P.npreds > MO_PLAN_MAX_PREDS || P.ninstr < 0 || P.ninstr > MO_PLAN_MAX_INSTR ||
        P.nkeys < 0 || P.nkeys > MO_PLAN_MAX_KEYS || P.naggs < 1 || P.naggs > MO_PLAN_MAX_AGGS) { set_error("plan: descriptor counts out of range"); return MO_RC_INVALID_ARGUMENT; }
    int keybytes = 0;
    auto tbytes = [](int T) { return (T == MO_T_BOOL || T == MO_T_INT8 || T == MO_T_UINT8) ? 1 : (T == MO_T_INT16 || T == MO_T_UINT16) ? 2 : (T == MO_T_INT32 || T == MO_T_UINT32 || T == MO_T_FLOAT32 || T == MO_T_DATE) ? 4 : 8; };
    for (int c = 0; c < P.ncols; c++) {
        const int T = P.col_type[c];
        if (!((T >= MO_T_INT8 && T <= MO_T_INT64) || (T >= MO_T_UINT8 && T <= MO_T_UINT64) || T == MO_T_BOOL || T == MO_T_FLOAT32 || T == MO_T_FLOAT64 || (T >= MO_T_DATE && T <= MO_T_TIMESTAMP))) { set_error("plan: column %d has unsupported type %d", c, T); return MO_RC_INVALID_ARGUMENT; }
        if (args[2 + c].dataSz < (uint64_t)tbytes(T) * len) { set_error("plan: column %d shorter than len", c); return MO_RC_INVALID_ARGUMENT; }
    }
    for (int j = 0; j < P.npreds; j++) if (P.pred[j].col < 0 || P.pred[j].col >= P.ncols || P.pred[j].op < 0 || P.pred[j].op > 6) { set_error("plan: predicate %d malformed", j); return MO_RC_INVALID_ARGUMENT; }
    for (int i = 0; i < P.ninstr; i++) {
        const mo_plan_instr_t &in = P.instr[i];
        const int lim = P.ncols + i;   // operands: columns or EARLIER instructions (SSA)
        const bool ok = in.op == MO_PLAN_OP_CONST || (in.op == MO_PLAN_OP_COL && in.a >= 0 && in.a < P.ncols) ||
                        (in.op >= MO_PLAN_OP_ADD && in.op <= MO_PLAN_OP_DIV && in.a >= 0 && in.a < lim && in.b >= 0 && in.b < lim);
        if (!ok) { set_error("plan: instruction %d malformed", i); return MO_RC_INVALID_ARGUMENT; }
    }
    for (int k = 0; k < P.nkeys; k++) {
        if (P.key_col[k] < 0 || P.key_col[k] >= P.ncols) { set_error("plan: key column %d out of range", k); return MO_RC_INVALID_ARGUMENT; }
        keybytes += tbytes(P.col_type[P.key_col[k]]) + (P.has_null_keys ? 1 : 0);
    }
    if (keybytes > 8) { set_error("plan: %d key bytes exceed the 8-byte IntHashMap key (group/exec2.go:73-118)", keybytes); return MO_RC_INVALID_ARGUMENT; }
    for (int a = 0; a < P.naggs; a++) {
        const mo_plan_agg_t &g = P.agg[a];
        if (g.kind < MO_AGG_SUM || g.kind > MO_AGG_AVG || g.value >= P.ncols + P.ninstr || (g.value < 0 && g.kind != MO_AGG_COUNT)) { set_error("plan: aggregate %d malformed", a); return MO_RC_INVALID_ARGUMENT; }
    }
    const size_t rec = sizeof(mo_plan_group_t) + sizeof(mo_plan_agg_value_t) * (size_t)P.naggs;
    if (!args[0].pdata || args[0].dataSz < sizeof(mo_plan_result_header_t) + rec) { set_error("plan: result buffer too small for one group"); return MO_RC_INVALID_ARGUMENT; }
    const uint64_t res_groups = (args[0].dataSz - sizeof(mo_plan_result_header_t)) / rec;
    {
        bool answered = false;
        const int rc = plan_try_specialised(t, P, args, len, res_groups, &answered);
        if (rc || answered) return rc;
    }
    Stager st(t);
    PlanCols C;
    for (int c = 0; c < MO_PLAN_MAX_COLS; c++) { C.data[c] = nullptr; C.nulls[c] = nullptr; }
    for (int c = 0; c < P.ncols; c++) {
        C.data[c] = (const uint8_t *)st.in(args[2 + c].pdata, (size_t)tbytes(P.col_type[c]) * len);
        C.nulls[c] = (const uint64_t *)st.in(args[2 + c].pnulls, args[2 + c].pnulls ? ((len + 63) / 64) * 8 : 0);
    }
    uint8_t *dres = (uint8_t *)st.out(args[0].pdata, sizeof(mo_plan_result_header_t) + rec * res_groups);
    // global table: twice the groups the caller's buffer can take (min 1024 slots)
    uint64_t cap = 1024;
    while (cap < 2 * res_groups && cap < (1ull << 30)) cap <<= 1;
    PlanGlobal G;
    G.mask = cap - 1;
    G.key = (uint64_t *)st.tmp((cap + 1) * 8); G.first_row = (unsigned long long *)st.tmp((cap + 1) * 8); G.rows = (unsigned long long *)st.tmp((cap + 1) * 8);
    G.acc = (double *)st.tmp((cap + 1) * 8 * P.naggs); G.cnt = (unsigned long long *)st.tmp((cap + 1) * 8 * P.naggs);
    uint32_t *used = (uint32_t *)st.tmp((cap + 1) * 4);
    unsigned long long *nused = (unsigned long long *)st.tmp(16);
    mo_plan_t *dP = (mo_plan_t *)st.tmp(sizeof(mo_plan_t));
    PlanAux *dX = (PlanAux *)st.tmp(sizeof(PlanAux));
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    G.overflow = (unsigned *)(nused + 1);
    MOB_CUDA_TRY(cudaMemsetAsync(nused, 0, 16, t.stream));
    // the descriptor travels through the thread's pinned staging buffer (the caller's copy may be pageable and short-lived)
    if (sizeof(mo_plan_t) + sizeof(PlanAux) > t.pinned_sz) { st.finish(); set_error("plan: descriptor larger than the staging buffer"); return MO_RC_INTERNAL_ERROR; }
    // decode once on the host: the domain of every column slot (raw int64 or float64), which predicates compare as integers, how the group
    // key reads its columns, whether per-aggregate counts are needed
    PlanAux X;
    memset(&X, 0, sizeof X);
    {
        auto is_float = [](int T) { return T == MO_T_FLOAT32 || T == MO_T_FLOAT64; };
        bool value_use[MO_PLAN_MAX_COLS] = {false}, f64dom[MO_PLAN_MAX_COLS];
        for (int i = 0; i < P.ninstr; i++) {
            const mo_plan_instr_t &in = P.instr[i];
            if (in.op == MO_PLAN_OP_CONST) continue;
            if (in.a < P.ncols) value_use[in.a] = true;
            if (in.op >= MO_PLAN_OP_ADD && in.b < P.ncols) value_use[in.b] = true;
        }
        for (int a = 0; a < P.naggs; a++) if (P.agg[a].value >= 0 && P.agg[a].value < P.ncols) value_use[P.agg[a].value] = true;
        for (int c = 0; c < P.ncols; c++) { f64dom[c] = is_float(P.col_type[c]) || value_use[c]; X.raw_phys[c] = -1; }
        // A predicate on an integer column compares the value with the float64 constant exactly (what the reference computes once the planner
        // has cast the constant to the column type): x > c <=> x > floor(c), x >= c <=> x >= ceil(c), == a non-integral c never holds.  The
        // integral bound is then compared in the 64-bit integer domain of the slot (unsigned for UINT64); a bound outside it decides the
        // predicate for every row.  A NaN constant follows IEEE: only != holds.
        const double two63 = 9223372036854775808.0, two64 = 18446744073709551616.0, two53 = 9007199254740992.0;
        int nphys = P.ncols;
        for (int j = 0; j < P.npreds; j++) {
            const mo_plan_pred_t &q = P.pred[j];
            const int c = q.col, T = P.col_type[c];
            X.pred_slot[j] = c;
            X.pred_mode[j] = 0;
            if (is_float(T)) continue;
            const bool uns = T == MO_T_UINT64;
            const double dmin = uns ? 0.0 : -two63, dmax = uns ? two64 : two63;   // the domain is [dmin, dmax)
            auto to_int = [&](double t) { return uns ? (long long)(unsigned long long)t : (long long)t; };
            int mode = uns ? 2 : 1;
            double lo = 0.0, hi = 0.0;
            if (q.op == 6) {
                lo = std::ceil(q.lo); hi = std::floor(q.hi);
                if (q.lo != q.lo || q.hi != q.hi || lo >= dmax || hi < dmin) mode = 3;
                else { lo = lo < dmin ? dmin : lo; X.ilo[j] = to_int(lo); X.ihi[j] = hi >= dmax ? (uns ? -1ll : 0x7fffffffffffffffll) : to_int(hi); }
            } else if (q.lo != q.lo) {
                mode = q.op == 1 ? 4 : 3;
            } else {
                lo = (q.op == 2 || q.op == 5) ? std::floor(q.lo) : (q.op == 3 || q.op == 4) ? std::ceil(q.lo) : q.lo;
                if ((q.op == 0 || q.op == 1) && lo != std::floor(lo)) mode = q.op == 1 ? 4 : 3;     // == a non-integral constant
                else if (lo >= dmax) mode = (q.op == 1 || q.op == 4 || q.op == 5) ? 4 : 3;            // above every value (also +inf)
                else if (lo < dmin) mode = (q.op == 1 || q.op == 2 || q.op == 3) ? 4 : 3;             // below every value (also -inf)
                else X.ilo[j] = to_int(lo);
            }
            X.pred_mode[j] = mode;
            if (!f64dom[c] || mode > 2) continue;
            // the column's slot holds float64(x): exact for a bound below 2^53 in magnitude (rounding is monotonic and c +- 1 are
            // representable), so the float64 compare with the original constant is kept; larger bounds read a raw copy of the column
            if (std::fabs(lo) < two53 && (q.op != 6 || std::fabs(hi) < two53)) { X.pred_mode[j] = 0; continue; }
            if (X.raw_phys[c] < 0) X.raw_phys[c] = nphys++;
            X.pred_slot[j] = X.raw_phys[c];
        }
        X.key_nulls = 0;
        for (int k = 0; k < P.nkeys; k++) if (args[2 + P.key_col[k]].pnulls) X.key_nulls |= 1u << P.key_col[k];
        for (int c = 0; c < P.ncols; c++) {
            const int T = P.col_type[c];
            X.sz[c] = tbytes(T);
            X.ext[c] = T == MO_T_INT8 ? 1 : T == MO_T_INT16 ? 2 : (T == MO_T_INT32 || T == MO_T_DATE) ? 3 : 0;
            X.tof[c] = T == MO_T_FLOAT32 ? 3 : T == MO_T_FLOAT64 ? 0 : !f64dom[c] ? 0 : T == MO_T_UINT64 ? 2 : 1;
        }
        int shift = 0;
        for (int k = 0; k < P.nkeys; k++) {
            const int c = P.key_col[k], T = P.col_type[c];
            X.key_mode[k] = T == MO_T_FLOAT32 ? 3 : T == MO_T_FLOAT64 ? 4 : !f64dom[c] ? 0 : X.sz[c] < 8 ? 1 : 2;
            X.key_shift[k] = shift < 64 ? shift : 63;
            shift += 8 * X.sz[c];
        }
        // an aggregate input can be NULL iff a nullable column or a division feeds it (null-ness only flows forward through the SSA program)
        bool maybe[MO_PLAN_MAX_COLS + MO_PLAN_MAX_INSTR];
        for (int c = 0; c < P.ncols; c++) maybe[c] = args[2 + c].pnulls != nullptr;
        for (int i = 0; i < P.ninstr; i++) {
            const mo_plan_instr_t &in = P.instr[i];
            maybe[P.ncols + i] = in.op == MO_PLAN_OP_CONST ? false : in.op == MO_PLAN_OP_COL ? maybe[in.a] : (in.op == MO_PLAN_OP_DIV || maybe[in.a] || maybe[in.b]);
        }
        for (int a = 0; a < P.naggs; a++) if (P.agg[a].value >= 0 && maybe[P.agg[a].value]) X.need_cnt = 1;
    }
    {
        // liveness-based slot allocation: the SSA program gives every node its own value slot; in shared memory a slot is reused once its value is
        // dead.  Times: 0 load, 1 filter, 2 group keys, 3 + i expression node i, 3 + ninstr aggregates.
        const int nv = P.ncols + P.ninstr, t_agg = 3 + P.ninstr;
        int last[MO_PLAN_MAX_COLS + MO_PLAN_MAX_INSTR];
        for (int v = 0; v < nv; v++) last[v] = v < P.ncols ? 0 : -1;
        auto use = [&](int v, int when) { if (v >= 0 && v < nv && last[v] < when) last[v] = when; };
        for (int j = 0; j < P.npreds; j++) use(P.pred[j].col, 1);
        for (int k = 0; k < P.nkeys; k++) use(P.key_col[k], 2);
        for (int i = 0; i < P.ninstr; i++) {
            const mo_plan_instr_t &in = P.instr[i];
            if (in.op != MO_PLAN_OP_CONST) use(in.a, 3 + i);
            if (in.op >= MO_PLAN_OP_ADD) use(in.b, 3 + i);
        }
        for (int a = 0; a < P.naggs; a++) use(P.agg[a].value, t_agg);
        bool busy[2 * MO_PLAN_MAX_COLS + MO_PLAN_MAX_INSTR] = {false};
        int nphys = P.ncols;
        for (int c = 0; c < P.ncols; c++) { X.phys[c] = c; busy[c] = true; }
        for (int c = 0; c < P.ncols; c++) if (X.raw_phys[c] >= 0) { busy[X.raw_phys[c]] = true; nphys = std::max(nphys, X.raw_phys[c] + 1); }
        for (int i = 0; i < P.ninstr; i++) {
            const int now = 3 + i, dst = P.ncols + i;
            if (i == 0) for (int c = 0; c < P.ncols; c++) if (X.raw_phys[c] >= 0) busy[X.raw_phys[c]] = false;   // raw copies die with the filter
            // values whose last reader is this node or an earlier phase give their slot back (a node may overwrite its own operand: every
            // (thread, row) cell is read before it is written)
            for (int v = 0; v < dst; v++) if (busy[X.phys[v]] && last[v] <= now) {
                busy[X.phys[v]] = false; last[v] = 1 << 30;   // released once
            }
            int p = 0;
            while (p < nphys && busy[p]) p++;
            if (p == nphys) nphys++;
            X.phys[dst] = p; busy[p] = true;
            if (last[dst] < 0) last[dst] = now;             // a node nobody reads: its slot is free again after it
        }
        X.nphys = nphys;
    }
    MOB_CUDA_TRY(cudaStreamSynchronize(t.stream));
    memcpy(t.pinned, &P, sizeof P);
    memcpy((char *)t.pinned + sizeof P, &X, sizeof X);
    MOB_CUDA_TRY(cudaMemcpyAsync(dP, t.pinned, sizeof P, cudaMemcpyHostToDevice, t.stream));
    MOB_CUDA_TRY(cudaMemcpyAsync(dX, (char *)t.pinned + sizeof P, sizeof X, cudaMemcpyHostToDevice, t.stream));
    const unsigned igrid = (unsigned)((cap + 1 + 255) / 256 > (uint64_t)num_sms() * 8 ? (uint64_t)num_sms() * 8 : (cap + 1 + 255) / 256);
    plan_init_kernel<<<igrid, 256, 0, t.stream>>>(G, P.naggs, dP);
    MOB_LAUNCH_CHECK();
    const size_t smem = (size_t)X.nphys * R * kThreads * 8 + (size_t)kCtaSlots * (24 + 16 * (size_t)P.naggs) +
                        (size_t)kPriv * kThreads * ((size_t)P.naggs * (X.need_cnt ? 12 : 8) + 12);
    static size_t attr_smem = 0;
    if (smem > attr_smem) { MOB_CUDA_TRY(cudaFuncSetAttribute(plan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr_smem = smem; }
    if (len) {
        int ctas = 1;   // exactly the resident CTAs: the rows are dealt statically over the grid, a partial second wave would double the time
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, plan_kernel, kThreads, smem) != cudaSuccess || ctas < 1) ctas = 1;
        int grid = num_sms() * ctas;
        const uint64_t work = (len + (uint64_t)kThreads * R - 1) / ((uint64_t)kThreads * R);
        if ((uint64_t)grid > work) grid = (int)work;
        cudaEventRecord(t.kev0, t.stream);
        plan_kernel<<<grid, kThreads, smem, t.stream>>>(dP, dX, C, len, G);
        cudaEventRecord(t.kev1, t.stream);
        MOB_LAUNCH_CHECK();
    }
    plan_collect_kernel<<<igrid, 256, 0, t.stream>>>(G, used, nused);
    MOB_LAUNCH_CHECK();
    plan_emit_kernel<<<num_sms() * 2, 256, 0, t.stream>>>(G, dP, used, nused, dres, res_groups, 8192);
    MOB_LAUNCH_CHECK();
    if (st.resident()) return st.complete();   // asynchronous form: header.overflow reports a full table
    mo_plan_result_header_t H;
    int rc = read_back(t, &H, dres, sizeof H);
    int frc = st.complete();
    if (rc) return rc;
    if (H.overflow) { set_error("plan: more groups (%lld) than the result buffer holds (%llu)", (long long)H.ngroups, (unsigned long long)res_groups); return MO_RC_INVALID_ARGUMENT; }
    return frc;
}

}  // namespace mob
