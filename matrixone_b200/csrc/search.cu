// search.cu -- batched exact nearest-neighbour search: brute-force top-k, IVF-flat list probes, top-k merge.
//
// Reference: GoBruteForceIndex.Search (pkg/vectorindex/brute_force/brute_force.go:248-341) = for every query, the metric
// function over every dataset row + FastMaxHeap (pkg/vectorindex/index.go:171-250); IvfflatSearchIndex.Search
// (pkg/vectorindex/ivfflat/search.go:509-630) = the same over the centroid table (nprobe) and then over the probed lists.
//
// Exact kernel (this file): a register-tiled distance kernel whose per-(query,row) accumulation replays the Go loop
// operation by operation -- 8-element chunks ((t0+t1)+(t2+t3))+(t4+t5))+(t6+t7), sum += chunk, fp32 accumulator, no
// FMA contraction -- so distances are BIT-EXACT with metric.L2DistanceSq / InnerProduct / L1Distance / CosineDistance.
// A CTA owns a 64-query tile and a contiguous range of dataset rows; x tiles (64 rows x 32 floats) and q tiles are
// double-buffered in shared memory ([k][row] for x so a thread reads 4 rows with one LDS.128, rows of one warp are
// consecutive => conflict-free; q reads are warp broadcasts).  The running top-k of the 64 queries lives in shared
// memory; a distance becomes a candidate only if it beats the query's current k-th best, so after the first tiles
// the selection cost vanishes against the 768x3 flops per pair.  Partial lists of the row ranges (and of the GPUs in a
// multi-GPU run) are merged by topk_merge_kernel.  Ordering is total: (distance, row id) ascending.
//
// CTAs that share a row range are adjacent in blockIdx, so the dataset is read from HBM about once (L2 reuse) and the
// query block (Q x dim x 4 B = 30 MB at the BASELINE shape) stays L2 resident.
// Work per launch: Q*N*dim element-pairs, 3 fp32 ops each (sub, mul, add) => 3*Q*N*dim flop; bytes N*dim*4 + Q*dim*4.
#include "common.cuh"
#include "search_internal.cuh"
#include "bloom_internal.cuh"
#include <cstring>
#include <cfloat>
#include <cmath>

using namespace mob;

namespace {

constexpr int kThreads = 256;
constexpr int TQ = 64, TX = 64, KC = 32;
constexpr int QP = KC + 4;          // q tile pitch (floats)
constexpr int KMAX = 64;            // largest k served by the fused kernel
constexpr unsigned FULL = 0xffffffffu;

struct SearchSmem {
    float xs[2][KC][TX];
    float qs[2][TQ][QP];
    float ld[KMAX][TQ];             // per-query sorted list, [rank][query]
    int li[KMAX][TQ];
    float thr_d[TQ]; int thr_i[TQ]; int lcnt[TQ];
    float qnorm[TQ];
    unsigned char cand_row[TQ][TX + 4]; float cand_d[TQ][TX + 1];   // per-query candidate lists of the current tile (padded: bank-conflict free across queries)
    int qcnt[TQ];
};

__device__ __forceinline__ bool lex_less(float d, int i, float d2, int i2) { return d < d2 || (d == d2 && i < i2); }

// metric ids follow include/mo_b200.h
template <int METRIC>
__device__ __forceinline__ void chunk8(const float *q, const float *x, float &acc) {
    if (METRIC == MO_METRIC_IP || METRIC == MO_METRIC_COS) {
        if (METRIC == MO_METRIC_IP) {   // InnerProduct, distance_func.go:184-195
            float s = __fadd_rn(__fmul_rn(q[0], x[0]), __fmul_rn(q[1], x[1]));
#pragma unroll
            for (int j = 2; j < 8; j++) s = __fadd_rn(s, __fmul_rn(q[j], x[j]));
            acc = __fadd_rn(acc, s);
        } else {                        // CosineDistance dot product: 4-wide chunks, distance_func.go:238-246
            float s = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(q[0], x[0]), __fmul_rn(q[1], x[1])), __fmul_rn(q[2], x[2])), __fmul_rn(q[3], x[3]));
            acc = __fadd_rn(acc, s);
            s = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(q[4], x[4]), __fmul_rn(q[5], x[5])), __fmul_rn(q[6], x[6])), __fmul_rn(q[7], x[7]));
            acc = __fadd_rn(acc, s);
        }
    } else if (METRIC == MO_METRIC_L1) { // L1Distance, distance_func.go:135-143
#pragma unroll
        for (int j = 0; j < 8; j++) acc = __fadd_rn(acc, fabsf(__fsub_rn(q[j], x[j])));
    } else {                             // L2DistanceSq, distance_func.go:69-86
        float t[8];
#pragma unroll
        for (int j = 0; j < 8; j++) { float d = __fsub_rn(q[j], x[j]); t[j] = __fmul_rn(d, d); }
        float s = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(t[0], t[1]), __fadd_rn(t[2], t[3])), __fadd_rn(t[4], t[5])), __fadd_rn(t[6], t[7]));
        acc = __fadd_rn(acc, s);
    }
}
template <int METRIC>
__device__ __forceinline__ void tail1(float q, float x, float &acc) {   // remainder loops of the Go functions
    if (METRIC == MO_METRIC_IP || METRIC == MO_METRIC_COS) acc = __fadd_rn(acc, __fmul_rn(q, x));
    else if (METRIC == MO_METRIC_L1) acc = __fadd_rn(acc, fabsf(__fsub_rn(q, x)));
    else { float d = __fsub_rn(q, x); acc = __fadd_rn(acc, __fmul_rn(d, d)); }
}

// One work item = (query tile, row range).  qidx (optional) gathers query rows; slot_of (optional) gives the output slot of
// each local query (IVF: slot = query*nprobe + probe rank); otherwise slot = range * nq + query.
struct WorkDesc {
    const float *data; int64_t n;            // rows of this item: data[(row_begin + r) * dim]
    int64_t row_begin, row_end;
    const float *queries; int64_t nq_total;
    const int32_t *qidx;                     // local query -> global query row (nullptr: q0 + local)
    int64_t q0; int nq_local;
    const int64_t *slot_of;                  // local query -> output slot (nullptr: range*nq_total + q)
    int64_t range;
    const float *xnorm, *qnorm;              // COS: squared norms (exact Go order)
    const uint32_t *admit;                   // nullable: bit r of word r / 32 = row r may be listed (filtered search)
};

template <int METRIC>
__global__ void __launch_bounds__(kThreads, 2)
bf_topk_kernel(const WorkDesc *__restrict__ items, int dim, int k, float *__restrict__ part_d, int32_t *__restrict__ part_i) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    SearchSmem &S = *reinterpret_cast<SearchSmem *>(smem_raw);
    const WorkDesc W = items[blockIdx.x];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const bool al4 = (dim & 3) == 0 && ((((uintptr_t)W.data) | ((uintptr_t)W.queries)) & 15) == 0;

    if (tid < TQ) { S.lcnt[tid] = 0; S.thr_d[tid] = INFINITY; S.thr_i[tid] = 0x7fffffff; S.qcnt[tid] = 0; }
    if (METRIC == MO_METRIC_COS && tid < TQ) {
        int64_t gq = tid < W.nq_local ? (W.qidx ? W.qidx[tid] : W.q0 + tid) : -1;
        S.qnorm[tid] = gq >= 0 ? W.qnorm[gq] : 0.f;
    }
    __syncthreads();

    // fill mapping
    const int fx_row = tid & 63, fx_kq = tid >> 6;           // x: rows consecutive across lanes, kq in {fx_kq, fx_kq+4}
    const int fq_q = tid >> 2, fq_kq = (tid & 3) * 2;        // q: 4 lanes per query row, kq in {fq_kq, fq_kq+1}
    const int64_t gq_fill = fq_q < W.nq_local ? (W.qidx ? (int64_t)W.qidx[fq_q] : W.q0 + fq_q) : -1;
    const int nsteps = (dim + KC - 1) / KC;

    auto gload = [&](const float *base, int64_t row, bool valid, int kk) -> float4 {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (!valid) return v;
        const float *p = base + row * (int64_t)dim + kk;
        if (al4) { if (kk < dim) v = __ldg(reinterpret_cast<const float4 *>(p)); }
        else {
            if (kk < dim) v.x = __ldg(p);
            if (kk + 1 < dim) v.y = __ldg(p + 1);
            if (kk + 2 < dim) v.z = __ldg(p + 2);
            if (kk + 3 < dim) v.w = __ldg(p + 3);
        }
        return v;
    };

    for (int64_t row0 = W.row_begin; row0 < W.row_end; row0 += TX) {
        __syncwarp();   // the per-query insertion loop below diverges; make sure every warp starts a tile converged
        float acc[4][4];
#pragma unroll
        for (int a = 0; a < 4; a++)
#pragma unroll
            for (int b = 0; b < 4; b++) acc[a][b] = 0.f;

        const int64_t xrow = row0 + fx_row;
        const bool xvalid = xrow < W.row_end;
        float4 px[2], pq[2];
        // prologue: step 0 -> buffer 0
        px[0] = gload(W.data, xrow, xvalid, 4 * fx_kq); px[1] = gload(W.data, xrow, xvalid, 4 * (fx_kq + 4));
        pq[0] = gload(W.queries, gq_fill, gq_fill >= 0, 4 * fq_kq); pq[1] = gload(W.queries, gq_fill, gq_fill >= 0, 4 * (fq_kq + 1));
        auto sstore = [&](int buf) {
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int kq = fx_kq + 4 * h;
                S.xs[buf][4 * kq + 0][fx_row] = px[h].x; S.xs[buf][4 * kq + 1][fx_row] = px[h].y;
                S.xs[buf][4 * kq + 2][fx_row] = px[h].z; S.xs[buf][4 * kq + 3][fx_row] = px[h].w;
                *reinterpret_cast<float4 *>(&S.qs[buf][fq_q][4 * (fq_kq + h)]) = pq[h];
            }
        };
        sstore(0);
        __syncthreads();
        for (int s = 0; s < nsteps; s++) {
            const int buf = s & 1;
            if (s + 1 < nsteps) {
                const int k1 = (s + 1) * KC;
                px[0] = gload(W.data, xrow, xvalid, k1 + 4 * fx_kq); px[1] = gload(W.data, xrow, xvalid, k1 + 4 * (fx_kq + 4));
                pq[0] = gload(W.queries, gq_fill, gq_fill >= 0, k1 + 4 * fq_kq); pq[1] = gload(W.queries, gq_fill, gq_fill >= 0, k1 + 4 * (fq_kq + 1));
            }
            const int k0 = s * KC;
#pragma unroll
            for (int c = 0; c < KC / 8; c++) {
                const int kb = k0 + 8 * c;
                if (kb >= dim) break;
                float qv[4][8], xv[8][4];
#pragma unroll
                for (int a = 0; a < 4; a++) {
                    float4 u = *reinterpret_cast<const float4 *>(&S.qs[buf][4 * ty + a][8 * c]);
                    float4 w = *reinterpret_cast<const float4 *>(&S.qs[buf][4 * ty + a][8 * c + 4]);
                    qv[a][0] = u.x; qv[a][1] = u.y; qv[a][2] = u.z; qv[a][3] = u.w; qv[a][4] = w.x; qv[a][5] = w.y; qv[a][6] = w.z; qv[a][7] = w.w;
                }
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    float4 u = *reinterpret_cast<const float4 *>(&S.xs[buf][8 * c + j][4 * tx]);
                    xv[j][0] = u.x; xv[j][1] = u.y; xv[j][2] = u.z; xv[j][3] = u.w;
                }
                if (kb + 8 <= dim) {
#pragma unroll
                    for (int a = 0; a < 4; a++)
#pragma unroll
                        for (int b = 0; b < 4; b++) {
                            float xx[8];
#pragma unroll
                            for (int j = 0; j < 8; j++) xx[j] = xv[j][b];
                            chunk8<METRIC>(qv[a], xx, acc[a][b]);
                        }
                } else {
                    // dim % 8 tail: COS uses 4-wide chunks first (distance_func.go:238-254), the rest element by element
                    int j0 = 0;
                    if (METRIC == MO_METRIC_COS && kb + 4 <= dim) {
#pragma unroll
                        for (int a = 0; a < 4; a++)
#pragma unroll
                            for (int b = 0; b < 4; b++) {
                                float s4 = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(qv[a][0], xv[0][b]), __fmul_rn(qv[a][1], xv[1][b])), __fmul_rn(qv[a][2], xv[2][b])), __fmul_rn(qv[a][3], xv[3][b]));
                                acc[a][b] = __fadd_rn(acc[a][b], s4);
                            }
                        j0 = 4;
                    }
                    for (int j = j0; kb + j < dim; j++)
#pragma unroll
                        for (int a = 0; a < 4; a++)
#pragma unroll
                            for (int b = 0; b < 4; b++) tail1<METRIC>(qv[a][j], xv[j][b], acc[a][b]);
                }
            }
            if (s + 1 < nsteps) sstore(buf ^ 1);
            __syncthreads();
        }

        // ---- candidates
#pragma unroll
        for (int a = 0; a < 4; a++) {
            const int ql = 4 * ty + a;
            if (ql >= W.nq_local) continue;
            const float td = S.thr_d[ql]; const int ti = S.thr_i[ql];
#pragma unroll
            for (int b = 0; b < 4; b++) {
                const int rl = 4 * tx + b;
                const int64_t row = row0 + rl;
                if (row >= W.row_end || (W.admit && !((W.admit[row >> 5] >> (row & 31)) & 1u))) continue;
                float d = acc[a][b];
                if (METRIC == MO_METRIC_IP) d = -d;
                if (METRIC == MO_METRIC_COS) {     // distance_func.go:264-284
                    const double den = sqrt((double)S.qnorm[ql]) * sqrt((double)W.xnorm[row]);
                    if (den == 0.0) d = 1.0f;
                    else { double sim = (double)d / den; sim = sim > 1.0 ? 1.0 : (sim < -1.0 ? -1.0 : sim); d = (float)(1.0 - sim); }
                }
                if (lex_less(d, (int)row, td, ti)) {
                    const int slot = atomicAdd(&S.qcnt[ql], 1);
                    S.cand_row[ql][slot] = (unsigned char)rl;
                    S.cand_d[ql][slot] = d;
                }
            }
        }
        __syncthreads();
        // every query thread inserts its own candidates (lanes work in parallel; the slot order inside a list is arbitrary but
        // the result is not: (distance, row) is a total order)
        if (tid < W.nq_local) {
            const int ql = tid;
            const int nc = S.qcnt[ql];
            int cnt = S.lcnt[ql];
            for (int c = 0; c < nc; c++) {
                const float d = S.cand_d[ql][c]; const int id = (int)(row0 + S.cand_row[ql][c]);
                int pos;
                if (cnt < k) pos = cnt++;
                else { if (!lex_less(d, id, S.ld[k - 1][ql], S.li[k - 1][ql])) continue; pos = k - 1; }
                while (pos > 0 && lex_less(d, id, S.ld[pos - 1][ql], S.li[pos - 1][ql])) {
                    S.ld[pos][ql] = S.ld[pos - 1][ql]; S.li[pos][ql] = S.li[pos - 1][ql]; pos--;
                }
                S.ld[pos][ql] = d; S.li[pos][ql] = id;
            }
            S.lcnt[ql] = cnt;
            if (cnt >= k) { S.thr_d[ql] = S.ld[k - 1][ql]; S.thr_i[ql] = S.li[k - 1][ql]; }
            S.qcnt[ql] = 0;
        }
        __syncthreads();
    }

    // ---- write the partial lists
    if (tid < W.nq_local) {
        const int ql = tid;
        const int64_t gq = W.qidx ? (int64_t)W.qidx[ql] : W.q0 + ql;
        const int64_t slot = W.slot_of ? W.slot_of[ql] : W.range * W.nq_total + gq;
        const int cnt = S.lcnt[ql];
        for (int j = 0; j < k; j++) {
            part_d[slot * k + j] = j < cnt ? S.ld[j][ql] : INFINITY;
            part_i[slot * k + j] = j < cnt ? S.li[j][ql] : -1;
        }
    }
}

// squared norms in the exact CosineDistance order (4-wide chunks, then elements), one warp per row
__global__ void cos_norm_kernel(const float *__restrict__ v, int64_t n, int dim, float *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < n; r += nwarps) {
        const float *p = v + r * dim;
        const int nch = dim >> 2;
        float sum = 0.f;
        for (int base = 0; base < nch; base += 32) {
            const int c = base + lane;
            float s = 0.f;
            if (c < nch) {
                const float a0 = p[4 * c], a1 = p[4 * c + 1], a2 = p[4 * c + 2], a3 = p[4 * c + 3];
                s = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(a0, a0), __fmul_rn(a1, a1)), __fmul_rn(a2, a2)), __fmul_rn(a3, a3));
            }
            const int m = min(32, nch - base);
            for (int l = 0; l < m; l++) sum = __fadd_rn(sum, __shfl_sync(FULL, s, l));
        }
        for (int i = nch << 2; i < dim; i++) sum = __fadd_rn(sum, __fmul_rn(p[i], p[i]));
        if (lane == 0) out[r] = sum;
    }
}

// COS: the squared norms of the rows and of the queries that bf_topk_kernel divides by (other metrics: none)
int cos_norms(ThreadCtx &t, int metric, const float *ddata, int64_t n, const float *dq, int64_t nq, int dim, float **xnorm, float **qnorm) {
    *xnorm = *qnorm = nullptr;
    if (metric != MO_METRIC_COS) return MO_RC_SUCCESS;
    *xnorm = (float *)arena_alloc(t, sizeof(float) * (size_t)(n > 0 ? n : 1));
    *qnorm = (float *)arena_alloc(t, sizeof(float) * (size_t)nq);
    if (!*xnorm || !*qnorm) return MO_RC_INTERNAL_ERROR;
    if (n > 0) { cos_norm_kernel<<<num_sms() * 8, 256, 0, t.stream>>>(ddata, n, dim, *xnorm); MOB_LAUNCH_CHECK(); }
    cos_norm_kernel<<<num_sms() * 8, 256, 0, t.stream>>>(dq, nq, dim, *qnorm); MOB_LAUNCH_CHECK();
    return MO_RC_SUCCESS;
}

__global__ void gather_rows_kernel(const float *__restrict__ src, const int *__restrict__ idx, int m, int dim, float *__restrict__ dst) {
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < (int64_t)m * dim; e += (int64_t)gridDim.x * blockDim.x)
        dst[e] = src[(int64_t)idx[e / dim] * dim + e % dim];
}
__global__ void scatter_results_kernel(const int64_t *__restrict__ sk, const double *__restrict__ sd, const int *__restrict__ idx, int m, int k,
                                       int64_t *__restrict__ out_k, double *__restrict__ out_d) {
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < m * k; e += gridDim.x * blockDim.x) {
        const int q = idx[e / k];
        out_k[(size_t)q * k + e % k] = sk[e]; out_d[(size_t)q * k + e % k] = sd[e];
    }
}

// ---- filtered search ---------------------------------------------------------------------------------------------------------
// admission mask: bit r of 32-bit word r / 32 = row r is admitted; one lane per row, one ballot per word, the admitted rows are
// counted in the same pass.  The key of row r is row_ids[r] (IVF: the primary key) or key_base + r (brute force).
//   KEY_BITMAP: bitmap_test_with_len (cgo/bitmap.h:55-63): bit `key` of words[0, nwords) -- a key at or past 64 * nwords (or < 0) is rejected
//   KEY_BLOOM:  bloomfilter_test of the key's 8 little-endian bytes against the filter's device mirror
__global__ void filter_admit_kernel(int kind, const uint64_t *__restrict__ words, uint64_t nwords, uint64_t nbits, uint32_t nhash, uint64_t seed,
                                    int64_t n, int64_t key_base, const int64_t *__restrict__ row_ids, uint32_t *__restrict__ admit,
                                    unsigned long long *count) {
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r - lane < n; r += stride) {   // r - lane: the warp's first row, uniform
        bool ok = false;
        if (r < n) {
            const int64_t key = row_ids ? row_ids[r] : key_base + r;
            if (kind == MO_SEARCH_FILTER_KEY_BITMAP) ok = ((uint64_t)key >> 6) < nwords && ((words[(uint64_t)key >> 6] >> (key & 63)) & 1ull);
            else ok = nbits != 0 && bloom_test_hash(words, nbits, nhash, bloom_key_hash(reinterpret_cast<const uint8_t *>(&key), 8, seed));
        }
        const unsigned w = __ballot_sync(0xffffffffu, ok);
        if (lane == 0) { admit[(r - lane) >> 5] = w; if (w) atomicAdd(count, (unsigned long long)__popc(w)); }
    }
}
// compacted set: local row -> key (brute force; the compaction keeps the row order, so the key order of ties is the local order)
__global__ void filter_remap_keys_kernel(int64_t *keys, int64_t cnt, const int32_t *__restrict__ idx, int64_t key_base) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < cnt; i += (int64_t)gridDim.x * blockDim.x)
        if (keys[i] >= 0) keys[i] = key_base + idx[keys[i]];
}
__global__ void filter_gather_ids_kernel(const int64_t *__restrict__ src, const int32_t *__restrict__ idx, int64_t m, int64_t *__restrict__ dst) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) dst[i] = src[idx[i]];
}
// IVF list boundaries of the compacted entries: list l starts at the number of admitted rows before offsets[l] (idx is ascending)
__global__ void filter_offsets_kernel(const int64_t *__restrict__ offsets, int64_t nlist, const int32_t *__restrict__ idx, int64_t m, int64_t *__restrict__ out) {
    for (int64_t l = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; l <= nlist; l += (int64_t)gridDim.x * blockDim.x) {
        int64_t lo = 0, hi = m;
        while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if (idx[mid] < offsets[l]) lo = mid + 1; else hi = mid; }
        out[l] = lo;
    }
}

// merge nlists sorted (dist,id) lists of length k per query into the final keys/distances.
// in_i holds LOCAL ids when id_map/key_base describe the translation, or final int64 keys when in_k is given.
__global__ void topk_merge_kernel(int64_t nq, int k, int nlists, int64_t list_stride /* in queries */, const float *__restrict__ in_d,
                                  const int32_t *__restrict__ in_i, const double *__restrict__ in_d64, const int64_t *__restrict__ in_k,
                                  const int64_t *__restrict__ id_map, int64_t key_base, int sqrt_out, int slot_major,
                                  int64_t *__restrict__ out_k, double *__restrict__ out_d) {
    const int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (q >= nq) return;
    int head[64];
    for (int l = 0; l < nlists; l++) head[l] = 0;
    // list l of query q starts at: slot_major ? (q*nlists + l)*k : (l*list_stride + q)*k
    int produced = 0;
    int64_t *ok = out_k + q * k; double *od = out_d + q * k;
    // count available entries first to implement the reference's front padding (brute_force.go:319-331)
    int avail = 0;
    for (int l = 0; l < nlists; l++) {
        const int64_t base = slot_major ? ((q * nlists + l) * (int64_t)k) : ((l * list_stride + q) * (int64_t)k);
        for (int j = 0; j < k; j++) { const bool has = in_k ? in_k[base + j] >= 0 : in_i[base + j] >= 0; avail += has; }
    }
    const int total = avail < k ? avail : k;
    const int pad = k - total;
    // limit == 1 over an empty dataset leaves the running minimum untouched: key -1, distance MaxFloat32 (brute_force.go:289-303)
    for (int j = 0; j < pad; j++) { ok[j] = -1; od[j] = (k == 1 && !slot_major) ? (double)3.40282346638528859811704183484516925440e+38f : 0.0; }
    while (produced < total) {
        int best = -1; double bd = 0; int64_t bk = 0;
        for (int l = 0; l < nlists; l++) {
            const int64_t base = slot_major ? ((q * nlists + l) * (int64_t)k) : ((l * list_stride + q) * (int64_t)k);
            int64_t key = -1; double d = 0;
            while (head[l] < k) {   // skip padding entries (front-padded final lists, back-padded partial lists)
                const int64_t idx = base + head[l];
                if (in_k) { key = in_k[idx]; d = in_d64[idx]; }
                else { const int32_t li = in_i[idx]; key = li < 0 ? -1 : (id_map ? id_map[li] : (int64_t)li + key_base); d = (double)in_d[idx]; }
                if (key >= 0) break;
                head[l]++;
            }
            if (head[l] >= k) continue;
            if (best < 0 || d < bd || (d == bd && key < bk)) { best = l; bd = d; bk = key; }
        }
        if (best < 0) break;
        head[best]++;
        ok[pad + produced] = bk;
        od[pad + produced] = sqrt_out ? sqrt(bd) : bd;
        produced++;
    }
}

template <int METRIC>
int launch_bf(ThreadCtx &t, const WorkDesc *ditems, int nitems, int dim, int k, float *part_d, int32_t *part_i) {
    static bool attr_set = false;
    if (!attr_set) {
        MOB_CUDA_TRY(cudaFuncSetAttribute(bf_topk_kernel<METRIC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SearchSmem)));
        attr_set = true;
    }
    const bool timed = t.kev_prio <= 1;   // a tensor-core candidate pass of the same call stays the reported kernel
    if (timed) { t.kev_prio = 1; cudaEventRecord(t.kev0, t.stream); }
    bf_topk_kernel<METRIC><<<nitems, kThreads, sizeof(SearchSmem), t.stream>>>(ditems, dim, k, part_d, part_i);
    if (timed) cudaEventRecord(t.kev1, t.stream);
    MOB_LAUNCH_CHECK();
    return MO_RC_SUCCESS;
}

int launch_bf_metric(ThreadCtx &t, int metric, const WorkDesc *ditems, int nitems, int dim, int k, float *part_d, int32_t *part_i) {
    switch (metric) {
    case MO_METRIC_L2: case MO_METRIC_L2SQ: return launch_bf<MO_METRIC_L2SQ>(t, ditems, nitems, dim, k, part_d, part_i);
    case MO_METRIC_IP: return launch_bf<MO_METRIC_IP>(t, ditems, nitems, dim, k, part_d, part_i);
    case MO_METRIC_COS: return launch_bf<MO_METRIC_COS>(t, ditems, nitems, dim, k, part_d, part_i);
    case MO_METRIC_L1: return launch_bf<MO_METRIC_L1>(t, ditems, nitems, dim, k, part_d, part_i);
    }
    set_error("search: unknown metric %d", metric);
    return MO_RC_INVALID_ARGUMENT;
}

int read_filter(ThreadCtx &t, const mo_xcall_args_t &a, mo_search_filter_t *F) {
    if (int rc = read_param(t, a, F, sizeof *F, sizeof *F, "filtered search: filter descriptor")) return rc;
    if (F->kind != MO_SEARCH_FILTER_KEY_BITMAP && F->kind != MO_SEARCH_FILTER_KEY_BLOOM) { set_error("filtered search: unknown filter kind %d", F->kind); return MO_RC_INVALID_ARGUMENT; }
    if (!F->filter) { set_error("filtered search: null filter"); return MO_RC_INVALID_ARGUMENT; }
    if (F->kind == MO_SEARCH_FILTER_KEY_BLOOM) {
        const bloomfilter_t *bf = (const bloomfilter_t *)F->filter;
        if (memcmp(bf->magic, "XXBF", 4) != 0 || bf->k > MAX_K_SEED) { set_error("filtered search: not a bloom filter (bad magic or k)"); return MO_RC_INVALID_ARGUMENT; }
    }
    return MO_RC_SUCCESS;
}

// the admission mask of n rows (keys: row_ids[r], or key_base + r without row_ids) in the call's arena, and the admitted count
int filter_admission(ThreadCtx &t, Stager &st, const mo_search_filter_t &F, int64_t n, int64_t key_base, const int64_t *row_ids,
                     uint32_t **admit, int64_t *admitted) {
    const uint64_t *words; uint64_t nwords = 0, nbits = 0, seed = 0; uint32_t nhash = 0;
    if (F.kind == MO_SEARCH_FILTER_KEY_BITMAP) {
        nwords = F.nwords;
        words = nwords ? (const uint64_t *)st.in(F.filter, (size_t)nwords * 8) : nullptr;   // no words: every key is rejected
    } else {   // the filter's own device mirror: bits added on the device are seen
        const bloomfilter_t *bf = (const bloomfilter_t *)F.filter;
        words = bloom_mirror(t, bf, false);
        if (!words) return MO_RC_INTERNAL_ERROR;
        nbits = bf->nbits; nhash = bf->k; seed = bf->seed;
    }
    *admit = (uint32_t *)arena_alloc(t, (size_t)((n + 31) / 32 + 1) * 4);
    unsigned long long *dcount = (unsigned long long *)arena_alloc(t, 8);
    if (st.failed || !*admit || !dcount) return MO_RC_INTERNAL_ERROR;
    MOB_CUDA_TRY(cudaMemsetAsync(dcount, 0, 8, t.stream));
    if (n > 0) {
        int64_t grid = (n + 255) / 256;
        if (grid > num_sms() * 8ll) grid = num_sms() * 8ll;
        filter_admit_kernel<<<(unsigned)grid, 256, 0, t.stream>>>(F.kind, words, nwords, nbits, nhash, seed, n, key_base, row_ids, *admit, dcount);
        MOB_LAUNCH_CHECK();
    }
    unsigned long long h = 0;
    int rc = read_back(t, &h, dcount, 8);
    *admitted = (int64_t)h;
    g_search_stats.filter_admitted = (int)h;
    return rc;
}

// the admitted rows of ddata, in order: *idx = their row numbers, *sub = the rows
int filter_gather(ThreadCtx &t, const float *ddata, int64_t n, int dim, const uint32_t *admit, int64_t m, int32_t **idx, float **sub) {
    *idx = (int32_t *)arena_alloc(t, (size_t)(m > 0 ? m : 1) * 4);
    *sub = (float *)arena_alloc(t, (size_t)(m > 0 ? m : 1) * dim * 4);
    unsigned long long *dtotal = (unsigned long long *)arena_alloc(t, 8);
    if (!*idx || !*sub || !dtotal) return MO_RC_INTERNAL_ERROR;
    int rc = compact_bits(t, admit, (uint64_t)n, *idx, dtotal);
    if (rc) return rc;
    if (m > 0) { gather_rows_kernel<<<num_sms() * 8, 256, 0, t.stream>>>(ddata, *idx, (int)m, dim, *sub); MOB_LAUNCH_CHECK(); }
    g_search_stats.filter_compacted = 1;
    return MO_RC_SUCCESS;
}

}  // namespace

namespace mob {

// Core: brute-force top-k of nq queries against rows [0,n) of ddata, results (keys + key_base, float64 distances) to
// device buffers out_k/out_d (nq*k).  All pointers are device pointers.
int bruteforce_topk_device(ThreadCtx &t, const float *ddata, int64_t n, int dim, const float *dq, int64_t nq, int k, int metric,
                           int64_t key_base, int sqrt_out, int64_t *out_k, double *out_d, const uint32_t *admit) {
    if (k <= 0 || nq <= 0) return MO_RC_SUCCESS;
    if (k > KMAX) { set_error("search: k=%d exceeds the fused kernel limit %d", k, KMAX); return MO_RC_INVALID_ARGUMENT; }
    if (n >= (1ll << 31)) { set_error("search: more than 2^31 rows per shard"); return MO_RC_INVALID_ARGUMENT; }
    const int nqt = (int)((nq + TQ - 1) / TQ);
    const int64_t ntiles = (n + TX - 1) / TX;
    int64_t R = (4ll * 2 * num_sms() + nqt - 1) / nqt;       // >= 4 waves of 2 CTAs/SM
    if (R > ntiles) R = ntiles;
    if (R > 64) R = 64;
    if (R < 1) R = 1;
    const int64_t tiles_per = (ntiles + R - 1) / R;
    R = n > 0 ? (ntiles + tiles_per - 1) / tiles_per : 1;
    const int nitems = (int)(R * nqt);
    float *xnorm, *qnorm;
    int rc = cos_norms(t, metric, ddata, n, dq, nq, dim, &xnorm, &qnorm);
    if (rc) return rc;
    std::vector<WorkDesc> items((size_t)nitems);
    for (int64_t r = 0; r < R; r++)
        for (int qt = 0; qt < nqt; qt++) {
            WorkDesc &w = items[(size_t)(r * nqt + qt)];   // CTAs sharing a row range are adjacent => L2 reuse of x
            w.data = ddata; w.n = n;
            w.row_begin = r * tiles_per * TX; w.row_end = (r + 1) * tiles_per * TX < n ? (r + 1) * tiles_per * TX : n;
            if (w.row_begin > n) w.row_begin = n;
            w.queries = dq; w.nq_total = nq; w.qidx = nullptr; w.q0 = (int64_t)qt * TQ;
            w.nq_local = (int)(nq - w.q0 < TQ ? nq - w.q0 : TQ);
            w.slot_of = nullptr; w.range = r; w.xnorm = xnorm; w.qnorm = qnorm; w.admit = admit;
        }
    WorkDesc *ditems = (WorkDesc *)arena_alloc(t, sizeof(WorkDesc) * (size_t)nitems);
    float *part_d = (float *)arena_alloc(t, sizeof(float) * (size_t)(R * nq * k));
    int32_t *part_i = (int32_t *)arena_alloc(t, sizeof(int32_t) * (size_t)(R * nq * k));
    if (!ditems || !part_d || !part_i) return MO_RC_INTERNAL_ERROR;
    MOB_CUDA_TRY(cudaMemcpyAsync(ditems, items.data(), sizeof(WorkDesc) * (size_t)nitems, cudaMemcpyHostToDevice, t.stream));
    MOB_CUDA_TRY(cudaStreamSynchronize(t.stream));   // items is pageable host memory about to go out of scope
    rc = launch_bf_metric(t, metric, ditems, nitems, dim, k, part_d, part_i);
    if (rc) return rc;
    topk_merge_kernel<<<(unsigned)((nq + 127) / 128), 128, 0, t.stream>>>(nq, k, (int)R, nq, part_d, part_i, nullptr, nullptr, nullptr, key_base, sqrt_out, 0, out_k, out_d);
    MOB_LAUNCH_CHECK();
    return MO_RC_SUCCESS;
}

// the tensor-core path where it applies, else the exact kernel; admit (nullable) restricts the rows that may be listed
static int bruteforce_search(ThreadCtx &t, const mo_search_params_t &P, const float *ddata, int64_t n, const float *dq, int64_t key_base,
                             int64_t *ok, double *od, const uint32_t *admit) {
    if (tc_search_applicable(n, (int)P.dim, P.nq, P.k, P.metric))
        return bruteforce_topk_tc_device(t, ddata, n, (int)P.dim, dq, P.nq, P.k, key_base, P.sqrt_out, ok, od, true, (int)P.metric, admit);
    return bruteforce_topk_device(t, ddata, n, (int)P.dim, dq, P.nq, P.k, P.metric, key_base, P.sqrt_out, ok, od, admit);
}

// MO_XCALL_BRUTEFORCE_TOPK_F32 (farg == nullptr) and MO_XCALL_BRUTEFORCE_TOPK_FILTERED_F32 (farg = the filter descriptor)
static int bruteforce_call(mo_xcall_args_t *args, uint64_t len, const mo_xcall_args_t *farg) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    SearchReadGuard guard;   // prepared operands stay alive until this call returns
    mo_search_params_t P;
    int rc = read_param(t, args[4], &P, sizeof P, sizeof P, "search: params");
    if (rc) return rc;
    if (P.nq != (int64_t)len) { set_error("search: len != params.nq"); return MO_RC_INVALID_ARGUMENT; }
    if (P.k == 0 || P.nq == 0) return MO_RC_SUCCESS;   // brute_force.go:262-264
    if (args[2].dataSz < (uint64_t)P.n * P.dim * 4 || args[3].dataSz < (uint64_t)P.nq * P.dim * 4 ||
        args[0].dataSz < (uint64_t)P.nq * P.k * 8 || args[1].dataSz < (uint64_t)P.nq * P.k * 8) {
        set_error("search: buffer sizes do not match params"); return MO_RC_INVALID_ARGUMENT;
    }
    mo_search_filter_t F;
    if (farg && (rc = read_filter(t, *farg, &F)) != 0) return rc;
    Stager st(t);
    const float *ddata = (const float *)st.in(args[2].pdata, (size_t)P.n * P.dim * 4);
    const float *dq = (const float *)st.in(args[3].pdata, (size_t)P.nq * P.dim * 4);
    int64_t *ok = (int64_t *)st.out(args[0].pdata, (size_t)P.nq * P.k * 8);
    double *od = (double *)st.out(args[1].pdata, (size_t)P.nq * P.k * 8);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    g_search_stats = SearchStats();   // the statistics describe this search, also when it does not reach the tensor cores
    if (!farg) {
        rc = bruteforce_search(t, P, ddata, P.n, dq, P.key_base, ok, od, nullptr);
    } else {
        uint32_t *admit; int64_t m = 0;
        rc = filter_admission(t, st, F, P.n, P.key_base, nullptr, &admit, &m);
        if (!rc && filter_compact_wanted(P.n, m, false)) {
            // few admitted rows: search the gathered rows (local ids 0..m-1), then local id -> key
            int32_t *idx; float *sub;
            rc = filter_gather(t, ddata, P.n, (int)P.dim, admit, m, &idx, &sub);
            if (!rc) rc = bruteforce_search(t, P, sub, m, dq, 0, ok, od, nullptr);
            if (!rc) {
                filter_remap_keys_kernel<<<num_sms() * 4, 256, 0, t.stream>>>(ok, P.nq * P.k, idx, P.key_base);
                if (cudaGetLastError() != cudaSuccess) { set_error("filtered search: key remap launch failed"); rc = MO_RC_INTERNAL_ERROR; }
                g_launches++;
            }
        } else if (!rc) {
            g_search_stats.filter_compacted = 0;
            rc = bruteforce_search(t, P, ddata, P.n, dq, P.key_base, ok, od, admit);
        }
    }
    int frc = st.finish();
    return rc ? rc : frc;
}

int xcall_bruteforce(mo_xcall_args_t *args, uint64_t len) { return bruteforce_call(args, len, nullptr); }
int xcall_bruteforce_filtered(mo_xcall_args_t *args, uint64_t len) { return bruteforce_call(args, len, &args[5]); }

// merge of per-shard lists: in keys/dists are [nshards][nq][k] (final keys, f64 distances, -1 = missing)
int xcall_topk_merge(mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    mo_search_params_t P;
    int rc = read_param(t, args[4], &P, sizeof P, sizeof P, "search: params");
    if (rc) return rc;
    const int64_t nshards = P.n;
    if (P.nq != (int64_t)len || nshards < 1 || nshards > 64) { set_error("merge: bad params"); return MO_RC_INVALID_ARGUMENT; }
    if (P.k == 0 || P.nq == 0) return MO_RC_SUCCESS;
    Stager st(t);
    const size_t per = (size_t)P.nq * P.k * 8;
    const int64_t *ik = (const int64_t *)st.in(args[2].pdata, per * nshards);
    const double *id = (const double *)st.in(args[3].pdata, per * nshards);
    int64_t *ok = (int64_t *)st.out(args[0].pdata, per);
    double *od = (double *)st.out(args[1].pdata, per);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    topk_merge_kernel<<<(unsigned)((P.nq + 127) / 128), 128, 0, t.stream>>>(P.nq, P.k, (int)nshards, P.nq, nullptr, nullptr, id, ik, nullptr, 0, 0, 0, ok, od);
    MOB_LAUNCH_CHECK();
    return st.finish();
}

}  // namespace mob

// =========================================================================================================
// IVF-flat probe
// =========================================================================================================
namespace {

// (query, probe rank) -> bucket of its list.  Order inside a bucket is arbitrary (atomics) but results do not depend on it:
// every (query, list) pair is scanned independently and exactly, and lands in the fixed slot query*nprobe + rank.
// list sharding (whole lists per GPU): a probed list that is empty on this shard contributes nothing -- drop the pair before it is
// bucketed, so neither its residual operand nor its work unit is ever built
__global__ void ivf_mask_empty_kernel(int64_t *probes, int64_t npairs, const int64_t *__restrict__ offsets) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < npairs; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t l = probes[i];
        if (l >= 0 && offsets[l + 1] <= offsets[l]) probes[i] = -1;
    }
}
__global__ void ivf_count_kernel(const int64_t *probes, int64_t npairs, int *cnt) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < npairs; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t l = probes[i];
        if (l >= 0) atomicAdd(&cnt[l], 1);
    }
}
__global__ void ivf_fill_kernel(const int64_t *probes, int64_t npairs, int nprobe, const int *start, int *cursor,
                                int32_t *bucket_q, int32_t *bucket_l, int64_t *bucket_slot, int32_t *pair_pos) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < npairs; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t l = probes[i];
        if (l < 0) { pair_pos[i] = -1; continue; }
        const int pos = start[l] + atomicAdd(&cursor[l], 1);
        bucket_q[pos] = (int32_t)(i / nprobe);
        bucket_l[pos] = (int32_t)l;
        bucket_slot[pos] = i;
        pair_pos[i] = pos;
    }
}

}  // namespace

namespace mob {

int redo_queries(ThreadCtx &t, const std::vector<int> &redo, const float *dq, int dim, int k, int64_t *out_k, double *out_d,
                 const std::function<int(const float *sub, int64_t m, int64_t *sk, double *sd)> &next) {
    if (redo.empty()) return MO_RC_SUCCESS;
    const int m = (int)redo.size();
    int *didx = (int *)arena_alloc(t, sizeof(int) * (size_t)m);
    float *sub = (float *)arena_alloc(t, sizeof(float) * (size_t)m * dim);
    int64_t *sk = (int64_t *)arena_alloc(t, sizeof(int64_t) * (size_t)m * k);
    double *sd = (double *)arena_alloc(t, sizeof(double) * (size_t)m * k);
    if (!didx || !sub || !sk || !sd) return MO_RC_INTERNAL_ERROR;
    MOB_CUDA_TRY(cudaMemcpyAsync(didx, redo.data(), sizeof(int) * (size_t)m, cudaMemcpyHostToDevice, t.stream));
    MOB_CUDA_TRY(cudaStreamSynchronize(t.stream));
    gather_rows_kernel<<<num_sms() * 4, 256, 0, t.stream>>>(dq, didx, m, dim, sub);
    MOB_LAUNCH_CHECK();
    int rc = next(sub, m, sk, sd);
    if (rc) return rc;
    scatter_results_kernel<<<(unsigned)((m * k + 255) / 256), 256, 0, t.stream>>>(sk, sd, didx, m, k, out_k, out_d);
    MOB_LAUNCH_CHECK();
    return MO_RC_SUCCESS;
}

struct IvfJob {
    const float *dcent; int64_t nlist; const float *ddata; int64_t n; int dim; const std::vector<int64_t> *offsets; const int64_t *doffsets;
    const int64_t *drowids;
    int k, nprobe, metric, sqrt_out;
    const uint32_t *admit;   // filtered search, masked scan: admitted list-ordered rows (nullptr: all)
};

// level 0: tensor-core candidate pass over whole lists (one-term product when the ladder allows it, else three-term), level 1: the
// queries it could not prove, three-term product with every list cut into sub-ranges, level 2: whatever is still unproven
// through the exact kernel.  Each level answers its queries exactly or hands them down; results are scattered back into the
// caller's rows.
static int ivf_search_level(ThreadCtx &t, const IvfJob &J, int level, const float *dq, int64_t nq, int64_t *ok, double *od) {
    IvfPlan plan;
    int rc = ivf_make_plan(t, J.dcent, J.nlist, J.dim, dq, nq, J.nprobe, J.metric, plan, J.doffsets);
    if (rc) return rc;
    if (level >= 2 || !tc_ivf_applicable(J.n, J.dim, nq, J.k, J.nprobe, J.metric, level == 1)) {
        if (level > 0) g_search_stats.fallbacks = (int)nq;
        return ivf_exact_scan(t, plan, J.ddata, J.n, J.dim, dq, nq, *J.offsets, J.drowids, J.k, J.metric, J.sqrt_out, ok, od, J.admit);
    }
    std::vector<int> redo;
    bool nonfinite = false;
    const int pass = level == 1 ? 2 : (tc_one_term_wanted(J.k, true) ? 0 : 1);
    rc = ivf_tc_scan(t, plan, J.ddata, J.n, J.dim, dq, nq, J.dcent, J.doffsets, *J.offsets, J.drowids, J.k, J.sqrt_out, pass, ok, od, redo, &nonfinite, J.admit);
    if (!rc && pass == 0 && !nonfinite) tc_one_term_report(nq, (int64_t)redo.size());
    if (rc) return rc;
    if (level == 0) { g_search_stats.refined = (int)redo.size(); g_search_stats.fallbacks = 0; }
    return redo_queries(t, redo, dq, J.dim, J.k, ok, od, [&](const float *sub, int64_t m, int64_t *sk, double *sd) {
        return ivf_search_level(t, J, nonfinite ? 2 : level + 1, sub, m, sk, sd);
    });
}

// IvfflatSearchIndex.Search (pkg/vectorindex/ivfflat/search.go:509-630):
//   findCentroids (:292-311)  = exact top-nprobe over the centroid table (same kernel, k = nprobe)
//   list scan + ORDER BY LIMIT (:572-592) = exact top-k over the rows of the probed lists
// args: see MO_XCALL_IVF_TOPK_F32 in include/mo_b200.h.
static int ivf_call(mo_xcall_args_t *args, uint64_t len, const mo_xcall_args_t *farg) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    SearchReadGuard guard;
    mo_search_params_t P;
    int rc = read_param(t, args[4], &P, sizeof P, sizeof P, "search: params");
    if (rc) return rc;
    if (P.nq != (int64_t)len) { set_error("ivf: len != params.nq"); return MO_RC_INVALID_ARGUMENT; }
    if (P.k == 0 || P.nq == 0) return MO_RC_SUCCESS;
    if (P.k > KMAX) { set_error("ivf: k=%d exceeds the fused kernel limit %d", P.k, KMAX); return MO_RC_INVALID_ARGUMENT; }
    int nprobe = P.nprobe < 1 ? 1 : P.nprobe;
    if (nprobe > P.nlist) nprobe = (int)P.nlist;
    if (nprobe > KMAX) { set_error("ivf: nprobe=%d exceeds the limit %d", nprobe, KMAX); return MO_RC_INVALID_ARGUMENT; }
    const int dim = (int)P.dim;
    if (args[2].dataSz < (uint64_t)P.n * dim * 4 || args[3].dataSz < (uint64_t)P.nq * dim * 4 || args[5].dataSz < (uint64_t)P.nlist * dim * 4 ||
        args[6].dataSz < (uint64_t)(P.nlist + 1) * 8 || args[7].dataSz < (uint64_t)P.n * 8 ||
        args[0].dataSz < (uint64_t)P.nq * P.k * 8 || args[1].dataSz < (uint64_t)P.nq * P.k * 8) {
        set_error("ivf: buffer sizes do not match params"); return MO_RC_INVALID_ARGUMENT;
    }
    mo_search_filter_t F;
    if (farg && (rc = read_filter(t, *farg, &F)) != 0) return rc;
    Stager st(t);
    const float *ddata = (const float *)st.in(args[2].pdata, (size_t)P.n * dim * 4);
    const float *dq = (const float *)st.in(args[3].pdata, (size_t)P.nq * dim * 4);
    const float *dcent = (const float *)st.in(args[5].pdata, (size_t)P.nlist * dim * 4);
    const int64_t *drowids = (const int64_t *)st.in(args[7].pdata, (size_t)P.n * 8);
    const int64_t *doffsets = (const int64_t *)st.in(args[6].pdata, (size_t)(P.nlist + 1) * 8);
    int64_t *ok = (int64_t *)st.out(args[0].pdata, (size_t)P.nq * P.k * 8);
    double *od = (double *)st.out(args[1].pdata, (size_t)P.nq * P.k * 8);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    std::vector<int64_t> offsets((size_t)P.nlist + 1);
    if (is_device_ptr(args[6].pdata)) { MOB_CUDA_TRY(cudaMemcpyAsync(offsets.data(), args[6].pdata, offsets.size() * 8, cudaMemcpyDeviceToHost, t.stream)); MOB_CUDA_TRY(cudaStreamSynchronize(t.stream)); }
    else memcpy(offsets.data(), args[6].pdata, offsets.size() * 8);

    IvfJob job{dcent, P.nlist, ddata, P.n, dim, &offsets, doffsets, drowids, (int)P.k, nprobe, (int)P.metric, (int)P.sqrt_out, nullptr};
    g_search_stats = SearchStats();
    if (!farg) {
        rc = ivf_search_level(t, job, 0, dq, P.nq, ok, od);
    } else {
        // the probes depend only on the centroids: both paths probe the lists the unfiltered search probes
        uint32_t *admit; int64_t m = 0;
        rc = filter_admission(t, st, F, P.n, 0, drowids, &admit, &m);
        std::vector<int64_t> sub_offsets((size_t)P.nlist + 1);
        if (!rc && filter_compact_wanted(P.n, m, true)) {
            // few admitted rows: a compacted index -- the admitted entries in list order, their primary keys, and list boundaries
            // rebuilt from them (lists without an admitted row become empty, and their probes are dropped)
            int32_t *idx; float *sub;
            int64_t *sub_ids = (int64_t *)arena_alloc(t, (size_t)(m > 0 ? m : 1) * 8), *dsub_off = (int64_t *)arena_alloc(t, sub_offsets.size() * 8);
            rc = sub_ids && dsub_off ? filter_gather(t, ddata, P.n, dim, admit, m, &idx, &sub) : MO_RC_INTERNAL_ERROR;
            if (!rc) {
                if (m > 0) filter_gather_ids_kernel<<<num_sms() * 4, 256, 0, t.stream>>>(drowids, idx, m, sub_ids);
                filter_offsets_kernel<<<(unsigned)((P.nlist + 256) / 256), 256, 0, t.stream>>>(doffsets, P.nlist, idx, m, dsub_off);
                g_launches += m > 0 ? 2 : 1;
                if (cudaGetLastError() != cudaSuccess) { set_error("filtered search: compaction launch failed"); rc = MO_RC_INTERNAL_ERROR; }
            }
            if (!rc && (cudaMemcpyAsync(sub_offsets.data(), dsub_off, sub_offsets.size() * 8, cudaMemcpyDeviceToHost, t.stream) != cudaSuccess ||
                        cudaStreamSynchronize(t.stream) != cudaSuccess)) { set_error("filtered search: list boundaries download failed"); rc = MO_RC_INTERNAL_ERROR; }
            if (!rc) {
                IvfJob sj{dcent, P.nlist, sub, m, dim, &sub_offsets, dsub_off, sub_ids, (int)P.k, nprobe, (int)P.metric, (int)P.sqrt_out, nullptr};
                rc = ivf_search_level(t, sj, 0, dq, P.nq, ok, od);
            }
        } else if (!rc) {
            g_search_stats.filter_compacted = 0;
            job.admit = admit;
            rc = ivf_search_level(t, job, 0, dq, P.nq, ok, od);
        }
    }
    int frc = st.finish();
    return rc ? rc : frc;
}

int xcall_ivf(mo_xcall_args_t *args, uint64_t len) { return ivf_call(args, len, nullptr); }
int xcall_ivf_filtered(mo_xcall_args_t *args, uint64_t len) { return ivf_call(args, len, &args[8]); }

// 1. probes[q][rank] = list id by ascending centroid distance (findCentroids, ivfflat/search.go:292-311): the exact top-nprobe kernel
// 2. invert: list -> bucket of (query, slot) pairs
int ivf_make_plan(ThreadCtx &t, const float *dcent, int64_t nlist, int dim, const float *dq, int64_t nq, int nprobe, int metric, IvfPlan &plan,
                  const int64_t *doffsets) {
    plan.nprobe = nprobe;
    plan.npairs = nq * nprobe;
    const int64_t npairs = plan.npairs;
    plan.probes = (int64_t *)arena_alloc(t, (size_t)npairs * 8);
    double *probe_d = (double *)arena_alloc(t, (size_t)npairs * 8);
    int *cnt = (int *)arena_alloc(t, (size_t)nlist * 4 * 3);
    plan.bucket_q = (int32_t *)arena_alloc(t, (size_t)npairs * 4);
    plan.bucket_slot = (int64_t *)arena_alloc(t, (size_t)npairs * 8);
    plan.pair_pos = (int32_t *)arena_alloc(t, (size_t)npairs * 4);
    plan.bucket_l = (int32_t *)arena_alloc(t, (size_t)npairs * 4);
    if (!plan.probes || !probe_d || !cnt || !plan.bucket_q || !plan.bucket_slot || !plan.pair_pos || !plan.bucket_l) return MO_RC_INTERNAL_ERROR;
    // exact either way: the tensor-core pass proves its top-nprobe complete or re-runs the query through the exact kernel
    int rc;
    if (tc_probe_applicable(nlist, dim, nq, nprobe, metric)) {
        rc = bruteforce_topk_tc_device(t, dcent, nlist, dim, dq, nq, nprobe, 0, 0, plan.probes, probe_d, false);
    } else {
        g_search_stats.probe_kused = 0;   // (an earlier level of the ladder may have probed on the tensor cores)
        rc = bruteforce_topk_device(t, dcent, nlist, dim, dq, nq, nprobe, metric, 0, 0, plan.probes, probe_d);
    }
    if (rc) return rc;
    int *dstart = cnt + nlist, *cursor = cnt + 2 * nlist;
    if (doffsets) { ivf_mask_empty_kernel<<<num_sms() * 4, 256, 0, t.stream>>>(plan.probes, npairs, doffsets); MOB_LAUNCH_CHECK(); }
    MOB_CUDA_TRY(cudaMemsetAsync(cnt, 0, (size_t)nlist * 4 * 3, t.stream));
    ivf_count_kernel<<<num_sms() * 4, 256, 0, t.stream>>>(plan.probes, npairs, cnt);
    MOB_LAUNCH_CHECK();
    plan.hcnt.assign((size_t)nlist, 0); plan.hstart.assign((size_t)nlist, 0);
    MOB_CUDA_TRY(cudaMemcpyAsync(plan.hcnt.data(), cnt, (size_t)nlist * 4, cudaMemcpyDeviceToHost, t.stream));
    MOB_CUDA_TRY(cudaStreamSynchronize(t.stream));
    int run = 0;
    for (int64_t l = 0; l < nlist; l++) { plan.hstart[(size_t)l] = run; run += plan.hcnt[(size_t)l]; }
    plan.nvalid = run;   // bucket entries [0, nvalid) are defined; pairs of missing / empty lists have none
    MOB_CUDA_TRY(cudaMemcpyAsync(dstart, plan.hstart.data(), (size_t)nlist * 4, cudaMemcpyHostToDevice, t.stream));
    ivf_fill_kernel<<<num_sms() * 4, 256, 0, t.stream>>>(plan.probes, npairs, nprobe, dstart, cursor, plan.bucket_q, plan.bucket_l, plan.bucket_slot, plan.pair_pos);
    MOB_LAUNCH_CHECK();
    MOB_CUDA_TRY(cudaStreamSynchronize(t.stream));   // hstart (pageable host memory) must stay valid until the copy above is done
    return MO_RC_SUCCESS;
}

// 3. (list, 64-query tile) work items through the exact kernel; 4. merge the nprobe partial lists of each query, local row -> primary
// key through row_ids, optional sqrt (DistanceTransformIvfflat)
int ivf_exact_scan(ThreadCtx &t, const IvfPlan &plan, const float *ddata, int64_t n, int dim, const float *dq, int64_t nq,
                   const std::vector<int64_t> &offsets, const int64_t *drowids, int k, int metric, int sqrt_out, int64_t *ok, double *od,
                   const uint32_t *admit) {
    const int64_t nlist = (int64_t)offsets.size() - 1;
    const int64_t npairs = plan.npairs;
    float *xnorm, *qnorm;
    int rc = cos_norms(t, metric, ddata, n, dq, nq, dim, &xnorm, &qnorm);
    if (rc) return rc;
    std::vector<WorkDesc> items;
    for (int64_t l = 0; l < nlist; l++) {
        const int c = plan.hcnt[(size_t)l];
        if (c == 0 || offsets[(size_t)l + 1] <= offsets[(size_t)l]) continue;
        for (int q0 = 0; q0 < c; q0 += TQ) {
            WorkDesc w;
            w.data = ddata; w.n = n; w.row_begin = offsets[(size_t)l]; w.row_end = offsets[(size_t)l + 1];
            w.queries = dq; w.nq_total = nq; w.qidx = plan.bucket_q + plan.hstart[(size_t)l] + q0; w.q0 = 0;
            w.nq_local = c - q0 < TQ ? c - q0 : TQ;
            w.slot_of = plan.bucket_slot + plan.hstart[(size_t)l] + q0; w.range = 0; w.xnorm = xnorm; w.qnorm = qnorm; w.admit = admit;
            items.push_back(w);
        }
    }
    float *part_d = (float *)arena_alloc(t, sizeof(float) * (size_t)(npairs * k));
    int32_t *part_i = (int32_t *)arena_alloc(t, sizeof(int32_t) * (size_t)(npairs * k));
    WorkDesc *ditems = (WorkDesc *)arena_alloc(t, sizeof(WorkDesc) * (items.size() ? items.size() : 1));
    if (!part_d || !part_i || !ditems) return MO_RC_INTERNAL_ERROR;
    MOB_CUDA_TRY(cudaMemsetAsync(part_i, 0xff, sizeof(int32_t) * (size_t)(npairs * k), t.stream));   // -1 = empty slot
    if (!items.empty()) {
        MOB_CUDA_TRY(cudaMemcpyAsync(ditems, items.data(), sizeof(WorkDesc) * items.size(), cudaMemcpyHostToDevice, t.stream));
        MOB_CUDA_TRY(cudaStreamSynchronize(t.stream));
        rc = launch_bf_metric(t, metric, ditems, (int)items.size(), dim, k, part_d, part_i);
        if (rc) return rc;
    }
    topk_merge_kernel<<<(unsigned)((nq + 127) / 128), 128, 0, t.stream>>>(nq, k, plan.nprobe, nq, part_d, part_i, nullptr, nullptr, drowids, 0, sqrt_out, 1, ok, od);
    MOB_LAUNCH_CHECK();
    return MO_RC_SUCCESS;
}

}  // namespace mob
