// distance.cu -- row-wise vector distances over MatrixOne varlena columns, behind XCall.
//
//   ids 0..3   (reference ids, cgo/mo.c:49-52): semantics of cgo/xcall.c:23-134 -- float diff, squares summed in
//              double, optional sqrt; dim taken from the first cell of arg 1; rows null in the result bitmap skipped.
//              This replaces cgo/cuda/mocl.cu:4-86 (one thread per row, uncoalesced, += into global memory).
//   ids 100..109 (new): the Go metric functions of pkg/vectorindex/metric/distance_func.go as wrapped by
//              pkg/vectorize/moarray/external.go:171-260 (what l2_distance / inner_product / cosine_distance /
//              cosine_similarity evaluate per row).  BIT-EXACT: the accumulator has the element type and the
//              8-way (cosine: 4-way) unrolled association of the Go source is reproduced operation by operation.
//
// Mapping: LANE per row, warp-transposed.  A warp takes 32 consecutive rows; it copies one 128-byte slice of each of them per
// step with cp.async (16 bytes per lane per instruction, 8 lanes cover a row slice: fully coalesced, no registers held while
// the bytes are in flight) into a per-warp shared-memory ring, and every lane then walks ITS row's slice serially in exactly
// the order of the Go loop -- no shuffles, ~100 warp instructions per row instead of ~520 (one warp per row replayed the
// serial `sum += chunk` chain with 96 shuffle+add pairs and was instruction/MIO-bound at 0.55 of the HBM rate; cosine with
// its three chains at 0.19).  The ring (5 stages, or 3 when both operands are per-row) is what keeps ~128 KB per SM in flight.
// Algorithmic bytes per row = 2 * dim * sizeof(T) (one side const: dim * sizeof(T)) + 24 per varlena cell + 8 for the result.
#include "column.cuh"
#include "godist.cuh"
#include <cstring>

using namespace mob;

namespace {

constexpr int kThreads = 128;   // 4 warps; every warp owns a shared-memory ring

constexpr unsigned ST_DIM = 1u, ST_AREA = 2u, ST_ZERO = 4u, ST_EMPTY = 8u;

using Ref = VarlenaRef;

using namespace mob::godist;

template <typename T, int KIND, bool TWO>
__global__ void __launch_bounds__(kThreads)
rowdist_kernel(double *__restrict__ res, const uint64_t *__restrict__ rnulls, uint64_t n, const __grid_constant__ Operand x1,
               const __grid_constant__ Operand x2, unsigned *status) {
    using Cfg = RingCfg<TWO>;
    using Acc = RowAcc<T, KIND>;
    constexpr int NST = Cfg::kStages;
    extern __shared__ __align__(16) unsigned char dist_smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    unsigned char *ring = dist_smem + (size_t)wib * NST * Cfg::kStageBytes;
    const uint64_t warp = (blockIdx.x * (uint64_t)kThreads + threadIdx.x) >> 5;
    const uint64_t nwarps = ((uint64_t)gridDim.x * kThreads) >> 5;
    int xc_dim = 0;
    if (Acc::kXc) {  // dim = c1.len / sizeof(T) from the FIRST cell of arg 1, xcall.c:40,55
        Ref r0 = varlena_ref((const uint8_t *)x1.data, 0, x1.area, x1.area_sz);
        xc_dim = r0.ok ? (int)(r0.len / sizeof(T)) : 0;
    }
    // the per-row ("x") side is arg 1 unless only arg 1 is const; every kind is symmetric in its operands bit for bit
    // ((a-b)^2 == (b-a)^2, products commute, the cosine denominator sqrt(n1)*sqrt(n2) commutes)
    const bool swap = !TWO && x1.cst && !x2.cst;
    unsigned st = 0;
    for (uint64_t base = warp * 32; base < n; base += nwarps * 32) {
        const uint64_t i = base + lane;
        const bool live = i < n && !bm_test(rnulls, i);
        int dim = 0; bool good = false;
        const uint8_t *px = nullptr, *pq = nullptr;
        if (live) {
            Ref a = varlena_ref((const uint8_t *)x1.data, x1.cst ? 0 : i, x1.area, x1.area_sz);
            Ref b = Acc::kOne ? a : varlena_ref((const uint8_t *)x2.data, x2.cst ? 0 : i, x2.area, x2.area_sz);
            if (!a.ok || !b.ok) st |= ST_AREA;
            else if (Acc::kOne && a.len < sizeof(T)) st |= ST_EMPTY;   // "cannot normalize empty vector", distance_func.go:413-415
            else if (Acc::kXc) {
                if ((uint64_t)xc_dim * sizeof(T) > a.len || (uint64_t)xc_dim * sizeof(T) > b.len) st |= ST_DIM;   // would read out of bounds
                else { dim = xc_dim; good = true; }
            } else {
                if (a.len != b.len) st |= ST_DIM;   // moerr.NewArrayInvalidOpNoCtx, external.go:182-184
                else { dim = (int)(a.len / sizeof(T)); good = true; }
            }
            px = swap ? b.ptr : a.ptr; pq = swap ? a.ptr : b.ptr;
        }
        if (!good) dim = 0;
        Acc acc = row_batch<T, KIND, TWO>(ring, lane, px, pq, dim, good);
        if (good) {
            double out; bool write = true;
            if (KIND == K_XC_L2) out = sqrt(acc.dsum);
            else if (KIND == K_XC_L2SQ) out = acc.dsum;
            else if (KIND == K_GO_NORM) out = sqrt(acc.dsum);                    // norm := math.Sqrt(sumSquares), distance_func.go:422
            else if (KIND == K_GO_L2SQ || KIND == K_GO_L1) out = (double)acc.sum;
            else if (KIND == K_GO_L2) out = (double)(T)sqrt((double)acc.sum);  // distance_func.go:35-42
            else if (KIND == K_GO_IP) out = (double)(-acc.sum);               // InnerProduct returns -sum, distance_func.go:172-205
            else {
                const double den = sqrt((double)acc.n1) * sqrt((double)acc.n2);
                if (KIND == K_GO_COSDIST) {
                    if (dim == 0) out = 0.0;
                    else if (den == 0.0) out = (double)(T)1.0;        // distance_func.go:268-271
                    else {
                        double sim = (double)acc.sum / den;
                        sim = sim > 1.0 ? 1.0 : (sim < -1.0 ? -1.0 : sim);
                        out = (double)(T)(1.0 - sim);
                    }
                } else {
                    if (dim == 0) out = 0.0;
                    else if (den == 0.0) { st |= ST_ZERO; write = false; out = 0.0; }   // "one of the vector is zero", distance_func.go:342-345
                    else {
                        double sim = (double)acc.sum / den;
                        sim = sim > 1.0 ? 1.0 : (sim < -1.0 ? -1.0 : sim);
                        double c = (double)(T)sim;
                        const float f = (float)c;                        // moarray.CosineSimilarity snap, external.go:252-257
                        if (f == 1.0f) c = 1.0; else if (f == -1.0f) c = -1.0;
                        out = c;
                    }
                }
            }
            if (write) res[i] = out;
        }
    }
    st = __reduce_or_sync(FULL, st);
    if (lane == 0 && st) atomicOr(status, st);
}

// argument k's cells and area, its size and data checked by the caller.  Only the result's bitmap says which rows are NULL, so the argument's is not staged; and a zero-byte area
// still bounds an empty value at offset 0, as it always has here.
int stage_vectors(Stager &st, const mo_xcall_args_t &arg, uint64_t len, const char *what, int k, Operand &o) {
    mo_xcall_args_t a = arg;
    a.pnulls = nullptr;
    if (int rc = stage_operand(st, a, MO_VARLENA_SZ, len, what, k, o)) return rc;
    if (!o.area) o.area = a.parea;
    return MO_RC_SUCCESS;
}

template <typename T, int KIND>
int run_rowdist(mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (len == 0) return MO_RC_SUCCESS;
    if (!args[0].pdata || args[0].dataSz < 8 * len) { set_error("distance: result vector shorter than len"); return MO_RC_INVALID_ARGUMENT; }
    for (int k = 1; k <= 2; k++) {
        if (!is_const(args[k], MO_VARLENA_SZ, len) && args[k].dataSz < 24 * len) { set_error("distance: argument vector shorter than len"); return MO_RC_INVALID_ARGUMENT; }
        if (!args[k].pdata) { set_error("distance: argument %d has no data", k); return MO_RC_INVALID_ARGUMENT; }
    }
    Stager st(t);
    Operand x1, x2;
    if (int rc = stage_vectors(st, args[1], len, "distance", 1, x1)) return rc;
    if (int rc = stage_vectors(st, args[2], len, "distance", 2, x2)) return rc;
    const uint64_t *rn = (const uint64_t *)st.in(args[0].pnulls, args[0].pnulls ? ((len + 63) / 64) * 8 : 0);
    double *res = (double *)st.out(args[0].pdata, 8 * len, args[0].pnulls != nullptr);
    unsigned *dstatus = (unsigned *)st.tmp(4);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    MOB_CUDA_TRY(cudaMemsetAsync(dstatus, 0, 4, t.stream));
    const bool two = !x1.cst && !x2.cst;
    const uint64_t warps = (len + 31) / 32;
    uint64_t blocks = (warps + kThreads / 32 - 1) / (kThreads / 32);
    const uint64_t cap = (uint64_t)num_sms() * 2;   // 2 CTAs per SM by shared memory (95 / 111 KB each)
    if (blocks > cap) blocks = cap;
    const size_t smem = (size_t)(kThreads / 32) * (two ? RingCfg<true>::kStages * RingCfg<true>::kStageBytes : RingCfg<false>::kStages * RingCfg<false>::kStageBytes);
    static bool attr1 = false, attr2 = false;
    if (two && !attr2) { MOB_CUDA_TRY(cudaFuncSetAttribute(rowdist_kernel<T, KIND, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr2 = true; }
    if (!two && !attr1) { MOB_CUDA_TRY(cudaFuncSetAttribute(rowdist_kernel<T, KIND, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr1 = true; }
    cudaEventRecord(t.kev0, t.stream);
    if (two) rowdist_kernel<T, KIND, true><<<(unsigned)blocks, kThreads, smem, t.stream>>>(res, rn, len, x1, x2, dstatus);
    else rowdist_kernel<T, KIND, false><<<(unsigned)blocks, kThreads, smem, t.stream>>>(res, rn, len, x1, x2, dstatus);
    cudaEventRecord(t.kev1, t.stream);
    MOB_LAUNCH_CHECK();
    unsigned status = 0;
    int rc = read_back(t, &status, dstatus, 4);
    int frc = st.finish();
    if (rc) return rc;
    if (frc) return frc;
    if (status & ST_AREA) { set_error("distance: varlena cell points outside its area"); return MO_RC_INVALID_ARGUMENT; }
    if (status & ST_DIM) { set_error("distance: vector dimension not matched"); return MO_RC_INVALID_ARGUMENT; }
    if (status & ST_ZERO) { set_error("cosine similarity: one of the vector is zero"); return MO_RC_INTERNAL_ERROR; }
    return MO_RC_SUCCESS;
}

// ---- NormalizeL2Array (moarray/external.go:262-285 == metric.NormalizeL2, distance_func.go:411-434): a VECTOR-valued result -------------
// Pass 1 = rowdist_kernel<T, K_GO_NORM> (the row's norm, float64, summed strictly in index order by the row's lane).  Pass 2 below: one warp
// per row writes normalized[i] = T(float64(val) / norm) (norm == 0: the row is copied), and the result's varlena cell.  Layout of the
// result: the cell of row i has the SAME (offset, length) as the input's cell -- the result area mirrors the input area, inline cells stay
// inline -- so no prefix sum over lengths is needed and a const input yields a const-shaped result (every cell points at the one vector).
// Algorithmic bytes per row: 2 reads + 1 write of dim * sizeof(T) (the second read is served from L2 when the rows are short), 48 of cells.
//
// Whether a row below i is not NULL (the warp of row i asks; all lanes get the answer).  A const input's vector is written by the first
// row that is not NULL: row 0 may be NULL.  The words below i are scanned downwards from i, so over all rows of a call the scans read
// each bitmap word about once.
__device__ __forceinline__ bool live_below(const uint64_t *rnulls, uint64_t i, int lane) {
    if (i == 0) return false;
    if (!rnulls) return true;
    const uint64_t top = (i - 1) >> 6;
    for (uint64_t b = 0; b <= top; b += 32) {
        bool hit = false;
        if (b + lane <= top) {
            const uint64_t w = top - b - lane;
            uint64_t live = ~rnulls[w];
            const uint64_t below = i - (w << 6);          // rows of word w that are below i
            if (below < 64) live &= (1ull << below) - 1;
            hit = live != 0;
        }
        if (__any_sync(FULL, hit)) return true;
    }
    return false;
}

template <typename T>
__global__ void __launch_bounds__(256)
normalize_write_kernel(uint8_t *__restrict__ ocells, uint8_t *__restrict__ oarea, const uint64_t *__restrict__ rnulls, uint64_t n,
                       const __grid_constant__ Operand in, const double *__restrict__ norms) {
    const int lane = threadIdx.x & 31;
    const uint64_t warp = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5, nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t i = warp; i < n; i += nwarps) {
        uint8_t *oc = ocells + 24 * i;
        if (bm_test(rnulls, i)) { if (lane < 24) oc[lane] = 0; continue; }          // NULL row: an empty inline cell
        const uint8_t *c = (const uint8_t *)in.data + 24 * (in.cst ? 0 : i);
        const Ref a = varlena_ref((const uint8_t *)in.data, in.cst ? 0 : i, in.area, in.area_sz);
        if (!a.ok || a.len < sizeof(T)) continue;                                   // reported by pass 1
        const int dim = (int)(a.len / sizeof(T));
        const double norm = norms[i];
        if (a.inl) {   // <= 23 bytes: the vector lives in the cell
            if (lane == 0) oc[0] = c[0];
            if (lane >= 1 && lane < 24 && lane > (int)a.len) oc[lane] = 0;
            if (lane < dim) {
                const T v = load1<T>(a.ptr + (size_t)lane * sizeof(T));
                const T o = norm == 0.0 ? v : (T)__ddiv_rn((double)v, norm);
                uint8_t b[sizeof(T)]; memcpy(b, &o, sizeof(T));
#pragma unroll
                for (int k = 0; k < (int)sizeof(T); k++) oc[1 + lane * sizeof(T) + k] = b[k];
            }
            // bytes between dim * sizeof(T) and a.len (a length that is not a multiple of the element size) are copied
            if (lane < (int)a.len - dim * (int)sizeof(T)) oc[1 + dim * sizeof(T) + lane] = a.ptr[dim * sizeof(T) + lane];
            continue;
        }
        if (lane < 24) oc[lane] = c[lane];
        if (in.cst && live_below(rnulls, i, lane)) continue;                        // a const input: one vector, written once
        uint8_t *dst = oarea + (a.ptr - in.area);
        if (((((uintptr_t)a.ptr) | ((uintptr_t)dst)) & 15) == 0) {
            constexpr int EPV = 16 / (int)sizeof(T);
            const int nv = dim / EPV;
            for (int v = lane; v < nv; v += 32) {
                const int4 raw = ld_stream16(a.ptr + 16 * (size_t)v);
                T x[EPV]; memcpy(x, &raw, 16);
#pragma unroll
                for (int k = 0; k < EPV; k++) x[k] = norm == 0.0 ? x[k] : (T)__ddiv_rn((double)x[k], norm);
                int4 o; memcpy(&o, x, 16);
                *reinterpret_cast<int4 *>(dst + 16 * (size_t)v) = o;
            }
            for (int e = nv * EPV + lane; e < dim; e += 32) {
                const T v = load1<T>(a.ptr + (size_t)e * sizeof(T));
                const T o = norm == 0.0 ? v : (T)__ddiv_rn((double)v, norm);
                memcpy(dst + (size_t)e * sizeof(T), &o, sizeof(T));
            }
        } else {
            for (int e = lane; e < dim; e += 32) {
                const T v = load1<T>(a.ptr + (size_t)e * sizeof(T));
                const T o = norm == 0.0 ? v : (T)__ddiv_rn((double)v, norm);
                uint8_t b[sizeof(T)]; memcpy(b, &o, sizeof(T));
#pragma unroll
                for (int k = 0; k < (int)sizeof(T); k++) dst[(size_t)e * sizeof(T) + k] = b[k];
            }
        }
    }
}

template <typename T>
int run_normalize(mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (len == 0) return MO_RC_SUCCESS;
    if (!args[0].pdata || args[0].dataSz < 24 * len) { set_error("normalize_l2: result vector shorter than len"); return MO_RC_INVALID_ARGUMENT; }
    if (!is_const(args[1], MO_VARLENA_SZ, len) && args[1].dataSz < 24 * len) { set_error("normalize_l2: argument vector shorter than len"); return MO_RC_INVALID_ARGUMENT; }
    if (!args[1].pdata) { set_error("normalize_l2: argument 1 has no data"); return MO_RC_INVALID_ARGUMENT; }
    if (args[1].areaSz && (!args[0].parea || args[0].areaSz < args[1].areaSz)) { set_error("normalize_l2: the result area must be at least as large as the argument's (it mirrors its layout)"); return MO_RC_INVALID_ARGUMENT; }
    Stager st(t);
    Operand x;
    if (int rc = stage_vectors(st, args[1], len, "normalize_l2", 1, x)) return rc;
    const uint64_t *rn = (const uint64_t *)st.in(args[0].pnulls, args[0].pnulls ? ((len + 63) / 64) * 8 : 0);
    uint8_t *ocells = (uint8_t *)st.out(args[0].pdata, 24 * len);
    uint8_t *oarea = args[1].areaSz ? (uint8_t *)st.out(args[0].parea, args[1].areaSz, true) : nullptr;
    double *norms = (double *)st.tmp(8 * len);
    unsigned *dstatus = (unsigned *)st.tmp(4);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    MOB_CUDA_TRY(cudaMemsetAsync(dstatus, 0, 4, t.stream));
    const uint64_t warps = (len + 31) / 32;
    uint64_t blocks = (warps + kThreads / 32 - 1) / (kThreads / 32);
    if (blocks > (uint64_t)num_sms() * 2) blocks = (uint64_t)num_sms() * 2;
    const size_t smem = (size_t)(kThreads / 32) * RingCfg<false>::kStages * RingCfg<false>::kStageBytes;
    static bool attr = false;
    if (!attr) { MOB_CUDA_TRY(cudaFuncSetAttribute(rowdist_kernel<T, K_GO_NORM, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = true; }
    cudaEventRecord(t.kev0, t.stream);
    rowdist_kernel<T, K_GO_NORM, false><<<(unsigned)blocks, kThreads, smem, t.stream>>>(norms, rn, len, x, x, dstatus);
    MOB_LAUNCH_CHECK();
    uint64_t wblocks = (len + 7) / 8;
    if (wblocks > (uint64_t)num_sms() * 8) wblocks = (uint64_t)num_sms() * 8;
    normalize_write_kernel<T><<<(unsigned)wblocks, 256, 0, t.stream>>>(ocells, oarea, rn, len, x, norms);
    cudaEventRecord(t.kev1, t.stream);
    MOB_LAUNCH_CHECK();
    unsigned status = 0;
    int rc = read_back(t, &status, dstatus, 4);
    int frc = st.finish();
    if (rc) return rc;
    if (frc) return frc;
    if (status & ST_AREA) { set_error("normalize_l2: varlena cell points outside its area"); return MO_RC_INVALID_ARGUMENT; }
    if (status & ST_EMPTY) { set_error("cannot normalize empty vector"); return MO_RC_INTERNAL_ERROR; }
    return MO_RC_SUCCESS;
}

}  // namespace

namespace mob {

int xcall_rowdist(int64_t funcId, mo_xcall_args_t *args, uint64_t len) {
    switch (funcId) {
    case MO_XCALL_L2DISTANCE_F32: return run_rowdist<float, K_XC_L2>(args, len);
    case MO_XCALL_L2DISTANCE_F64: return run_rowdist<double, K_XC_L2>(args, len);
    case MO_XCALL_L2DISTANCE_SQ_F32: return run_rowdist<float, K_XC_L2SQ>(args, len);
    case MO_XCALL_L2DISTANCE_SQ_F64: return run_rowdist<double, K_XC_L2SQ>(args, len);
    case MO_XCALL_GO_L2_F32: return run_rowdist<float, K_GO_L2>(args, len);
    case MO_XCALL_GO_L2_F64: return run_rowdist<double, K_GO_L2>(args, len);
    case MO_XCALL_GO_L2SQ_F32: return run_rowdist<float, K_GO_L2SQ>(args, len);
    case MO_XCALL_GO_L2SQ_F64: return run_rowdist<double, K_GO_L2SQ>(args, len);
    case MO_XCALL_GO_IP_F32: return run_rowdist<float, K_GO_IP>(args, len);
    case MO_XCALL_GO_IP_F64: return run_rowdist<double, K_GO_IP>(args, len);
    case MO_XCALL_GO_COSDIST_F32: return run_rowdist<float, K_GO_COSDIST>(args, len);
    case MO_XCALL_GO_COSDIST_F64: return run_rowdist<double, K_GO_COSDIST>(args, len);
    case MO_XCALL_GO_COSSIM_F32: return run_rowdist<float, K_GO_COSSIM>(args, len);
    case MO_XCALL_GO_COSSIM_F64: return run_rowdist<double, K_GO_COSSIM>(args, len);
    case MO_XCALL_GO_L1_F32: return run_rowdist<float, K_GO_L1>(args, len);
    case MO_XCALL_GO_L1_F64: return run_rowdist<double, K_GO_L1>(args, len);
    case MO_XCALL_GO_NORMALIZE_L2_F32: return run_normalize<float>(args, len);
    case MO_XCALL_GO_NORMALIZE_L2_F64: return run_normalize<double>(args, len);
    }
    return -1;
}

}  // namespace mob
