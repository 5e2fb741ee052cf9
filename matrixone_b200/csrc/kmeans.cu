// kmeans.cu -- Elkan k-means (the IVF index build's clustering), dense variant, on the GPU with the reference's results.
//
// Reference: pkg/vectorindex/ivfflat/kmeans/elkans/clusterer.go -- Cluster :330-356, elkansCluster :358-392, initBounds :458-512,
// computeCentroidDistances :516-575, assignData :579-676, recalculateCentroids :679-727, updateBounds :730-762.  The distance is metric.L2Distance for
// every metric (ResolveKmeansDistanceFnForDense, distance_func.go:452-476).  Given the initial centroids every step is deterministic: the per-vector
// loops are independent (the reference's worker pools only partition rows) and recalculateCentroids sums a cluster's members serially, in row order,
// in the element type.  So the results -- centroids bit for bit, assignments, iteration count -- can be reproduced by keeping each of those orders:
//
//   distances     godist::go_l2sq: one warp per (vector, centroid) pair replays the Go loop's 8-way association and its serial chunk chain
//   assignData    one warp per vector walks the centroids in order with the vector's (upper, assignment, recompute) in registers, exactly the
//                 reference's branch sequence; a distance is computed by the whole warp only where the reference computes it
//   recalculate   members of every cluster in ROW ORDER through the stable grouping of join.cu (radix sort by cluster id), then one thread per
//                 (cluster, dimension) adds them in that order; 1 / T(count) scaling as metric.ScaleInPlace; an empty cluster takes `dim` values of
//                 the caller's rnd.Float32() stream (clusterer.go:700-707), in cluster order
//   updateBounds  elementwise, Go's math.Max(x, 0) semantics (-0 -> +0)
//
// InitCentroids (random draws from Go's PCG / kmeans++, initializer.go) stays with the caller: the op takes the initial centroids.
// Memory: lower bounds n x k elements in HBM (the reference keeps the same matrix).  The pass is compute-light after the first iterations (most
// (vector, centroid) pairs are pruned by the bounds); initBounds is the n x k x dim part.
#include "common.cuh"
#include "godist.cuh"
#include <cstring>
#include <vector>

namespace mob {

int group_rows_stable(ThreadCtx &t, const uint64_t *groups, uint64_t len, uint64_t ngroups, uint64_t **starts, uint32_t **rows, uint64_t **scal_out);   // join.cu

namespace {

constexpr int kThreads = 256;
using godist::FULL;

template <typename T>
__device__ __forceinline__ T l2dist(const T *p, const T *q, int dim, int lane) {   // metric.L2Distance: T(math.Sqrt(float64(L2DistanceSq)))
    const bool al = ((((uintptr_t)p) | ((uintptr_t)q)) & 15) == 0;
    const T s = godist::go_l2sq<T>(reinterpret_cast<const uint8_t *>(p), reinterpret_cast<const uint8_t *>(q), dim, lane, al, false, false);
    return (T)sqrt((double)s);
}
__device__ __forceinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double div_rn(double a, double b) { return __ddiv_rn(a, b); }
template <typename T> __device__ __forceinline__ T go_max0(T s) { return s > (T)0 ? s : (s != s ? s : (T)0); }   // T(math.Max(float64(s), 0))

template <typename T>
__global__ void __launch_bounds__(kThreads) km_init_bounds_kernel(const T *__restrict__ vec, int64_t n, int dim, const T *__restrict__ cent, int k,
                                                                  T *__restrict__ lower, T *__restrict__ upper, uint8_t *__restrict__ recompute, int32_t *__restrict__ assign) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * (int64_t)kThreads + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * kThreads) >> 5;
    for (int64_t x = warp; x < n; x += nwarps) {
        T minDist = sizeof(T) == 4 ? (T)3.40282346638528859811704183484516925440e+38 : (T)1.79769313486231570814527423731704356798070e+308;
        int closest = 0;
        for (int c = 0; c < k; c++) {
            const T d = l2dist(vec + x * dim, cent + (int64_t)c * dim, dim, lane);
            if (lane == 0) lower[x * k + c] = d;
            if (d < minDist) { minDist = d; closest = c; }
        }
        if (lane == 0) { upper[x] = minDist; assign[x] = closest; recompute[x] = 1; }
    }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) km_pair_dists_kernel(const T *__restrict__ cent, int k, int dim, T *__restrict__ half) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * (int64_t)kThreads + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * kThreads) >> 5;
    for (int64_t pr = warp; pr < (int64_t)k * k; pr += nwarps) {
        const int i = (int)(pr / k), j = (int)(pr % k);
        if (j <= i) continue;
        T d = l2dist(cent + (int64_t)i * dim, cent + (int64_t)j * dim, dim, lane);
        d = d * (T)0.5;
        if (lane == 0) { half[(int64_t)i * k + j] = d; half[(int64_t)j * k + i] = d; }
    }
}
template <typename T>
__global__ void __launch_bounds__(kThreads) km_min_half_kernel(const T *__restrict__ half, int k, T *__restrict__ minhalf) {
    for (int i = blockIdx.x * kThreads + threadIdx.x; i < k; i += gridDim.x * kThreads) {
        T cur = (T)3.40282346638528859811704183484516925440e+38;   // T(math.MaxFloat32), clusterer.go:565
        for (int j = 0; j < k; j++) {
            if (j == i) continue;
            const double a = (double)cur, b = (double)half[(int64_t)i * k + j];
            cur = (T)(b < a ? b : (b != b ? b : a));                 // math.Min
        }
        minhalf[i] = cur;
    }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) km_assign_kernel(const T *__restrict__ vec, int64_t n, int dim, const T *__restrict__ cent, int k, const T *__restrict__ half,
                                                             const T *__restrict__ minhalf, T *__restrict__ lower, T *__restrict__ upper, uint8_t *__restrict__ recompute,
                                                             int32_t *__restrict__ assign, unsigned long long *changes) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * (int64_t)kThreads + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * kThreads) >> 5;
    unsigned long long mychanges = 0;
    for (int64_t x = warp; x < n; x += nwarps) {
        T up = upper[x]; int a = assign[x]; bool rec = recompute[x] != 0;
        if (up <= minhalf[a]) continue;                                              // step 2: u(x) <= s(c(x))
        T *lx = lower + x * k;
        const T *vx = vec + x * dim;
        for (int c = 0; c < k; c++) {
            if (c == a) continue;
            if (!(up > lx[c] && up > half[(int64_t)a * k + c])) continue;            // step 3 (ii), (iii)
            T dxcx;
            if (rec) {
                rec = false;
                dxcx = l2dist(vx, cent + (int64_t)a * dim, dim, lane);
                up = dxcx;
                if (lane == 0) lx[a] = dxcx;
                __syncwarp();
                if (up <= lx[c]) continue;
                if (up <= half[(int64_t)a * k + c]) continue;
            } else dxcx = up;
            if (dxcx > lx[c] || dxcx > half[(int64_t)a * k + c]) {
                const T dxc = l2dist(vx, cent + (int64_t)c * dim, dim, lane);
                if (lane == 0) lx[c] = dxc;
                __syncwarp();
                if (dxc < dxcx) { up = dxc; a = c; mychanges++; }
            }
        }
        if (lane == 0) { upper[x] = up; assign[x] = a; recompute[x] = rec ? 1 : 0; }
    }
    if (lane == 0 && mychanges) atomicAdd(changes, mychanges);
}

__global__ void __launch_bounds__(kThreads) km_groups_kernel(const int32_t *__restrict__ assign, int64_t n, uint64_t *__restrict__ groups) {
    for (int64_t x = blockIdx.x * (int64_t)kThreads + threadIdx.x; x < n; x += (int64_t)gridDim.x * kThreads) groups[x] = (uint64_t)assign[x] + 1;
}

// empty clusters consume the caller's rnd stream in cluster order: rnd_base[c] = dim * (number of empty clusters before c); one thread (k is small)
__global__ void km_empty_prefix_kernel(const uint64_t *__restrict__ starts, int k, int dim, int64_t *__restrict__ rnd_base, int64_t rnd_len, int *__restrict__ status) {
    if (blockIdx.x || threadIdx.x) return;
    int64_t used = 0;
    for (int c = 0; c < k; c++) {
        rnd_base[c] = used;
        if (starts[c + 1] == starts[c]) used += dim;
    }
    if (used > rnd_len) *status = 1;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) km_recalc_kernel(const T *__restrict__ vec, int dim, int k, const uint64_t *__restrict__ starts, const uint32_t *__restrict__ rows,
                                                             const float *__restrict__ rnd, const int64_t *__restrict__ rnd_base, int64_t rnd_len, T *__restrict__ newc) {
    const int64_t total = (int64_t)k * dim;
    for (int64_t e = blockIdx.x * (int64_t)kThreads + threadIdx.x; e < total; e += (int64_t)gridDim.x * kThreads) {
        const int c = (int)(e / dim), i = (int)(e % dim);
        const uint64_t s0 = starts[c], s1 = starts[c + 1];
        if (s1 == s0) {                                                               // empty: T(rnd.Float32())
            const int64_t r = rnd_base[c] + i;
            newc[e] = r < rnd_len ? (T)rnd[r] : (T)0;
            continue;
        }
        T sum = 0;
        for (uint64_t m = s0; m < s1; m++) sum = godist::add_rn(sum, vec[(int64_t)rows[m] * dim + i]);   // newCentroids[cx][i] += vec[i], members in row order
        const T scale = div_rn((T)1.0, (T)(int64_t)(s1 - s0));                          // metric.ScaleInPlace(v, 1.0 / T(count))
        newc[e] = godist::mul_rn(sum, scale);
    }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) km_shift_kernel(const T *__restrict__ cent, const T *__restrict__ newc, int k, int dim, T *__restrict__ shift) {
    const int lane = threadIdx.x & 31;
    const int warp = (blockIdx.x * kThreads + threadIdx.x) >> 5, nwarps = (gridDim.x * kThreads) >> 5;
    for (int c = warp; c < k; c += nwarps) {
        const T d = l2dist(cent + (int64_t)c * dim, newc + (int64_t)c * dim, dim, lane);
        if (lane == 0) shift[c] = d;
    }
}
template <typename T>
__global__ void __launch_bounds__(kThreads) km_update_bounds_kernel(int64_t n, int k, const T *__restrict__ shift, const int32_t *__restrict__ assign, T *__restrict__ lower,
                                                                    T *__restrict__ upper, uint8_t *__restrict__ recompute) {
    const int64_t total = n * k;
    for (int64_t e = blockIdx.x * (int64_t)kThreads + threadIdx.x; e < total; e += (int64_t)gridDim.x * kThreads) {
        const int c = (int)(e % k);
        lower[e] = go_max0(godist::sub_rn(lower[e], shift[c]));
        if (c == 0) { const int64_t x = e / k; upper[x] = godist::add_rn(upper[x], shift[assign[x]]); recompute[x] = 1; }
    }
}
__global__ void __launch_bounds__(kThreads) km_assign_out_kernel(const int32_t *__restrict__ assign, int64_t n, int64_t *__restrict__ out) {
    for (int64_t x = blockIdx.x * (int64_t)kThreads + threadIdx.x; x < n; x += (int64_t)gridDim.x * kThreads) out[x] = assign[x];
}

inline unsigned grid_for(int64_t items, int per_block = kThreads) {
    int64_t g = (items + per_block - 1) / per_block;
    const int64_t mx = (int64_t)num_sms() * 8;
    return (unsigned)(g > mx ? mx : (g > 0 ? g : 1));
}

template <typename T>
int run_kmeans(mo_xcall_args_t *args) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    mo_kmeans_params_t P;
    if (int rc = read_param(t, args[3], &P, sizeof P, sizeof P, "kmeans: mo_kmeans_params_t")) return rc;
    const int64_t n = P.n, dim = P.dim, k = P.k;
    if (n < 1 || dim < 1 || k < 1 || k > n || dim > (1 << 20) || k > (1 << 20) || P.max_iter < 1) { set_error("kmeans: bad shape n=%lld dim=%lld k=%lld max_iter=%lld", (long long)n, (long long)dim, (long long)k, (long long)P.max_iter); return MO_RC_INVALID_ARGUMENT; }
    if (args[0].dataSz < (uint64_t)(k * dim) * sizeof(T) || args[1].dataSz < (uint64_t)n * 8 || !args[2].pdata || args[2].dataSz < 8 || args[4].dataSz < (uint64_t)(n * dim) * sizeof(T)) { set_error("kmeans: buffers too small"); return MO_RC_INVALID_ARGUMENT; }
    Stager st(t);
    T *cent = (T *)st.out(args[0].pdata, (size_t)(k * dim) * sizeof(T), true);
    int64_t *assign_out = (int64_t *)st.out(args[1].pdata, (size_t)n * 8);
    const T *vec = (const T *)st.in(args[4].pdata, (size_t)(n * dim) * sizeof(T));
    const int64_t rnd_len = args[5].pdata ? (int64_t)(args[5].dataSz / 4) : 0;
    const float *rnd = (const float *)st.in(args[5].pdata, (size_t)rnd_len * 4);
    T *lower = (T *)st.tmp((size_t)(n * k) * sizeof(T)), *upper = (T *)st.tmp((size_t)n * sizeof(T)), *half = (T *)st.tmp((size_t)(k * k) * sizeof(T));
    T *minhalf = (T *)st.tmp((size_t)k * sizeof(T)), *next = (T *)st.tmp((size_t)(k * dim) * sizeof(T)), *shift = (T *)st.tmp((size_t)k * sizeof(T));
    uint8_t *recompute = (uint8_t *)st.tmp((size_t)n);
    int32_t *assign = (int32_t *)st.tmp((size_t)n * 4);
    uint64_t *groups = (uint64_t *)st.tmp((size_t)n * 8);
    int64_t *rnd_base = (int64_t *)st.tmp((size_t)k * 8);
    unsigned long long *dchanges = (unsigned long long *)st.tmp(16);
    int *dstatus = (int *)(dchanges + 1);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    MOB_CUDA_TRY(cudaMemsetAsync(half, 0, (size_t)(k * k) * sizeof(T), t.stream));
    MOB_CUDA_TRY(cudaMemsetAsync(dchanges, 0, 16, t.stream));
    cudaEventRecord(t.kev0, t.stream);
    km_init_bounds_kernel<T><<<grid_for(n * 32), kThreads, 0, t.stream>>>(vec, n, (int)dim, cent, (int)k, lower, upper, recompute, assign);
    MOB_LAUNCH_CHECK();
    int64_t iter = 0, rnd_used = 0;
    int rc = MO_RC_SUCCESS;
    // every iteration allocates scratch for the stable grouping from the arena: remember the mark and rewind (the arena is a bump allocator)
    for (;; iter++) {
        km_pair_dists_kernel<T><<<grid_for(k * k * 32), kThreads, 0, t.stream>>>(cent, (int)k, (int)dim, half);
        MOB_LAUNCH_CHECK();
        km_min_half_kernel<T><<<grid_for(k), kThreads, 0, t.stream>>>(half, (int)k, minhalf);
        MOB_LAUNCH_CHECK();
        MOB_CUDA_TRY(cudaMemsetAsync(dchanges, 0, 8, t.stream));
        km_assign_kernel<T><<<grid_for(n * 32), kThreads, 0, t.stream>>>(vec, n, (int)dim, cent, (int)k, half, minhalf, lower, upper, recompute, assign, dchanges);
        MOB_LAUNCH_CHECK();
        km_groups_kernel<<<grid_for(n), kThreads, 0, t.stream>>>(assign, n, groups);
        MOB_LAUNCH_CHECK();
        const ArenaMark mark = arena_mark(t);
        uint64_t *starts, *scal; uint32_t *rows;
        rc = group_rows_stable(t, groups, (uint64_t)n, (uint64_t)k, &starts, &rows, &scal);
        if (rc) break;
        km_empty_prefix_kernel<<<1, 32, 0, t.stream>>>(starts, (int)k, (int)dim, rnd_base, rnd_len - rnd_used, dstatus);
        MOB_LAUNCH_CHECK();
        km_recalc_kernel<T><<<grid_for(k * dim), kThreads, 0, t.stream>>>(vec, (int)dim, (int)k, starts, rows, rnd + rnd_used, rnd_base, rnd_len - rnd_used, next);
        MOB_LAUNCH_CHECK();
        km_shift_kernel<T><<<grid_for(k * 32), kThreads, 0, t.stream>>>(cent, next, (int)k, (int)dim, shift);
        MOB_LAUNCH_CHECK();
        km_update_bounds_kernel<T><<<grid_for(n * k), kThreads, 0, t.stream>>>(n, (int)k, shift, assign, lower, upper, recompute);
        MOB_LAUNCH_CHECK();
        MOB_CUDA_TRY(cudaMemcpyAsync(cent, next, (size_t)(k * dim) * sizeof(T), cudaMemcpyDeviceToDevice, t.stream));
        // host decisions of this iteration: changes, the rnd stream, how many empty clusters consumed it
        struct { unsigned long long changes; int status; int pad; } h;
        rc = read_back(t, &h, dchanges, 16);
        if (rc) break;
        if (h.status) { set_error("kmeans: an empty cluster needs %lld random values, the rnd vector is exhausted", (long long)dim); rc = MO_RC_INVALID_ARGUMENT; break; }
        // count the consumed random values: starts of the empty clusters (k is small: read the starts back only when rnd is in use)
        if (rnd_len > rnd_used) {
            std::vector<uint64_t> hs((size_t)k + 1);
            rc = read_back(t, hs.data(), starts, (size_t)(k + 1) * 8);
            if (rc) break;
            for (int64_t c = 0; c < k; c++) if (hs[(size_t)c + 1] == hs[(size_t)c]) rnd_used += dim;
        }
        arena_rewind(t, mark);
        if (iter != 0 && (iter == P.max_iter || h.changes == 0)) break;               // isConverged, clusterer.go:765-775
    }
    if (rc) { st.finish(); return rc; }
    km_assign_out_kernel<<<grid_for(n), kThreads, 0, t.stream>>>(assign, n, assign_out);
    cudaEventRecord(t.kev1, t.stream);
    MOB_LAUNCH_CHECK();
    int frc = st.finish();
    if (frc) return frc;
    const int64_t iters = iter + 1;
    return write_param(t, args[2].pdata, &iters, 8);
}

}  // namespace

// MO_XCALL_KMEANS_ELKAN_F32 / _F64: args [0] centroids T[k * dim] (in: initial, out: final) ; [1] assignments int64[n] (out) ; [2] int64 iterations (out) ;
// [3] mo_kmeans_params_t ; [4] vectors T[n * dim] ; [5] rnd float32[] (optional: the rnd.Float32() stream empty clusters draw from)
int xcall_kmeans(int64_t funcId, mo_xcall_args_t *args, uint64_t len) {
    (void)len;
    return funcId == MO_XCALL_KMEANS_ELKAN_F32 ? run_kmeans<float>(args) : run_kmeans<double>(args);
}

}  // namespace mob
