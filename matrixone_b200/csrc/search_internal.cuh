// search_internal.cuh -- declarations shared by search.cu (exact kernels) and tcsearch.cu (tensor-core candidate pass)
#pragma once
#include "common.cuh"
#include <functional>
#include <vector>

namespace mob {

// IVF probe plan: which lists every query scans, inverted into per-list buckets of (query, slot) pairs
struct IvfPlan {
    int nprobe = 0;
    int64_t npairs = 0;            // nq * nprobe
    int64_t nvalid = 0;            // pairs that landed in a bucket (npairs minus missing / empty lists)
    int64_t *probes = nullptr;     // [nq][nprobe] list ids by ascending centroid distance (-1 = none)       (device)
    int32_t *bucket_q = nullptr;   // [npairs] query of every bucket entry, entries of one list are contiguous  (device)
    int32_t *bucket_l = nullptr;   // [npairs] list of every bucket entry                                        (device)
    int64_t *bucket_slot = nullptr;// [npairs] q * nprobe + rank of every bucket entry                          (device)
    int32_t *pair_pos = nullptr;   // [npairs] inverse map: position of pair (q, rank) in the buckets, -1 = none (device)
    std::vector<int> hcnt, hstart; // per list: bucket size / first position                                    (host)
};

// admit (filtered search, nullable): bit r of 32-bit word r / 32 set = row r may be listed; rows are dataset rows (brute force) or
// list-ordered entries (IVF).  With nullptr every path computes exactly what it computes without a filter.
int bruteforce_topk_device(ThreadCtx &t, const float *ddata, int64_t n, int dim, const float *dq, int64_t nq, int k, int metric,
                           int64_t key_base, int sqrt_out, int64_t *out_k, double *out_d, const uint32_t *admit = nullptr);
int ivf_make_plan(ThreadCtx &t, const float *dcent, int64_t nlist, int dim, const float *dq, int64_t nq, int nprobe, int metric, IvfPlan &plan,
                  const int64_t *doffsets = nullptr);   // doffsets: drop the pairs of lists that are empty here (list-sharded index)
int ivf_exact_scan(ThreadCtx &t, const IvfPlan &plan, const float *ddata, int64_t n, int dim, const float *dq, int64_t nq,
                   const std::vector<int64_t> &offsets, const int64_t *drowids, int k, int metric, int sqrt_out, int64_t *ok, double *od,
                   const uint32_t *admit = nullptr);

// held (shared) by every search entry point for the duration of the call; see g_search_rw in tcsearch.cu
struct SearchReadGuard { SearchReadGuard(); ~SearchReadGuard(); SearchReadGuard(const SearchReadGuard &) = delete; SearchReadGuard &operator=(const SearchReadGuard &) = delete; };

bool tc_search_applicable(int64_t n, int dim, int64_t nq, int k, int metric);
bool tc_probe_applicable(int64_t nlist, int dim, int64_t nq, int nprobe, int metric);
// record_stats = false: a helper search inside another call (IVF centroid probe) leaves the fallback counter and kernel timer alone
// and records only probe_kused
int bruteforce_topk_tc_device(ThreadCtx &t, const float *ddata, int64_t n, int dim, const float *dq, int64_t nq, int k,
                              int64_t key_base, int sqrt_out, int64_t *out_k, double *out_d, bool record_stats = true, int metric = MO_METRIC_L2SQ,
                              const uint32_t *admit = nullptr);
bool tc_ivf_applicable(int64_t n, int dim, int64_t nq, int k, int nprobe, int metric, bool refine);
// returns the queries whose completeness proof failed in `redo` (their rows of ok/od are still filled with best-effort results).
// pass 0 = one-term product, 1 = three-term, 2 = three-term over list sub-ranges.  *nonfinite: Inf/NaN input, the error bound
// does not apply, redo = all.
int ivf_tc_scan(ThreadCtx &t, const IvfPlan &plan, const float *ddata, int64_t n, int dim, const float *dq, int64_t nq,
                const float *dcent, const int64_t *doffsets, const std::vector<int64_t> &offsets, const int64_t *drowids, int k, int sqrt_out,
                int pass, int64_t *ok, double *od, std::vector<int> &redo, bool *nonfinite, const uint32_t *admit = nullptr);
bool tc_one_term_wanted(int k, bool record);   // ladder policy shared by brute force and IVF
// filtered search: gather the `admitted` rows of `n` and search only them (true), or scan all rows under the admission mask (false)
bool filter_compact_wanted(int64_t n, int64_t admitted, bool ivf);
// order-preserving compaction (colops.cu): the indices of the set bits of bits[0, n) (32 rows per word), ascending; *dtotal = their count
int compact_bits(ThreadCtx &t, const uint32_t *bits, uint64_t n, int32_t *sels, unsigned long long *dtotal);
void tc_one_term_report(int64_t nq, int64_t failed);

// the next level of a precision ladder for the queries in `redo` (rows of dq): they are gathered into one sub-batch, next(sub, m, sk, sd)
// answers it, and its keys and distances are scattered back into their rows of out_k / out_d
int redo_queries(ThreadCtx &t, const std::vector<int> &redo, const float *dq, int dim, int k, int64_t *out_k, double *out_d,
                 const std::function<int(const float *sub, int64_t m, int64_t *sk, double *sd)> &next);

// statistics of the last search on this thread (MoB200_SetTuning "get_tc_*"); xcall_bruteforce and xcall_ivf reset them at entry
struct SearchStats {
    int kused = 0;        // K columns per (query, row) pair the search's first candidate pass multiplied (0: it ran no candidate pass)
    int probe_kused = 0;  // IVF: K columns of the last pass of the centroid probe (0: the probe ran on the exact kernel)
    int refined = -1;     // queries the first tensor-core level could not prove (brute force: only a one-term level records it)
    int fallbacks = -1;   // queries that ended in the exact kernel (-1: the search did not reach the tensor cores)
    int filter_admitted = -1;   // filtered search: rows the filter admitted (-1: no filter)
    int filter_compacted = -1;  // filtered search: 1 = the admitted rows were gathered and searched, 0 = masked scan of every row
};
extern thread_local SearchStats g_search_stats;

}  // namespace mob
