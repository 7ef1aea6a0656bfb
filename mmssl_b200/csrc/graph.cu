// Graph preparation for the SpMM operator: torch sparse COO (int64 indices, fp32 values, possibly
// unsorted / with duplicate coordinates) -> CSR with int32 indices, for A and for A^T, plus the
// nnz-balanced work plan the SpMM kernel consumes.  All device-side, no host synchronisation.
//
// Replaces what ATen does inside torch.sparse.mm on every call of the reference
// (Models.py:69-73, :203-208: coalesce + COO->CSR conversion before cuSPARSE) with a one-time,
// cached conversion (see mmssl_b200/graph.py).  Graph normalisation itself (main.py:89-103) is
// provided as mmssl_csr_row_normalize.
#include <cub/cub.cuh>

#include "common.cuh"
#include "../../include/mmssl_b200.h"

namespace mmssl {

__global__ void make_keys_kernel(const int64_t* __restrict__ rows, const int64_t* __restrict__ cols, int64_t nnz,
                                 int transpose, uint64_t* __restrict__ keys, uint32_t* __restrict__ idx) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= nnz) return;
    const uint64_t r = (uint64_t)(transpose ? cols[i] : rows[i]);
    const uint64_t c = (uint64_t)(transpose ? rows[i] : cols[i]);
    keys[i] = (r << 32) | (c & 0xffffffffull);
    idx[i] = (uint32_t)i;
}

__global__ void scatter_sorted_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ idx,
                                      const float* __restrict__ vals, int64_t nnz, int32_t* __restrict__ colidx,
                                      float* __restrict__ out_vals) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= nnz) return;
    colidx[i] = (int32_t)(keys[i] & 0xffffffffull);
    out_vals[i] = vals[idx[i]];
}

// rowptr[r] = first position whose key >= (r << 32); rowptr[n_rows] = nnz.
__global__ void rowptr_kernel(const uint64_t* __restrict__ keys, int64_t nnz, int64_t n_rows,
                              int32_t* __restrict__ rowptr) {
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r > n_rows) return;
    const uint64_t target = (uint64_t)r << 32;
    int64_t lo = 0, hi = nnz;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (keys[mid] < target) lo = mid + 1; else hi = mid;
    }
    rowptr[r] = (int32_t)lo;
}

__global__ void fill_i32_kernel(int32_t* p, int64_t n, int32_t v) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

static inline int ceil_log2(uint64_t v) {
    int b = 0;
    while ((1ull << b) < v) ++b;
    return b;
}

struct CsrWs {
    uint64_t* keys_in; uint64_t* keys_out; uint32_t* idx_in; uint32_t* idx_out; void* cub_tmp; size_t cub_bytes;
    size_t total;
};

static cudaError_t carve_csr_ws(int64_t nnz, int64_t n_rows, void* base, CsrWs* w) {
    size_t cub_bytes = 0;
    const int end_bit = 32 + ceil_log2((uint64_t)(n_rows > 1 ? n_rows : 2));
    cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                                                    (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)nnz, 0, end_bit);
    if (e != cudaSuccess) return e;
    auto up = [](size_t v) { return (v + 255) & ~(size_t)255; };
    size_t off = 0;
    char* b = (char*)base;
    w->keys_in = (uint64_t*)(b + off); off += up(sizeof(uint64_t) * nnz);
    w->keys_out = (uint64_t*)(b + off); off += up(sizeof(uint64_t) * nnz);
    w->idx_in = (uint32_t*)(b + off); off += up(sizeof(uint32_t) * nnz);
    w->idx_out = (uint32_t*)(b + off); off += up(sizeof(uint32_t) * nnz);
    w->cub_tmp = (void*)(b + off); off += up(cub_bytes);
    w->cub_bytes = cub_bytes;
    w->total = off + 256;
    return cudaSuccess;
}

// ---------------------------------------------------------------- SpMM work plan
// item = {row, begin, end, split}: split = -1 -> the item covers the whole row (<= kSplitThreshold
// non-zeros); otherwise the index of the row in the split-row table {first partial slot, #segments,
// segment length, 0}.  Long rows are cut into segments that different lane groups process
// concurrently (the critical path of a small graph is its longest serial row walk); the last group
// to finish reduces the partial sums in segment order, so results stay deterministic.
// Rows up to kHeavyThreshold: segments of 32, partial sums reduced in segment order (deterministic).
// Heavier rows (the head of a power-law degree distribution): segments of 64 that accumulate with
// 128-bit float atomics into a dedicated zeroed row -- a serial reduction over hundreds of partials
// would otherwise be the kernel's critical path.  (Summation order of those few rows is not fixed.)
// Defaults chosen by measurement on the earlier hardware (tools/probe.py plan; not re-tuned for the H100): the kernel's duration on a small graph is its longest item --
// an item of 64 non-zeros is 8 dependent gather batches of 8 -- so rows are cut earlier than the first version did (64 / 32).
struct PlanCuts { int split_threshold, seg_len, heavy_threshold, heavy_seg_len; };
static PlanCuts g_cuts = {64, 32, 1024, 64};
__host__ __device__ __forceinline__ int plan_seg_len(int len, const PlanCuts c) { return len <= c.heavy_threshold ? c.seg_len : c.heavy_seg_len; }
int4 spmm_plan_cuts() { return make_int4(g_cuts.split_threshold, g_cuts.seg_len, g_cuts.heavy_threshold, g_cuts.heavy_seg_len); }

__global__ void plan_count_kernel(const int32_t* __restrict__ rowptr, int64_t n_rows,
                                  int32_t* __restrict__ n_items, int32_t* __restrict__ is_split,
                                  int32_t* __restrict__ n_segs, const PlanCuts cuts) {
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r >= n_rows) return;
    const int len = rowptr[r + 1] - rowptr[r];
    const bool split = len > cuts.split_threshold;
    const int sl = plan_seg_len(len, cuts);
    const int segs = split ? (len + sl - 1) / sl : 0;
    n_items[r] = split ? segs : 1;
    is_split[r] = split ? 1 : 0;
    n_segs[r] = segs;
}

__global__ void plan_fill_kernel(const int32_t* __restrict__ rowptr, int64_t n_rows,
                                 const int32_t* __restrict__ item_off, const int32_t* __restrict__ split_off,
                                 const int32_t* __restrict__ seg_off, const int32_t* __restrict__ is_split,
                                 int4* __restrict__ items, int4* __restrict__ split_table, int32_t* __restrict__ totals,
                                 const PlanCuts cuts) {
    const int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= n_rows) return;
    const int b = rowptr[r], e = rowptr[r + 1];
    const int sl = plan_seg_len(e - b, cuts);
    const int segs = is_split[r] ? (e - b + sl - 1) / sl : 0;
    if (!is_split[r]) {
        if (lane == 0) items[item_off[r]] = make_int4((int)r, b, e, -1);
    } else {
        const int s = split_off[r];
        for (int k = lane; k < segs; k += 32) {
            const int sb = b + k * sl;
            items[item_off[r] + k] = make_int4((int)r, sb, min(e, sb + sl), s);
        }
        if (lane == 0) split_table[s] = make_int4(seg_off[r], segs, sl, (e - b) > cuts.heavy_threshold ? 1 : 0);
    }
    if (r == n_rows - 1 && lane == 0) {
        totals[0] = item_off[r] + (is_split[r] ? segs : 1);   // number of work items
        totals[1] = split_off[r] + is_split[r];               // number of split rows
        totals[2] = seg_off[r] + segs;                        // number of partial-sum slots
    }
}


// ---------------------------------------------------------------- work plan of the staged-gather SpMM (spmm_bulk.cu)
// BUCKETS of at most 32 consecutive non-zeros (one per lane of the warp that owns the bucket) and at most 8 rows, that never cut
// a row of <= 32 non-zeros:
//   * rows of <= 32 non-zeros ("short", empty rows included) are grouped by the 32-aligned window their first position falls
//     in; the rows of one window form a run (a longer row in between ends it).  A run spans at most 63 positions and only its
//     last row can end more than 32 positions after the run's first one: that row gets a bucket of its own, the others share
//     buckets of up to 8 rows;
//   * a row of more than 32 non-zeros is cut into chunks of 32 from its start, one bucket each; split-row table entry
//     {first partial slot, #chunks, 0, heavy}: heavy (> 32 chunks) rows accumulate with vector reductions.
//   bucket = {first row, #rows, first position, #positions}, {split-row index or -1, chunk index, 0, 0}, in row order.
constexpr int kBulkBucket = 32;
constexpr int kBulkRows = 8;
constexpr int kBulkHeavySegs = 32;

__global__ void bulk_runflag_kernel(const int32_t* __restrict__ rowptr, int64_t n_rows, int32_t* __restrict__ run_flag) {
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r >= n_rows) return;
    const int b = rowptr[r], e = rowptr[r + 1];
    bool start = (r == 0) || (e - b) > kBulkBucket;
    if (!start) {
        const int pb = rowptr[r - 1];
        start = (b - pb) > kBulkBucket || (b / kBulkBucket) != (pb / kBulkBucket);
    }
    run_flag[r] = start ? 1 : 0;
}

__global__ void bulk_runfirst_kernel(const int32_t* __restrict__ run_flag, const int32_t* __restrict__ run_excl, int64_t n_rows,
                                     int32_t* __restrict__ run_first) {
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r < n_rows && run_flag[r]) run_first[run_excl[r]] = (int32_t)r;
}

__global__ void bulk_count_kernel(const int32_t* __restrict__ rowptr, int64_t n_rows, const int32_t* __restrict__ run_flag,
                                  const int32_t* __restrict__ run_excl, const int32_t* __restrict__ run_first,
                                  int32_t* __restrict__ n_bk, int32_t* __restrict__ is_split, int32_t* __restrict__ n_segs) {
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r >= n_rows) return;
    const int b = rowptr[r], e = rowptr[r + 1];
    if (e - b > kBulkBucket) {
        const int chunks = (e - b + kBulkBucket - 1) / kBulkBucket;
        n_bk[r] = chunks; is_split[r] = 1; n_segs[r] = chunks;
        return;
    }
    const int rs = run_first[run_excl[r] + run_flag[r] - 1];      // first row of this row's run
    const bool straddler = (e - rowptr[rs]) > kBulkBucket;
    n_bk[r] = (r == rs || straddler || ((r - rs) % kBulkRows) == 0) ? 1 : 0;
    is_split[r] = 0; n_segs[r] = 0;
}

__global__ void bulk_fill_kernel(const int32_t* __restrict__ rowptr, int64_t n_rows, const int32_t* __restrict__ n_bk,
                                 const int32_t* __restrict__ bk_off, const int32_t* __restrict__ split_off,
                                 const int32_t* __restrict__ seg_off, const int32_t* __restrict__ is_split, int4* __restrict__ buckets,
                                 int4* __restrict__ split_table, int32_t* __restrict__ totals) {
    const int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= n_rows) return;
    const int b = rowptr[r], e = rowptr[r + 1];
    const int nb = n_bk[r], o = bk_off[r];
    if (is_split[r]) {
        const int s = split_off[r];
        for (int k = lane; k < nb; k += 32) {
            buckets[2 * (o + k)] = make_int4((int)r, 1, b + k * kBulkBucket, min(kBulkBucket, e - (b + k * kBulkBucket)));
            buckets[2 * (o + k) + 1] = make_int4(s, k, 0, 0);
        }
        if (lane == 0) split_table[s] = make_int4(seg_off[r], nb, 0, nb > kBulkHeavySegs ? 1 : 0);
    } else if (nb == 1 && lane == 0) {
        buckets[2 * o] = make_int4((int)r, 0, b, 0);          // #rows / #positions: bulk_extent_kernel (needs the next bucket's first row)
        buckets[2 * o + 1] = make_int4(-1, 0, 0, 0);
    }
    if (r == n_rows - 1 && lane == 0) {
        totals[0] = o + nb;                                    // buckets
        totals[1] = split_off[r] + is_split[r];                // split rows
        totals[2] = seg_off[r] + (is_split[r] ? nb : 0);       // partial-sum slots
    }
}

__global__ void bulk_extent_kernel(const int32_t* __restrict__ rowptr, int64_t n_rows, const int32_t* __restrict__ totals,
                                   int32_t* __restrict__ buckets) {
    const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int total = totals[0];
    if (k >= total) return;
    if (buckets[8 * k + 4] >= 0) return;                       // chunk of a long row: complete
    const int row0 = buckets[8 * k];
    const int r1 = (k + 1 < total) ? buckets[8 * (k + 1)] : (int)n_rows;
    buckets[8 * k + 1] = r1 - row0;
    buckets[8 * k + 3] = rowptr[r1] - rowptr[row0];
}

__global__ void row_normalize_kernel(const int32_t* __restrict__ rowptr, int64_t n_rows, float* __restrict__ vals) {
    // D_row^{-1/2} * A with the reference's +1e-8 inside the power (main.py:90-93), in double.
    const int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= n_rows) return;
    const int b = rowptr[r], e = rowptr[r + 1];
    double s = 0.0;
    for (int k = b + lane; k < e; k += 32) s += (double)vals[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const double scale = 1.0 / sqrt(s + 1e-8);   // rows with sum 0 have no entries to scale
    for (int k = b + lane; k < e; k += 32) vals[k] = (float)((double)vals[k] * scale);
}

}  // namespace mmssl

using namespace mmssl;

extern "C" int64_t mmssl_csr_workspace_bytes(int64_t nnz, int64_t n_rows) {
    if (nnz <= 0) return 256;
    CsrWs w;
    if (carve_csr_ws(nnz, n_rows, nullptr, &w) != cudaSuccess) return -1;
    return (int64_t)w.total;
}

extern "C" int mmssl_csr_from_coo(const int64_t* rows, const int64_t* cols, const float* vals, int64_t nnz,
                                  int64_t n_rows, int64_t n_cols, int transpose, int32_t* rowptr, int32_t* colidx,
                                  float* out_vals, void* workspace, int64_t workspace_bytes, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    MMSSL_REQUIRE(n_rows >= 0 && n_cols >= 0 && nnz >= 0, "negative size");
    MMSSL_REQUIRE(n_rows < (1ll << 31) - 1 && n_cols < (1ll << 31) - 1 && nnz < (1ll << 31) - 1,
                  "sizes must fit int32 (shard the graph across ranks first)");
    const int T = 256;
    if (nnz == 0) {
        fill_i32_kernel<<<(unsigned)((n_rows + 1 + T - 1) / T), T, 0, stream>>>(rowptr, n_rows + 1, 0);
        MMSSL_LAUNCH_OK();
        return 0;
    }
    CsrWs w;
    MMSSL_CUDA(carve_csr_ws(nnz, n_rows, workspace, &w));
    MMSSL_REQUIRE((int64_t)w.total <= workspace_bytes, "workspace too small (see mmssl_csr_workspace_bytes)");
    const unsigned gb = (unsigned)((nnz + T - 1) / T);
    make_keys_kernel<<<gb, T, 0, stream>>>(rows, cols, nnz, transpose, w.keys_in, w.idx_in);
    MMSSL_LAUNCH_OK();
    const int end_bit = 32 + ceil_log2((uint64_t)(n_rows > 1 ? n_rows : 2));
    size_t cub_bytes = w.cub_bytes;
    MMSSL_CUDA(cub::DeviceRadixSort::SortPairs(w.cub_tmp, cub_bytes, (const uint64_t*)w.keys_in, w.keys_out,
                                               (const uint32_t*)w.idx_in, w.idx_out, (int)nnz, 0, end_bit, stream));
    scatter_sorted_kernel<<<gb, T, 0, stream>>>(w.keys_out, w.idx_out, vals, nnz, colidx, out_vals);
    MMSSL_LAUNCH_OK();
    rowptr_kernel<<<(unsigned)((n_rows + 1 + T - 1) / T), T, 0, stream>>>(w.keys_out, nnz, n_rows, rowptr);
    MMSSL_LAUNCH_OK();
    return 0;
}

extern "C" int mmssl_spmm_plan_set_cuts(int split_threshold, int seg_len, int heavy_threshold, int heavy_seg_len) {
    MMSSL_REQUIRE(split_threshold >= 1 && seg_len >= 1 && heavy_seg_len >= 1 && heavy_threshold >= split_threshold, "bad cuts");
    g_cuts = {split_threshold, seg_len, heavy_threshold, heavy_seg_len};
    return 0;
}
static int64_t min_seg() { return g_cuts.seg_len < g_cuts.heavy_seg_len ? g_cuts.seg_len : g_cuts.heavy_seg_len; }
// a split row of len non-zeros has <= len / seg + 1 segments and there are <= nnz / (threshold + 1) split rows
extern "C" int64_t mmssl_spmm_plan_segs_cap(int64_t nnz) { return nnz / min_seg() + nnz / g_cuts.split_threshold + 2; }
extern "C" int64_t mmssl_spmm_plan_splits_cap(int64_t nnz) { return nnz / g_cuts.split_threshold + 2; }
extern "C" int64_t mmssl_spmm_plan_items_cap(int64_t n_rows, int64_t nnz) { return n_rows + mmssl_spmm_plan_segs_cap(nnz); }

extern "C" int64_t mmssl_spmm_plan_workspace_bytes(int64_t n_rows) {
    size_t cub_bytes = 0;
    if (n_rows <= 0) return 256;
    if (cub::DeviceScan::ExclusiveSum(nullptr, cub_bytes, (const int32_t*)nullptr, (int32_t*)nullptr, (int)n_rows) != cudaSuccess)
        return -1;
    return (int64_t)(6 * ((sizeof(int32_t) * n_rows + 255) & ~(size_t)255) + cub_bytes + 512);
}

extern "C" int mmssl_spmm_plan(const int32_t* rowptr, int64_t n_rows, int64_t nnz, int32_t* items4,
                               int64_t items_cap, int32_t* split_table4, int32_t* counters, int64_t splits_cap,
                               int32_t* totals3, void* workspace, int64_t workspace_bytes, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    MMSSL_REQUIRE(items_cap >= mmssl_spmm_plan_items_cap(n_rows, nnz), "items_cap too small");
    MMSSL_REQUIRE(splits_cap >= mmssl_spmm_plan_splits_cap(nnz), "splits_cap too small");
    const int T = 256;
    // all items start as {-1,-1,-1,-1}: the SpMM kernel skips row < 0
    MMSSL_CUDA(cudaMemsetAsync(items4, 0xff, sizeof(int4) * items_cap, stream));
    MMSSL_CUDA(cudaMemsetAsync(counters, 0, sizeof(int32_t) * splits_cap, stream));
    MMSSL_CUDA(cudaMemsetAsync(totals3, 0, sizeof(int32_t) * 3, stream));
    if (n_rows == 0) return 0;
    size_t cub_bytes = 0;
    MMSSL_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, cub_bytes, (const int32_t*)nullptr, (int32_t*)nullptr, (int)n_rows));
    const size_t arr = (sizeof(int32_t) * n_rows + 255) & ~(size_t)255;
    MMSSL_REQUIRE((int64_t)(6 * arr + cub_bytes + 256) <= workspace_bytes, "workspace too small");
    char* b = (char*)workspace;
    int32_t* n_items = (int32_t*)(b);
    int32_t* is_split = (int32_t*)(b + arr);
    int32_t* n_segs = (int32_t*)(b + 2 * arr);
    int32_t* item_off = (int32_t*)(b + 3 * arr);
    int32_t* split_off = (int32_t*)(b + 4 * arr);
    int32_t* seg_off = (int32_t*)(b + 5 * arr);
    void* cub_tmp = (void*)(b + 6 * arr);
    plan_count_kernel<<<(unsigned)((n_rows + T - 1) / T), T, 0, stream>>>(rowptr, n_rows, n_items, is_split, n_segs, g_cuts);
    MMSSL_LAUNCH_OK();
    MMSSL_CUDA(cub::DeviceScan::ExclusiveSum(cub_tmp, cub_bytes, n_items, item_off, (int)n_rows, stream));
    MMSSL_CUDA(cub::DeviceScan::ExclusiveSum(cub_tmp, cub_bytes, is_split, split_off, (int)n_rows, stream));
    MMSSL_CUDA(cub::DeviceScan::ExclusiveSum(cub_tmp, cub_bytes, n_segs, seg_off, (int)n_rows, stream));
    const int64_t threads = n_rows * 32;
    plan_fill_kernel<<<(unsigned)((threads + T - 1) / T), T, 0, stream>>>(rowptr, n_rows, item_off, split_off, seg_off,
                                                                         is_split, (int4*)items4, (int4*)split_table4,
                                                                         totals3, g_cuts);
    MMSSL_LAUNCH_OK();
    return 0;
}


extern "C" int64_t mmssl_spmm_bulk_plan_splits_cap(int64_t nnz) { return nnz / (kBulkBucket + 1) + 2; }
extern "C" int64_t mmssl_spmm_bulk_plan_segs_cap(int64_t nnz) { return nnz / kBulkBucket + mmssl_spmm_bulk_plan_splits_cap(nnz) + 2; }
extern "C" int64_t mmssl_spmm_bulk_plan_buckets_cap(int64_t n_rows, int64_t nnz) { return n_rows / kBulkRows + nnz / 8 + 16; }
extern "C" int64_t mmssl_spmm_bulk_plan_workspace_bytes(int64_t n_rows) {
    size_t cub_bytes = 0;
    if (n_rows <= 0) return 256;
    if (cub::DeviceScan::ExclusiveSum(nullptr, cub_bytes, (const int32_t*)nullptr, (int32_t*)nullptr, (int)n_rows) != cudaSuccess)
        return -1;
    return (int64_t)(9 * ((sizeof(int32_t) * n_rows + 255) & ~(size_t)255) + cub_bytes + 512);
}

extern "C" int mmssl_spmm_bulk_plan(const int32_t* rowptr, int64_t n_rows, int64_t nnz, int32_t* split_table4, int32_t* counters,
                                    int64_t splits_cap, int32_t* buckets8, int64_t buckets_cap, int32_t* totals3, void* workspace,
                                    int64_t workspace_bytes, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    MMSSL_REQUIRE(splits_cap >= mmssl_spmm_bulk_plan_splits_cap(nnz), "splits_cap too small");
    MMSSL_REQUIRE(buckets_cap >= mmssl_spmm_bulk_plan_buckets_cap(n_rows, nnz), "buckets_cap too small");
    const int T = 256;
    MMSSL_CUDA(cudaMemsetAsync(counters, 0, sizeof(int32_t) * splits_cap, stream));
    MMSSL_CUDA(cudaMemsetAsync(totals3, 0, sizeof(int32_t) * 3, stream));
    MMSSL_CUDA(cudaMemsetAsync(buckets8, 0, sizeof(int4) * 2 * buckets_cap, stream));      // unused entries: 0 rows -> skipped
    if (n_rows == 0) return 0;
    size_t cub_bytes = 0;
    MMSSL_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, cub_bytes, (const int32_t*)nullptr, (int32_t*)nullptr, (int)n_rows));
    const size_t arr = (sizeof(int32_t) * n_rows + 255) & ~(size_t)255;
    MMSSL_REQUIRE((int64_t)(9 * arr + cub_bytes + 256) <= workspace_bytes, "workspace too small (mmssl_spmm_bulk_plan_workspace_bytes)");
    char* b = (char*)workspace;
    int32_t* run_flag = (int32_t*)(b);
    int32_t* run_excl = (int32_t*)(b + arr);
    int32_t* run_first = (int32_t*)(b + 2 * arr);
    int32_t* n_bk = (int32_t*)(b + 3 * arr);
    int32_t* is_split = (int32_t*)(b + 4 * arr);
    int32_t* n_segs = (int32_t*)(b + 5 * arr);
    int32_t* bk_off = (int32_t*)(b + 6 * arr);
    int32_t* split_off = (int32_t*)(b + 7 * arr);
    int32_t* seg_off = (int32_t*)(b + 8 * arr);
    void* cub_tmp = (void*)(b + 9 * arr);
    const unsigned gr = (unsigned)((n_rows + T - 1) / T);
    bulk_runflag_kernel<<<gr, T, 0, stream>>>(rowptr, n_rows, run_flag);
    MMSSL_LAUNCH_OK();
    MMSSL_CUDA(cub::DeviceScan::ExclusiveSum(cub_tmp, cub_bytes, run_flag, run_excl, (int)n_rows, stream));
    bulk_runfirst_kernel<<<gr, T, 0, stream>>>(run_flag, run_excl, n_rows, run_first);
    MMSSL_LAUNCH_OK();
    bulk_count_kernel<<<gr, T, 0, stream>>>(rowptr, n_rows, run_flag, run_excl, run_first, n_bk, is_split, n_segs);
    MMSSL_LAUNCH_OK();
    MMSSL_CUDA(cub::DeviceScan::ExclusiveSum(cub_tmp, cub_bytes, n_bk, bk_off, (int)n_rows, stream));
    MMSSL_CUDA(cub::DeviceScan::ExclusiveSum(cub_tmp, cub_bytes, is_split, split_off, (int)n_rows, stream));
    MMSSL_CUDA(cub::DeviceScan::ExclusiveSum(cub_tmp, cub_bytes, n_segs, seg_off, (int)n_rows, stream));
    const int64_t threads = n_rows * 32;
    bulk_fill_kernel<<<(unsigned)((threads + T - 1) / T), T, 0, stream>>>(rowptr, n_rows, n_bk, bk_off, split_off, seg_off, is_split,
                                                                         (int4*)buckets8, (int4*)split_table4, totals3);
    MMSSL_LAUNCH_OK();
    bulk_extent_kernel<<<(unsigned)((buckets_cap + T - 1) / T), T, 0, stream>>>(rowptr, n_rows, totals3, buckets8);
    MMSSL_LAUNCH_OK();
    return 0;
}

extern "C" int mmssl_csr_row_normalize(const int32_t* rowptr, int64_t n_rows, float* vals, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (n_rows == 0) return 0;
    const int T = 256;
    const int64_t threads = n_rows * 32;
    row_normalize_kernel<<<(unsigned)((threads + T - 1) / T), T, 0, stream>>>(rowptr, n_rows, vals);
    MMSSL_LAUNCH_OK();
    return 0;
}
