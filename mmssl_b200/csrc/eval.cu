// Evaluation path -- SURVEY section 8f "next" row 3.  What the reference does per epoch in Trainer.test
// (main.py:301-306 -> utility/batch_test.py:112-169): dense scores of a user batch against all items, per
// user drop the training items, rank the rest, keep the max(Ks) best (heapq.nlargest: equal scores keep the
// LOWER item id first, batch_test.py:21-27), mark the held-out positives among them and compute
// precision / recall / ndcg / hit ratio at every K (batch_test.py:67-80, utility/metrics.py).
//
// One fused kernel, no [users x items] score matrix in HBM:
//   * CTA = 128 threads x 8 users.  The 8 user vectors sit in shared memory; every thread owns one item per
//     sweep, reads its row once (float4, coalesced across the row over the k loop, item table is L2 resident)
//     and scores it against the 8 users -> the item table is re-read users/8 times instead of users times.
//   * selection = "threshold + candidate buffer": a score enters the user's 512-slot shared buffer only if
//     its key beats the current max(Ks)-th best key; when a buffer may overflow on the next sweep, a warp
//     bitonic-sorts it, keeps the best max(Ks) and raises the threshold.  Expected appends per user are
//     ~K(1 + ln(I/K)), so a handful of sorts per user.  Keys are (orderable fp32 score, ~item id) packed in
//     64 bits and unique, so the result does not depend on append order: bit-deterministic.
//   * training-item masking and hit marking are binary searches in the (sorted) CSR rows, done only for
//     scores that already beat the threshold.
//   * metrics in fp64 like numpy; per-user rows are then averaged by a fixed-order reduction kernel.
//
// Full mode (--test_flag full, batch_test.py:38-68: roc_auc_score over every non-training item) is the kFull
// instantiation of the same kernel and the same sweep.  Before it, one warp per user scores the user's positives
// with the sweep's own dot product and sorts their keys (in shared memory, or in a workspace slot for long held-out
// rows).  Every sweep then builds 128-bit train / held-out masks from cursors in the sorted rows (O(deg + |held|) per
// user in total), classifies every item, and counts 2 #{s_p > s} + #{s_p == s} for each negative with two binary
// searches in the positives.  The counts are 64-bit integers, so the per-user AUC is exact and bit-deterministic.
#include "common.cuh"
#include "../../include/mmssl_b200.h"

#include <math_constants.h>

namespace mmssl {

constexpr int kEvalUsers = 8;      // users per CTA
constexpr int kEvalThreads = 128;  // items per sweep
constexpr int kEvalCap = 512;      // candidate keys per user
constexpr int kEvalMaxK = 64;      // max(Ks)
constexpr int kEvalMaxKs = 8;

struct EvalKs {
    int n;
    int kmax;
    int k[kEvalMaxKs];
};

// Larger key == better: higher score first, then lower item id.  fp32 -> order-preserving u32.
__device__ __forceinline__ uint64_t eval_key(float s, uint32_t item) {
    uint32_t b = __float_as_uint(s);
    b = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
    return ((uint64_t)b << 32) | (uint64_t)(0xFFFFFFFFu - item);
}
__device__ __forceinline__ float eval_key_score(uint64_t key) {
    uint32_t b = (uint32_t)(key >> 32);
    b = (b & 0x80000000u) ? (b & 0x7FFFFFFFu) : ~b;
    return __uint_as_float(b);
}

__device__ __forceinline__ bool row_contains(const int64_t* __restrict__ idx, int64_t lo, int64_t hi, int64_t x) {
    const int64_t end = hi;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg(idx + mid) < x) lo = mid + 1; else hi = mid;
    }
    return lo < end && __ldg(idx + lo) == x;
}

// Warp-cooperative bitonic sort (descending) of n (a power of two) keys in shared memory.
__device__ __forceinline__ void warp_sort_desc(uint64_t* a, int n, int lane) {
    for (int k = 2; k <= n; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = lane; i < n; i += 32) {
                const int p = i ^ j;
                if (p > i) {
                    const uint64_t x = a[i], y = a[p];
                    const bool desc = (i & k) == 0;
                    if (desc ? (x < y) : (x > y)) { a[i] = y; a[p] = x; }
                }
            }
            __syncwarp();
        }
    }
}

// Every warp sorts the buffers of its users, keeps the best kmax keys and raises the threshold.  Call at a
// block-uniform point, between two __syncthreads().
__device__ __forceinline__ void eval_compact(uint64_t (*keys)[kEvalCap], int* cnt, uint64_t* thr, int kmax, int warp, int lane) {
    for (int u = warp; u < kEvalUsers; u += kEvalThreads / 32) {
        const int n = cnt[u];
        int np2 = 64;
        while (np2 < n) np2 <<= 1;
        for (int i = n + lane; i < np2; i += 32) keys[u][i] = 0ull;      // 0 sorts below every real key
        __syncwarp();
        warp_sort_desc(keys[u], np2, lane);
        if (lane == 0 && n >= kmax) { thr[u] = keys[u][kmax - 1]; cnt[u] = kmax; }
        __syncwarp();
    }
}

// Scores of one item row against NU user vectors (stride d floats in shared memory).  The sweep and the full-mode
// positives both score through this function, so a positive's score is bitwise the score the sweep computes for it:
// same fmaf chain, same float4 grouping, same "+ 0.0f" (-0 -> +0: equal scores must tie).
template <int NU>
__device__ __forceinline__ void eval_dot(const float* __restrict__ row, const float* uvec, int d, float (&s)[NU]) {
#pragma unroll
    for (int u = 0; u < NU; ++u) s[u] = 0.f;
#pragma unroll 4
    for (int k4 = 0; k4 < (d >> 2); ++k4) {
        const float4 x = ldg4(row + 4 * k4);
#pragma unroll
        for (int u = 0; u < NU; ++u) {
            const float4 y = ld4(uvec + u * d + 4 * k4);
            s[u] = fmaf(x.x, y.x, s[u]);
            s[u] = fmaf(x.y, y.y, s[u]);
            s[u] = fmaf(x.z, y.z, s[u]);
            s[u] = fmaf(x.w, y.w, s[u]);
        }
    }
#pragma unroll
    for (int u = 0; u < NU; ++u) s[u] = s[u] + 0.0f;
}

// ---- full mode (test_flag == 'full', batch_test.py:38-68): per-user ROC-AUC over all non-training items.
constexpr int kEvalPosStage = 128;   // positives per user sorted in shared memory; longer held rows use the workspace

// fp32 -> u32 with the same order; equal floats (after "+ 0.0f") give equal keys.
__device__ __forceinline__ uint32_t eval_ord(float s) {
    const uint32_t b = __float_as_uint(s);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// Warp-cooperative bitonic sort (ascending) of n (a power of two) u32 keys in shared or global memory.
__device__ __forceinline__ void warp_sort_asc_u32(uint32_t* a, int n, int lane) {
    for (int k = 2; k <= n; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = lane; i < n; i += 32) {
                const int p = i ^ j;
                if (p > i) {
                    const uint32_t x = a[i], y = a[p];
                    const bool asc = (i & k) == 0;
                    if (asc ? (x > y) : (x < y)) { a[i] = y; a[p] = x; }
                }
            }
            __syncwarp();
        }
    }
}

// First index in the ascending a[0, n) whose key is > x (strict == false: >= x).
__device__ __forceinline__ int eval_bound(const uint32_t* a, int n, uint32_t x, bool strict) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (strict ? a[mid] <= x : a[mid] < x) lo = mid + 1; else hi = mid;
    }
    return lo;
}

template <bool kFull>
__global__ void __launch_bounds__(kEvalThreads, kFull ? 2 : 0) eval_rank_kernel(
    const float* __restrict__ user_emb, int64_t ldu, const float* __restrict__ item_emb, int64_t ldi, int64_t n_items, int d,
    const int64_t* __restrict__ users, int64_t n_eval, const int64_t* __restrict__ tr_ptr, const int64_t* __restrict__ tr_idx,
    const int64_t* __restrict__ he_ptr, const int64_t* __restrict__ he_idx, EvalKs ks, int32_t* __restrict__ ranked,
    float* __restrict__ ranked_scores, int32_t* __restrict__ hits_out, double* __restrict__ per_user, float* __restrict__ scores_out,
    double* __restrict__ auc_out, uint32_t* pos_ws, const int64_t* __restrict__ pos_ws_off) {
    extern __shared__ __align__(16) unsigned char eval_smem[];
    uint64_t (*keys)[kEvalCap] = reinterpret_cast<uint64_t (*)[kEvalCap]>(eval_smem);
    float* uvec = reinterpret_cast<float*>(eval_smem + sizeof(uint64_t) * kEvalUsers * kEvalCap);
    __shared__ int cnt[kEvalUsers];
    __shared__ uint64_t thr[kEvalUsers];
    __shared__ int64_t uid[kEvalUsers], tb[kEvalUsers], te[kEvalUsers];
    __shared__ double disc[kEvalMaxK];
    // full mode only: sorted positive keys (pkeys -> the stage or the user's workspace slot), their count, the
    // train / held-out membership masks of the current 128-item sweep, the row cursors behind them, distinct
    // training items seen, the non-finite-score flag and 2 x (pairs ordered right) + (tied pairs).
    __shared__ uint32_t pstage[kFull ? kEvalUsers : 1][kFull ? kEvalPosStage : 1];
    __shared__ uint32_t* pkeys[kEvalUsers];
    __shared__ int npos[kEvalUsers], ntrain[kEvalUsers], bad[kEvalUsers];
    __shared__ uint32_t trmask[kEvalUsers][kEvalThreads / 32], hemask[kEvalUsers][kEvalThreads / 32];
    __shared__ int64_t tcur[kEvalUsers], hcur[kEvalUsers];
    __shared__ unsigned long long num[kEvalUsers];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int64_t tile0 = (int64_t)blockIdx.x * kEvalUsers;
    if (tid < kEvalUsers) {
        const int64_t g = tile0 + tid;
        const int64_t u = g < n_eval ? users[g] : -1;
        uid[tid] = u;
        cnt[tid] = 0;
        thr[tid] = 0ull;
        tb[tid] = u >= 0 ? tr_ptr[u] : 0;
        te[tid] = u >= 0 ? tr_ptr[u + 1] : 0;
        if constexpr (kFull) {
            tcur[tid] = tb[tid];
            hcur[tid] = u >= 0 ? he_ptr[u] : 0;
            ntrain[tid] = 0;
            bad[tid] = 0;
            num[tid] = 0ull;
        }
    }
    if (tid < kEvalMaxK) disc[tid] = 1.0 / log2((double)(tid + 2));      // metrics.py:54
    __syncthreads();
    for (int i = tid; i < kEvalUsers * d; i += kEvalThreads) {
        const int uu = i / d, c = i - uu * d;
        uvec[i] = uid[uu] >= 0 ? user_emb[uid[uu] * ldu + c] : 0.f;
    }
    __syncthreads();

    if constexpr (kFull) {
        // Positives = distinct held-out ids in [0, n_items) that are not training items.  One warp per user scores
        // them, packs their keys in id order, pads to a power of two with the largest key and sorts ascending.
        for (int u = warp; u < kEvalUsers; u += kEvalThreads / 32) {
            if (uid[u] < 0) continue;                                    // warp-uniform
            const int64_t hb = he_ptr[uid[u]], he = he_ptr[uid[u] + 1];
            uint32_t* buf = he - hb <= kEvalPosStage ? pstage[u] : pos_ws + pos_ws_off[tile0 + u];
            int n = 0;
            for (int64_t b = hb; b < he; b += 32) {
                const int64_t i = b + lane;
                bool ok = false;
                uint32_t key = 0u;
                if (i < he) {
                    const int64_t x = he_idx[i];
                    ok = x >= 0 && x < n_items && (i == hb || he_idx[i - 1] != x) && !row_contains(tr_idx, tb[u], te[u], x);
                    if (ok) {
                        float s[1];
                        eval_dot<1>(item_emb + x * ldi, uvec + u * d, d, s);
                        key = eval_ord(s[0]);
                    }
                }
                const unsigned m = __ballot_sync(0xffffffffu, ok);
                if (ok) buf[n + __popc(m & ((1u << lane) - 1u))] = key;
                n += __popc(m);
            }
            int np2 = 1;
            while (np2 < n) np2 <<= 1;
            for (int i = n + lane; i < np2; i += 32) buf[i] = 0xFFFFFFFFu;
            __syncwarp();
            warp_sort_asc_u32(buf, np2, lane);
            if (lane == 0) { pkeys[u] = buf; npos[u] = n; }
        }
    }

    unsigned long long pairs[kFull ? kEvalUsers : 1];                   // this thread's share of num[]
#pragma unroll
    for (int u = 0; u < (kFull ? kEvalUsers : 1); ++u) pairs[u] = 0ull;
    for (int64_t base = 0; base < n_items; base += kEvalThreads) {
        if constexpr (kFull) {
            // membership masks of items [base, base + 128): thread u walks user u's training row, thread 8 + u its
            // held-out row (both sorted), so every id is visited once over the whole sweep
            if (tid < 2 * kEvalUsers) {
                const int u = tid % kEvalUsers;
                const bool is_tr = tid < kEvalUsers;
                uint32_t* mk = is_tr ? trmask[u] : hemask[u];
#pragma unroll
                for (int w = 0; w < kEvalThreads / 32; ++w) mk[w] = 0u;
                if (uid[u] >= 0) {
                    const int64_t* idx = is_tr ? tr_idx : he_idx;
                    const int64_t end = is_tr ? te[u] : he_ptr[uid[u] + 1];
                    int64_t c = is_tr ? tcur[u] : hcur[u];
                    for (; c < end; ++c) {
                        const int64_t x = idx[c];
                        if (x >= base + kEvalThreads) break;
                        if (x >= base && x < n_items) mk[(x - base) >> 5] |= 1u << ((x - base) & 31);
                    }
                    if (is_tr) {
                        tcur[u] = c;
#pragma unroll
                        for (int w = 0; w < kEvalThreads / 32; ++w) ntrain[u] += __popc(mk[w]);
                    } else {
                        hcur[u] = c;
                    }
                }
            }
            __syncthreads();
        }
        const int64_t j = base + tid;
        if (j < n_items) {
            float acc[kEvalUsers];
            eval_dot<kEvalUsers>(item_emb + j * ldi, uvec, d, acc);
#pragma unroll
            for (int u = 0; u < kEvalUsers; ++u) {
                if (uid[u] < 0) continue;
                const float s = acc[u];
                if (scores_out) scores_out[(tile0 + u) * n_items + j] = s;
                const uint64_t key = eval_key(s, (uint32_t)j);
                bool keep = key > thr[u];
                if constexpr (kFull) {
                    const bool train = (trmask[u][warp] >> lane) & 1u;
                    keep = keep && !train;
                    if (!train) {
                        if ((__float_as_uint(s) & 0x7F800000u) == 0x7F800000u) bad[u] = 1;       // NaN / inf: sklearn raises
                        if (!((hemask[u][warp] >> lane) & 1u)) {         // a negative: 2 #{s_p > s} + #{s_p == s}
                            const uint32_t o = eval_ord(s);
                            const int n = npos[u];
                            const int lt = eval_bound(pkeys[u], n, o, false);
                            const int le = lt < n && pkeys[u][lt] == o ? eval_bound(pkeys[u], n, o, true) : lt;
                            pairs[u] += 2ull * (unsigned long long)(n - le) + (unsigned long long)(le - lt);
                        }
                    }
                } else {
                    keep = keep && !row_contains(tr_idx, tb[u], te[u], j);
                }
                if (keep) {
                    const int pos = atomicAdd(&cnt[u], 1);               // < kEvalCap: cnt <= Cap-128 at sweep start
                    keys[u][pos] = key;
                }
            }
        }
        __syncthreads();
        const int need = __syncthreads_or(tid < kEvalUsers && cnt[tid] > kEvalCap - kEvalThreads);
        if (need) {
            eval_compact(keys, cnt, thr, ks.kmax, warp, lane);
            __syncthreads();
        }
    }
    eval_compact(keys, cnt, thr, ks.kmax, warp, lane);
    __syncthreads();

    if constexpr (kFull) {
#pragma unroll
        for (int u = 0; u < kEvalUsers; ++u) {
            unsigned long long v = pairs[u];
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if (lane == 0 && v) atomicAdd(&num[u], v);                   // integer sums: exact in any order
        }
        __syncthreads();
        if (tid < kEvalUsers && uid[tid] >= 0) {
            const int64_t n_cand = n_items - ntrain[tid], P = npos[tid], N = n_cand - P;
            double a;
            if (n_cand == 0 || bad[tid]) a = 0.0;                        // sklearn raises (no sample, NaN / inf), metrics.auc -> 0
            else if (P == 0 || N == 0) a = CUDART_NAN;                   // one class: sklearn warns and returns NaN
            else a = (double)num[tid] / (2.0 * (double)P * (double)N);
            auc_out[tile0 + tid] = a;
        }
    }

    for (int u = warp; u < kEvalUsers; u += kEvalThreads / 32) {
        if (uid[u] < 0) continue;                                        // warp-uniform
        const int64_t g = tile0 + u;
        const int m = min(cnt[u], ks.kmax);                              // length of the hit list (batch_test.py:29-34)
        const int64_t hb = he_ptr[uid[u]], he = he_ptr[uid[u] + 1];
        uint64_t H = 0ull;
        for (int half = 0; half < 2; ++half) {
            const int pos = lane + 32 * half;
            bool hit = false;
            int32_t item = -1;
            float sc = 0.f;
            if (pos < m) {
                const uint64_t key = keys[u][pos];
                item = (int32_t)(0xFFFFFFFFu - (uint32_t)key);
                sc = eval_key_score(key);
                hit = row_contains(he_idx, hb, he, (int64_t)item);
            }
            if (pos < ks.kmax) {
                ranked[g * ks.kmax + pos] = item;
                if (ranked_scores) ranked_scores[g * ks.kmax + pos] = sc;
                if (hits_out) hits_out[g * ks.kmax + pos] = pos < m ? (int32_t)hit : -1;
            }
            H |= (uint64_t)__ballot_sync(0xffffffffu, hit) << (32 * half);
        }
        if (lane == 0) {
            const int nh_all = __popcll(H);
            const double n_pos = (double)(he - hb);
            double* o = per_user + g * 4 * ks.n;
            for (int q = 0; q < ks.n; ++q) {
                const int kk = min(ks.k[q], m);
                const uint64_t Hk = kk >= 64 ? H : (H & ((1ull << kk) - 1ull));
                const int nh = __popcll(Hk);
                double dcg = 0.0, idcg = 0.0;
                for (int i = 0; i < kk; ++i) {
                    if ((Hk >> i) & 1ull) dcg += disc[i];
                    if (i < nh_all) idcg += disc[i];                     // ideal = the retrieved hits sorted first (metrics.py:70)
                }
                o[0 * ks.n + q] = kk > 0 ? (double)nh / (double)kk : CUDART_NAN;          // metrics.py:17-18
                o[1 * ks.n + q] = n_pos > 0.0 ? (double)nh / n_pos : 0.0;                 // metrics.py:78-83
                o[2 * ks.n + q] = idcg > 0.0 ? dcg / idcg : 0.0;                          // metrics.py:70-73
                o[3 * ks.n + q] = nh > 0 ? 1.0 : 0.0;                                     // metrics.py:85-90
            }
        }
    }
}

// result[m] = (sum over users of per_user[u][m]) / n, fixed order (batch_test.py:159-163).
__global__ void __launch_bounds__(256) eval_reduce_kernel(const double* __restrict__ per_user, int64_t n, int n_metrics,
                                                          double* __restrict__ result) {
    __shared__ double sh[256];
    const int m = blockIdx.x, tid = threadIdx.x;
    double s = 0.0;
    for (int64_t i = tid; i < n; i += 256) s += per_user[i * n_metrics + m];
    sh[tid] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (tid < o) sh[tid] += sh[tid + o];
        __syncthreads();
    }
    if (tid == 0) result[m] = n > 0 ? sh[0] / (double)n : 0.0;
}

}  // namespace mmssl

using namespace mmssl;

template <bool kFull>
static int eval_rank_launch(const float* user_emb, int64_t ldu, const float* item_emb, int64_t ldi, int64_t n_items, int d,
                            const int64_t* users, int64_t n_eval, const int64_t* train_indptr, const int64_t* train_indices,
                            const int64_t* held_indptr, const int64_t* held_indices, const int32_t* ks_host, int n_ks,
                            int32_t* ranked, float* ranked_scores, int32_t* hits, double* per_user, float* scores_out,
                            double* auc_per_user, uint32_t* pos_ws, const int64_t* pos_ws_off, void* stream_) {
    MMSSL_REQUIRE(d >= 4 && d <= 256 && (d & 3) == 0, "embedding width must be a multiple of 4, at most 256");
    MMSSL_REQUIRE((ldi & 3) == 0 && aligned16(item_emb), "item table rows must be 16-byte aligned");
    MMSSL_REQUIRE(n_items >= 0 && n_items < (1ll << 31), "bad item count");
    MMSSL_REQUIRE(n_ks >= 1 && n_ks <= kEvalMaxKs && ks_host != nullptr, "1..8 cut-offs");
    MMSSL_REQUIRE(ranked != nullptr && per_user != nullptr, "ranked / per_user outputs are required");
    MMSSL_REQUIRE(!kFull || (auc_per_user != nullptr && pos_ws_off != nullptr), "auc_per_user / pos_ws_off are required");
    EvalKs ks;
    ks.n = n_ks;
    ks.kmax = 0;
    for (int q = 0; q < kEvalMaxKs; ++q) ks.k[q] = 0;
    for (int q = 0; q < n_ks; ++q) {
        MMSSL_REQUIRE(ks_host[q] >= 1 && ks_host[q] <= kEvalMaxK, "every K must be in 1..64");
        ks.k[q] = ks_host[q];
        ks.kmax = ks_host[q] > ks.kmax ? ks_host[q] : ks.kmax;
    }
    if (n_eval == 0) return 0;
    const size_t smem = sizeof(uint64_t) * kEvalUsers * kEvalCap + sizeof(float) * kEvalUsers * (size_t)d;
    const unsigned grid = (unsigned)((n_eval + kEvalUsers - 1) / kEvalUsers);
    eval_rank_kernel<kFull><<<grid, kEvalThreads, smem, (cudaStream_t)stream_>>>(
        user_emb, ldu, item_emb, ldi, n_items, d, users, n_eval, train_indptr, train_indices, held_indptr, held_indices, ks,
        ranked, ranked_scores, hits, per_user, scores_out, auc_per_user, pos_ws, pos_ws_off);
    MMSSL_LAUNCH_OK();
    return 0;
}

extern "C" int mmssl_eval_rank(const float* user_emb, int64_t ldu, const float* item_emb, int64_t ldi, int64_t n_items, int d,
                               const int64_t* users, int64_t n_eval, const int64_t* train_indptr, const int64_t* train_indices,
                               const int64_t* held_indptr, const int64_t* held_indices, const int32_t* ks_host, int n_ks,
                               int32_t* ranked, float* ranked_scores, int32_t* hits, double* per_user, float* scores_out,
                               void* stream_) {
    return eval_rank_launch<false>(user_emb, ldu, item_emb, ldi, n_items, d, users, n_eval, train_indptr, train_indices,
                                   held_indptr, held_indices, ks_host, n_ks, ranked, ranked_scores, hits, per_user, scores_out,
                                   nullptr, nullptr, nullptr, stream_);
}

extern "C" int mmssl_eval_full_stage(void) { return kEvalPosStage; }

extern "C" int mmssl_eval_rank_full(const float* user_emb, int64_t ldu, const float* item_emb, int64_t ldi, int64_t n_items, int d,
                                    const int64_t* users, int64_t n_eval, const int64_t* train_indptr, const int64_t* train_indices,
                                    const int64_t* held_indptr, const int64_t* held_indices, const int32_t* ks_host, int n_ks,
                                    int32_t* ranked, float* ranked_scores, int32_t* hits, double* per_user, float* scores_out,
                                    double* auc_per_user, uint32_t* pos_ws, const int64_t* pos_ws_off, void* stream_) {
    return eval_rank_launch<true>(user_emb, ldu, item_emb, ldi, n_items, d, users, n_eval, train_indptr, train_indices,
                                  held_indptr, held_indices, ks_host, n_ks, ranked, ranked_scores, hits, per_user, scores_out,
                                  auc_per_user, pos_ws, pos_ws_off, stream_);
}

extern "C" int mmssl_eval_reduce(const double* per_user, int64_t n_eval, int n_metrics, double* result, void* stream_) {
    MMSSL_REQUIRE(n_metrics >= 1 && n_metrics <= 4 * kEvalMaxKs, "bad metric count");
    eval_reduce_kernel<<<n_metrics, 256, 0, (cudaStream_t)stream_>>>(per_user, n_eval, n_metrics, result);
    MMSSL_LAUNCH_OK();
    return 0;
}
