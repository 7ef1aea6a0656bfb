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
//
// Up to 8 cut-offs of at most 64 run on eval_rank_kernel (512-key buffers, 64-bit hit mask).  Any other Ks (the reference
// takes any list) runs on eval_wide_kernel: the same tile, sweep and AUC code (eval_sweep, eval_positives, eval_auc_finish),
// buffers sized from max(Ks) in shared memory or a per-CTA workspace slot, an exact radix select as compaction, one radix
// sort at the end and the metrics of any number of cut-offs in one walk over the ranked list.
#include "common.cuh"
#include "../../include/mmssl_b200.h"

#include <math_constants.h>

namespace mmssl {

constexpr int kEvalUsers = 8;      // users per CTA
constexpr int kEvalThreads = 128;  // items per sweep
constexpr int kEvalCap = 512;      // candidate keys per user
constexpr int kEvalMaxK = 64;      // max(Ks)
constexpr int kEvalMaxKs = 8;
constexpr int kEvalWideMaxK = 1 << 26;  // wide path: any K up to this (buffer offsets stay int)

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

// Shared state of the 8 users of one tile.  Both selection stages (eval_rank_kernel, eval_wide_kernel) sweep through it.
struct EvalTile {
    int64_t uid[kEvalUsers], tb[kEvalUsers], te[kEvalUsers];
    int cnt[kEvalUsers];
    uint64_t thr[kEvalUsers];
    // full mode only: sorted positive keys (pkeys -> the stage or the user's workspace slot), their count, the train /
    // held-out membership masks of the current 128-item sweep, the row cursors behind them, distinct training items seen,
    // the non-finite-score flag and 2 x (pairs ordered right) + (tied pairs).
    uint32_t* pkeys[kEvalUsers];
    int npos[kEvalUsers], ntrain[kEvalUsers], bad[kEvalUsers];
    uint32_t trmask[kEvalUsers][kEvalThreads / 32], hemask[kEvalUsers][kEvalThreads / 32];
    int64_t tcur[kEvalUsers], hcur[kEvalUsers];
    unsigned long long num[kEvalUsers];
};

// Reads the user ids, row bounds and user vectors of the tile starting at tile0.  Call between two __syncthreads().
template <bool kFull>
__device__ __forceinline__ void eval_tile_begin(EvalTile& t, float* uvec, int64_t tile0, const float* __restrict__ user_emb,
                                                int64_t ldu, int d, const int64_t* __restrict__ users, int64_t n_eval,
                                                const int64_t* __restrict__ tr_ptr, const int64_t* __restrict__ he_ptr, int tid) {
    if (tid < kEvalUsers) {
        const int64_t g = tile0 + tid;
        const int64_t u = g < n_eval ? users[g] : -1;
        t.uid[tid] = u;
        t.cnt[tid] = 0;
        t.thr[tid] = 0ull;
        t.tb[tid] = u >= 0 ? tr_ptr[u] : 0;
        t.te[tid] = u >= 0 ? tr_ptr[u + 1] : 0;
        if constexpr (kFull) {
            t.tcur[tid] = t.tb[tid];
            t.hcur[tid] = u >= 0 ? he_ptr[u] : 0;
            t.ntrain[tid] = 0;
            t.bad[tid] = 0;
            t.num[tid] = 0ull;
        }
    }
    __syncthreads();
    for (int i = tid; i < kEvalUsers * d; i += kEvalThreads) {
        const int uu = i / d, c = i - uu * d;
        uvec[i] = t.uid[uu] >= 0 ? user_emb[t.uid[uu] * ldu + c] : 0.f;
    }
    __syncthreads();
}

// Full mode, before the sweep.  Positives = distinct held-out ids in [0, n_items) that are not training items.  One warp
// per user scores them, packs their keys in id order, pads to a power of two with the largest key and sorts ascending.
__device__ __forceinline__ void eval_positives(EvalTile& t, uint32_t (*pstage)[kEvalPosStage], const float* uvec,
                                               const float* __restrict__ item_emb, int64_t ldi, int64_t n_items, int d,
                                               const int64_t* __restrict__ tr_idx, const int64_t* __restrict__ he_ptr,
                                               const int64_t* __restrict__ he_idx, uint32_t* pos_ws,
                                               const int64_t* __restrict__ pos_ws_off, int64_t tile0, int warp, int lane) {
    for (int u = warp; u < kEvalUsers; u += kEvalThreads / 32) {
        if (t.uid[u] < 0) continue;                                      // warp-uniform
        const int64_t hb = he_ptr[t.uid[u]], he = he_ptr[t.uid[u] + 1];
        uint32_t* buf = he - hb <= kEvalPosStage ? pstage[u] : pos_ws + pos_ws_off[tile0 + u];
        int n = 0;
        for (int64_t b = hb; b < he; b += 32) {
            const int64_t i = b + lane;
            bool ok = false;
            uint32_t key = 0u;
            if (i < he) {
                const int64_t x = he_idx[i];
                ok = x >= 0 && x < n_items && (i == hb || he_idx[i - 1] != x) && !row_contains(tr_idx, t.tb[u], t.te[u], x);
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
        if (lane == 0) { t.pkeys[u] = buf; t.npos[u] = n; }
    }
}

// One 128-item sweep from item `base`: in full mode the membership masks first (thread u walks user u's training row,
// thread 8 + u its held-out row, both sorted, so every id is visited once over the whole sweep), then every thread scores
// its item against the 8 users, skips training items, counts the AUC pairs of negatives into `pairs` (full mode) and appends
// every key that beats the user's threshold to the user's buffer keys[u * cap, ...).  Ends without a barrier.
template <bool kFull>
__device__ __forceinline__ void eval_sweep(EvalTile& t, int64_t base, const float* uvec, const float* __restrict__ item_emb,
                                           int64_t ldi, int64_t n_items, int d, const int64_t* __restrict__ tr_idx,
                                           const int64_t* __restrict__ he_ptr, const int64_t* __restrict__ he_idx,
                                           float* __restrict__ scores_out, int64_t tile0,
                                           unsigned long long (&pairs)[kFull ? kEvalUsers : 1], uint64_t* keys, int cap, int tid) {
    const int warp = tid >> 5, lane = tid & 31;
    if constexpr (kFull) {
        if (tid < 2 * kEvalUsers) {
            const int u = tid % kEvalUsers;
            const bool is_tr = tid < kEvalUsers;
            uint32_t* mk = is_tr ? t.trmask[u] : t.hemask[u];
#pragma unroll
            for (int w = 0; w < kEvalThreads / 32; ++w) mk[w] = 0u;
            if (t.uid[u] >= 0) {
                const int64_t* idx = is_tr ? tr_idx : he_idx;
                const int64_t end = is_tr ? t.te[u] : he_ptr[t.uid[u] + 1];
                int64_t c = is_tr ? t.tcur[u] : t.hcur[u];
                for (; c < end; ++c) {
                    const int64_t x = idx[c];
                    if (x >= base + kEvalThreads) break;
                    if (x >= base && x < n_items) mk[(x - base) >> 5] |= 1u << ((x - base) & 31);
                }
                if (is_tr) {
                    t.tcur[u] = c;
#pragma unroll
                    for (int w = 0; w < kEvalThreads / 32; ++w) t.ntrain[u] += __popc(mk[w]);
                } else {
                    t.hcur[u] = c;
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
            if (t.uid[u] < 0) continue;
            const float s = acc[u];
            if (scores_out) scores_out[(tile0 + u) * n_items + j] = s;
            const uint64_t key = eval_key(s, (uint32_t)j);
            bool keep = key > t.thr[u];
            if constexpr (kFull) {
                const bool train = (t.trmask[u][warp] >> lane) & 1u;
                keep = keep && !train;
                if (!train) {
                    if ((__float_as_uint(s) & 0x7F800000u) == 0x7F800000u) t.bad[u] = 1;     // NaN / inf: sklearn raises
                    if (!((t.hemask[u][warp] >> lane) & 1u)) {           // a negative: 2 #{s_p > s} + #{s_p == s}
                        const uint32_t o = eval_ord(s);
                        const int n = t.npos[u];
                        const int lt = eval_bound(t.pkeys[u], n, o, false);
                        const int le = lt < n && t.pkeys[u][lt] == o ? eval_bound(t.pkeys[u], n, o, true) : lt;
                        pairs[u] += 2ull * (unsigned long long)(n - le) + (unsigned long long)(le - lt);
                    }
                }
            } else {
                keep = keep && !row_contains(tr_idx, t.tb[u], t.te[u], j);
            }
            if (keep) {
                const int pos = atomicAdd(&t.cnt[u], 1);                 // < cap: cnt <= cap - 128 at sweep start
                keys[(size_t)u * cap + pos] = key;
            }
        }
    }
}

// Full mode, after the sweep: the per-user AUC from the integer pair counts.  Call at a block-uniform point.
__device__ __forceinline__ void eval_auc_finish(EvalTile& t, unsigned long long (&pairs)[kEvalUsers], int64_t tile0, int64_t n_items,
                                                double* __restrict__ auc_out, int tid) {
    const int lane = tid & 31;
#pragma unroll
    for (int u = 0; u < kEvalUsers; ++u) {
        unsigned long long v = pairs[u];
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0 && v) atomicAdd(&t.num[u], v);                     // integer sums: exact in any order
    }
    __syncthreads();
    if (tid < kEvalUsers && t.uid[tid] >= 0) {
        const int64_t n_cand = n_items - t.ntrain[tid], P = t.npos[tid], N = n_cand - P;
        double a;
        if (n_cand == 0 || t.bad[tid]) a = 0.0;                          // sklearn raises (no sample, NaN / inf), metrics.auc -> 0
        else if (P == 0 || N == 0) a = CUDART_NAN;                       // one class: sklearn warns and returns NaN
        else a = (double)t.num[tid] / (2.0 * (double)P * (double)N);
        auc_out[tile0 + tid] = a;
    }
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
    __shared__ EvalTile t;
    __shared__ double disc[kEvalMaxK];
    __shared__ uint32_t pstage[kFull ? kEvalUsers : 1][kFull ? kEvalPosStage : 1];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int64_t tile0 = (int64_t)blockIdx.x * kEvalUsers;
    if (tid < kEvalMaxK) disc[tid] = 1.0 / log2((double)(tid + 2));      // metrics.py:54
    eval_tile_begin<kFull>(t, uvec, tile0, user_emb, ldu, d, users, n_eval, tr_ptr, he_ptr, tid);
    if constexpr (kFull)
        eval_positives(t, pstage, uvec, item_emb, ldi, n_items, d, tr_idx, he_ptr, he_idx, pos_ws, pos_ws_off, tile0, warp, lane);

    unsigned long long pairs[kFull ? kEvalUsers : 1];                   // this thread's share of t.num[]
#pragma unroll
    for (int u = 0; u < (kFull ? kEvalUsers : 1); ++u) pairs[u] = 0ull;
    for (int64_t base = 0; base < n_items; base += kEvalThreads) {
        eval_sweep<kFull>(t, base, uvec, item_emb, ldi, n_items, d, tr_idx, he_ptr, he_idx, scores_out, tile0, pairs, keys[0],
                          kEvalCap, tid);
        __syncthreads();
        const int need = __syncthreads_or(tid < kEvalUsers && t.cnt[tid] > kEvalCap - kEvalThreads);
        if (need) {
            eval_compact(keys, t.cnt, t.thr, ks.kmax, warp, lane);
            __syncthreads();
        }
    }
    eval_compact(keys, t.cnt, t.thr, ks.kmax, warp, lane);
    __syncthreads();
    if constexpr (kFull) eval_auc_finish(t, pairs, tile0, n_items, auc_out, tid);

    for (int u = warp; u < kEvalUsers; u += kEvalThreads / 32) {
        if (t.uid[u] < 0) continue;                                      // warp-uniform
        const int64_t g = tile0 + u;
        const int m = min(t.cnt[u], ks.kmax);                            // length of the hit list (batch_test.py:29-34)
        const int64_t hb = he_ptr[t.uid[u]], he = he_ptr[t.uid[u] + 1];
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

// ---- wide path: max(Ks) > 64 or more than 8 cut-offs.  Same tile, same sweep; per-user candidate buffers of `cap` >=
// 2 ksel + 256 keys (ksel = min(max(Ks), n_items)) in shared memory or in the CTA's global workspace slot, compacted by
// an exact radix select and sorted once at the end by an LSD radix sort, both block-cooperative.
struct EvalRadix {
    int hist[256];                        // digit histogram of one pass
    int off[256];                         // scatter offsets per digit
    int wc[kEvalThreads / 32][256];       // keys per (warp, digit) in the current 128-key round; all zero between rounds
    int wsum[kEvalThreads / 32];
    uint64_t prefix;
    int want, last;
};

// The k-th largest of the n >= k unique keys in a[0, n): 8-bit MSD radix select over shared histograms, stopping early
// once the prefix names a single key.  Block-cooperative: call at a block-uniform point, after a __syncthreads().
__device__ __forceinline__ uint64_t eval_kth_key(const uint64_t* a, int n, int k, EvalRadix& r, int tid) {
    const int lane = tid & 31;
    if (tid == 0) { r.prefix = 0ull; r.want = k; }
    uint64_t mask = 0ull;
    for (int shift = 56;; shift -= 8) {
        for (int i = tid; i < 256; i += kEvalThreads) r.hist[i] = 0;
        __syncthreads();
        const uint64_t prefix = r.prefix;
        for (int i = tid; i < n; i += kEvalThreads) {
            const uint64_t x = a[i];
            if ((x & mask) == prefix) atomicAdd(&r.hist[(int)((x >> shift) & 255u)], 1);
        }
        __syncthreads();
        if (tid < 32) {                                                  // lane l owns digits 255 - 8l ... 248 - 8l
            const int want = r.want;                                     // read before the deciding lane writes it
            int h[8], s = 0;
#pragma unroll
            for (int q = 0; q < 8; ++q) { h[q] = r.hist[255 - 8 * lane - q]; s += h[q]; }
            int inc = s;
            for (int o = 1; o < 32; o <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += v;
            }
            int cum = inc - s;
            if (cum < want && want <= inc) {
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    if (cum < want && want <= cum + h[q]) {
                        r.prefix = prefix | ((uint64_t)(255 - 8 * lane - q) << shift);
                        r.want = want - cum;
                        r.last = h[q];
                    }
                    cum += h[q];
                }
            }
        }
        __syncthreads();
        mask |= 0xFFull << shift;
        if (shift == 0) break;                                           // the prefix is the whole key
        if (r.last == 1) {                                               // one key left with this prefix: fetch it
            const uint64_t p = r.prefix;
            __syncthreads();
            for (int i = tid; i < n; i += kEvalThreads)
                if ((a[i] & mask) == p) r.prefix = a[i];
            __syncthreads();
            break;
        }
    }
    return r.prefix;
}

// Keeps the keys >= T of a[0, n) at the front, in their order (each lands at or before its own index, and a round's
// reads finish before its writes).  Returns their count.
__device__ __forceinline__ int eval_keep_ge(uint64_t* a, int n, uint64_t T, EvalRadix& r, int tid) {
    const int warp = tid >> 5, lane = tid & 31;
    int base = 0;
    for (int r0 = 0; r0 < n; r0 += kEvalThreads) {
        const int i = r0 + tid;
        const uint64_t x = i < n ? a[i] : 0ull;
        const bool keep = i < n && x >= T;
        const unsigned b = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) r.wsum[warp] = __popc(b);
        __syncthreads();
        int off = base;
#pragma unroll
        for (int w = 0; w < kEvalThreads / 32; ++w) {
            const int c = r.wsum[w];
            if (w < warp) off += c;
            base += c;
        }
        if (keep) a[off + __popc(b & ((1u << lane) - 1u))] = x;
        __syncthreads();
    }
    return base;
}

// Sorts the m unique keys of a[0, m) best first: stable LSD radix sort on 8-bit digits between a and s[0, m); a pass
// whose digit is the same for every key is skipped.  Returns a or s, whichever holds the result.
__device__ __forceinline__ uint64_t* eval_sort_desc(uint64_t* a, uint64_t* s, int m, EvalRadix& r, int tid) {
    const int warp = tid >> 5, lane = tid & 31;
    for (int shift = 0; shift < 64; shift += 8) {
        for (int i = tid; i < 256; i += kEvalThreads) r.hist[i] = 0;
        __syncthreads();
        for (int i = tid; i < m; i += kEvalThreads) atomicAdd(&r.hist[255 - (int)((a[i] >> shift) & 255u)], 1);
        __syncthreads();
        const bool skip = m == 0 || r.hist[255 - (int)((a[0] >> shift) & 255u)] == m;
        if (tid < 32 && !skip) {                                         // exclusive scan; lane l owns digits 8l .. 8l + 7
            int h[8], sum = 0;
#pragma unroll
            for (int q = 0; q < 8; ++q) { h[q] = r.hist[8 * lane + q]; sum += h[q]; }
            int inc = sum;
            for (int o = 1; o < 32; o <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += v;
            }
            int e = inc - sum;
#pragma unroll
            for (int q = 0; q < 8; ++q) { r.off[8 * lane + q] = e; e += h[q]; }
        }
        __syncthreads();
        if (skip) continue;
        for (int r0 = 0; r0 < m; r0 += kEvalThreads) {
            const int i = r0 + tid;
            const bool ok = i < m;
            const uint64_t x = ok ? a[i] : 0ull;
            const int dg = 255 - (int)((x >> shift) & 255u);
            unsigned peers = __ballot_sync(0xffffffffu, ok);             // lanes holding a key with the same digit
#pragma unroll
            for (int bit = 0; bit < 8; ++bit) {
                const unsigned b = __ballot_sync(0xffffffffu, (dg >> bit) & 1);
                peers &= ((dg >> bit) & 1) ? b : ~b;
            }
            const int rank = __popc(peers & ((1u << lane) - 1u));
            const bool leader = ok && rank == 0;
            if (leader) r.wc[warp][dg] = __popc(peers);
            __syncthreads();
            if (ok) {
                int pos = r.off[dg] + rank;
                for (int w = 0; w < warp; ++w) pos += r.wc[w][dg];
                s[pos] = x;
            }
            __syncthreads();
            if (leader) { atomicAdd(&r.off[dg], __popc(peers)); r.wc[warp][dg] = 0; }
            __syncthreads();
        }
        uint64_t* tmp = a; a = s; s = tmp;
    }
    return a;
}

template <bool kFull>
__global__ void __launch_bounds__(kEvalThreads, 1) eval_wide_kernel(
    const float* __restrict__ user_emb, int64_t ldu, const float* __restrict__ item_emb, int64_t ldi, int64_t n_items, int d,
    const int64_t* __restrict__ users, int64_t n_eval, const int64_t* __restrict__ tr_ptr, const int64_t* __restrict__ tr_idx,
    const int64_t* __restrict__ he_ptr, const int64_t* __restrict__ he_idx, const int32_t* __restrict__ ks, int n_ks, int kmax,
    int ksel, int cap, uint64_t* key_ws, int32_t* __restrict__ ranked, float* __restrict__ ranked_scores,
    int32_t* __restrict__ hits_out, double* __restrict__ per_user, float* __restrict__ scores_out, double* __restrict__ auc_out,
    uint32_t* pos_ws, const int64_t* __restrict__ pos_ws_off) {
    extern __shared__ __align__(16) unsigned char eval_smem[];
    float* uvec = reinterpret_cast<float*>(eval_smem);
    // candidate buffers: after the user vectors (8 d floats, a multiple of 16 bytes), or the CTA's workspace slot
    uint64_t* const keys = key_ws ? key_ws + (size_t)blockIdx.x * kEvalUsers * cap
                                  : reinterpret_cast<uint64_t*>(eval_smem + sizeof(float) * kEvalUsers * (size_t)d);
    __shared__ EvalTile t;
    __shared__ EvalRadix r;
    __shared__ uint32_t pstage[kFull ? kEvalUsers : 1][kFull ? kEvalPosStage : 1];
    __shared__ uint64_t* sorted[kEvalUsers];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    for (int i = tid; i < (kEvalThreads / 32) * 256; i += kEvalThreads) (&r.wc[0][0])[i] = 0;
    const int64_t n_tiles = (n_eval + kEvalUsers - 1) / kEvalUsers;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {  // a workspace slot serves one tile at a time
        const int64_t tile0 = tile * kEvalUsers;
        __syncthreads();
        eval_tile_begin<kFull>(t, uvec, tile0, user_emb, ldu, d, users, n_eval, tr_ptr, he_ptr, tid);
        if constexpr (kFull)
            eval_positives(t, pstage, uvec, item_emb, ldi, n_items, d, tr_idx, he_ptr, he_idx, pos_ws, pos_ws_off, tile0, warp, lane);

        unsigned long long pairs[kFull ? kEvalUsers : 1];
#pragma unroll
        for (int u = 0; u < (kFull ? kEvalUsers : 1); ++u) pairs[u] = 0ull;
        for (int64_t base = 0; base < n_items; base += kEvalThreads) {
            eval_sweep<kFull>(t, base, uvec, item_emb, ldi, n_items, d, tr_idx, he_ptr, he_idx, scores_out, tile0, pairs, keys, cap,
                              tid);
            __syncthreads();
            if (__syncthreads_or(tid < kEvalUsers && t.cnt[tid] > cap - kEvalThreads)) {
                for (int u = 0; u < kEvalUsers; ++u) {
                    const int n = t.cnt[u];                              // block-uniform
                    if (n <= ksel) continue;
                    const uint64_t T = eval_kth_key(keys + (size_t)u * cap, n, ksel, r, tid);
                    eval_keep_ge(keys + (size_t)u * cap, n, T, r, tid);
                    if (tid == 0) { t.thr[u] = T; t.cnt[u] = ksel; }
                    __syncthreads();
                }
            }
        }
        for (int u = 0; u < kEvalUsers; ++u) {                           // the ksel best, sorted once
            uint64_t* a = keys + (size_t)u * cap;
            int n = t.cnt[u];
            if (n > ksel) {
                eval_keep_ge(a, n, eval_kth_key(a, n, ksel, r, tid), r, tid);
                n = ksel;
            }
            uint64_t* res = eval_sort_desc(a, a + ksel, n, r, tid);
            if (tid == 0) { sorted[u] = res; t.cnt[u] = n; }
            __syncthreads();
        }
        if constexpr (kFull) eval_auc_finish(t, pairs, tile0, n_items, auc_out, tid);

        // One warp per user: mark the hits (their flags go to the other half of the buffer), then one walk over the
        // ranked list with a running hit count, fp64 DCG and ideal DCG (warp scans, carried from chunk to chunk); the lane
        // holding rank K - 1 writes the metrics at K.
        for (int u = warp; u < kEvalUsers; u += kEvalThreads / 32) {
            if (t.uid[u] < 0) continue;                                  // warp-uniform
            const int64_t g = tile0 + u;
            const int m = t.cnt[u];                                      // length of the hit list (batch_test.py:29-34)
            const uint64_t* sk = sorted[u];
            uint8_t* hitf = reinterpret_cast<uint8_t*>(sk == keys + (size_t)u * cap ? keys + (size_t)u * cap + ksel : keys + (size_t)u * cap);
            const int64_t hb = he_ptr[t.uid[u]], he = he_ptr[t.uid[u] + 1];
            int nh_all = 0;
            for (int pos = lane; pos < kmax; pos += 32) {
                bool hit = false;
                int32_t item = -1;
                float sc = 0.f;
                if (pos < m) {
                    const uint64_t key = sk[pos];
                    item = (int32_t)(0xFFFFFFFFu - (uint32_t)key);
                    sc = eval_key_score(key);
                    hit = row_contains(he_idx, hb, he, (int64_t)item);
                    hitf[pos] = (uint8_t)hit;
                    nh_all += hit;
                }
                ranked[g * kmax + pos] = item;
                if (ranked_scores) ranked_scores[g * kmax + pos] = sc;
                if (hits_out) hits_out[g * kmax + pos] = pos < m ? (int32_t)hit : -1;
            }
            for (int o = 16; o > 0; o >>= 1) nh_all += __shfl_xor_sync(0xffffffffu, nh_all, o);
            __syncwarp();
            const double n_pos = (double)(he - hb);
            double* o = per_user + g * 4 * n_ks;
            if (m == 0) {
                for (int q = lane; q < n_ks; q += 32) {
                    o[0 * n_ks + q] = CUDART_NAN;
                    o[1 * n_ks + q] = 0.0;
                    o[2 * n_ks + q] = 0.0;
                    o[3 * n_ks + q] = 0.0;
                }
            }
            int c_nh = 0;
            double c_dcg = 0.0, c_idcg = 0.0;
            for (int c = 0; c < m; c += 32) {
                const int pos = c + lane;
                const bool in = pos < m;
                const bool hit = in && hitf[pos];
                const double disc = in ? 1.0 / log2((double)(pos + 2)) : 0.0;      // metrics.py:54
                int nh = c_nh + __popc(__ballot_sync(0xffffffffu, hit) & (0xFFFFFFFFu >> (31 - lane)));
                double dcg = hit ? disc : 0.0, idcg = pos < nh_all ? disc : 0.0;     // ideal: retrieved hits first (metrics.py:70)
                for (int s = 1; s < 32; s <<= 1) {
                    const double x = __shfl_up_sync(0xffffffffu, dcg, s), y = __shfl_up_sync(0xffffffffu, idcg, s);
                    if (lane >= s) { dcg += x; idcg += y; }
                }
                dcg += c_dcg;
                idcg += c_idcg;
                if (in) {
                    for (int q = 0; q < n_ks; ++q) {
                        const int kk = min(__ldg(ks + q), m);
                        if (kk != pos + 1) continue;
                        o[0 * n_ks + q] = (double)nh / (double)kk;                         // metrics.py:17-18
                        o[1 * n_ks + q] = n_pos > 0.0 ? (double)nh / n_pos : 0.0;          // metrics.py:78-83
                        o[2 * n_ks + q] = idcg > 0.0 ? dcg / idcg : 0.0;                   // metrics.py:70-73
                        o[3 * n_ks + q] = nh > 0 ? 1.0 : 0.0;                              // metrics.py:85-90
                    }
                }
                c_nh = __shfl_sync(0xffffffffu, nh, 31);
                c_dcg = __shfl_sync(0xffffffffu, dcg, 31);
                c_idcg = __shfl_sync(0xffffffffu, idcg, 31);
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

// Wide path sizing.  ksel = min(kmax, n_items) keys survive per user; cap = 2 ksel + 256 rounded up to 128 leaves room
// for the sort's second buffer and for >= ksel + 128 appends between two compactions.  The buffers of a CTA's 8 users
// stay in shared memory while they fit in kEvalWideSmem bytes (two CTAs per SM), else each CTA owns one workspace slot
// of 8 cap keys and loops over tiles; the slot count is bounded by kEvalWideSlots and kEvalWideWsBytes.
constexpr size_t kEvalWideSmem = 112 * 1024;
constexpr int64_t kEvalWideSlots = 4 * 132;
constexpr int64_t kEvalWideWsBytes = 512ll << 20;

struct EvalWidePlan {
    int ksel, cap;
    size_t smem;
    int64_t grid, ws_keys;
};

static EvalWidePlan eval_wide_plan(int64_t n_eval, int kmax, int64_t n_items, int d) {
    EvalWidePlan p;
    p.ksel = (int)(kmax < n_items ? kmax : (n_items > 0 ? n_items : 1));
    p.cap = (2 * p.ksel + 256 + 127) / 128 * 128;
    const int64_t n_tiles = (n_eval + kEvalUsers - 1) / kEvalUsers;
    const size_t slot = sizeof(uint64_t) * kEvalUsers * (size_t)p.cap;
    const size_t uvec = sizeof(float) * kEvalUsers * (size_t)d;
    if (uvec + slot <= kEvalWideSmem) {
        p.smem = uvec + slot;
        p.grid = n_tiles;
        p.ws_keys = 0;
    } else {
        int64_t slots = kEvalWideWsBytes / (int64_t)slot;
        slots = slots < 1 ? 1 : (slots > kEvalWideSlots ? kEvalWideSlots : slots);
        p.smem = uvec;
        p.grid = n_tiles < slots ? n_tiles : slots;
        p.ws_keys = p.grid * kEvalUsers * (int64_t)p.cap;
    }
    return p;
}

extern "C" int64_t mmssl_eval_wide_workspace_bytes(int64_t n_eval, int kmax, int64_t n_items, int d) {
    if (n_eval <= 0 || kmax < 1 || kmax > kEvalWideMaxK || d < 4) return 0;
    return eval_wide_plan(n_eval, kmax, n_items, d).ws_keys * (int64_t)sizeof(uint64_t);
}

extern "C" int mmssl_eval_rank_wide(const float* user_emb, int64_t ldu, const float* item_emb, int64_t ldi, int64_t n_items, int d,
                                    const int64_t* users, int64_t n_eval, const int64_t* train_indptr, const int64_t* train_indices,
                                    const int64_t* held_indptr, const int64_t* held_indices, const int32_t* ks_host,
                                    const int32_t* ks_dev, int n_ks, int32_t* ranked, float* ranked_scores, int32_t* hits,
                                    double* per_user, float* scores_out, double* auc_per_user, uint32_t* pos_ws,
                                    const int64_t* pos_ws_off, uint64_t* key_ws, void* stream_) {
    MMSSL_REQUIRE(d >= 4 && d <= 256 && (d & 3) == 0, "embedding width must be a multiple of 4, at most 256");
    MMSSL_REQUIRE((ldi & 3) == 0 && aligned16(item_emb), "item table rows must be 16-byte aligned");
    MMSSL_REQUIRE(n_items >= 0 && n_items < (1ll << 31), "bad item count");
    MMSSL_REQUIRE(n_ks >= 1 && ks_host != nullptr && ks_dev != nullptr, "at least one cut-off, on the host and on the device");
    MMSSL_REQUIRE(ranked != nullptr && per_user != nullptr, "ranked / per_user outputs are required");
    MMSSL_REQUIRE(auc_per_user == nullptr || pos_ws_off != nullptr, "full mode needs pos_ws_off");
    int kmax = 0;
    for (int q = 0; q < n_ks; ++q) {
        MMSSL_REQUIRE(ks_host[q] >= 1 && ks_host[q] <= kEvalWideMaxK, "every K must be in 1..2^26");
        kmax = ks_host[q] > kmax ? ks_host[q] : kmax;
    }
    if (n_eval == 0) return 0;
    const EvalWidePlan p = eval_wide_plan(n_eval, kmax, n_items, d);
    MMSSL_REQUIRE(p.ws_keys == 0 || key_ws != nullptr, "key_ws (mmssl_eval_wide_workspace_bytes) is required");
    cudaStream_t st = (cudaStream_t)stream_;
    if (auc_per_user) {
        MMSSL_CUDA(cudaFuncSetAttribute(eval_wide_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem));
        eval_wide_kernel<true><<<(unsigned)p.grid, kEvalThreads, p.smem, st>>>(
            user_emb, ldu, item_emb, ldi, n_items, d, users, n_eval, train_indptr, train_indices, held_indptr, held_indices, ks_dev,
            n_ks, kmax, p.ksel, p.cap, p.ws_keys ? key_ws : nullptr, ranked, ranked_scores, hits, per_user, scores_out, auc_per_user,
            pos_ws, pos_ws_off);
    } else {
        MMSSL_CUDA(cudaFuncSetAttribute(eval_wide_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem));
        eval_wide_kernel<false><<<(unsigned)p.grid, kEvalThreads, p.smem, st>>>(
            user_emb, ldu, item_emb, ldi, n_items, d, users, n_eval, train_indptr, train_indices, held_indptr, held_indices, ks_dev,
            n_ks, kmax, p.ksel, p.cap, p.ws_keys ? key_ws : nullptr, ranked, ranked_scores, hits, per_user, scores_out, nullptr,
            nullptr, nullptr);
    }
    MMSSL_LAUNCH_OK();
    return 0;
}

extern "C" int mmssl_eval_reduce(const double* per_user, int64_t n_eval, int n_metrics, double* result, void* stream_) {
    MMSSL_REQUIRE(n_metrics >= 1, "bad metric count");
    eval_reduce_kernel<<<n_metrics, 256, 0, (cudaStream_t)stream_>>>(per_user, n_eval, n_metrics, result);
    MMSSL_LAUNCH_OK();
    return 0;
}
