// GPU triple sampler -- SURVEY section 8f "next" row 1.  Semantics of the reference's host sampler
// Data.sample (utility/load_data.py:153-191):
//   users : `batch` DISTINCT users drawn uniformly from the users that have >= 1 training item
//           (rd.sample without replacement, :154-155)
//   pos   : one uniform draw from the user's training items            (:160-171)
//   neg   : uniform item id, rejected while it is in the user's row    (:173-180)
// Batches of up to 1024 triples: one CTA (sample_triples_kernel).  Larger batches: a multi-CTA radix select over computed
// per-slot keys (select_pass_kernel and below), exact for any batch up to n_exist.
// One CTA (batch <= 1024).  Distinctness without atomics races: rounds of "draw, atomicMin-claim,
// check" -- the winner of a claim is the smallest thread id, so the result depends only on
// (seed, step), never on scheduling; the claim table cleans itself up.  Threads the 64 rounds leave unserved (batch close to
// n_exist) take the free slots of one sweep over the claim table (the claim finish), so the users are distinct at every
// batch <= n_exist.  Negatives: after 4096 rejected draws, a uniform draw from the row's complement.  Counter-based RNG
// (splitmix64 of (seed, step, thread, draw)), so the kernel is replayable inside a CUDA graph with
// the step number read from device memory.
// Row-sharded runs (ShardedTripleSampler): the same kernels with an owned slot range -- every rank selects the slots over the
// global n_exist, draws the triples of the slots whose users it holds and writes zeros elsewhere (draw_or_zero).
#include <cub/cub.cuh>

#include <algorithm>

#include "common.cuh"
#include "../../include/mmssl_b200.h"

namespace mmssl {

__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}
__device__ __forceinline__ uint32_t rnd32(uint64_t seed, uint32_t step, uint32_t tid, uint32_t draw) {
    return (uint32_t)(splitmix64(splitmix64(seed ^ ((uint64_t)step << 32 | tid)) + draw) >> 32);
}
// unbiased enough for sampling: 32-bit multiply-shift range reduction
__device__ __forceinline__ uint32_t below(uint32_t r, uint32_t n) { return (uint32_t)(((uint64_t)r * n) >> 32); }

constexpr int kClaimRounds = 64;                        // claim-by-minimum rounds before the claim finish
constexpr int kNegTries = 4096;                         // rejection draws of a negative before the complement draw
constexpr uint64_t kFinishStream = 0xBB67AE8584CAA73Bull;   // the claim finish's start slot, apart from the per-thread draws

// Triple t of the batch for the user of `slot`: one uniform positive from the user's row, one uniform negative rejected while it
// is in the row; `draw` is the next unused draw number of thread t.  Shared by both sampler paths.
// The rows are those of one block of users: the user of slot s is row0 + exist[s - slot_lo], whose row is indptr / indices of
// that local row (indices: GLOBAL item ids, int64 on one GPU, int32 in a row block).  The one-GPU sampler passes the whole
// matrix: slot_lo = row0 = 0.
template <typename IdxT>
__device__ __forceinline__ void draw_triple(const int64_t* __restrict__ indptr, const IdxT* __restrict__ indices,
                                            const int64_t* __restrict__ exist, int64_t slot, int64_t slot_lo, int64_t row0,
                                            int64_t n_items, uint64_t seed, uint32_t step, uint32_t t, uint32_t draw,
                                            int64_t* __restrict__ users, int64_t* __restrict__ pos, int64_t* __restrict__ neg) {
    const int64_t r = exist[slot - slot_lo];
    const int64_t b = indptr[r], e = indptr[r + 1];
    const uint32_t deg = (uint32_t)(e - b);
    const int64_t p = indices[b + below(rnd32(seed, step, t, draw++), deg)];
    int64_t ng = 0;
    bool in_row = true;
    for (int tries = 0; tries < kNegTries && in_row; ++tries) {
        ng = below(rnd32(seed, step, t, draw++), (uint32_t)n_items);
        int64_t lo = b, hi = e;             // binary search in the (sorted) row
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if ((int64_t)indices[mid] < ng) lo = mid + 1; else hi = mid;
        }
        in_row = lo < e && (int64_t)indices[lo] == ng;
    }
    if (in_row && (int64_t)deg < n_items) {
        // A dense row rejected every try: the j-th item missing from the row, uniform over the complement, so the mixture with
        // the rejection draws stays uniform.  Items below indices[b + m] missing from the row: indices[b + m] - m (sorted,
        // distinct), so the answer is j + (number of row items below it) = j + (first m with indices[b + m] - m > j).
        const int64_t j = below(rnd32(seed, step, t, draw++), (uint32_t)(n_items - deg));
        int64_t lo = 0, hi = deg;
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if ((int64_t)indices[b + mid] - mid <= j) lo = mid + 1; else hi = mid;
        }
        ng = j + lo;
    }
    users[t] = row0 + r; pos[t] = p; neg[t] = ng;
}

// Row-sharded form (kOwned): every rank runs the same slot selection over the GLOBAL n_exist, and thread t draws its triple only
// when its slot lies in the rank's range [slot_lo, slot_hi); every other entry is written as zero, so each entry of the batch has
// exactly one writer over the ranks and an integer sum over the ranks is the one-GPU batch.
template <typename IdxT, bool kOwned>
__device__ __forceinline__ void draw_or_zero(const int64_t* __restrict__ indptr, const IdxT* __restrict__ indices,
                                             const int64_t* __restrict__ exist, int64_t slot, int64_t slot_lo, int64_t slot_hi,
                                             int64_t row0, int64_t n_items, uint64_t seed, uint32_t step, uint32_t t, uint32_t draw,
                                             int64_t* __restrict__ users, int64_t* __restrict__ pos, int64_t* __restrict__ neg) {
    if (kOwned && (slot < slot_lo || slot >= slot_hi)) { users[t] = 0; pos[t] = 0; neg[t] = 0; return; }
    // the one-GPU instances see constant zeros: no new work in them
    draw_triple(indptr, indices, exist, slot, kOwned ? slot_lo : 0, kOwned ? row0 : 0, n_items, seed, step, t, draw, users, pos, neg);
}

// Threads of the block below this one whose `pred` holds (a block-wide exclusive count); `*total` (if given) = all of them.
// Every thread of the block calls it; warp_count is free again on return.
__device__ __forceinline__ int block_count_before(bool pred, int* warp_count, int* total) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, warps = (int)(blockDim.x >> 5);
    const unsigned m = __ballot_sync(0xffffffffu, pred);
    if (lane == 0) warp_count[w] = __popc(m);
    __syncthreads();
    int before = 0, all = 0;
    for (int k = 0; k < warps; ++k) {
        const int c = warp_count[k];
        before += k < w ? c : 0;
        all += c;
    }
    __syncthreads();
    if (total) *total = all;
    return before + __popc(m & ((1u << lane) - 1u));
}

template <typename IdxT, bool kOwned>
__global__ void __launch_bounds__(1024) sample_triples_kernel(const int64_t* __restrict__ indptr,
                                                              const IdxT* __restrict__ indices,
                                                              const int64_t* __restrict__ exist, int64_t slot_lo, int64_t slot_hi,
                                                              int64_t row0, int64_t n_exist, int64_t n_items, int batch, uint64_t seed,
                                                              const int32_t* __restrict__ step_dev, int32_t step_host,
                                                              int32_t* __restrict__ claim, int64_t* __restrict__ users,
                                                              int64_t* __restrict__ pos, int64_t* __restrict__ neg) {
    __shared__ int pending;
    __shared__ int warp_count[32];
    __shared__ int32_t given[1024];         // claim finish: the slot of the r-th thread still pending
    const int t = threadIdx.x;
    const uint32_t step = (uint32_t)(step_dev ? *step_dev : step_host);
    const bool with_replacement = batch > n_exist;
    uint32_t draw = 0;
    int64_t slot = -1;                      // index into `exist`
    bool done = t >= batch;
    if (with_replacement && !done) { slot = below(rnd32(seed, step, t, draw++), (uint32_t)n_exist); done = true; }
    // ---- distinct users: rounds of claim-by-minimum ----
    // claim[x]: INT_MAX = free, -1 = taken in an earlier round, otherwise the smallest contender id.
    int left = 0;
    for (int round = 0; round < kClaimRounds; ++round) {
        if (t == 0) pending = 0;
        __syncthreads();
        int64_t cand = -1;
        if (!done) {
            cand = below(rnd32(seed, step, t, draw++), (uint32_t)n_exist);
            atomicMin(&claim[cand], t);
        }
        __syncthreads();
        bool won = false;
        if (!done) {
            won = (claim[cand] == t);          // the smallest contender of a free slot wins it
            if (!won) atomicAdd(&pending, 1);
        }
        __syncthreads();
        left = pending;                        // read before thread 0 may reset it for the next round
        if (won) { slot = cand; done = true; claim[cand] = -1; }
        __syncthreads();
        if (left == 0) break;
    }
    // ---- claim finish (batch close to n_exist: the rounds are a coupon collector whose tail outlasts them) ----
    // One sweep over the claim table from a random start slot, cyclically: the free slots are handed out in that order to the
    // pending threads in thread order; it stops as soon as every pending thread has one, and at the latest after n_exist slots,
    // which hold at least `left` free ones (batch <= n_exist).  A uniform start keeps the batch invariant under a rotation of the
    // slots.  Runs only when the rounds did not finish (`left` is the same in every thread), so other batches keep their bits.
    if (left > 0) {
        const int64_t start = below(rnd32(seed ^ kFinishStream, step, 0, 0), (uint32_t)n_exist);
        int served = 0;
        for (int64_t c = 0; c < n_exist && served < left; c += blockDim.x) {
            int64_t x = c + t;
            bool free = false;
            if (x < n_exist) {
                x += start;
                if (x >= n_exist) x -= n_exist;
                free = claim[x] == 0x7fffffff;
            }
            int found;
            const int at = served + block_count_before(free, warp_count, &found);
            if (free && at < left) given[at] = (int32_t)x;
            served += found;
        }
        const int rank = block_count_before(!done, warp_count, nullptr);     // (its barriers also publish `given`)
        if (!done) { slot = given[rank]; done = true; }
    }
    if (t < batch && !with_replacement) claim[slot] = 0x7fffffff;   // leave the table clean
    if (t >= batch) return;
    draw_or_zero<IdxT, kOwned>(indptr, indices, exist, slot, slot_lo, slot_hi, row0, n_items, seed, step, t, draw, users, pos, neg);
}

__global__ void fill_claim_kernel(int32_t* claim, int64_t n) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) claim[i] = 0x7fffffff;
}

// ---- any batch size: exact selection of the `batch` smallest slot keys ----
// Slot s of `exist` gets the key (hash32(seed, step, s) << 32) | s: computed, never read, and unique.  The users of a batch are the
// slots of the `batch` smallest keys, in key order -- a uniformly random subset in a uniformly random order, like rd.sample.
// A radix select finds the batch-th smallest key one 8-bit digit at a time (at most 8 passes over the n_exist keys; a pass
// ends the select as soon as the threshold digit's bucket holds exactly the keys still needed, which at 1M users happens after
// two or three passes), the selected keys are compacted and sorted, and one thread per triple draws its positive and negative.
// Only integer counts are reduced, so the batch depends on (seed, step, batch) alone.
constexpr int kSelThreads = 256;               // = number of buckets of one 8-bit digit
constexpr int kSelMaxBlocks = 2 * kNumSMs;
constexpr uint64_t kKeyStream = 0x6A09E667F3BCC908ull;   // separates the key hashes from the per-thread draws

struct SelectState {
    uint64_t prefix;            // digits of the threshold key found so far
    int64_t need;               // selected keys still missing below the undecided digits
    int32_t shift;              // bit position of the last decided digit
    int32_t done;               // the keys with (key >> shift) <= (prefix >> shift) are exactly the batch
    uint32_t arrive;            // blocks finished with the current pass (zero between launches)
    uint32_t count;             // compaction cursor
    uint32_t hist[kSelThreads]; // bucket counts of the current pass (zero between launches)
};

__device__ __forceinline__ uint64_t slot_key(uint64_t seed, uint32_t step, uint32_t s) {
    const uint32_t h = (uint32_t)(splitmix64(splitmix64(seed ^ kKeyStream ^ ((uint64_t)step << 32 | s))) >> 32);
    return (uint64_t)h << 32 | s;
}

// One digit of the radix select.  Every block histograms the digit (bits [shift, shift + 8)) of the keys that agree with the
// threshold on the digits decided so far; the last block to finish picks the bucket that holds the batch-th smallest key and
// clears the histogram for the next pass.
__global__ void __launch_bounds__(kSelThreads) select_pass_kernel(uint64_t seed, const int32_t* __restrict__ step_dev, int32_t step_host,
                                                                  int64_t n_exist, int64_t batch, int pass, SelectState* st) {
    __shared__ uint32_t h[kSelThreads];
    __shared__ int last;
    const int t = threadIdx.x;
    if (pass > 0 && *(volatile int32_t*)&st->done) return;
    const uint32_t step = (uint32_t)(step_dev ? *step_dev : step_host);
    const int shift = 56 - 8 * pass;
    const uint64_t prefix = pass > 0 ? st->prefix : 0;
    h[t] = 0;
    __syncthreads();
    for (int64_t s = blockIdx.x * (int64_t)kSelThreads + t; s < n_exist; s += (int64_t)gridDim.x * kSelThreads) {
        const uint64_t key = slot_key(seed, step, (uint32_t)s);
        if (pass == 0 || (key >> (shift + 8)) == (prefix >> (shift + 8))) atomicAdd(&h[(key >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (h[t]) atomicAdd(&st->hist[t], h[t]);
    __threadfence();
    __syncthreads();
    if (t == 0) last = atomicAdd(&st->arrive, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!last) return;
    __threadfence();
    const int64_t need = pass > 0 ? st->need : batch;
    const uint32_t c = atomicExch(&st->hist[t], 0u);
    h[t] = c;
    __syncthreads();
    for (int o = 1; o < kSelThreads; o <<= 1) {           // inclusive scan of the bucket counts
        const uint32_t v = t >= o ? h[t - o] : 0u;
        __syncthreads();
        h[t] += v;
        __syncthreads();
    }
    const int64_t incl = h[t], excl = incl - c;
    if (excl < need && need <= incl) {                    // exactly one bucket
        st->prefix = prefix | ((uint64_t)t << shift);
        st->need = need - excl;
        st->shift = shift;
        st->done = (int64_t)c == need - excl;
    }
    if (t == 0) {
        st->arrive = 0;
        if (pass == 0) st->count = 0;
    }
}

// The selected keys, in any order (the sort that follows restores the key order).  They are written packed as
// hash << slot_bits | slot, slot_bits = bits of n_exist - 1: the same order as the 64-bit keys, so the sort can stop at
// bit 32 + slot_bits instead of 64 (six 8-bit passes instead of eight at Baby, seven at 1M users).
__host__ __device__ __forceinline__ int slot_bits(int64_t n_exist) {
    int b = 1;
    while ((1ll << b) < n_exist) ++b;
    return b;
}
__global__ void __launch_bounds__(kSelThreads) select_compact_kernel(uint64_t seed, const int32_t* __restrict__ step_dev, int32_t step_host,
                                                                     int64_t n_exist, int64_t batch, SelectState* st,
                                                                     uint64_t* __restrict__ keys, int32_t* __restrict__ slots) {
    const int sb = slot_bits(n_exist);
    const uint32_t step = (uint32_t)(step_dev ? *step_dev : step_host);
    const int shift = st->shift;
    const uint64_t lim = st->prefix >> shift;
    for (int64_t s = blockIdx.x * (int64_t)kSelThreads + threadIdx.x; s < n_exist; s += (int64_t)gridDim.x * kSelThreads) {
        const uint64_t key = slot_key(seed, step, (uint32_t)s);
        if ((key >> shift) <= lim) {
            const uint32_t p = atomicAdd(&st->count, 1u);
            if (p < batch) { keys[p] = (key >> 32) << sb | (uint64_t)s; slots[p] = (int32_t)s; }
        }
    }
}

// Triple t: the user of sorted slot t, or (batch > n_exist) a uniform slot with replacement, as in sample_triples_kernel
template <typename IdxT, bool kOwned>
__global__ void __launch_bounds__(256) sample_draw_kernel(const int64_t* __restrict__ indptr, const IdxT* __restrict__ indices,
                                                          const int64_t* __restrict__ exist, int64_t slot_lo, int64_t slot_hi,
                                                          int64_t row0, int64_t n_exist, int64_t n_items, int batch,
                                                          uint64_t seed, const int32_t* __restrict__ step_dev, int32_t step_host,
                                                          const int32_t* __restrict__ slots, int64_t* __restrict__ users,
                                                          int64_t* __restrict__ pos, int64_t* __restrict__ neg) {
    const int64_t t = blockIdx.x * 256ll + threadIdx.x;
    if (t >= batch) return;
    const uint32_t step = (uint32_t)(step_dev ? *step_dev : step_host);
    uint32_t draw = 0;
    const int64_t slot = slots ? (int64_t)slots[t] : (int64_t)below(rnd32(seed, step, (uint32_t)t, draw++), (uint32_t)n_exist);
    draw_or_zero<IdxT, kOwned>(indptr, indices, exist, slot, slot_lo, slot_hi, row0, n_items, seed, step, (uint32_t)t, draw, users, pos,
                               neg);
}

struct SelectWs {
    SelectState* st;
    uint64_t *keys_in, *keys_out;
    int32_t *slots_in, *slots_out;
    void* cub_tmp;
    size_t cub_bytes, total;
};

static cudaError_t select_carve(int64_t batch, int64_t n_exist, void* base, SelectWs* w) {
    size_t cub_bytes = 0;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                                                    (const int32_t*)nullptr, (int32_t*)nullptr, (int)batch, 0, 32 + slot_bits(n_exist));
    if (e != cudaSuccess) return e;
    auto up = [](size_t v) { return (v + 255) & ~(size_t)255; };
    size_t off = 0;
    char* b = (char*)base;
    w->st = (SelectState*)(b + off); off += up(sizeof(SelectState));
    w->keys_in = (uint64_t*)(b + off); off += up(sizeof(uint64_t) * batch);
    w->keys_out = (uint64_t*)(b + off); off += up(sizeof(uint64_t) * batch);
    w->slots_in = (int32_t*)(b + off); off += up(sizeof(int32_t) * batch);
    w->slots_out = (int32_t*)(b + off); off += up(sizeof(int32_t) * batch);
    w->cub_tmp = (void*)(b + off); off += up(cub_bytes);
    w->cub_bytes = cub_bytes;
    w->total = off;
    return cudaSuccess;
}

// The two sampler paths for one index type and ownership; the extern "C" entry points below only pick the instance.
template <typename IdxT, bool kOwned>
static int sample_one_cta(const int64_t* indptr, const IdxT* indices, const int64_t* exist, int64_t slot_lo, int64_t slot_hi, int64_t row0,
                          int64_t n_exist, int64_t n_items, int batch, uint64_t seed, const int32_t* step_dev, int32_t step_host,
                          int32_t* claim, int64_t* users, int64_t* pos, int64_t* neg, cudaStream_t st) {
    MMSSL_REQUIRE(batch >= 1 && batch <= 1024, "one sampler launch draws at most 1024 triples (larger batches: mmssl_sample_triples_multi)");
    MMSSL_REQUIRE(n_exist >= 1 && n_exist < (1ll << 31) && n_items >= 1 && n_items < (1ll << 31), "bad sizes");
    sample_triples_kernel<IdxT, kOwned><<<1, 1024, 0, st>>>(indptr, indices, exist, slot_lo, slot_hi, row0, n_exist, n_items, batch, seed,
                                                            step_dev, step_host, claim, users, pos, neg);
    MMSSL_LAUNCH_OK();
    return 0;
}

template <typename IdxT, bool kOwned>
static int sample_multi(const int64_t* indptr, const IdxT* indices, const int64_t* exist, int64_t slot_lo, int64_t slot_hi, int64_t row0,
                        int64_t n_exist, int64_t n_items, int batch, uint64_t seed, const int32_t* step_dev, int32_t step_host,
                        void* workspace, int64_t workspace_bytes, int64_t* users, int64_t* pos, int64_t* neg, cudaStream_t st) {
    MMSSL_REQUIRE(batch >= 1, "batch must be positive");
    MMSSL_REQUIRE(n_exist >= 1 && n_exist < (1ll << 31) && n_items >= 1 && n_items < (1ll << 31), "bad sizes");
    const int32_t* slots = nullptr;
    if (batch <= n_exist) {
        SelectWs w;
        MMSSL_CUDA(select_carve(batch, n_exist, workspace, &w));
        MMSSL_REQUIRE(workspace != nullptr && (int64_t)w.total <= workspace_bytes, "workspace too small (mmssl_sampler_workspace_bytes)");
        const unsigned blocks = (unsigned)std::min<int64_t>((n_exist + kSelThreads - 1) / kSelThreads, kSelMaxBlocks);
        for (int pass = 0; pass < 8; ++pass) {
            select_pass_kernel<<<blocks, kSelThreads, 0, st>>>(seed, step_dev, step_host, n_exist, batch, pass, w.st);
            MMSSL_LAUNCH_OK();
        }
        select_compact_kernel<<<blocks, kSelThreads, 0, st>>>(seed, step_dev, step_host, n_exist, batch, w.st, w.keys_in, w.slots_in);
        MMSSL_LAUNCH_OK();
        size_t cub_bytes = w.cub_bytes;
        MMSSL_CUDA(cub::DeviceRadixSort::SortPairs(w.cub_tmp, cub_bytes, w.keys_in, w.keys_out, w.slots_in, w.slots_out, batch, 0, 32 + slot_bits(n_exist), st));
        slots = w.slots_out;
    }
    sample_draw_kernel<IdxT, kOwned><<<(unsigned)((batch + 255) / 256), 256, 0, st>>>(indptr, indices, exist, slot_lo, slot_hi, row0, n_exist,
                                                                                      n_items, batch, seed, step_dev, step_host, slots, users,
                                                                                      pos, neg);
    MMSSL_LAUNCH_OK();
    return 0;
}

// The owned slot range of a rank: [slot_lo, slot_hi) inside [0, n_exist), exist[] holds slot_hi - slot_lo local rows.
static int check_owned(int64_t slot_lo, int64_t slot_hi, int64_t row0, int64_t n_exist) {
    MMSSL_REQUIRE(slot_lo >= 0 && slot_lo <= slot_hi && slot_hi <= n_exist && row0 >= 0, "owned slot range outside [0, n_exist)");
    return 0;
}

}  // namespace mmssl

using namespace mmssl;

extern "C" int mmssl_sampler_init(int32_t* claim, int64_t n_exist, void* stream_) {
    if (n_exist == 0) return 0;
    fill_claim_kernel<<<(unsigned)((n_exist + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(claim, n_exist);
    MMSSL_LAUNCH_OK();
    return 0;
}

extern "C" int mmssl_sample_triples(const int64_t* indptr, const int64_t* indices, const int64_t* exist, int64_t n_exist,
                                    int64_t n_items, int batch, uint64_t seed, const int32_t* step_dev, int32_t step_host,
                                    int32_t* claim, int64_t* users, int64_t* pos, int64_t* neg, void* stream_) {
    return sample_one_cta<int64_t, false>(indptr, indices, exist, 0, n_exist, 0, n_exist, n_items, batch, seed, step_dev, step_host, claim,
                                          users, pos, neg, (cudaStream_t)stream_);
}

extern "C" int64_t mmssl_sampler_workspace_bytes(int64_t n_exist, int batch) {
    if (batch < 1 || batch > n_exist) return 0;     // with replacement: no selection
    SelectWs w;
    if (select_carve(batch, n_exist, nullptr, &w) != cudaSuccess) return -1;
    return (int64_t)w.total;
}

extern "C" int mmssl_sample_triples_multi(const int64_t* indptr, const int64_t* indices, const int64_t* exist, int64_t n_exist,
                                          int64_t n_items, int batch, uint64_t seed, const int32_t* step_dev, int32_t step_host,
                                          void* workspace, int64_t workspace_bytes, int64_t* users, int64_t* pos, int64_t* neg,
                                          void* stream_) {
    return sample_multi<int64_t, false>(indptr, indices, exist, 0, n_exist, 0, n_exist, n_items, batch, seed, step_dev, step_host, workspace,
                                        workspace_bytes, users, pos, neg, (cudaStream_t)stream_);
}

extern "C" int mmssl_sample_triples_owned(const int64_t* indptr, const int32_t* indices, const int64_t* exist, int64_t slot_lo,
                                          int64_t slot_hi, int64_t row0, int64_t n_exist, int64_t n_items, int batch, uint64_t seed,
                                          const int32_t* step_dev, int32_t step_host, int32_t* claim, int64_t* users, int64_t* pos,
                                          int64_t* neg, void* stream_) {
    if (int rc = check_owned(slot_lo, slot_hi, row0, n_exist)) return rc;
    return sample_one_cta<int32_t, true>(indptr, indices, exist, slot_lo, slot_hi, row0, n_exist, n_items, batch, seed, step_dev, step_host,
                                         claim, users, pos, neg, (cudaStream_t)stream_);
}

extern "C" int mmssl_sample_triples_multi_owned(const int64_t* indptr, const int32_t* indices, const int64_t* exist, int64_t slot_lo,
                                                int64_t slot_hi, int64_t row0, int64_t n_exist, int64_t n_items, int batch, uint64_t seed,
                                                const int32_t* step_dev, int32_t step_host, void* workspace, int64_t workspace_bytes,
                                                int64_t* users, int64_t* pos, int64_t* neg, void* stream_) {
    if (int rc = check_owned(slot_lo, slot_hi, row0, n_exist)) return rc;
    return sample_multi<int32_t, true>(indptr, indices, exist, slot_lo, slot_hi, row0, n_exist, n_items, batch, seed, step_dev, step_host,
                                       workspace, workspace_bytes, users, pos, neg, (cudaStream_t)stream_);
}
