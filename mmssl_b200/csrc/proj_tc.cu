// Projection GEMM on the Hopper tensor cores (wgmma) fed by TMA, accumulators in registers.
//
//   partial[s][m][n] = sum_{k in slice s} (A_hi + A_lo)[m][k] * (B_hi + B_lo)[n][k]      (lo*lo dropped)
//
// replaces nn.Linear image_trans / text_trans forward (X = F W^T, Models.py:173-174) and its weight
// gradient (dW^T = F^T dX, autograd of the same lines).  fp32 contract (1e-4 rel) is met with a
// bf16 hi/lo operand split: three bf16 MMAs per product, fp32 accumulation in registers.  The
// feature matrix is constant (Models.py:46-47), so its split (and its transposed split for the
// weight gradient) is made once; both GEMMs then run the SAME K-major kernel.
//
// Shape of the work: HBM-bound (AI = 3*2*N/4 flop per byte of A at N = d), M is small (items) or
// medium (feature dim) -> split-K so that >= 2 waves of CTAs pull from HBM; partials are reduced in
// a fixed order by the epilogue kernels in proj_common.cu (deterministic, no float atomics).
//
// Kernel anatomy (one CTA = one 128 x N output tile of one K slice, 288 threads, tc_common.cuh):
//   warps 0-7: two consumer warpgroups, 64 rows each: wgmma.mma_async m64nNk16 from the swizzled smem tiles, each warp
//              releases a stage once its MMAs have completed; epilogue straight from the accumulator registers
//   warp 8   : TMA producer (cp.async.bulk.tensor.2d, SWIZZLE_128B, mbarrier complete_tx)
#include "tc_common.cuh"
#include "../../include/mmssl_b200.h"

namespace mmssl {

// N = 32 and 64: two CTAs are co-resident per SM (2 stages each: 160 / 192 KB of loads in flight),
// so one CTA's prologue / epilogue overlaps the other's main loop.
static constexpr int ctas_per_sm(int64_t n) { return n <= 64 ? 2 : 1; }
static bool proj_width_ok(int64_t n) { return n == 32 || n == 64 || n == 96 || n == 128 || n == 192 || n == 256; }

// kDeep: the one-CTA-per-SM instance of the grouped kernel at N = 32 / 64, which spends the whole SM's shared memory on its
// ring: 5 x 40 KB / 4 x 48 KB, so three to four k-blocks of F (32 KB each) are in flight per SM instead of one.
template <int N, bool kDeep = false>
struct GemmCfg {
    static constexpr int kTileBBytes = N * kBlockK * 2;
    static constexpr int kStageBytes = 2 * kTileABytes + 2 * kTileBBytes;   // 32 KB of A (hi + lo) + N * 256 B of B
    static constexpr int kCtasPerSm = kDeep ? 1 : ctas_per_sm(N);
    // 2 x 40 / 48 KB per CTA at N = 32 / 64; 3 x 56 / 64 KB at N = 96 / 128; 2 x 80 / 128 KB at N = 192 / 256
    static constexpr int kStages = kDeep ? (N <= 32 ? 5 : 4) : (N <= 64) ? 2 : (N <= 128 ? 3 : 2);
    static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
    static_assert(!kDeep || N <= 64, "the deep instance exists for N = 32 and 64 only");
    static_assert(kSmemBytes <= 227 * 1024, "shared memory of one CTA");
};
constexpr int kGroupMax = 2;                                                // problems of one grouped launch (image, text)

template <int N>
__global__ void __launch_bounds__(kThreads, GemmCfg<N>::kCtasPerSm)
gemm_bf16x3_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
                   const __grid_constant__ CUtensorMap tm_b_hi, const __grid_constant__ CUtensorMap tm_b_lo,
                   float* __restrict__ partial, int M, int total_kb, int kb_per_split) {
    using Cfg = GemmCfg<N>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::kStages * Cfg::kStageBytes);
    uint64_t* empty_bar = full_bar + Cfg::kStages;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m_tile = blockIdx.x, split = blockIdx.y;
    const int kb0 = split * kb_per_split;
    const int nkb = max(0, min(total_kb, kb0 + kb_per_split) - kb0);

    if (warp == kProducerWarp && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tm_a_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tm_a_lo) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tm_b_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tm_b_lo) : "memory");
        for (int s = 0; s < Cfg::kStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kConsumerWarps); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == kProducerWarp) {
        if (lane == 0) {
            for (int i = 0; i < nkb; ++i) {
                const int s = i % Cfg::kStages;
                const uint32_t ph = (uint32_t)(i / Cfg::kStages) & 1u;
                mbar_wait(&empty_bar[s], ph ^ 1u);
                uint8_t* st = smem + s * Cfg::kStageBytes;
                mbar_expect_tx(&full_bar[s], Cfg::kStageBytes);
                const int kx = (kb0 + i) * kBlockK;
                tma_load_2d(&tm_a_hi, &full_bar[s], st, kx, m_tile * kBlockM, kEvictFirst);
                tma_load_2d(&tm_a_lo, &full_bar[s], st + kTileABytes, kx, m_tile * kBlockM, kEvictFirst);
                tma_load_2d(&tm_b_hi, &full_bar[s], st + 2 * kTileABytes, kx, 0, kEvictLast);
                tma_load_2d(&tm_b_lo, &full_bar[s], st + 2 * kTileABytes + Cfg::kTileBBytes, kx, 0, kEvictLast);
            }
        }
    } else {
        float acc[N / 2];
#pragma unroll
        for (int j = 0; j < N / 2; ++j) acc[j] = 0.f;
        mma_kblocks<N, Cfg::kStages, Cfg::kStageBytes>(acc, smem, full_bar, empty_bar, 0, nkb);
        const int64_t row0 = (int64_t)m_tile * kBlockM + 64 * (warp >> 2);
        float* out = partial + ((int64_t)split * M) * N;
#pragma unroll
        for (int j = 0; j < N / 2; j += 2) {
            const int64_t row = row0 + frag_row(warp, lane, j);
            if (row < M) *reinterpret_cast<float2*>(out + row * N + frag_col(lane, j)) = make_float2(acc[j], acc[j + 1]);
        }
    }
}

static int choose_split(int64_t m, int64_t n, int64_t k) {
    // HBM-bound streaming GEMM: what matters is that all SMs pull from HBM for the whole kernel.
    // Pick the split-K that fills ONE wave of co-resident CTAs as completely as possible
    // (e.g. 56 M-tiles x 4 slices = 224 of 264 slots) instead of leaving a nearly empty tail wave.
    const int64_t total_kb = (k + kBlockK - 1) / kBlockK;
    const int64_t m_tiles = (m + kBlockM - 1) / kBlockM;
    const int64_t slots = (int64_t)kNumSMs * ctas_per_sm(n);
    int64_t split = slots / m_tiles;
    // accuracy: the tensor core's fp32 accumulate is not round-to-nearest and its error grows linearly with the number of MMAs
    // chained into one accumulator (gemm_wide.cu; the weight gradient at 200k items with 347 k-blocks per slice was 1e-4 off).  A slice is therefore at most kMaxChainKb k-blocks long; the slices are summed in fp32 by the epilogue.
    const int64_t need = (total_kb + kMaxChainKb - 1) / kMaxChainKb;
    if (split < need) split = need;
    if (split > kMaxSplit) split = kMaxSplit;
    if (split > total_kb) split = total_kb;
    if (split < 1) split = 1;
    // make every slice non-empty
    const int64_t per = (total_kb + split - 1) / split;
    split = (total_kb + per - 1) / per;
    return (int)split;
}

template <int N>
static int launch_gemm(const CUtensorMap& ah, const CUtensorMap& al, const CUtensorMap& bh, const CUtensorMap& bl,
                       float* partial, int64_t m, int64_t k, int split_k, cudaStream_t st) {
    using Cfg = GemmCfg<N>;
    static bool attr_done = false;
    if (!attr_done) {
        MMSSL_CUDA(cudaFuncSetAttribute(gemm_bf16x3_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
        attr_done = true;
    }
    const int total_kb = (int)((k + kBlockK - 1) / kBlockK);
    const int per = (total_kb + split_k - 1) / split_k;
    dim3 grid((unsigned)((m + kBlockM - 1) / kBlockM), (unsigned)split_k);
    gemm_bf16x3_kernel<N><<<grid, kThreads, Cfg::kSmemBytes, st>>>(ah, al, bh, bl, partial, (int)m, total_kb, per);
    MMSSL_LAUNCH_OK();
    return 0;
}

// ---- grouped, persistent variant: the image and text problems of one direction in one launch ----------------------------
//
// The work of a group is a list of units (problem, m_tile, K slice).  Each problem cuts its K into `split` slices of `per`
// k-blocks (the last one may be shorter), exactly as the kernel above does for the same split, so a unit writes the same
// partial[s][m][n] tile the single-problem kernel would.  One resident wave of CTAs walks the list: CTA b takes units
// b, b + gridDim.x, ... (a static schedule: the same CTA computes the same tile on every launch).  The TMA producer runs
// across unit boundaries: the stage ring and its mbarrier phases continue from one unit to the next, so the next unit's
// stages land while the consumers store the previous unit's accumulators.
//
// The unit list is not stored: it is a few classes of equal-length units (per problem: its full slices, then its shorter
// last slice), sorted longest first, and a unit's index decodes into (class, slice, m_tile) on the device and on the host.
struct GroupClass {
    float* partial;             // the problem's partial[split][m][n]
    int prob, m, m_tiles, per;  // problem index, rows, 128-row tiles, k-blocks per full slice
    int s0, u0, n_units, len;   // first slice of the class, first unit index, units (= slices * m_tiles), k-blocks per unit
};
struct GroupParams {
    CUtensorMap maps[kGroupMax][4];   // a_hi, a_lo, b_hi, b_lo of each problem
    GroupClass cls[2 * kGroupMax];
    int n_classes, n_units, n_problems;
};
struct GroupUnit { int cls, slice, m_tile, kb0, kb1; };

__host__ __device__ __forceinline__ GroupUnit group_unit(const GroupClass* cls, int n_classes, int u) {
    int c = 0;
    while (c + 1 < n_classes && u >= cls[c + 1].u0) ++c;
    const GroupClass& k = cls[c];
    const int j = u - k.u0;
    GroupUnit w;
    w.cls = c;
    w.slice = k.s0 + j / k.m_tiles;
    w.m_tile = j % k.m_tiles;
    w.kb0 = w.slice * k.per;
    w.kb1 = w.kb0 + k.len;
    return w;
}

template <int N, bool kDeep>
__global__ void __launch_bounds__(kThreads, GemmCfg<N, kDeep>::kCtasPerSm)
gemm_bf16x3_group_kernel(const __grid_constant__ GroupParams P) {
    using Cfg = GemmCfg<N, kDeep>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::kStages * Cfg::kStageBytes);
    uint64_t* empty_bar = full_bar + Cfg::kStages;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp == kProducerWarp && lane == 0) {
        for (int p = 0; p < P.n_problems; ++p)
            for (int t = 0; t < 4; ++t) asm volatile("prefetch.tensormap [%0];" ::"l"(&P.maps[p][t]) : "memory");
        for (int s = 0; s < Cfg::kStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kConsumerWarps); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == kProducerWarp) {
        if (lane == 0) {
            int it = 0;   // k-blocks issued by this CTA so far: stage it % kStages, phase (it / kStages) & 1
            for (int u = blockIdx.x; u < P.n_units; u += gridDim.x) {
                const GroupUnit w = group_unit(P.cls, P.n_classes, u);
                const CUtensorMap* tm = P.maps[P.cls[w.cls].prob];
                const int y = w.m_tile * kBlockM;
                for (int kb = w.kb0; kb < w.kb1; ++kb, ++it) {
                    const int s = it % Cfg::kStages;
                    mbar_wait(&empty_bar[s], ((uint32_t)(it / Cfg::kStages) & 1u) ^ 1u);
                    uint8_t* st = smem + s * Cfg::kStageBytes;
                    mbar_expect_tx(&full_bar[s], Cfg::kStageBytes);
                    const int kx = kb * kBlockK;
                    tma_load_2d(&tm[0], &full_bar[s], st, kx, y, kEvictFirst);
                    tma_load_2d(&tm[1], &full_bar[s], st + kTileABytes, kx, y, kEvictFirst);
                    tma_load_2d(&tm[2], &full_bar[s], st + 2 * kTileABytes, kx, 0, kEvictLast);
                    tma_load_2d(&tm[3], &full_bar[s], st + 2 * kTileABytes + Cfg::kTileBBytes, kx, 0, kEvictLast);
                }
            }
        }
    } else {
        int it = 0;
        for (int u = blockIdx.x; u < P.n_units; u += gridDim.x) {
            const GroupUnit w = group_unit(P.cls, P.n_classes, u);
            float acc[N / 2];
#pragma unroll
            for (int j = 0; j < N / 2; ++j) acc[j] = 0.f;
            mma_kblocks<N, Cfg::kStages, Cfg::kStageBytes>(acc, smem, full_bar, empty_bar, it, it + (w.kb1 - w.kb0));
            it += w.kb1 - w.kb0;
            const GroupClass& c = P.cls[w.cls];
            const int64_t row0 = (int64_t)w.m_tile * kBlockM + 64 * (warp >> 2);
            float* out = c.partial + ((int64_t)w.slice * c.m) * N;
#pragma unroll
            for (int j = 0; j < N / 2; j += 2) {
                const int64_t row = row0 + frag_row(warp, lane, j);
                if (row < c.m) *reinterpret_cast<float2*>(out + row * N + frag_col(lane, j)) = make_float2(acc[j], acc[j + 1]);
            }
        }
    }
}

// The classes of a group for the given splits, sorted longest first (stable: problem order, full slices before last slices).
// partial may be null (planning only).  Returns the number of classes.
static int group_classes(int np, const int64_t* m, const int64_t* n, const int64_t* k, const int* split, float* const* partial,
                         GroupClass* cls) {
    int nc = 0;
    for (int p = 0; p < np; ++p) {
        const int total_kb = (int)((k[p] + kBlockK - 1) / kBlockK);
        const int per = (total_kb + split[p] - 1) / split[p];
        const int last = total_kb - per * (split[p] - 1);
        const int m_tiles = (int)((m[p] + kBlockM - 1) / kBlockM);
        GroupClass c{partial ? partial[p] : nullptr, p, (int)m[p], m_tiles, per, 0, 0, 0, per};
        const int full = (last == per) ? split[p] : split[p] - 1;
        if (full > 0) { c.n_units = full * m_tiles; cls[nc++] = c; }
        if (full < split[p]) { c.s0 = full; c.len = last; c.n_units = m_tiles; cls[nc++] = c; }
    }
    for (int i = 1; i < nc; ++i)   // insertion sort, stable
        for (int j = i; j > 0 && cls[j].len > cls[j - 1].len; --j) { GroupClass t = cls[j]; cls[j] = cls[j - 1]; cls[j - 1] = t; }
    int u0 = 0;
    for (int i = 0; i < nc; ++i) { cls[i].u0 = u0; u0 += cls[i].n_units; }
    (void)n;
    return nc;
}

static int group_grid(int n_units, int n, int max_ctas) {
    int g = kNumSMs * ctas_per_sm(n);
    if (max_ctas > 0 && max_ctas < g) g = max_ctas;
    return n_units < g ? n_units : g;
}

// Estimated time of the round-robin schedule, in k-blocks of the busiest CTA.  A unit also costs its partial tile
// (128 x N fp32): written here and read again by the epilogue, about two k-blocks of A (128 x 64 bf16 hi + lo) per 64 of N.
static int64_t group_cost(const GroupClass* cls, int nc, int grid, int n) {
    const int64_t unit_cost = 2 * n / 64;
    int64_t load[kNumSMs * 2] = {0};
    for (int i = 0; i < nc; ++i) {
        const int64_t per_cta = cls[i].n_units / grid, rem = cls[i].n_units % grid, first = cls[i].u0 % grid;
        const int64_t c = cls[i].len + unit_cost;
        for (int b = 0; b < grid; ++b) {
            const int64_t off = (b - first + grid) % grid;
            load[b] += c * (per_cta + (off < rem ? 1 : 0));
        }
    }
    int64_t worst = 0;
    for (int b = 0; b < grid; ++b) worst = load[b] > worst ? load[b] : worst;
    return worst;
}

}  // namespace mmssl

using namespace mmssl;

extern "C" int64_t mmssl_gemm_bf16x3_workspace_floats(int64_t m, int64_t n, int64_t k, int* split_k_out) {
    const int split = choose_split(m, n, k);
    if (split_k_out) *split_k_out = split;
    return (int64_t)split * m * n;
}

extern "C" int mmssl_gemm_bf16x3(const uint16_t* a_hi, const uint16_t* a_lo, int64_t lda, const uint16_t* b_hi,
                                 const uint16_t* b_lo, int64_t ldb, int64_t m, int64_t n, int64_t k, int split_k,
                                 float* partial, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE(proj_width_ok(n), "n (embedding width) must be 32, 64, 96, 128, 192 or 256");
    MMSSL_REQUIRE(m >= 1 && k >= 1 && m < (1ll << 31) && k < (1ll << 31), "bad m / k");
    MMSSL_REQUIRE(lda % 8 == 0 && ldb % 8 == 0 && lda >= k && ldb >= k, "lda/ldb must be >= k and multiples of 8 (16-byte TMA strides)");
    MMSSL_REQUIRE(aligned16(a_hi) && aligned16(a_lo) && aligned16(b_hi) && aligned16(b_lo) && aligned16(partial), "alignment");
    const int total_kb = (int)((k + kBlockK - 1) / kBlockK);
    MMSSL_REQUIRE(split_k >= 1 && split_k <= total_kb, "split_k out of range");
    {
        const int per = (total_kb + split_k - 1) / split_k;
        MMSSL_REQUIRE((int64_t)per * (split_k - 1) < total_kb, "split_k leaves an empty K slice (use mmssl_gemm_bf16x3_workspace_floats)");
    }
    CUtensorMap ah, al, bh, bl;
    if (int rc = make_map(&ah, a_hi, m, lda, kBlockM)) return rc;
    if (int rc = make_map(&al, a_lo, m, lda, kBlockM)) return rc;
    if (int rc = make_map(&bh, b_hi, n, ldb, (int)n)) return rc;
    if (int rc = make_map(&bl, b_lo, n, ldb, (int)n)) return rc;
    switch (n) {
        case 32: return launch_gemm<32>(ah, al, bh, bl, partial, m, k, split_k, st);
        case 64: return launch_gemm<64>(ah, al, bh, bl, partial, m, k, split_k, st);
        case 96: return launch_gemm<96>(ah, al, bh, bl, partial, m, k, split_k, st);
        case 128: return launch_gemm<128>(ah, al, bh, bl, partial, m, k, split_k, st);
        case 192: return launch_gemm<192>(ah, al, bh, bl, partial, m, k, split_k, st);
        default: return launch_gemm<256>(ah, al, bh, bl, partial, m, k, split_k, st);
    }
}

namespace mmssl {

// Splits of a group: the plan of the estimated shortest round-robin schedule (group_cost).  The single-problem plans
// (choose_split) are tried first and kept unless another plan is strictly shorter, so a group whose problems already
// balance computes bitwise the partials of mmssl_gemm_bf16x3.  Every slice stays within kMaxChainKb k-blocks.
static void group_plan(int np, const int64_t* m, const int64_t* n, const int64_t* k, int max_ctas, int* split) {
    GroupClass cls[2 * kGroupMax];
    int cand[kGroupMax][kMaxChainKb], n_cand[kGroupMax];
    for (int p = 0; p < np; ++p) {
        split[p] = choose_split(m[p], n[p], k[p]);
        const int total_kb = (int)((k[p] + kBlockK - 1) / kBlockK);
        n_cand[p] = 0;
        for (int per = total_kb < kMaxChainKb ? total_kb : kMaxChainKb; per >= 1; --per) {   // fewest slices first
            const int s = (total_kb + per - 1) / per;
            if (s > kMaxSplit) break;
            if (n_cand[p] == 0 || cand[p][n_cand[p] - 1] != s) cand[p][n_cand[p]++] = s;
        }
    }
    auto cost = [&](const int* sp) {
        const int nc = group_classes(np, m, n, k, sp, nullptr, cls);
        const int units = cls[nc - 1].u0 + cls[nc - 1].n_units;
        return group_cost(cls, nc, group_grid(units, (int)n[0], max_ctas), (int)n[0]);
    };
    int64_t best = cost(split);
    int trial[kGroupMax];
    for (int i = 0; i < n_cand[0]; ++i)
        for (int j = 0; j < (np > 1 ? n_cand[1] : 1); ++j) {
            trial[0] = cand[0][i];
            if (np > 1) trial[1] = cand[1][j];
            const int64_t c = cost(trial);
            if (c < best) {
                best = c;
                for (int p = 0; p < np; ++p) split[p] = trial[p];
            }
        }
}

static int group_check_shapes(int np, const int64_t* m, const int64_t* n, const int64_t* k) {
    MMSSL_REQUIRE(np >= 1 && np <= kGroupMax, "a group holds one or two problems");
    for (int p = 0; p < np; ++p) {
        MMSSL_REQUIRE(proj_width_ok(n[p]), "n (embedding width) must be 32, 64, 96, 128, 192 or 256");
        MMSSL_REQUIRE(n[p] == n[0], "the problems of a group must have the same n");
        MMSSL_REQUIRE(m[p] >= 1 && k[p] >= 1 && m[p] < (1ll << 31) && k[p] < (1ll << 31), "bad m / k");
    }
    return 0;
}

template <int N, bool kDeep = false>
static int launch_group(const GroupParams& prm, int grid, cudaStream_t st) {
    using Cfg = GemmCfg<N, kDeep>;
    static bool attr_done = false;
    if (!attr_done) {
        MMSSL_CUDA(cudaFuncSetAttribute(gemm_bf16x3_group_kernel<N, kDeep>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
        attr_done = true;
    }
    gemm_bf16x3_group_kernel<N, kDeep><<<grid, kThreads, Cfg::kSmemBytes, st>>>(prm);
    MMSSL_LAUNCH_OK();
    return 0;
}

}  // namespace mmssl

extern "C" int64_t mmssl_gemm_bf16x3_group_plan(int n_problems, const int64_t* mnk, int max_ctas, int* split_out,
                                                int64_t* floats_out, int32_t* units_out, int64_t units_cap) {
    int64_t m[kGroupMax], n[kGroupMax], k[kGroupMax];
    if (n_problems < 1 || n_problems > kGroupMax || mnk == nullptr) {
        fail(__func__, "a group holds one or two problems");
        return -1;
    }
    for (int p = 0; p < n_problems; ++p) { m[p] = mnk[3 * p]; n[p] = mnk[3 * p + 1]; k[p] = mnk[3 * p + 2]; }
    if (group_check_shapes(n_problems, m, n, k)) return -1;
    int split[kGroupMax];
    group_plan(n_problems, m, n, k, max_ctas, split);
    GroupClass cls[2 * kGroupMax];
    const int nc = group_classes(n_problems, m, n, k, split, nullptr, cls);
    const int64_t units = cls[nc - 1].u0 + cls[nc - 1].n_units;
    for (int p = 0; p < n_problems; ++p) {
        if (split_out) split_out[p] = split[p];
        if (floats_out) floats_out[p] = (int64_t)split[p] * m[p] * n[p];
    }
    if (units_out)
        for (int64_t u = 0; u < units && u < units_cap; ++u) {
            const GroupUnit w = group_unit(cls, nc, (int)u);
            units_out[4 * u] = cls[w.cls].prob;
            units_out[4 * u + 1] = w.m_tile;
            units_out[4 * u + 2] = w.kb0;
            units_out[4 * u + 3] = w.kb1;
        }
    return units;
}

extern "C" int mmssl_gemm_bf16x3_group(int n_problems, const mmssl_gemm_problem_t* probs, int max_ctas, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE(n_problems >= 1 && n_problems <= kGroupMax && probs != nullptr, "a group holds one or two problems");
    MMSSL_REQUIRE(max_ctas >= 0, "max_ctas must be >= 0 (0 = one resident wave)");
    int64_t m[kGroupMax], n[kGroupMax], k[kGroupMax];
    int split[kGroupMax];
    float* partial[kGroupMax];
    GroupParams prm;
    memset(&prm, 0, sizeof(prm));
    for (int p = 0; p < n_problems; ++p) {
        const mmssl_gemm_problem_t& q = probs[p];
        m[p] = q.m; n[p] = q.n; k[p] = q.k; split[p] = q.split_k; partial[p] = q.partial;
    }
    if (int rc = group_check_shapes(n_problems, m, n, k)) return rc;
    for (int p = 0; p < n_problems; ++p) {
        const mmssl_gemm_problem_t& q = probs[p];
        MMSSL_REQUIRE(q.lda % 8 == 0 && q.ldb % 8 == 0 && q.lda >= q.k && q.ldb >= q.k,
                      "lda/ldb must be >= k and multiples of 8 (16-byte TMA strides)");
        MMSSL_REQUIRE(aligned16(q.a_hi) && aligned16(q.a_lo) && aligned16(q.b_hi) && aligned16(q.b_lo) && aligned16(q.partial),
                      "alignment");
        const int total_kb = (int)((q.k + kBlockK - 1) / kBlockK);
        MMSSL_REQUIRE(q.split_k >= 1 && q.split_k <= total_kb, "split_k out of range");
        const int per = (total_kb + q.split_k - 1) / q.split_k;
        MMSSL_REQUIRE((int64_t)per * (q.split_k - 1) < total_kb, "split_k leaves an empty K slice (use mmssl_gemm_bf16x3_group_plan)");
        MMSSL_REQUIRE(per <= kMaxChainKb, "a K slice is longer than kMaxChainKb k-blocks (use mmssl_gemm_bf16x3_group_plan)");
        MMSSL_REQUIRE((int64_t)q.split_k * ((q.m + kBlockM - 1) / kBlockM) < (1ll << 30), "too many units");
        if (int rc = make_map(&prm.maps[p][0], q.a_hi, q.m, q.lda, kBlockM)) return rc;
        if (int rc = make_map(&prm.maps[p][1], q.a_lo, q.m, q.lda, kBlockM)) return rc;
        if (int rc = make_map(&prm.maps[p][2], q.b_hi, q.n, q.ldb, (int)q.n)) return rc;
        if (int rc = make_map(&prm.maps[p][3], q.b_lo, q.n, q.ldb, (int)q.n)) return rc;
    }
    prm.n_problems = n_problems;
    prm.n_classes = group_classes(n_problems, m, n, k, split, partial, prm.cls);
    prm.n_units = prm.cls[prm.n_classes - 1].u0 + prm.cls[prm.n_classes - 1].n_units;
    const int grid = group_grid(prm.n_units, (int)n[0], max_ctas);
    // at most one CTA per SM (the engine's 132-CTA cap): the deep-ring instance, which fills the SM's shared memory alone
    const bool deep = grid <= kNumSMs;
    switch (n[0]) {
        case 32: return deep ? launch_group<32, true>(prm, grid, st) : launch_group<32>(prm, grid, st);
        case 64: return deep ? launch_group<64, true>(prm, grid, st) : launch_group<64>(prm, grid, st);
        case 96: return launch_group<96>(prm, grid, st);
        case 128: return launch_group<128>(prm, grid, st);
        case 192: return launch_group<192>(prm, grid, st);
        default: return launch_group<256>(prm, grid, st);
    }
}
