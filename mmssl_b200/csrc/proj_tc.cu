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

template <int N>
struct GemmCfg {
    static constexpr int kTileBBytes = N * kBlockK * 2;
    static constexpr int kStageBytes = 2 * kTileABytes + 2 * kTileBBytes;
    // N = 64: two CTAs are co-resident per SM (2 stages each = the same 192 KB of loads in flight),
    // so one CTA's prologue / epilogue overlaps the other's main loop.
    static constexpr int kCtasPerSm = (N == 64) ? 2 : 1;
    static constexpr int kStages = (N == 64) ? 2 : (N == 128 ? 3 : 2);
    static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
};

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
    const int64_t slots = (int64_t)kNumSMs * (n == 64 ? 2 : 1);
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
    MMSSL_REQUIRE(n == 64 || n == 128 || n == 256, "n (embedding width) must be 64, 128 or 256");
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
    if (n == 64) return launch_gemm<64>(ah, al, bh, bl, partial, m, k, split_k, st);
    if (n == 128) return launch_gemm<128>(ah, al, bh, bl, partial, m, k, split_k, st);
    return launch_gemm<256>(ah, al, bh, bl, partial, m, k, split_k, st);
}
