// General-width tensor-core GEMM for the GAN side of the full step (SURVEY 8f "next" row 2, DESIGN section 9):
//
//   C[m][n] = alpha * sum_k (A_hi + A_lo)[m][k] * (B_hi + B_lo)[n][k]  (+ C when beta == 1)       (lo*lo dropped)
//
// The Discriminator's first layer (Models.py:224-245, nn.Linear(n_items, n_items/4)) makes every D call of the reference's
// iteration a [2B, I] x [I, I/4] product, and the closed-form backward / gradient-penalty sweeps (oracle/gan_oracle.py) add
// its transposed variants: 11 such products per iteration (Baby: 2048 x 7050 x 1762 = 50.9 GFLOP each).  Compute-bound:
// wgmma, with the same bf16 hi/lo operand split as the projection (fp32 contract, 1e-4 relative), i.e. 3 MMAs per product.
//
// Same anatomy as proj_tc.cu (two consumer warpgroups with register accumulators, one TMA producer warp, tc_common.cuh), but
// tiled over N as well: CTA (m_tile, n_tile) owns a 128 x NT tile of C for the whole K range (no split-K: every shape on this
// path gives >= 100 tiles).
//
// Accumulation length is bounded: the tensor core's fp32 accumulate is not round-to-nearest, so its error grows with the
// number of MMAs chained into one accumulator.  The K range is therefore cut into passes of `chunk_kb` k-blocks (default 16 =
// 1024 of K = 192 chained MMAs); after each pass the consumer warps fold the accumulator into C with round-to-nearest fp32 adds
// (C (+)= alpha * pass; C is L2-resident) and start the next pass from zero.  Both operands are re-read from L2 by the other
// tiles of their row / column of the grid, so both are hinted evict-last.  Rows / columns beyond m / n: TMA zero-fills the
// loads, the epilogue masks the stores; C's leading dimension is arbitrary (I/4 is not a multiple of 4): column pairs are stored
// as 8-byte accesses when ldc is even, element by element otherwise.
//
// Executed on the CPU through a functional model of the PTX it issues (tests/cuemu/cuemu_ptx.cpp; tests/test_emu_tensor_core.py:
// multi-tile N, ragged edges, both epilogues, several passes); its GPU test is tests/test_gpu_zzz_gemm_wide.py.  mbar_wait traps
// instead of hanging.
#include "tc_common.cuh"
#include "../../include/mmssl_b200.h"

namespace mmssl {


template <int NT>
struct WideCfg {
    static constexpr int kTileBBytes = NT * kBlockK * 2;
    static constexpr int kStageBytes = 2 * kTileABytes + 2 * kTileBBytes;      // 96 KB at NT = 256, 64 KB at NT = 128
    static constexpr int kStages = (NT == 256) ? 2 : 3;
    static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
};

template <int NT>
__global__ void __launch_bounds__(kThreads, 1)
gemm_wide_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
                 const __grid_constant__ CUtensorMap tm_b_hi, const __grid_constant__ CUtensorMap tm_b_lo,
                 float* __restrict__ C, int64_t ldc, int M, int Ntot, int nkb, int chunk_kb, float alpha, int accumulate) {
    using Cfg = WideCfg<NT>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::kStages * Cfg::kStageBytes);
    uint64_t* empty_bar = full_bar + Cfg::kStages;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m_tile = blockIdx.x, n_tile = blockIdx.y;

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
                const int kx = i * kBlockK;
                tma_load_2d(&tm_a_hi, &full_bar[s], st, kx, m_tile * kBlockM, kEvictLast);
                tma_load_2d(&tm_a_lo, &full_bar[s], st + kTileABytes, kx, m_tile * kBlockM, kEvictLast);
                tma_load_2d(&tm_b_hi, &full_bar[s], st + 2 * kTileABytes, kx, n_tile * NT, kEvictLast);
                tma_load_2d(&tm_b_lo, &full_bar[s], st + 2 * kTileABytes + Cfg::kTileBBytes, kx, n_tile * NT, kEvictLast);
            }
        }
    } else {
        const int64_t row0 = (int64_t)m_tile * kBlockM + 64 * (warp >> 2);
        const int col0 = n_tile * NT;
        const bool pair_ok = (ldc % 2) == 0 && (reinterpret_cast<uintptr_t>(C) & 7u) == 0;   // every (row, even col) pair 8-byte aligned
        const int n_pass = (nkb + chunk_kb - 1) / chunk_kb;
        float acc[NT / 2];
        for (int pass = 0; pass < n_pass; ++pass) {
            const bool add_c = accumulate != 0 || pass > 0;       // later passes fold into what the earlier ones stored
#pragma unroll
            for (int j = 0; j < NT / 2; ++j) acc[j] = 0.f;
            mma_kblocks<NT, Cfg::kStages, Cfg::kStageBytes>(acc, smem, full_bar, empty_bar, pass * chunk_kb, min(nkb, (pass + 1) * chunk_kb));
#pragma unroll
            for (int j = 0; j < NT / 2; j += 2) {         // acc[j], acc[j + 1]: columns col, col + 1 of one row
                const int64_t row = row0 + frag_row(warp, lane, j);
                const int col = col0 + frag_col(lane, j);   // even
                if (row >= M || col >= Ntot) continue;
                float* out = C + row * ldc + col;
                if (pair_ok && col + 1 < Ntot) {            // 8-byte access: a lane quad covers 32 contiguous bytes of the row
                    float2 r = make_float2(alpha * acc[j], alpha * acc[j + 1]);
                    if (add_c) {
                        const float2 prev = *reinterpret_cast<const float2*>(out);
                        r.x += prev.x;
                        r.y += prev.y;
                    }
                    *reinterpret_cast<float2*>(out) = r;
                } else {
                    for (int e = 0; e < 2 && col + e < Ntot; ++e) {
                        float r = alpha * acc[j + e];
                        if (add_c) r += out[e];
                        out[e] = r;
                    }
                }
            }
        }
    }
}

template <int NT>
static int launch_wide(const CUtensorMap& ah, const CUtensorMap& al, const CUtensorMap& bh, const CUtensorMap& bl, float* c,
                       int64_t ldc, int64_t m, int64_t n, int64_t k, float alpha, int accumulate, int chunk_kb, cudaStream_t st) {
    using Cfg = WideCfg<NT>;
    static bool attr_done = false;
    if (!attr_done) {
        MMSSL_CUDA(cudaFuncSetAttribute(gemm_wide_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
        attr_done = true;
    }
    const int nkb = (int)((k + kBlockK - 1) / kBlockK);
    dim3 grid((unsigned)((m + kBlockM - 1) / kBlockM), (unsigned)((n + NT - 1) / NT));
    gemm_wide_kernel<NT><<<grid, kThreads, Cfg::kSmemBytes, st>>>(ah, al, bh, bl, c, ldc, (int)m, (int)n, nkb, chunk_kb, alpha, accumulate);
    MMSSL_LAUNCH_OK();
    return 0;
}

}  // namespace mmssl

using namespace mmssl;

// k-blocks (64 of K each) chained into one accumulator before the epilogue folds it into C (see the file header).
static int g_wide_chunk_kb = 16;

extern "C" int mmssl_gemm_wide_set_chunk(int k_blocks) {
    MMSSL_REQUIRE(k_blocks >= 1, "chunk must be >= 1 k-block");
    g_wide_chunk_kb = k_blocks;
    return 0;
}

extern "C" int mmssl_gemm_bf16x3_wide(const uint16_t* a_hi, const uint16_t* a_lo, int64_t lda, const uint16_t* b_hi,
                                      const uint16_t* b_lo, int64_t ldb, int64_t m, int64_t n, int64_t k, float alpha, int accumulate,
                                      float* c, int64_t ldc, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE(m >= 1 && n >= 1 && k >= 1 && m < (1ll << 31) && n < (1ll << 31) && k < (1ll << 31), "bad m / n / k");
    MMSSL_REQUIRE(m / kBlockM < 65535 * 32768ll && (n + 127) / 128 <= 65535, "grid too large");
    MMSSL_REQUIRE(lda % 8 == 0 && ldb % 8 == 0 && lda >= k && ldb >= k, "lda/ldb must be >= k and multiples of 8 (16-byte TMA strides)");
    MMSSL_REQUIRE(aligned16(a_hi) && aligned16(a_lo) && aligned16(b_hi) && aligned16(b_lo), "operand alignment");
    MMSSL_REQUIRE(c != nullptr && ldc >= n && (reinterpret_cast<uintptr_t>(c) & 3u) == 0, "bad output");
    const int nt = n > 128 ? 256 : 128;
    CUtensorMap ah, al, bh, bl;
    if (int rc = make_map(&ah, a_hi, m, lda, kBlockM)) return rc;
    if (int rc = make_map(&al, a_lo, m, lda, kBlockM)) return rc;
    if (int rc = make_map(&bh, b_hi, n, ldb, nt)) return rc;
    if (int rc = make_map(&bl, b_lo, n, ldb, nt)) return rc;
    if (nt == 256) return launch_wide<256>(ah, al, bh, bl, c, ldc, m, n, k, alpha, accumulate, g_wide_chunk_kb, st);
    return launch_wide<128>(ah, al, bh, bl, c, ldc, m, n, k, alpha, accumulate, g_wide_chunk_kb, st);
}
