// InfoNCE on the tensor cores (VERDICT r1 #6; reference: sim / batched_contrastive_loss, main.py:211-249, calls :411-412).
//
// For a batch of n <= 2048 rows the two similarity matrices  a a^T  and  a b^T  (a = normalised z1 rows, b = normalised z2 rows)
// are n x n x d contractions: 0.27 GFLOP at n = 1024, d = 64 -- tensor-core work.  The fp32 contract (1e-4) is kept the way the
// projection keeps it: operands as bf16 hi + lo pairs, three MMAs per product, fp32 accumulation in registers (K = d <= 256: 48
// chained MMAs at most, far below the lengths where the accumulate error shows, gemm_wide.cu).  |s / tau| <= 2, so a 1e-5
// error in s is 2e-5 in exp(s / tau).
//
//   forward  nce_stats_tc_kernel: CTA (it, jt, m) owns ONE 128 x 128 tile of  S_R = A_i A_j^T (m = 0),  S_B = A_i B_j^T (1)  or
//            S_T = B_i A_j^T (2: the transposed block of a b^T that the backward needs row-major) in the registers of its two
//            wgmma warpgroups -- 192 CTAs at n = 1024, two per SM; operands by TMA (SWIZZLE_128B); the same warps then compute
//            exp -> row sums, diagonal, and the exponentials themselves stored as bf16 hi / lo matrices E_R, E_B, E_T (12 MB at
//            n = 1024: L2-resident).
//            nce_finalize_kernel (loss.cu) turns the sums into loss rows and backward coefficients u, v as before.
//   backward with P_ij = -(u_i + u_j) R_ij / tau (i != j), Q_ij = B_ij (-u_i + [i == j] v_i) / tau:
//              dL/da_i = sum_j P_ij a_j + Q_ij b_j = -(1/tau) [ u_i (E_R a)_i + (E_R (u.a))_i + u_i (E_B b)_i ] + diagonal terms
//              dL/db_j = sum_i Q_ij a_i           = -(1/tau) (E_T (u.a))_j + diagonal term
//            i.e. three products of the stored exponentials with [a | u.a], b and u.a: nce_operands_kernel writes those operands
//            transposed (K-major over the batch) as bf16 hi / lo, the products run on the projection's split-K wgmma kernel
//            (mmssl_gemm_bf16x3), nce_combine_kernel sums the K slices and applies the coefficients.
// Larger batches (B = 16384: the exponentials would take 3 TB) and d = 256 (operand width 512) stay on the CUDA-core kernels.
#include <cuda_bf16.h>

#include "tc_common.cuh"
#include "../../include/mmssl_b200.h"

namespace mmssl {

int nce_finalize_launch(int64_t n, int64_t ntj, float* stats, float* coef, const float* g_loss, float* loss_part, cudaStream_t st);   // loss.cu
int nce_prepare_split_launch(const float* z1, int64_t ldz1, const float* z2, int64_t ldz2, const int64_t* idx, int64_t n, int d, float* a,
                             float* b, float* na, float* nb, uint16_t* a_hi, uint16_t* a_lo, uint16_t* b_hi, uint16_t* b_lo, cudaStream_t st);   // loss.cu

constexpr int kNceTile = 128;
constexpr int kNceMaxN = 2048;
constexpr int kNceStageBytes = 4 * kTileABytes;                     // row operand, column operand  x  hi, lo : 64 KB
constexpr int kNceRows = 16, kNceRowPitch = 272;                    // epilogue staging: a warp's 16 rows x (256 B + 16 B pad), hi and lo
constexpr int kNceEpiBytes = kConsumerWarps * 2 * kNceRows * kNceRowPitch;   // 68 KB, laid over the operand tiles (dead once the MMAs completed)
constexpr int kNceSmemBytes = kNceEpiBytes + 256 + 1024;            // 2 CTAs per SM

// bf16 pair (x in the low half) with one cvt.rn.bf16x2; its two halves widened back to fp32 are shifts
__device__ __forceinline__ uint32_t pack_bf16(float x, float y) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(x, y);
    return *reinterpret_cast<const uint32_t*>(&h);
}
__device__ __forceinline__ float fast_exp2(float x) {      // MUFU.EX2: |x| <= 2.9 here (|s / tau| <= 2), relative error ~2e-7
    float y;
    asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// stats layout (loss.cu): [diagR n][diagB n][loss n][unused n][partR ntj*n][partB ntj*n],  ntj = 2 * gridDim.y
constexpr int kNceThreads = kThreads;   // warps 0-7 two wgmma warpgroups + epilogue, warp 8 TMA producer

__global__ void __launch_bounds__(kNceThreads, 2)
nce_stats_tc_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
                    const __grid_constant__ CUtensorMap tm_b_hi, const __grid_constant__ CUtensorMap tm_b_lo, int64_t n, int nkb,
                    float inv_tau, float* __restrict__ stats, uint16_t* __restrict__ e_hi, uint16_t* __restrict__ e_lo, int64_t lde) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    static_assert(kNceEpiBytes >= kNceStageBytes, "staging lies over the operand tiles");
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kNceEpiBytes);
    uint64_t* empty_bar = full_bar + 1;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int it = blockIdx.x, jt = blockIdx.y;
    const int mat = blockIdx.z;                                   // 0: S_R = A_i A_j^T   1: S_B = A_i B_j^T   2: S_T = B_i A_j^T

    if (warp == kProducerWarp && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tm_a_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tm_a_lo) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tm_b_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tm_b_lo) : "memory");
        mbar_init(full_bar, 1); mbar_init(empty_bar, kConsumerWarps);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    float acc[kNceTile / 2];
    if (warp == kProducerWarp) {
        if (lane == 0) {
            for (int kb = 0; kb < nkb; ++kb) {
                mbar_wait(empty_bar, ((uint32_t)kb & 1u) ^ 1u);
                mbar_expect_tx(full_bar, kNceStageBytes);
                const int kx = kb * kBlockK;
                const CUtensorMap* rh = (mat == 2) ? &tm_b_hi : &tm_a_hi;      // row operand (tile it)
                const CUtensorMap* rl = (mat == 2) ? &tm_b_lo : &tm_a_lo;
                const CUtensorMap* ch = (mat == 1) ? &tm_b_hi : &tm_a_hi;      // column operand (tile jt)
                const CUtensorMap* cl = (mat == 1) ? &tm_b_lo : &tm_a_lo;
                tma_load_2d(rh, full_bar, smem + 0 * kTileABytes, kx, it * kNceTile, kEvictLast);
                tma_load_2d(rl, full_bar, smem + 1 * kTileABytes, kx, it * kNceTile, kEvictLast);
                tma_load_2d(ch, full_bar, smem + 2 * kTileABytes, kx, jt * kNceTile, kEvictLast);
                tma_load_2d(cl, full_bar, smem + 3 * kTileABytes, kx, jt * kNceTile, kEvictLast);
            }
        }
    } else {
#pragma unroll
        for (int j = 0; j < kNceTile / 2; ++j) acc[j] = 0.f;
        mma_kblocks<kNceTile, 1, kNceStageBytes>(acc, smem, full_bar, empty_bar, 0, nkb);     // hi hi + hi lo + lo hi
    }
    __syncthreads();            // every MMA has read the operand tiles: the staging area may overwrite them
    if (warp == kProducerWarp) return;

    // A warp owns 16 rows x 128 columns of the tile (rows r and r + 8 per lane, wgmma fragment layout).  Exponentials, their row
    // sums per column half (the two partials of this column tile in the stats layout) and the diagonal; the exponentials go to
    // global memory as bf16 hi / lo through a shared-memory staging tile (row pitch 272 B: conflict-free both ways) so that
    // 16 lanes write one 256-byte row segment.
    const int64_t rbase = (int64_t)it * kNceTile + 64 * (warp >> 2) + 16 * (warp & 3);
    const int64_t j0 = (int64_t)jt * kNceTile;
    const int64_t ntj = 2 * (int64_t)gridDim.y;                   // row-sum partials: one per (column tile, half)
    const float scale = inv_tau * 1.4426950408889634f;          // exp(x) = exp2(x log2 e)
    const bool plain = (int64_t)(it + 1) * kNceTile <= n && (int64_t)(jt + 1) * kNceTile <= n && it != jt;   // CTA-uniform
    float* diag = mat < 2 ? stats + mat * n : nullptr;
    uint8_t* stage_hi = smem + warp * (2 * kNceRows * kNceRowPitch);
    uint8_t* stage_lo = stage_hi + kNceRows * kNceRowPitch;
    float part[2][2] = {{0.f, 0.f}, {0.f, 0.f}};                  // [row r / r + 8][column half]
#pragma unroll
    for (int j = 0; j < kNceTile / 2; j += 2) {
        const int rr = (j >> 1) & 1, h = j >= kNceTile / 4 ? 1 : 0;
        const int rl = (lane >> 2) + 8 * rr, cl = frag_col(lane, j);
        const int64_t i = rbase + rl, col = j0 + cl;
        float e0, e1;
        if (plain) {            // interior tiles off the diagonal (most of them) skip the bounds and diagonal tests
            e0 = fast_exp2(acc[j] * scale);
            e1 = fast_exp2(acc[j + 1] * scale);
        } else {
            e0 = (i < n && col < n) ? fast_exp2(acc[j] * scale) : 0.f;
            e1 = (i < n && col + 1 < n) ? fast_exp2(acc[j + 1] * scale) : 0.f;
            if (diag != nullptr && i < n) {
                if (i == col) diag[i] = e0;
                if (i == col + 1) diag[i] = e1;
            }
        }
        part[rr][h] += e0 + e1;
        const uint32_t hp = pack_bf16(e0, e1);
        *reinterpret_cast<uint32_t*>(stage_hi + rl * kNceRowPitch + cl * 2) = hp;
        *reinterpret_cast<uint32_t*>(stage_lo + rl * kNceRowPitch + cl * 2) =
            pack_bf16(e0 - __uint_as_float(hp << 16), e1 - __uint_as_float(hp & 0xffff0000u));
    }
#pragma unroll
    for (int rr = 0; rr < 2; ++rr)
#pragma unroll
        for (int h = 0; h < 2; ++h) part[rr][h] = group_sum<4>(part[rr][h], group_mask<4>());
    if (mat < 2 && (lane & 3) == 0) {
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
            const int64_t i = rbase + (lane >> 2) + 8 * rr;
            if (i < n) {
                stats[4 * n + mat * ntj * n + (2 * jt) * n + i] = part[rr][0];
                stats[4 * n + mat * ntj * n + (2 * jt + 1) * n + i] = part[rr][1];
            }
        }
    }
    __syncwarp();
    // rows up to the padded height are written (zeros beyond n): the backward's GEMMs read them as K padding
    uint16_t* ghi = e_hi + (int64_t)mat * lde * lde + rbase * lde + j0;
    uint16_t* glo = e_lo + (int64_t)mat * lde * lde + rbase * lde + j0;
#pragma unroll
    for (int r0 = 0; r0 < kNceRows; r0 += 2) {
        const int r = r0 + (lane >> 4), ch = lane & 15;
        *reinterpret_cast<uint4*>(ghi + (int64_t)r * lde + ch * 8) = *reinterpret_cast<const uint4*>(stage_hi + r * kNceRowPitch + ch * 16);
        *reinterpret_cast<uint4*>(glo + (int64_t)r * lde + ch * 8) = *reinterpret_cast<const uint4*>(stage_lo + r * kNceRowPitch + ch * 16);
    }
}

// Transposed bf16 hi / lo operands of the backward products, K-major over the batch (zero beyond n):
//   op1[c][i] = a[i][c] (c < d),  op1[d + c][i] = u_i a[i][c];    op2[c][i] = b[i][c]
__global__ void nce_operands_kernel(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ coef, int64_t n,
                                    int d, uint16_t* __restrict__ op1_hi, uint16_t* __restrict__ op1_lo, uint16_t* __restrict__ op2_hi,
                                    uint16_t* __restrict__ op2_lo, int64_t ldn) {
    __shared__ float ta[32][33], tb[32][33];
    __shared__ float us[32];
    const int64_t i0 = blockIdx.x * 32ll;
    const int c0 = blockIdx.y * 32;
    for (int k = threadIdx.y; k < 32; k += blockDim.y) {
        const int64_t i = i0 + k;
        const int c = c0 + threadIdx.x;
        ta[k][threadIdx.x] = (i < n) ? a[i * d + c] : 0.f;
        tb[k][threadIdx.x] = (i < n) ? b[i * d + c] : 0.f;
    }
    if (threadIdx.y == 0) us[threadIdx.x] = (i0 + threadIdx.x < n) ? coef[i0 + threadIdx.x] : 0.f;
    __syncthreads();
    for (int k = threadIdx.y; k < 32; k += blockDim.y) {
        const int c = c0 + k;
        const int64_t i = i0 + threadIdx.x;
        if (i >= ldn) continue;
        const float va = ta[threadIdx.x][k], vb = tb[threadIdx.x][k], vu = va * us[threadIdx.x];
        const __nv_bfloat16 ha = __float2bfloat16_rn(va), hb = __float2bfloat16_rn(vb), hu = __float2bfloat16_rn(vu);
        op1_hi[(int64_t)c * ldn + i] = __bfloat16_as_ushort(ha);
        op1_lo[(int64_t)c * ldn + i] = __bfloat16_as_ushort(__float2bfloat16_rn(va - __bfloat162float(ha)));
        op1_hi[(int64_t)(d + c) * ldn + i] = __bfloat16_as_ushort(hu);
        op1_lo[(int64_t)(d + c) * ldn + i] = __bfloat16_as_ushort(__float2bfloat16_rn(vu - __bfloat162float(hu)));
        op2_hi[(int64_t)c * ldn + i] = __bfloat16_as_ushort(hb);
        op2_lo[(int64_t)c * ldn + i] = __bfloat16_as_ushort(__float2bfloat16_rn(vb - __bfloat162float(hb)));
    }
}

// ga[i] = -(1/tau) [ u_i (G1a_i - R_ii a_i) + (G1ua_i - R_ii u_i a_i) + u_i G2_i ] + (v_i/tau) B_ii b_i
// gb[j] = -(1/tau) G3_j + (v_j/tau) B_jj a_j          G1 = E_R [a | u.a] (width 2d), G2 = E_B b, G3 = E_T (u.a): sums of K slices
__global__ void __launch_bounds__(256) nce_combine_kernel(const float* __restrict__ g1, int s1, const float* __restrict__ g2, int s2,
                                                          const float* __restrict__ g3, int s3, const float* __restrict__ a,
                                                          const float* __restrict__ b, const float* __restrict__ coef,
                                                          const float* __restrict__ stats, int64_t n, int d4, float inv_tau,
                                                          float* __restrict__ ga, float* __restrict__ gb) {
    const int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (t >= n * d4) return;
    const int64_t i = t / d4;
    const int c = (int)(t - i * d4) * 4;
    const int d = d4 * 4;
    float4 xa = f4zero(), xua = f4zero(), x2 = f4zero(), x3 = f4zero();
    const bool do_a = blockIdx.y == 0;             // blockIdx.y: 0 -> ga, 1 -> gb (independent halves of the work)
    if (do_a) {
        for (int s0 = 0; s0 < s1; s0 += 4) {        // 12 independent loads in flight, summed in slice order
            float4 pa[4], pu[4], p2[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const bool ok = s0 + q < s1;
                const float* p = g1 + ((int64_t)(ok ? s0 + q : 0) * n + i) * (2 * d);
                pa[q] = ok ? ld4(p + c) : f4zero();
                pu[q] = ok ? ld4(p + d + c) : f4zero();
                p2[q] = (s0 + q < s2) ? ld4(g2 + ((int64_t)(s0 + q) * n + i) * d + c) : f4zero();
            }
#pragma unroll
            for (int q = 0; q < 4; ++q) { xa = add4(xa, pa[q]); xua = add4(xua, pu[q]); x2 = add4(x2, p2[q]); }
        }
    } else {
        for (int s0 = 0; s0 < s3; s0 += 8) {
            float4 p3[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) p3[q] = (s0 + q < s3) ? ld4(g3 + ((int64_t)(s0 + q) * n + i) * d + c) : f4zero();
#pragma unroll
            for (int q = 0; q < 8; ++q) x3 = add4(x3, p3[q]);
        }
    }
    const float u = coef[i], v = coef[n + i], rii = stats[i], bii = stats[n + i];
    const float4 av = ld4(a + i * d + c), bv = ld4(b + i * d + c);
    float4 o, w;
    o.x = -inv_tau * (u * (xa.x - rii * av.x) + (xua.x - rii * u * av.x) + u * x2.x) + inv_tau * v * bii * bv.x;
    o.y = -inv_tau * (u * (xa.y - rii * av.y) + (xua.y - rii * u * av.y) + u * x2.y) + inv_tau * v * bii * bv.y;
    o.z = -inv_tau * (u * (xa.z - rii * av.z) + (xua.z - rii * u * av.z) + u * x2.z) + inv_tau * v * bii * bv.z;
    o.w = -inv_tau * (u * (xa.w - rii * av.w) + (xua.w - rii * u * av.w) + u * x2.w) + inv_tau * v * bii * bv.w;
    w.x = -inv_tau * x3.x + inv_tau * v * bii * av.x;
    w.y = -inv_tau * x3.y + inv_tau * v * bii * av.y;
    w.z = -inv_tau * x3.z + inv_tau * v * bii * av.z;
    w.w = -inv_tau * x3.w + inv_tau * v * bii * av.w;
    if (do_a) st4(ga + i * d + c, o); else st4(gb + i * d + c, w);
}

struct NceWs {
    uint16_t *a_hi, *a_lo, *b_hi, *b_lo;        // [n][d]
    uint16_t *e_hi, *e_lo;                       // [3][lde][lde]  (E_R, E_B, E_T)
    uint16_t *op1_hi, *op1_lo, *op2_hi, *op2_lo; // [2d][lde], [d][lde]
    float *g1, *g2, *g3;                         // K-slice partials of the three products
    int s1, s2, s3;
    int64_t lde;
    size_t total;
};

static void nce_carve(int64_t n, int d, void* base, NceWs* w) {
    auto up = [](size_t v) { return (v + 255) & ~(size_t)255; };
    const int64_t lde = (n + kNceTile - 1) / kNceTile * kNceTile;
    size_t off = 0;
    char* b = (char*)base;
    auto take = [&](size_t bytes) { char* p = b + off; off += up(bytes); return p; };
    w->lde = lde;
    w->a_hi = (uint16_t*)take(2 * n * d); w->a_lo = (uint16_t*)take(2 * n * d);
    w->b_hi = (uint16_t*)take(2 * n * d); w->b_lo = (uint16_t*)take(2 * n * d);
    w->e_hi = (uint16_t*)take(2 * 3 * lde * lde); w->e_lo = (uint16_t*)take(2 * 3 * lde * lde);
    w->op1_hi = (uint16_t*)take(2 * 2 * d * lde); w->op1_lo = (uint16_t*)take(2 * 2 * d * lde);
    w->op2_hi = (uint16_t*)take(2 * d * lde); w->op2_lo = (uint16_t*)take(2 * d * lde);
    // K slices of the backward products: the three run side by side (8 M-tiles each), so 8 slices each fill the machine; more
    // slices only add partial-sum traffic for the combine kernel
    int sk = 0;
    mmssl_gemm_bf16x3_workspace_floats(n, d, n, &sk);
    const int64_t total_kb = (n + kBlockK - 1) / kBlockK;
    if (sk > 8) sk = 8;
    { const int64_t per = (total_kb + sk - 1) / sk; sk = (int)((total_kb + per - 1) / per); }
    w->s1 = w->s2 = w->s3 = sk;
    w->g1 = (float*)take(4 * (size_t)sk * n * 2 * d); w->g2 = (float*)take(4 * (size_t)sk * n * d); w->g3 = (float*)take(4 * (size_t)sk * n * d);
    w->total = off + 256;
}

}  // namespace mmssl

using namespace mmssl;

extern "C" int mmssl_infonce_tc_supported(int64_t n, int d) { return (n >= 1 && n <= kNceMaxN && (d == 64 || d == 128)) ? 1 : 0; }

extern "C" int64_t mmssl_infonce_tc_workspace_bytes(int64_t n, int d) {
    if (!mmssl_infonce_tc_supported(n, d)) return 0;
    NceWs w;
    nce_carve(n, d, nullptr, &w);
    return (int64_t)w.total;
}

// a, b: the normalised rows written by mmssl_infonce_prepare; stats / coef / loss_part as for mmssl_infonce_stats.
static int nce_stats_tc_impl(const float* a, const float* b, int64_t n, int d, float inv_tau, float* stats, float* coef,
                             const float* g_loss, float* loss_part, void* workspace, int64_t workspace_bytes, int presplit, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE(mmssl_infonce_tc_supported(n, d), "tensor-core InfoNCE: n <= 2048 and d in {64, 128} (use mmssl_infonce_stats)");
    MMSSL_REQUIRE(workspace != nullptr && aligned16(workspace), "workspace missing");
    NceWs w;
    nce_carve(n, d, workspace, &w);
    MMSSL_REQUIRE((int64_t)w.total <= workspace_bytes, "workspace too small (mmssl_infonce_tc_workspace_bytes)");
    if (!presplit) {
        if (int rc = mmssl_split_bf16(a, d, n, d, w.a_hi, w.a_lo, d, stream_)) return rc;
        if (int rc = mmssl_split_bf16(b, d, n, d, w.b_hi, w.b_lo, d, stream_)) return rc;
    }
    CUtensorMap ah, al, bh, bl;
    if (int rc = make_map(&ah, w.a_hi, n, d, kNceTile)) return rc;
    if (int rc = make_map(&al, w.a_lo, n, d, kNceTile)) return rc;
    if (int rc = make_map(&bh, w.b_hi, n, d, kNceTile)) return rc;
    if (int rc = make_map(&bl, w.b_lo, n, d, kNceTile)) return rc;
    static bool attr_done = false;
    if (!attr_done) {
        MMSSL_CUDA(cudaFuncSetAttribute(nce_stats_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kNceSmemBytes));
        attr_done = true;
    }
    const unsigned nt = (unsigned)(w.lde / kNceTile);
    nce_stats_tc_kernel<<<dim3(nt, nt, 3), kNceThreads, kNceSmemBytes, st>>>(ah, al, bh, bl, n, d / kBlockK, inv_tau, stats, w.e_hi, w.e_lo, w.lde);
    MMSSL_LAUNCH_OK();
    return nce_finalize_launch(n, 2 * (int64_t)nt, stats, coef, g_loss, loss_part, st);
}

extern "C" int mmssl_infonce_stats_tc(const float* a, const float* b, int64_t n, int d, float inv_tau, float* stats, float* coef,
                                      const float* g_loss, float* loss_part, void* workspace, int64_t workspace_bytes, void* stream_) {
    return nce_stats_tc_impl(a, b, n, d, inv_tau, stats, coef, g_loss, loss_part, workspace, workspace_bytes, 0, stream_);
}

// mmssl_infonce_prepare + operand split in one kernel, then the statistics: z1 / z2 rows (gathered through idx) -> a, b, norms,
// bf16 hi / lo of a and b in the workspace -> mmssl_infonce_stats_tc's work.
extern "C" int mmssl_infonce_forward_tc(const float* z1, int64_t ldz1, const float* z2, int64_t ldz2, const int64_t* idx, int64_t n,
                                        int d, float inv_tau, float* a, float* b, float* na, float* nb, float* stats, float* coef,
                                        const float* g_loss, float* loss_part, void* workspace, int64_t workspace_bytes, void* stream_) {
    MMSSL_REQUIRE(mmssl_infonce_tc_supported(n, d), "tensor-core InfoNCE: n <= 2048 and d in {64, 128}");
    MMSSL_REQUIRE(workspace != nullptr && aligned16(workspace), "workspace missing");
    NceWs w;
    nce_carve(n, d, workspace, &w);
    MMSSL_REQUIRE((int64_t)w.total <= workspace_bytes, "workspace too small (mmssl_infonce_tc_workspace_bytes)");
    if (int rc = nce_prepare_split_launch(z1, ldz1, z2, ldz2, idx, n, d, a, b, na, nb, w.a_hi, w.a_lo, w.b_hi, w.b_lo, (cudaStream_t)stream_)) return rc;
    return nce_stats_tc_impl(a, b, n, d, inv_tau, stats, coef, g_loss, loss_part, workspace, workspace_bytes, 1, stream_);
}

// ga, gb (written, not accumulated) from the exponentials mmssl_infonce_stats_tc left in `workspace`.
// phase: -1 everything on `stream`; 0 transposed operands; 1, 2, 3 one product each (independent: may run on three streams);
// 4 combine.
extern "C" int mmssl_infonce_grad_tc(const float* a, const float* b, int64_t n, int d, float inv_tau, const float* coef,
                                     const float* stats, float* ga, float* gb, void* workspace, int64_t workspace_bytes, int phase,
                                     void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE(mmssl_infonce_tc_supported(n, d), "tensor-core InfoNCE: n <= 2048 and d in {64, 128} (use mmssl_infonce_grad)");
    NceWs w;
    nce_carve(n, d, workspace, &w);
    MMSSL_REQUIRE(workspace != nullptr && (int64_t)w.total <= workspace_bytes, "workspace too small");
    MMSSL_REQUIRE(phase >= -1 && phase <= 4, "phase");
    const auto on = [&](int p) { return phase == -1 || phase == p; };
    if (on(0)) {
        dim3 grid((unsigned)((w.lde + 31) / 32), (unsigned)(d / 32));
        nce_operands_kernel<<<grid, dim3(32, 8), 0, st>>>(a, b, coef, n, d, w.op1_hi, w.op1_lo, w.op2_hi, w.op2_lo, w.lde);
        MMSSL_LAUNCH_OK();
    }
    const int64_t ee = w.lde * w.lde;
    if (on(1)) if (int rc = mmssl_gemm_bf16x3(w.e_hi, w.e_lo, w.lde, w.op1_hi, w.op1_lo, w.lde, n, 2 * d, n, w.s1, w.g1, stream_)) return rc;
    if (on(2)) if (int rc = mmssl_gemm_bf16x3(w.e_hi + ee, w.e_lo + ee, w.lde, w.op2_hi, w.op2_lo, w.lde, n, d, n, w.s2, w.g2, stream_)) return rc;
    if (on(3)) if (int rc = mmssl_gemm_bf16x3(w.e_hi + 2 * ee, w.e_lo + 2 * ee, w.lde, w.op1_hi + (int64_t)d * w.lde, w.op1_lo + (int64_t)d * w.lde,
                                              w.lde, n, d, n, w.s3, w.g3, stream_)) return rc;
    if (on(4)) {
        const int64_t tot = n * (d / 4);
        nce_combine_kernel<<<dim3((unsigned)((tot + 255) / 256), 2), 256, 0, st>>>(w.g1, w.s1, w.g2, w.s2, w.g3, w.s3, a, b, coef, stats, n, d / 4, inv_tau, ga, gb);
        MMSSL_LAUNCH_OK();
    }
    return 0;
}
