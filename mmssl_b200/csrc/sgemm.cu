// CUDA-core fp32 GEMM (64x64x16 tiles, 4x4 per thread).  Not the projection's production path
// (that is the wgmma kernel in proj_tc.cu); used for the small d x d mixing GEMMs of the
// "attention" closed form (Models.py:139-169, SURVEY appendix B.1), their gradients, and as the
// independent verification path for the tensor-core projection.
#include "common.cuh"
#include "../../include/mmssl_b200.h"

namespace mmssl {

constexpr int BM = 64, BN = 64, BK = 16;

template <bool TA, bool TB>
__global__ void __launch_bounds__(256) sgemm_kernel(int64_t M, int64_t N, int64_t K, float alpha,
                                                    const float* __restrict__ A, int64_t lda,
                                                    const float* __restrict__ B, int64_t ldb, float beta,
                                                    float* __restrict__ C, int64_t ldc, int64_t k_per_split) {
    __shared__ __align__(16) float As[BK][BM + 4];
    __shared__ __align__(16) float Bs[BK][BN + 4];
    const int t = threadIdx.x;
    const int64_t m0 = blockIdx.x * (int64_t)BM, n0 = blockIdx.y * (int64_t)BN;
    const int64_t kbeg = blockIdx.z * k_per_split;
    const int64_t kend = min(K, kbeg + k_per_split);
    const int ty = t / 16, tx = t % 16;
    float acc[4][4] = {};
    for (int64_t k0 = kbeg; k0 < kend; k0 += BK) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            int mm, kk;
            if (!TA) { kk = t % 16; mm = t / 16 + 16 * i; } else { mm = t % 64; kk = t / 64 + 4 * i; }
            const int64_t gm = m0 + mm, gk = k0 + kk;
            float v = 0.f;
            if (gm < M && gk < kend) v = TA ? A[gk * lda + gm] : A[gm * lda + gk];
            As[kk][mm] = v;
            int nn, kb;
            if (!TB) { nn = t % 64; kb = t / 64 + 4 * i; } else { kb = t % 16; nn = t / 16 + 16 * i; }
            const int64_t gn = n0 + nn, gkb = k0 + kb;
            float w = 0.f;
            if (gn < N && gkb < kend) w = TB ? B[gn * ldb + gkb] : B[gkb * ldb + gn];
            Bs[kb][nn] = w;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            const float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
            const float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
            const float av[4] = {a.x, a.y, a.z, a.w};
            const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int64_t gm = m0 + ty * 4 + i;
        if (gm >= M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int64_t gn = n0 + tx * 4 + j;
            if (gn >= N) continue;
            float* cp = C + gm * ldc + gn;
            if (gridDim.z > 1) atomicAdd(cp, alpha * acc[i][j]);
            else *cp = alpha * acc[i][j] + (beta != 0.f ? beta * (*cp) : 0.f);
        }
    }
}

// ---- large shapes (the GAN side's n x I x I/4 products when the tensor-core route is not selected): 128 x 128 x 8 tiles,
// 8 x 8 outputs per thread in two 4-wide strips per dimension (A reads broadcast inside a half-warp, B reads are 256
// contiguous bytes: conflict-free), the next tile's global loads issued before the current tile's FMAs (register double
// buffering).  Same argument meaning and split-K semantics as sgemm_kernel.
constexpr int LM = 128, LN = 128, LK = 8;

template <bool TA, bool TB>
__global__ void __launch_bounds__(256) sgemm_large_kernel(int64_t M, int64_t N, int64_t K, float alpha,
                                                          const float* __restrict__ A, int64_t lda,
                                                          const float* __restrict__ B, int64_t ldb, float beta,
                                                          float* __restrict__ C, int64_t ldc, int64_t k_per_split) {
    __shared__ __align__(16) float As[LK][LM + 4];
    __shared__ __align__(16) float Bs[LK][LN + 4];
    const int t = threadIdx.x;
    const int64_t m0 = blockIdx.x * (int64_t)LM, n0 = blockIdx.y * (int64_t)LN;
    const int64_t kbeg = blockIdx.z * k_per_split;
    const int64_t kend = min(K, kbeg + k_per_split);
    const int ty = t / 16, tx = t % 16;
    // this thread's 4 elements of the A tile and of the B tile: consecutive along the operand's contiguous dimension
    int a_m[4], a_k[4], b_n[4], b_k[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        if (!TA) { a_k[i] = (t % 2) * 4 + i; a_m[i] = t / 2; } else { a_k[i] = t / 32; a_m[i] = (t % 32) * 4 + i; }
        if (TB) { b_k[i] = (t % 2) * 4 + i; b_n[i] = t / 2; } else { b_k[i] = t / 32; b_n[i] = (t % 32) * 4 + i; }
    }
    auto load = [&](int64_t k0, float (&ra)[4], float (&rb)[4]) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int64_t gm = m0 + a_m[i], gk = k0 + a_k[i];
            ra[i] = (gm < M && gk < kend) ? (TA ? A[gk * lda + gm] : A[gm * lda + gk]) : 0.f;
            const int64_t gn = n0 + b_n[i], gkb = k0 + b_k[i];
            rb[i] = (gn < N && gkb < kend) ? (TB ? B[gn * ldb + gkb] : B[gkb * ldb + gn]) : 0.f;
        }
    };
    float acc[8][8] = {};
    float ra[4], rb[4];
    if (kbeg < kend) load(kbeg, ra, rb);
    for (int64_t k0 = kbeg; k0 < kend; k0 += LK) {
#pragma unroll
        for (int i = 0; i < 4; ++i) { As[a_k[i]][a_m[i]] = ra[i]; Bs[b_k[i]][b_n[i]] = rb[i]; }
        __syncthreads();
        if (k0 + LK < kend) load(k0 + LK, ra, rb);            // in flight while the FMAs below run
#pragma unroll
        for (int kk = 0; kk < LK; ++kk) {
            const float4 a0 = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[kk][64 + ty * 4]);
            const float4 b0 = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
            const float4 b1 = *reinterpret_cast<const float4*>(&Bs[kk][64 + tx * 4]);
            const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int64_t gm = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
        if (gm >= M) continue;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int64_t gn = n0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4));
            if (gn >= N) continue;
            float* cp = C + gm * ldc + gn;
            if (gridDim.z > 1) atomicAdd(cp, alpha * acc[i][j]);
            else *cp = alpha * acc[i][j] + (beta != 0.f ? beta * (*cp) : 0.f);
        }
    }
}

}  // namespace mmssl

using namespace mmssl;

extern "C" int mmssl_sgemm(int trans_a, int trans_b, int64_t m, int64_t n, int64_t k, float alpha, const float* a,
                           int64_t lda, const float* b, int64_t ldb, float beta, float* c, int64_t ldc, int split_k,
                           void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE(m >= 0 && n >= 0 && k >= 0 && split_k >= 1, "bad sizes");
    if (m == 0 || n == 0) return 0;
    // Large products (both output dimensions beyond every embedding width of the hot path) take the 128 x 128 kernel; the
    // d x d mixing GEMMs, the simt projection path and everything else keep the 64 x 64 kernel they were validated with.
    const bool large = m >= 128 && n >= 512;
    const int bm = large ? LM : BM, bn = large ? LN : BN;
    dim3 grid((unsigned)((m + bm - 1) / bm), (unsigned)((n + bn - 1) / bn), (unsigned)split_k);
    MMSSL_REQUIRE(grid.y <= 65535 && grid.z <= 65535, "grid too large");
    int64_t kps = (k + split_k - 1) / split_k;
    kps = (kps + BK - 1) / BK * BK;
    if (kps == 0) kps = BK;
    if (large) {
#define LAUNCH_L(TA, TB) sgemm_large_kernel<TA, TB><<<grid, 256, 0, st>>>(m, n, k, alpha, a, lda, b, ldb, beta, c, ldc, kps)
        if (!trans_a && !trans_b) LAUNCH_L(false, false);
        else if (!trans_a && trans_b) LAUNCH_L(false, true);
        else if (trans_a && !trans_b) LAUNCH_L(true, false);
        else LAUNCH_L(true, true);
#undef LAUNCH_L
        MMSSL_LAUNCH_OK();
        return 0;
    }
#define LAUNCH(TA, TB) sgemm_kernel<TA, TB><<<grid, 256, 0, st>>>(m, n, k, alpha, a, lda, b, ldb, beta, c, ldc, kps)
    if (!trans_a && !trans_b) LAUNCH(false, false);
    else if (!trans_a && trans_b) LAUNCH(false, true);
    else if (trans_a && !trans_b) LAUNCH(true, false);
    else LAUNCH(true, true);
#undef LAUNCH
    MMSSL_LAUNCH_OK();
    return 0;
}
