// Helpers around the projection GEMMs (nn.Linear image_trans / text_trans, Models.py:28-31,173-174):
//  * fp32 -> (bf16 hi, bf16 lo) operand split (x ~= hi + lo with ~16 mantissa bits) so the wgmma
//    kernel can reach fp32-level accuracy with three bf16 MMAs per product;
//  * split-K reduction epilogues: bias + dropout mask for the forward, transpose for the weight grad.
#include <cuda_bf16.h>

#include "common.cuh"
#include "../../include/mmssl_b200.h"

namespace mmssl {

__device__ __forceinline__ void split2(float x, uint16_t& hi, uint16_t& lo) {
    const __nv_bfloat16 h = __float2bfloat16_rn(x);
    const float r = x - __bfloat162float(h);
    const __nv_bfloat16 l = __float2bfloat16_rn(r);
    hi = __bfloat16_as_ushort(h);
    lo = __bfloat16_as_ushort(l);
}

// hi/lo [rows][ldo] <- x [rows][ldx]; columns in [cols, ldo) are zero-filled (TMA-friendly padding)
__global__ void split_bf16_kernel(const float* __restrict__ x, int64_t ldx, int64_t rows, int64_t cols,
                                  uint16_t* __restrict__ hi, uint16_t* __restrict__ lo, int64_t ldo) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= rows * ldo) return;
    const int64_t r = i / ldo, c = i - r * ldo;
    uint16_t h = 0, l = 0;
    if (c < cols) split2(x[r * ldx + c], h, l);
    hi[i] = h;
    lo[i] = l;
}

// hi/lo [cols][ldo] <- (x * mask)[rows][cols] transposed, through a 32x32 smem tile.  colsum != NULL: additionally
// colsum[c] += sum over the tile's rows of (x * mask)[r][c]  (the bias gradient db = colsum(dX * mask) of the projection's
// backward rides along: the tile is in shared memory anyway; one float reduction per column per 32-row tile).
__global__ void split_bf16_t_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ mask,
                                    int64_t ldm, int64_t rows, int64_t cols, uint16_t* __restrict__ hi,
                                    uint16_t* __restrict__ lo, int64_t ldo, float* __restrict__ colsum) {
    __shared__ float tile[32][33];
    const int64_t r0 = blockIdx.x * 32ll, c0 = blockIdx.y * 32ll;
    for (int k = threadIdx.y; k < 32; k += blockDim.y) {
        const int64_t r = r0 + k, c = c0 + threadIdx.x;
        float v = 0.f;
        if (r < rows && c < cols) {
            v = x[r * ldx + c];
            if (mask) v *= mask[r * ldm + c];
        }
        tile[k][threadIdx.x] = v;
    }
    __syncthreads();
    if (colsum != nullptr && threadIdx.y == 0 && c0 + threadIdx.x < cols) {
        float sacc = 0.f;
#pragma unroll 8
        for (int k = 0; k < 32; ++k) sacc += tile[k][threadIdx.x];      // rows beyond `rows` hold zeros
        atomicAdd(colsum + c0 + threadIdx.x, sacc);
    }
    for (int k = threadIdx.y; k < 32; k += blockDim.y) {
        const int64_t c = c0 + k, r = r0 + threadIdx.x;   // output row = input column
        if (c < cols && r < ldo) {
            uint16_t h = 0, l = 0;
            if (r < rows) split2(tile[threadIdx.x][k], h, l);
            hi[c * ldo + r] = h;
            lo[c * ldo + r] = l;
        }
    }
}

__global__ void proj_epilogue_kernel(const float* __restrict__ partial, int split_k, int64_t m, int n4,
                                     const float* __restrict__ bias, const float* __restrict__ mask, int64_t ldm,
                                     float* __restrict__ y, int64_t ldy, float* __restrict__ y_pre, int64_t ldyp) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= m * n4) return;
    const int64_t r = i / n4;
    const int c = (int)(i - r * n4) * 4;
    const int64_t n = (int64_t)n4 * 4;
    float4 acc = bias ? ld4(bias + c) : f4zero();
    int s = 0;
    for (; s + 4 <= split_k; s += 4) {   // 4 independent loads in flight, summed in slice order
        const float4 p0 = ld4(partial + ((int64_t)(s + 0) * m + r) * n + c);
        const float4 p1 = ld4(partial + ((int64_t)(s + 1) * m + r) * n + c);
        const float4 p2 = ld4(partial + ((int64_t)(s + 2) * m + r) * n + c);
        const float4 p3 = ld4(partial + ((int64_t)(s + 3) * m + r) * n + c);
        acc = add4(add4(add4(add4(acc, p0), p1), p2), p3);
    }
    for (; s < split_k; ++s) acc = add4(acc, ld4(partial + ((int64_t)s * m + r) * n + c));
    if (y_pre) st4(y_pre + r * ldyp + c, acc);
    if (mask) {
        const float4 mv = ld4(mask + r * ldm + c);
        acc.x *= mv.x; acc.y *= mv.y; acc.z *= mv.z; acc.w *= mv.w;
    }
    st4(y + r * ldy + c, acc);
}

// dw[nn][mm] (+)= sum_s partial[s][mm][nn]; 32x32 smem transpose
__global__ void wgrad_epilogue_kernel(const float* __restrict__ partial, int split_k, int64_t m, int64_t n,
                                      float* __restrict__ dw, int64_t ldw, int accumulate) {
    __shared__ float tile[32][33];
    const int64_t m0 = blockIdx.x * 32ll, n0 = blockIdx.y * 32ll;
    for (int k = threadIdx.y; k < 32; k += blockDim.y) {
        const int64_t mm = m0 + k, nn = n0 + threadIdx.x;
        float v = 0.f;
        if (mm < m && nn < n) {
            int s = 0;
            for (; s + 4 <= split_k; s += 4) {   // independent loads first, fixed summation order
                const float p0 = partial[((int64_t)(s + 0) * m + mm) * n + nn];
                const float p1 = partial[((int64_t)(s + 1) * m + mm) * n + nn];
                const float p2 = partial[((int64_t)(s + 2) * m + mm) * n + nn];
                const float p3 = partial[((int64_t)(s + 3) * m + mm) * n + nn];
                v = (((v + p0) + p1) + p2) + p3;
            }
            for (; s < split_k; ++s) v += partial[((int64_t)s * m + mm) * n + nn];
        }
        tile[k][threadIdx.x] = v;
    }
    __syncthreads();
    for (int k = threadIdx.y; k < 32; k += blockDim.y) {
        const int64_t nn = n0 + k, mm = m0 + threadIdx.x;
        if (nn < n && mm < m) {
            float* o = dw + nn * ldw + mm;
            *o = tile[threadIdx.x][k] + (accumulate ? *o : 0.f);
        }
    }
}

}  // namespace mmssl

using namespace mmssl;

extern "C" int mmssl_split_bf16(const float* x, int64_t ldx, int64_t rows, int64_t cols, uint16_t* hi, uint16_t* lo,
                                int64_t ldo, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE(ldo >= cols, "ldo < cols");
    const int64_t tot = rows * ldo;
    if (tot == 0) return 0;
    split_bf16_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(x, ldx, rows, cols, hi, lo, ldo);
    MMSSL_LAUNCH_OK();
    return 0;
}

static int split_t_launch(const float* x, int64_t ldx, const float* mask, int64_t ldm, int64_t rows, int64_t cols, uint16_t* hi,
                          uint16_t* lo, int64_t ldo, float* colsum, cudaStream_t st) {
    MMSSL_REQUIRE(ldo >= rows, "ldo < rows");
    if (colsum != nullptr) MMSSL_CUDA(cudaMemsetAsync(colsum, 0, sizeof(float) * cols, st));
    if (cols == 0 || ldo == 0) return 0;
    dim3 grid((unsigned)((ldo + 31) / 32), (unsigned)((cols + 31) / 32));
    split_bf16_t_kernel<<<grid, dim3(32, 8), 0, st>>>(x, ldx, mask, ldm, rows, cols, hi, lo, ldo, colsum);
    MMSSL_LAUNCH_OK();
    return 0;
}

extern "C" int mmssl_split_bf16_t(const float* x, int64_t ldx, const float* mask, int64_t ldm, int64_t rows,
                                  int64_t cols, uint16_t* hi, uint16_t* lo, int64_t ldo, void* stream_) {
    return split_t_launch(x, ldx, mask, ldm, rows, cols, hi, lo, ldo, nullptr, (cudaStream_t)stream_);
}

extern "C" int mmssl_split_bf16_t_colsum(const float* x, int64_t ldx, const float* mask, int64_t ldm, int64_t rows,
                                         int64_t cols, uint16_t* hi, uint16_t* lo, int64_t ldo, float* colsum, void* stream_) {
    MMSSL_REQUIRE(colsum != nullptr, "colsum output missing");
    return split_t_launch(x, ldx, mask, ldm, rows, cols, hi, lo, ldo, colsum, (cudaStream_t)stream_);
}

extern "C" int mmssl_proj_epilogue(const float* partial, int split_k, int64_t m, int64_t n, const float* bias,
                                   const float* mask, int64_t ldm, float* y, int64_t ldy, float* y_pre, int64_t ldyp,
                                   void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE(n % 4 == 0 && aligned16(partial) && aligned16(y) && ldy % 4 == 0, "alignment");
    MMSSL_REQUIRE((mask == nullptr || (aligned16(mask) && ldm % 4 == 0)) && (bias == nullptr || aligned16(bias)), "alignment");
    MMSSL_REQUIRE(y_pre == nullptr || (aligned16(y_pre) && ldyp % 4 == 0), "alignment");
    const int64_t tot = m * (n / 4);
    if (tot == 0) return 0;
    proj_epilogue_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(partial, split_k, m, (int)(n / 4), bias, mask, ldm,
                                                                       y, ldy, y_pre, ldyp);
    MMSSL_LAUNCH_OK();
    return 0;
}

extern "C" int mmssl_wgrad_epilogue(const float* partial, int split_k, int64_t m, int64_t n, float* dw, int64_t ldw,
                                    int accumulate, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (m == 0 || n == 0) return 0;
    dim3 grid((unsigned)((m + 31) / 32), (unsigned)((n + 31) / 32));
    wgrad_epilogue_kernel<<<grid, dim3(32, 8), 0, st>>>(partial, split_k, m, n, dw, ldw, accumulate);
    MMSSL_LAUNCH_OK();
    return 0;
}
