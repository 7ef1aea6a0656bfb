// Row-wise fused glue of MMSSL.forward / backward: everything between the SpMMs that is not a GEMM.
// One lane group (width_shape in common.cuh: 8 to 32 lanes) owns one row, float4 per lane, shuffle reductions;
// all kernels are HBM/L2-bound streaming passes.
//   id_fuse      Models.py:196-197   u0 = E + id_cat_rate * normalize(z)
//   combine      Models.py:213-218   uf = mean_k(u_k) + model_cat_rate*(normalize(Uv)+normalize(Ut))
//                                    (+ the sums of squares main.py:252-257 needs, for free)
//   softmax_bwd  backward of Models.py:203-204
#include "common.cuh"
#include "../../include/mmssl_b200.h"

namespace mmssl {

constexpr float kNormEps = 1e-12f;   // F.normalize default eps

template <int G, int C>
struct RowIdx {
    int64_t row;
    int lane;
    unsigned mask;
    __device__ __forceinline__ RowIdx() {
        mask = group_mask<G>();
        lane = threadIdx.x & (G - 1);
        row = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / G;
    }
    __device__ __forceinline__ int col(int c) const { return lane * 4 + c * 4 * G; }
};

template <int G, int C>
__device__ __forceinline__ void load_row(float4 (&v)[C], const float* base, int64_t ld, const RowIdx<G, C>& ix) {
#pragma unroll
    for (int c = 0; c < C; ++c) v[c] = ld4(base + ix.row * ld + ix.col(c));
}
template <int G, int C>
__device__ __forceinline__ void store_row(const float4 (&v)[C], float* base, int64_t ld, const RowIdx<G, C>& ix) {
#pragma unroll
    for (int c = 0; c < C; ++c) st4(base + ix.row * ld + ix.col(c), v[c]);
}
template <int G, int C>
__device__ __forceinline__ float row_dot(const float4 (&a)[C], const float4 (&b)[C], unsigned mask) {
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < C; ++c) s += dot4(a[c], b[c]);
    return group_sum<G>(s, mask);
}

// normalize-backward for one row: returns rate * d/dx [x / max(|x|, eps)] applied to g
template <int G, int C>
__device__ __forceinline__ void normalize_bwd_row(float4 (&out)[C], const float4 (&x)[C], const float4 (&g)[C],
                                                  float rate, unsigned mask) {
    const float ss = row_dot<G, C>(x, x, mask);
    const float nrm = sqrtf(ss);
    if (nrm > kNormEps) {
        const float inv = 1.f / nrm;
        const float dot = row_dot<G, C>(x, g, mask) * inv;   // <xn, g>
#pragma unroll
        for (int c = 0; c < C; ++c) {
            out[c].x = rate * inv * (g[c].x - x[c].x * inv * dot);
            out[c].y = rate * inv * (g[c].y - x[c].y * inv * dot);
            out[c].z = rate * inv * (g[c].z - x[c].z * inv * dot);
            out[c].w = rate * inv * (g[c].w - x[c].w * inv * dot);
        }
    } else {   // clamp_min(eps) branch of F.normalize: derivative is g / eps
        const float k = rate / kNormEps;
#pragma unroll
        for (int c = 0; c < C; ++c) out[c] = scale4(g[c], k);
    }
}

template <int G, int C>
__global__ void __launch_bounds__(256) id_fuse_fwd_kernel(const float* __restrict__ z, int64_t ldz,
                                                          const float* __restrict__ e, int64_t lde, int64_t n,
                                                          float rate, float* __restrict__ out, int64_t ldo,
                                                          float* __restrict__ zn, float* __restrict__ nrm_out) {
    pdl_wait();
    RowIdx<G, C> ix;
    if (ix.row >= n) return;
    float4 zv[C], ev[C];
    load_row<G, C>(zv, z, ldz, ix);
    load_row<G, C>(ev, e, lde, ix);
    const float nrm = sqrtf(row_dot<G, C>(zv, zv, ix.mask));
    const float inv = 1.f / fmaxf(nrm, kNormEps);
#pragma unroll
    for (int c = 0; c < C; ++c) {
        zv[c] = scale4(zv[c], inv);
        fma4(ev[c], rate, zv[c]);
    }
    store_row<G, C>(ev, out, ldo, ix);
    store_row<G, C>(zv, zn, (int64_t)(4 * G * C), ix);
    if (ix.lane == 0) nrm_out[ix.row] = nrm;
}

template <int G, int C>
__global__ void __launch_bounds__(256) id_fuse_bwd_kernel(const float* __restrict__ g, int64_t ldg,
                                                          const float* __restrict__ zn, const float* __restrict__ nrm,
                                                          int64_t n, float rate, float* __restrict__ dz, int64_t lddz) {
    pdl_wait();
    RowIdx<G, C> ix;
    if (ix.row >= n) return;
    float4 gv[C], nv[C], o[C];
    load_row<G, C>(gv, g, ldg, ix);
    load_row<G, C>(nv, zn, (int64_t)(4 * G * C), ix);
    const float nr = nrm[ix.row];
    if (nr > kNormEps) {
        const float dot = row_dot<G, C>(nv, gv, ix.mask);
        const float k = rate / nr;
#pragma unroll
        for (int c = 0; c < C; ++c) {
            o[c].x = k * (gv[c].x - nv[c].x * dot); o[c].y = k * (gv[c].y - nv[c].y * dot);
            o[c].z = k * (gv[c].z - nv[c].z * dot); o[c].w = k * (gv[c].w - nv[c].w * dot);
        }
    } else {
        const float k = rate / kNormEps;
#pragma unroll
        for (int c = 0; c < C; ++c) o[c] = scale4(gv[c], k);
    }
    store_row<G, C>(o, dz, lddz, ix);
}

template <int G, int C>
__global__ void __launch_bounds__(256) combine_fwd_kernel(const float* __restrict__ s, int64_t lds,
                                                          const float* __restrict__ a, int64_t lda,
                                                          const float* __restrict__ b, int64_t ldb, int64_t n,
                                                          float inv_layers, float rate, float* __restrict__ out,
                                                          int64_t ldo, float* __restrict__ sumsq_partials) {
    pdl_wait();
    __shared__ float red[32];
    RowIdx<G, C> ix;
    float ss = 0.f;
    if (ix.row < n) {
        float4 sv[C], av[C], bv[C];
        load_row<G, C>(sv, s, lds, ix);
        load_row<G, C>(av, a, lda, ix);
        load_row<G, C>(bv, b, ldb, ix);
        const float sa = row_dot<G, C>(av, av, ix.mask);
        const float sb = row_dot<G, C>(bv, bv, ix.mask);
        const float ia = rate / fmaxf(sqrtf(sa), kNormEps);
        const float ib = rate / fmaxf(sqrtf(sb), kNormEps);
#pragma unroll
        for (int c = 0; c < C; ++c) {
            sv[c] = scale4(sv[c], inv_layers);
            fma4(sv[c], ia, av[c]);
            fma4(sv[c], ib, bv[c]);
        }
        store_row<G, C>(sv, out, ldo, ix);
        if (ix.lane == 0) ss = sa + sb;
    }
    if (sumsq_partials != nullptr) {
        const float tot = block_sum(ss, red);
        if (threadIdx.x == 0) sumsq_partials[blockIdx.x] = tot;
    }
}

template <int G, int C>
__global__ void __launch_bounds__(256) combine_bwd_kernel(const float* __restrict__ g, int64_t ldg,
                                                          const float* __restrict__ a, int64_t lda,
                                                          const float* __restrict__ b, int64_t ldb,
                                                          const float* __restrict__ ga_ext, int64_t ldgae,
                                                          const float* __restrict__ gb_ext, int64_t ldgbe, int64_t n,
                                                          float rate, float reg_coef, float* __restrict__ ga,
                                                          int64_t ldga, float* __restrict__ gb, int64_t ldgb) {
    pdl_wait();
    RowIdx<G, C> ix;
    if (ix.row >= n) return;
    float4 gv[C], xv[C], o[C];
    load_row<G, C>(gv, g, ldg, ix);
    // a
    load_row<G, C>(xv, a, lda, ix);
    normalize_bwd_row<G, C>(o, xv, gv, rate, ix.mask);
#pragma unroll
    for (int c = 0; c < C; ++c) fma4(o[c], reg_coef, xv[c]);
    if (ga_ext != nullptr) {
        float4 ev[C];
        load_row<G, C>(ev, ga_ext, ldgae, ix);
#pragma unroll
        for (int c = 0; c < C; ++c) o[c] = add4(o[c], ev[c]);
    }
    store_row<G, C>(o, ga, ldga, ix);
    // b
    load_row<G, C>(xv, b, ldb, ix);
    normalize_bwd_row<G, C>(o, xv, gv, rate, ix.mask);
#pragma unroll
    for (int c = 0; c < C; ++c) fma4(o[c], reg_coef, xv[c]);
    if (gb_ext != nullptr) {
        float4 ev[C];
        load_row<G, C>(ev, gb_ext, ldgbe, ix);
#pragma unroll
        for (int c = 0; c < C; ++c) o[c] = add4(o[c], ev[c]);
    }
    store_row<G, C>(o, gb, ldgb, ix);
}

template <int G, int C>
__global__ void __launch_bounds__(256) softmax_bwd_kernel(const float* __restrict__ y, int64_t ldy,
                                                          const float* __restrict__ g, int64_t ldg, int64_t n,
                                                          float alpha, float* __restrict__ t, int64_t ldt) {
    pdl_wait();
    RowIdx<G, C> ix;
    if (ix.row >= n) return;
    float4 yv[C], gv[C];
    load_row<G, C>(yv, y, ldy, ix);
    load_row<G, C>(gv, g, ldg, ix);
#pragma unroll
    for (int c = 0; c < C; ++c) gv[c] = scale4(gv[c], alpha);
    const float dot = row_dot<G, C>(yv, gv, ix.mask);
#pragma unroll
    for (int c = 0; c < C; ++c) {
        gv[c].x = yv[c].x * (gv[c].x - dot); gv[c].y = yv[c].y * (gv[c].y - dot);
        gv[c].z = yv[c].z * (gv[c].z - dot); gv[c].w = yv[c].w * (gv[c].w - dot);
    }
    store_row<G, C>(gv, t, ldt, ix);
}

// ---- plain element-wise passes over strided [n, d] matrices (d % 4 == 0) ----
__global__ void axpby_kernel(const float* __restrict__ x, int64_t ldx, int64_t n, int d4, float alpha,
                             const float* __restrict__ alpha_dev, float beta, float* __restrict__ y, int64_t ldy) {
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n * d4) return;
    const int64_t r = i / d4;
    const int c = (int)(i - r * d4) * 4;
    float4 xv = ld4(x + r * ldx + c);
    if (alpha_dev != nullptr) alpha *= *alpha_dev;
    float4 o = scale4(xv, alpha);
    if (beta != 0.f) {
        const float4 yv = ld4(y + r * ldy + c);
        fma4(o, beta, yv);
    }
    st4(y + r * ldy + c, o);
}

__global__ void mul_mask_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ m, int64_t ldm,
                                int64_t n, int d4, float* __restrict__ y, int64_t ldy) {
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n * d4) return;
    const int64_t r = i / d4;
    const int c = (int)(i - r * d4) * 4;
    float4 xv = ld4(x + r * ldx + c);
    if (m != nullptr) {
        const float4 mv = ld4(m + r * ldm + c);
        xv.x *= mv.x; xv.y *= mv.y; xv.z *= mv.z; xv.w *= mv.w;
    }
    st4(y + r * ldy + c, xv);
}

constexpr int kSumsqElemsPerBlock = 256 * 4 * 8;   // 8 float4 per thread
__global__ void __launch_bounds__(256) sumsq_kernel(const float* __restrict__ x, int64_t ldx, int64_t n, int d4,
                                                    float* __restrict__ partials) {
    pdl_wait();
    __shared__ float red[32];
    const int64_t total = n * d4;
    float s = 0.f;
    const int64_t base = blockIdx.x * (int64_t)(256 * 8);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int64_t i = base + k * 256 + threadIdx.x;
        if (i < total) {
            const int64_t r = i / d4;
            const int c = (int)(i - r * d4) * 4;
            const float4 v = ld4(x + r * ldx + c);
            s += dot4(v, v);
        }
    }
    const float tot = block_sum(s, red);
    if (threadIdx.x == 0) partials[blockIdx.x] = tot;
}

// column sums of (g * mask): one block handles a strip of rows, then one atomic per column
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ g, int64_t ldg,
                                                     const float* __restrict__ m, int64_t ldm, int64_t rows, int n,
                                                     int rows_per_block, float* __restrict__ out) {
    pdl_wait();
    extern __shared__ float sm[];   // [256/n_threads_per_row ...] simple: [blockDim.x]
    const int tpr = n;               // threads per row (n <= 256, blockDim.x multiple of n)
    const int rl = threadIdx.x / tpr;
    const int col = threadIdx.x - rl * tpr;
    const int rstep = blockDim.x / tpr;
    const int64_t r0 = blockIdx.x * (int64_t)rows_per_block;
    const int64_t r1 = min(rows, r0 + rows_per_block);
    float s = 0.f;
    for (int64_t r = r0 + rl; r < r1; r += rstep) {
        float v = g[r * ldg + col];
        if (m != nullptr) v *= m[r * ldm + col];
        s += v;
    }
    sm[threadIdx.x] = s;
    __syncthreads();
    if (rl == 0) {
        for (int k = 1; k < rstep; ++k) s += sm[k * tpr + col];
        atomicAdd(out + col, s);
    }
}

static inline unsigned row_blocks(int64_t n, int g) { return (unsigned)((n * g + 255) / 256); }

}  // namespace mmssl

using namespace mmssl;
#define ROW_ALIGN_OK(p, ld) (aligned16(p) && ((ld) % 4 == 0))

extern "C" int mmssl_id_fuse_fwd(const float* z, int64_t ldz, const float* e, int64_t lde, int64_t n, int d, float rate,
                                 float* out, int64_t ldo, float* zn, float* nrm, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE(ROW_ALIGN_OK(z, ldz) && ROW_ALIGN_OK(e, lde) && ROW_ALIGN_OK(out, ldo) && aligned16(zn), "alignment");
    if (n == 0) return 0;
    return dispatch_width(d, [&](auto G, auto C) {
        MMSSL_CUDA_LAUNCH((id_fuse_fwd_kernel<decltype(G)::value, decltype(C)::value>), dim3(row_blocks(n, decltype(G)::value)), dim3(256), 0, st, z, ldz, e, lde, n, rate, out, ldo, zn, nrm);
        MMSSL_LAUNCH_OK();
        return 0;
    }, __func__);
}

extern "C" int mmssl_id_fuse_bwd(const float* g, int64_t ldg, const float* zn, const float* nrm, int64_t n, int d,
                                 float rate, float* dz, int64_t lddz, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE(ROW_ALIGN_OK(g, ldg) && ROW_ALIGN_OK(dz, lddz) && aligned16(zn), "alignment");
    if (n == 0) return 0;
    return dispatch_width(d, [&](auto G, auto C) {
        MMSSL_CUDA_LAUNCH((id_fuse_bwd_kernel<decltype(G)::value, decltype(C)::value>), dim3(row_blocks(n, decltype(G)::value)), dim3(256), 0, st, g, ldg, zn, nrm, n, rate, dz, lddz);
        MMSSL_LAUNCH_OK();
        return 0;
    }, __func__);
}

extern "C" int64_t mmssl_combine_partials(int64_t n, int d) { return (n * width_shape(d).g + 255) / 256; }

extern "C" int mmssl_combine_fwd(const float* s, int64_t lds, const float* a, int64_t lda, const float* b, int64_t ldb,
                                 int64_t n, int d, float inv_layers, float rate, float* out, int64_t ldo,
                                 float* sumsq_partials, int64_t n_partials, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE(ROW_ALIGN_OK(s, lds) && ROW_ALIGN_OK(a, lda) && ROW_ALIGN_OK(b, ldb) && ROW_ALIGN_OK(out, ldo), "alignment");
    MMSSL_REQUIRE(sumsq_partials == nullptr || n_partials >= mmssl_combine_partials(n, d), "sumsq_partials too small");
    if (n == 0) return 0;
    return dispatch_width(d, [&](auto G, auto C) {
        MMSSL_CUDA_LAUNCH((combine_fwd_kernel<decltype(G)::value, decltype(C)::value>), dim3(row_blocks(n, decltype(G)::value)), dim3(256), 0, st, s, lds, a, lda, b, ldb, n, inv_layers,
                                                                                   rate, out, ldo, sumsq_partials);
        MMSSL_LAUNCH_OK();
        return 0;
    }, __func__);
}

extern "C" int mmssl_combine_bwd(const float* g, int64_t ldg, const float* a, int64_t lda, const float* b, int64_t ldb,
                                 const float* ga_ext, int64_t ldgae, const float* gb_ext, int64_t ldgbe, int64_t n, int d,
                                 float rate, float reg_coef, float* ga, int64_t ldga, float* gb, int64_t ldgb,
                                 void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE(ROW_ALIGN_OK(g, ldg) && ROW_ALIGN_OK(a, lda) && ROW_ALIGN_OK(b, ldb) && ROW_ALIGN_OK(ga, ldga) &&
                      ROW_ALIGN_OK(gb, ldgb), "alignment");
    MMSSL_REQUIRE((ga_ext == nullptr || ROW_ALIGN_OK(ga_ext, ldgae)) && (gb_ext == nullptr || ROW_ALIGN_OK(gb_ext, ldgbe)), "alignment");
    if (n == 0) return 0;
    return dispatch_width(d, [&](auto G, auto C) {
        MMSSL_CUDA_LAUNCH((combine_bwd_kernel<decltype(G)::value, decltype(C)::value>), dim3(row_blocks(n, decltype(G)::value)), dim3(256), 0, st, g, ldg, a, lda, b, ldb, ga_ext, ldgae,
                                                                                   gb_ext, ldgbe, n, rate, reg_coef, ga,
                                                                                   ldga, gb, ldgb);
        MMSSL_LAUNCH_OK();
        return 0;
    }, __func__);
}

extern "C" int mmssl_softmax_bwd(const float* y, int64_t ldy, const float* g, int64_t ldg, int64_t n, int d, float alpha,
                                 float* t, int64_t ldt, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE(ROW_ALIGN_OK(y, ldy) && ROW_ALIGN_OK(g, ldg) && ROW_ALIGN_OK(t, ldt), "alignment");
    if (n == 0) return 0;
    return dispatch_width(d, [&](auto G, auto C) {
        MMSSL_CUDA_LAUNCH((softmax_bwd_kernel<decltype(G)::value, decltype(C)::value>), dim3(row_blocks(n, decltype(G)::value)), dim3(256), 0, st, y, ldy, g, ldg, n, alpha, t, ldt);
        MMSSL_LAUNCH_OK();
        return 0;
    }, __func__);
}

extern "C" int mmssl_axpby(const float* x, int64_t ldx, int64_t n, int d, float alpha, const float* alpha_dev, float beta,
                           float* y, int64_t ldy, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE(d % 4 == 0 && ROW_ALIGN_OK(x, ldx) && ROW_ALIGN_OK(y, ldy), "alignment");
    const int64_t tot = n * (d / 4);
    if (tot == 0) return 0;
    MMSSL_CUDA_LAUNCH((axpby_kernel), dim3((unsigned)((tot + 255) / 256)), dim3(256), 0, st, x, ldx, n, d / 4, alpha, alpha_dev, beta, y, ldy);
    MMSSL_LAUNCH_OK();
    return 0;
}

extern "C" int mmssl_mul_mask(const float* x, int64_t ldx, const float* mask, int64_t ldm, int64_t n, int d, float* y,
                              int64_t ldy, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE(d % 4 == 0 && ROW_ALIGN_OK(x, ldx) && ROW_ALIGN_OK(y, ldy) && (mask == nullptr || ROW_ALIGN_OK(mask, ldm)), "alignment");
    const int64_t tot = n * (d / 4);
    if (tot == 0) return 0;
    MMSSL_CUDA_LAUNCH((mul_mask_kernel), dim3((unsigned)((tot + 255) / 256)), dim3(256), 0, st, x, ldx, mask, ldm, n, d / 4, y, ldy);
    MMSSL_LAUNCH_OK();
    return 0;
}

extern "C" int64_t mmssl_sumsq_blocks(int64_t n, int d) { return (n * (d / 4) + 256 * 8 - 1) / (256 * 8); }

extern "C" int mmssl_sumsq(const float* x, int64_t ldx, int64_t n, int d, float* partials, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE(d % 4 == 0 && ROW_ALIGN_OK(x, ldx), "alignment");
    const int64_t blocks = mmssl_sumsq_blocks(n, d);
    if (blocks == 0) return 0;
    MMSSL_CUDA_LAUNCH((sumsq_kernel), dim3((unsigned)blocks), dim3(256), 0, st, x, ldx, n, d / 4, partials);
    MMSSL_LAUNCH_OK();
    return 0;
}

extern "C" int mmssl_colsum(const float* g, int64_t ldg, const float* mask, int64_t ldm, int64_t rows, int n, float* out,
                            int accumulate, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE(n >= 1 && n <= 256, "n must be 1..256");
    if (!accumulate) MMSSL_CUDA(cudaMemsetAsync(out, 0, sizeof(float) * n, st));
    if (rows == 0) return 0;
    const int rows_per_block = 64;
    const unsigned blocks = (unsigned)((rows + rows_per_block - 1) / rows_per_block);
    const unsigned threads = (256 / n) * n;      // a whole number of rows per pass (256 when n divides it; 192 at n = 96)
    MMSSL_CUDA_LAUNCH((colsum_kernel), dim3(blocks), dim3(threads), 256 * sizeof(float), st, g, ldg, mask, ldm, rows, n, rows_per_block, out);
    MMSSL_LAUNCH_OK();
    return 0;
}
