// Fused id-fusion kernels (reference Models.py:139-169 "attention" closed form + :188-197):
//   forward : m = coef*(Ya [+ Yb]) ; z = m * Wsum ; out = E + rate * z / max(|z|, eps)
//   backward: dz = rate * d(normalize)(g) ; dY = coef * dz * Wsum^T (+ external grads) ;
//             dWsum += m^T dz  (one partial tile per block, reduced in a fixed order)
// with Wsum = sum_h Wcat[h*d:(h+1)*d, :]  (SURVEY appendix B.1) and dWcat[h] = dWsum for every head.
//
// Each block owns a tile of TR = 32 or 64 rows and runs register-tiled (4x4 per thread) products against the
// d x d matrix staged in shared memory, with the row-wise normalisation / its backward fused as
// prologue / epilogue.  (A first version walked rows one by one and re-read the whole matrix from
// shared memory per row: shared-memory-bandwidth bound.)
// Shared memory is 24 KB per block at d = 64 (matrix 16 KB + one 8 KB row tile; the backward keeps its second tile in the
// matrix's place until the matrix is needed): these kernels run beside the projection GEMMs, whose two ~97 KB CTAs leave ~30 KB
// of an SM -- with 32 / 48 KB blocks they would wait for the GEMM to drain.
#include <cstdlib>

#include "common.cuh"
#include "../../include/mmssl_b200.h"

namespace mmssl {

constexpr float kNormEps = 1e-12f;
// rows per block tile TR (template parameter): 32 for tables under kSmallRows rows (latency-bound: more, smaller blocks; 24 KB of
// shared memory at d = 64), 64 above (throughput-bound: half as many matrix reloads and partial dWsum tiles -- at 1M rows, d = 128
// the 32-row tiles cost 2 GB more of partial-tile traffic).  threads = (TR / 4) (ty: rows ty*4..+3) x 16 (tx: columns)
constexpr int64_t kSmallRows = 100000;
__host__ __device__ constexpr int tile_rows(int64_t n) { return n < kSmallRows ? 32 : 64; }

// wsum[k][c] = sum_h wcat[h][k][c] ; wsum_t[c][k] = the same transposed
__global__ void wsum_kernel(const float* __restrict__ wcat, int d, int heads, float* __restrict__ wsum,
                            float* __restrict__ wsum_t) {
    pdl_wait();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= d * d) return;
    float s = 0.f;
    for (int h = 0; h < heads; ++h) s += wcat[(int64_t)h * d * d + i];
    wsum[i] = s;
    const int k = i / d, c = i - k * d;
    wsum_t[c * d + k] = s;
}

// acc[i][cc][j] += sum_k A[ty*4+i][k] * B[k][cc*64 + tx*4 + j]   (A: [TR][D] smem, B: [D][D] smem)
template <int D>
__device__ __forceinline__ void tile_mm(float (&acc)[4][D / 64][4], const float* __restrict__ A,
                                        const float* __restrict__ B, int ty, int tx) {
#pragma unroll 4
    for (int k = 0; k < D; ++k) {
        float a[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) a[i] = A[(ty * 4 + i) * D + k];
#pragma unroll
        for (int cc = 0; cc < D / 64; ++cc) {
            const float4 b = *reinterpret_cast<const float4*>(B + k * D + cc * 64 + tx * 4);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                acc[i][cc][0] = fmaf(a[i], b.x, acc[i][cc][0]); acc[i][cc][1] = fmaf(a[i], b.y, acc[i][cc][1]);
                acc[i][cc][2] = fmaf(a[i], b.z, acc[i][cc][2]); acc[i][cc][3] = fmaf(a[i], b.w, acc[i][cc][3]);
            }
        }
    }
}

// sum over the 16 threads (tx) that share a row
__device__ __forceinline__ float row16_sum(float v) {
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o, 16);
    return v;
}

template <int D, int TR>
__global__ void __launch_bounds__(TR * 4) id_fuse2_fwd_kernel(const float* __restrict__ ya, int64_t lda,
                                                           const float* __restrict__ yb, int64_t ldb, float coef,
                                                           const float* __restrict__ wsum, const float* __restrict__ e,
                                                           int64_t lde, int64_t n, float rate, float* __restrict__ out,
                                                           int64_t ldo, float* __restrict__ zn, float* __restrict__ nrm) {
    pdl_wait();
    constexpr int NT = TR * 4;
    extern __shared__ __align__(16) float sm[];
    float* Ws = sm;              // [D][D]
    float* Ms = sm + D * D;      // [TR][D]
    const int64_t r0 = blockIdx.x * (int64_t)TR;
    for (int i = threadIdx.x; i < D * D / 4; i += NT)
        reinterpret_cast<float4*>(Ws)[i] = __ldg(reinterpret_cast<const float4*>(wsum) + i);
    for (int i = threadIdx.x; i < TR * D / 4; i += NT) {
        const int r = i / (D / 4), c = (i - r * (D / 4)) * 4;
        float4 m = f4zero();
        if (r0 + r < n) {
            m = ld4(ya + (r0 + r) * lda + c);
            if (yb != nullptr) m = add4(m, ld4(yb + (r0 + r) * ldb + c));
            m = scale4(m, coef);
        }
        *reinterpret_cast<float4*>(Ms + r * D + c) = m;
    }
    __syncthreads();
    const int ty = threadIdx.x / 16, tx = threadIdx.x % 16;
    float acc[4][D / 64][4] = {};
    tile_mm<D>(acc, Ms, Ws, ty, tx);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float ss = 0.f;
#pragma unroll
        for (int cc = 0; cc < D / 64; ++cc)
#pragma unroll
            for (int j = 0; j < 4; ++j) ss = fmaf(acc[i][cc][j], acc[i][cc][j], ss);
        ss = row16_sum(ss);
        const float nr = sqrtf(ss);
        const float inv = 1.f / fmaxf(nr, kNormEps);
        const int64_t row = r0 + ty * 4 + i;
        if (row < n) {
#pragma unroll
            for (int cc = 0; cc < D / 64; ++cc) {
                const int c = cc * 64 + tx * 4;
                const float4 z = make_float4(acc[i][cc][0] * inv, acc[i][cc][1] * inv, acc[i][cc][2] * inv, acc[i][cc][3] * inv);
                float4 o = ld4(e + row * lde + c);
                fma4(o, rate, z);
                st4(out + row * ldo + c, o);
                st4(zn + row * D + c, z);
            }
            if (tx == 0) nrm[row] = nr;
        }
    }
}

template <int D, int TR>
__global__ void __launch_bounds__(TR * 4) id_fuse2_bwd_kernel(const float* __restrict__ g, int64_t ldg,
                                                          const float* __restrict__ zn, const float* __restrict__ nrm,
                                                          const float* __restrict__ ya, int64_t lda,
                                                          const float* __restrict__ yb, int64_t ldb, float coef,
                                                          const float* __restrict__ wsum_t, int64_t n, float rate,
                                                          const float* __restrict__ ext_a, int64_t ldea,
                                                          const float* __restrict__ ext_b, int64_t ldeb,
                                                          float* __restrict__ out_a, int64_t ldoa,
                                                          float* __restrict__ out_b, int64_t ldob,
                                                          float* __restrict__ dw_part) {
    pdl_wait();
    constexpr int NTY = TR / 4, NT = TR * 4;
    extern __shared__ __align__(16) float sm[];
    float* Zs = sm;                   // [TR][D]  dz rows
    float* Xs = sm + TR * D;          // first [TR][D] m rows (dWsum product), then [D][D]: Wt[c][k] = Wsum[k][c] (dY product)
    float* Ms = Xs;
    float* Wt = Xs;
    const int64_t r0 = blockIdx.x * (int64_t)TR;
    // dz (normalize backward) and m, one 16-lane group per row: lane owns float4 slices c = cc*64 + tx*4
    const int ty = threadIdx.x / 16, tx = threadIdx.x % 16;
    for (int rl = ty; rl < TR; rl += NTY) {
        const int64_t row = r0 + rl;
        float4 gv[D / 64], nv[D / 64];
        float dot = 0.f;
        const bool on = row < n;
#pragma unroll
        for (int cc = 0; cc < D / 64; ++cc) {
            const int c = cc * 64 + tx * 4;
            gv[cc] = on ? ld4(g + row * ldg + c) : f4zero();
            nv[cc] = on ? ld4(zn + row * D + c) : f4zero();
            dot += dot4(gv[cc], nv[cc]);
        }
        dot = row16_sum(dot);
        const float nr = on ? nrm[row] : 1.f;
#pragma unroll
        for (int cc = 0; cc < D / 64; ++cc) {
            const int c = cc * 64 + tx * 4;
            float4 dz;
            if (nr > kNormEps) {
                const float k = rate / nr;
                dz = make_float4(k * (gv[cc].x - nv[cc].x * dot), k * (gv[cc].y - nv[cc].y * dot),
                                 k * (gv[cc].z - nv[cc].z * dot), k * (gv[cc].w - nv[cc].w * dot));
            } else {
                dz = scale4(gv[cc], rate / kNormEps);
            }
            float4 m = f4zero();
            if (on) {
                m = ld4(ya + row * lda + c);
                if (yb != nullptr) m = add4(m, ld4(yb + row * ldb + c));
                m = scale4(m, coef);
            }
            *reinterpret_cast<float4*>(Zs + rl * D + c) = dz;
            *reinterpret_cast<float4*>(Ms + rl * D + c) = m;
        }
    }
    __syncthreads();
    // partial dWsum tile = M^T DZ : thread owns k = kc*TR + ty*4 + i, c = cc*64 + tx*4 + j
    float* part = dw_part + (int64_t)blockIdx.x * D * D;
#pragma unroll 1
    for (int kc = 0; kc < D / TR; ++kc) {
        float acc[4][D / 64][4] = {};
#pragma unroll 4
        for (int r = 0; r < TR; ++r) {
            const float4 a = *reinterpret_cast<const float4*>(Ms + r * D + kc * TR + ty * 4);
            const float av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
            for (int cc = 0; cc < D / 64; ++cc) {
                const float4 b = *reinterpret_cast<const float4*>(Zs + r * D + cc * 64 + tx * 4);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    acc[i][cc][0] = fmaf(av[i], b.x, acc[i][cc][0]); acc[i][cc][1] = fmaf(av[i], b.y, acc[i][cc][1]);
                    acc[i][cc][2] = fmaf(av[i], b.z, acc[i][cc][2]); acc[i][cc][3] = fmaf(av[i], b.w, acc[i][cc][3]);
                }
            }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int cc = 0; cc < D / 64; ++cc)
                st4(part + (kc * TR + ty * 4 + i) * D + cc * 64 + tx * 4,
                    make_float4(acc[i][cc][0], acc[i][cc][1], acc[i][cc][2], acc[i][cc][3]));
    }
    __syncthreads();                  // every thread is done with the m rows: the matrix takes their place
    for (int i = threadIdx.x; i < D * D / 4; i += NT)
        reinterpret_cast<float4*>(Wt)[i] = __ldg(reinterpret_cast<const float4*>(wsum_t) + i);
    __syncthreads();
    // dY tile = coef * DZ * Wsum^T
    {
        float acc[4][D / 64][4] = {};
        tile_mm<D>(acc, Zs, Wt, ty, tx);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int64_t row = r0 + ty * 4 + i;
            if (row >= n) continue;
#pragma unroll
            for (int cc = 0; cc < D / 64; ++cc) {
                const int c = cc * 64 + tx * 4;
                const float4 dy = make_float4(coef * acc[i][cc][0], coef * acc[i][cc][1], coef * acc[i][cc][2], coef * acc[i][cc][3]);
                float4 da = dy, db = dy;
                if (ext_a) da = add4(da, ld4(ext_a + row * ldea + c));
                if (out_b == nullptr) {
                    if (ext_b) da = add4(da, ld4(ext_b + row * ldeb + c));
                    st4(out_a + row * ldoa + c, da);
                } else {
                    if (ext_b) db = add4(db, ld4(ext_b + row * ldeb + c));
                    st4(out_a + row * ldoa + c, da);
                    st4(out_b + row * ldob + c, db);
                }
            }
        }
    }
}

// dWcat[h*d*d + i] = sum over the partial tiles of both sides (fixed order), for every head h.
// block = 32 outputs x 32 slices of the partial-tile list (a slice walks its ~26 tiles of Baby's 829 in batches of 8 independent
// loads); slices are combined in order.  (A first version used 64 outputs x 4 slices: 13 dependent batches per thread.)
constexpr int kRedOut = 32, kRedSlices = 32;
__global__ void __launch_bounds__(kRedOut * kRedSlices) dwcat_reduce_kernel(const float* __restrict__ part_u, int nu,
                                                                            const float* __restrict__ part_i, int ni, int d, int heads,
                                                                            float* __restrict__ dwcat) {
    pdl_wait();
    __shared__ float red[kRedSlices][kRedOut];
    const int o = threadIdx.x % kRedOut, sl = threadIdx.x / kRedOut;
    const int i = blockIdx.x * kRedOut + o;
    const int64_t dd = (int64_t)d * d;
    const int nt = nu + ni;
    const int per = (nt + kRedSlices - 1) / kRedSlices;
    const int b0 = min(nt, sl * per), b1 = min(nt, b0 + per);
    float s = 0.f;
    if (i < dd) {
        int b = b0;
        for (; b + 8 <= b1; b += 8) {
            float v[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const int t = b + q;
                v[q] = (t < nu) ? part_u[t * dd + i] : part_i[(t - nu) * dd + i];
            }
#pragma unroll
            for (int q = 0; q < 8; ++q) s += v[q];
        }
        for (; b < b1; ++b) s += (b < nu) ? part_u[b * dd + i] : part_i[(b - nu) * dd + i];
    }
    red[sl][o] = s;
    __syncthreads();
    if (sl == 0 && i < dd) {
        float tot = red[0][o];
#pragma unroll
        for (int q = 1; q < kRedSlices; ++q) tot += red[q][o];
        for (int h = 0; h < heads; ++h) dwcat[h * dd + i] = tot;
    }
}

}  // namespace mmssl

using namespace mmssl;

extern "C" int mmssl_wsum(const float* wcat, int d, int heads, float* wsum, float* wsum_t, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_CUDA_LAUNCH((wsum_kernel), dim3((d * d + 255) / 256), dim3(256), 0, st, wcat, d, heads, wsum, wsum_t);
    MMSSL_LAUNCH_OK();
    return 0;
}

static int idfuse_carveout() {          // percent of the SM's L1 / shared array; MMSSL_IDFUSE_CARVEOUT: experiment knob
    const char* e = getenv("MMSSL_IDFUSE_CARVEOUT");       // (asking for the GEMMs' configuration, 100, changed nothing on the earlier hardware)
    return e ? atoi(e) : (int)cudaSharedmemCarveoutDefault;
}

extern "C" int mmssl_id_fuse2_blocks(int64_t n) { return (int)((n + tile_rows(n) - 1) / tile_rows(n)); }

template <int D, int TR>
static int launch_fwd_t(const float* ya, int64_t lda, const float* yb, int64_t ldb, float coef, const float* wsum,
                      const float* e, int64_t lde, int64_t n, float rate, float* out, int64_t ldo, float* zn, float* nrm,
                      cudaStream_t st) {
    const int smem = (D * D + TR * D) * 4;
    static bool attr = false;
    if (!attr) {
        MMSSL_CUDA(cudaFuncSetAttribute(id_fuse2_fwd_kernel<D, TR>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        MMSSL_CUDA(cudaFuncSetAttribute(id_fuse2_fwd_kernel<D, TR>, cudaFuncAttributePreferredSharedMemoryCarveout, idfuse_carveout()));
        attr = true;
    }
    MMSSL_CUDA_LAUNCH((id_fuse2_fwd_kernel<D, TR>), dim3((unsigned)((n + TR - 1) / TR)), dim3(TR * 4), smem, st, ya, lda, yb, ldb, coef, wsum, e, lde, n, rate, out, ldo, zn, nrm);
    MMSSL_LAUNCH_OK();
    return 0;
}

template <int D>
static int launch_fwd(const float* ya, int64_t lda, const float* yb, int64_t ldb, float coef, const float* wsum,
                      const float* e, int64_t lde, int64_t n, float rate, float* out, int64_t ldo, float* zn, float* nrm,
                      cudaStream_t st) {
    if (tile_rows(n) == 32) return launch_fwd_t<D, 32>(ya, lda, yb, ldb, coef, wsum, e, lde, n, rate, out, ldo, zn, nrm, st);
    return launch_fwd_t<D, 64>(ya, lda, yb, ldb, coef, wsum, e, lde, n, rate, out, ldo, zn, nrm, st);
}

extern "C" int mmssl_id_fuse2_fwd(const float* ya, int64_t lda, const float* yb, int64_t ldb, float coef, const float* wsum,
                                  const float* e, int64_t lde, int64_t n, int d, float rate, float* out, int64_t ldo,
                                  float* zn, float* nrm, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE(d == 64 || d == 128, "fused id-fusion supports d = 64 or 128 (d = 256 uses the GEMM path)");
    MMSSL_REQUIRE(aligned16(ya) && lda % 4 == 0 && (yb == nullptr || (aligned16(yb) && ldb % 4 == 0)) && aligned16(e) &&
                      lde % 4 == 0 && aligned16(out) && ldo % 4 == 0 && aligned16(zn) && aligned16(wsum), "alignment");
    if (n == 0) return 0;
    if (d == 64) return launch_fwd<64>(ya, lda, yb, ldb, coef, wsum, e, lde, n, rate, out, ldo, zn, nrm, st);
    return launch_fwd<128>(ya, lda, yb, ldb, coef, wsum, e, lde, n, rate, out, ldo, zn, nrm, st);
}

template <int D, int TR>
static int launch_bwd_t(const float* g, int64_t ldg, const float* zn, const float* nrm, const float* ya, int64_t lda,
                      const float* yb, int64_t ldb, float coef, const float* wsum_t, int64_t n, float rate, const float* ext_a,
                      int64_t ldea, const float* ext_b, int64_t ldeb, float* out_a, int64_t ldoa, float* out_b, int64_t ldob,
                      float* dw_part, cudaStream_t st) {
    const int smem = (TR * D + (D * D > TR * D ? D * D : TR * D)) * 4;
    static bool attr = false;
    if (!attr) {
        MMSSL_CUDA(cudaFuncSetAttribute(id_fuse2_bwd_kernel<D, TR>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        MMSSL_CUDA(cudaFuncSetAttribute(id_fuse2_bwd_kernel<D, TR>, cudaFuncAttributePreferredSharedMemoryCarveout, idfuse_carveout()));
        attr = true;
    }
    MMSSL_CUDA_LAUNCH((id_fuse2_bwd_kernel<D, TR>), dim3((unsigned)((n + TR - 1) / TR)), dim3(TR * 4), smem, st, g, ldg, zn, nrm, ya, lda, yb, ldb, coef, wsum_t, n, rate,
                                                                            ext_a, ldea, ext_b, ldeb, out_a, ldoa, out_b, ldob, dw_part);
    MMSSL_LAUNCH_OK();
    return 0;
}

template <int D>
static int launch_bwd(const float* g, int64_t ldg, const float* zn, const float* nrm, const float* ya, int64_t lda,
                      const float* yb, int64_t ldb, float coef, const float* wsum_t, int64_t n, float rate, const float* ext_a,
                      int64_t ldea, const float* ext_b, int64_t ldeb, float* out_a, int64_t ldoa, float* out_b, int64_t ldob,
                      float* dw_part, cudaStream_t st) {
    if (tile_rows(n) == 32)
        return launch_bwd_t<D, 32>(g, ldg, zn, nrm, ya, lda, yb, ldb, coef, wsum_t, n, rate, ext_a, ldea, ext_b, ldeb, out_a, ldoa, out_b, ldob, dw_part, st);
    return launch_bwd_t<D, 64>(g, ldg, zn, nrm, ya, lda, yb, ldb, coef, wsum_t, n, rate, ext_a, ldea, ext_b, ldeb, out_a, ldoa, out_b, ldob, dw_part, st);
}

extern "C" int mmssl_id_fuse2_bwd(const float* g, int64_t ldg, const float* zn, const float* nrm, const float* ya,
                                  int64_t lda, const float* yb, int64_t ldb, float coef, const float* wsum_t, int64_t n, int d,
                                  float rate, const float* ext_a, int64_t ldea, const float* ext_b, int64_t ldeb,
                                  float* out_a, int64_t ldoa, float* out_b, int64_t ldob, float* dw_part, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE(d == 64 || d == 128, "fused id-fusion supports d = 64 or 128 (d = 256 uses the GEMM path)");
    MMSSL_REQUIRE(aligned16(g) && ldg % 4 == 0 && aligned16(zn) && aligned16(ya) && lda % 4 == 0 && aligned16(out_a) &&
                      ldoa % 4 == 0 && aligned16(dw_part) && aligned16(wsum_t), "alignment");
    MMSSL_REQUIRE((yb == nullptr || (aligned16(yb) && ldb % 4 == 0)) && (ext_a == nullptr || (aligned16(ext_a) && ldea % 4 == 0)) &&
                      (ext_b == nullptr || (aligned16(ext_b) && ldeb % 4 == 0)) && (out_b == nullptr || (aligned16(out_b) && ldob % 4 == 0)), "alignment");
    if (n == 0) return 0;
    if (d == 64)
        return launch_bwd<64>(g, ldg, zn, nrm, ya, lda, yb, ldb, coef, wsum_t, n, rate, ext_a, ldea, ext_b, ldeb, out_a, ldoa, out_b, ldob, dw_part, st);
    return launch_bwd<128>(g, ldg, zn, nrm, ya, lda, yb, ldb, coef, wsum_t, n, rate, ext_a, ldea, ext_b, ldeb, out_a, ldoa, out_b, ldob, dw_part, st);
}

extern "C" int mmssl_dwcat_reduce(const float* part_u, int nu, const float* part_i, int ni, int d, int heads, float* dwcat,
                                  void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_CUDA_LAUNCH((dwcat_reduce_kernel), dim3((d * d + kRedOut - 1) / kRedOut), dim3(kRedOut * kRedSlices), 0, st, part_u, nu, part_i, ni, d, heads, dwcat);
    MMSSL_LAUNCH_OK();
    return 0;
}
