// Fused loss kernels of the MMSSL hot step: BPR (main.py:368-371, :499-511), InfoNCE
// (main.py:211-249) and the final loss assembly (main.py:420 without the GAN term).
// Gather + dot + log-sigmoid / exp-softmax with warp-level reductions; forward value and the
// gradient w.r.t. the embedding tables come out of the same pass (the gradient seeds of the scalar
// losses are read from device scalars so nothing syncs with the host).
#include <cuda_bf16.h>

#include "common.cuh"
#include "../../include/mmssl_b200.h"

namespace mmssl {

constexpr float kNormEps = 1e-12f;

__device__ __forceinline__ void atomic_add4(float* p, const float4& v) {
    atomicAdd(reinterpret_cast<float4*>(p), v);   // sm_90+: one 128-bit reduction
}

// --------------------------------------------------------------------------- BPR
template <int G, int C>
__global__ void __launch_bounds__(256) bpr_kernel(const float* __restrict__ uf, int64_t ldu,
                                                  const float* __restrict__ pf, int64_t ldp,
                                                  const float* __restrict__ nf, int64_t ldn,
                                                  const int64_t* __restrict__ users, const int64_t* __restrict__ pos,
                                                  const int64_t* __restrict__ neg, int64_t batch, int mode,
                                                  float reg_coef, const float* __restrict__ g_mf,
                                                  const float* __restrict__ g_emb, float* __restrict__ part,
                                                  float* __restrict__ g_u, int64_t ldgu, float* __restrict__ g_p,
                                                  int64_t ldgp, float* __restrict__ g_n, int64_t ldgn) {
    pdl_wait();
    __shared__ float red[2][32];
    const unsigned mask = group_mask<G>();
    const int lane = threadIdx.x & (G - 1);
    const int64_t k = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / G;
    float sp = 0.f, rg = 0.f;
    if (k < batch) {
        const int64_t iu = users ? users[k] : k, ip = pos ? pos[k] : k, in_ = neg ? neg[k] : k;
        float4 u[C], p[C], n[C];
        float dpn = 0.f, ss = 0.f;
#pragma unroll
        for (int c = 0; c < C; ++c) {
            const int col = lane * 4 + c * 4 * G;
            u[c] = ld4(uf + iu * ldu + col);
            p[c] = ld4(pf + ip * ldp + col);
            n[c] = ld4(nf + in_ * ldn + col);
            const float4 df = make_float4(p[c].x - n[c].x, p[c].y - n[c].y, p[c].z - n[c].z, p[c].w - n[c].w);
            dpn += dot4(u[c], df);
            ss += dot4(u[c], u[c]) + dot4(p[c], p[c]) + dot4(n[c], n[c]);
        }
        const float x = group_sum<G>(dpn, mask);   // pos_score - neg_score
        ss = group_sum<G>(ss, mask);
        if (lane == 0) {
            sp = fmaxf(-x, 0.f) + log1pf(expf(-fabsf(x)));   // -logsigmoid(x)
            rg = 0.5f * ss;
        }
        if (mode & 2) {
            const float gm = g_mf ? *g_mf : 1.f;
            const float ge = g_emb ? *g_emb : 1.f;
            const float sig = 1.f / (1.f + expf(x));   // sigmoid(-x)
            const float dx = -sig * gm / (float)batch;
            const float wr = ge * reg_coef;
#pragma unroll
            for (int c = 0; c < C; ++c) {
                const int col = lane * 4 + c * 4 * G;
                float4 gu, gp, gn;
                gu.x = dx * (p[c].x - n[c].x) + wr * u[c].x; gu.y = dx * (p[c].y - n[c].y) + wr * u[c].y;
                gu.z = dx * (p[c].z - n[c].z) + wr * u[c].z; gu.w = dx * (p[c].w - n[c].w) + wr * u[c].w;
                gp.x = dx * u[c].x + wr * p[c].x; gp.y = dx * u[c].y + wr * p[c].y;
                gp.z = dx * u[c].z + wr * p[c].z; gp.w = dx * u[c].w + wr * p[c].w;
                gn.x = -dx * u[c].x + wr * n[c].x; gn.y = -dx * u[c].y + wr * n[c].y;
                gn.z = -dx * u[c].z + wr * n[c].z; gn.w = -dx * u[c].w + wr * n[c].w;
                if (users) atomic_add4(g_u + iu * ldgu + col, gu); else st4(g_u + iu * ldgu + col, add4(ld4(g_u + iu * ldgu + col), gu));
                if (pos) atomic_add4(g_p + ip * ldgp + col, gp); else st4(g_p + ip * ldgp + col, add4(ld4(g_p + ip * ldgp + col), gp));
                if (neg) atomic_add4(g_n + in_ * ldgn + col, gn); else st4(g_n + in_ * ldgn + col, add4(ld4(g_n + in_ * ldgn + col), gn));
            }
        }
    }
    if (mode & 1) {
        const float a = block_sum(sp, red[0]);
        const float b = block_sum(rg, red[1]);
        if (threadIdx.x == 0) { part[2 * blockIdx.x] = a; part[2 * blockIdx.x + 1] = b; }
    }
}

// --------------------------------------------------------------------------- InfoNCE
template <int G, int C>
__global__ void __launch_bounds__(256) nce_prepare_kernel(const float* __restrict__ z1, int64_t ldz1,
                                                          const float* __restrict__ z2, int64_t ldz2,
                                                          const int64_t* __restrict__ idx, int64_t n,
                                                          float* __restrict__ a, float* __restrict__ b,
                                                          float* __restrict__ na, float* __restrict__ nb,
                                                          float* __restrict__ ga, float* __restrict__ gb,
                                                          uint16_t* __restrict__ a_hi = nullptr, uint16_t* __restrict__ a_lo = nullptr,
                                                          uint16_t* __restrict__ b_hi = nullptr, uint16_t* __restrict__ b_lo = nullptr) {
    pdl_wait();
    const unsigned mask = group_mask<G>();
    const int lane = threadIdx.x & (G - 1);
    const int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / G;
    if (i >= n) return;
    const int64_t src = idx ? idx[i] : i;
    const int d = 4 * G * C;
    float4 v[C], w[C];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int c = 0; c < C; ++c) {
        const int col = lane * 4 + c * 4 * G;
        v[c] = ld4(z1 + src * ldz1 + col);
        w[c] = ld4(z2 + src * ldz2 + col);
        s1 += dot4(v[c], v[c]);
        s2 += dot4(w[c], w[c]);
    }
    const float n1 = sqrtf(group_sum<G>(s1, mask)), n2 = sqrtf(group_sum<G>(s2, mask));
    const float i1 = 1.f / fmaxf(n1, kNormEps), i2 = 1.f / fmaxf(n2, kNormEps);
#pragma unroll
    for (int c = 0; c < C; ++c) {
        const int col = lane * 4 + c * 4 * G;
        const float4 av = scale4(v[c], i1), bv = scale4(w[c], i2);
        st4(a + i * d + col, av);
        st4(b + i * d + col, bv);
        if (ga) st4(ga + i * d + col, f4zero());
        if (gb) st4(gb + i * d + col, f4zero());
        if (a_hi) {     // bf16 hi / lo operands of the tensor-core path (loss_tc.cu), [n][d] K-major
            auto split4 = [](const float4& x, uint16_t* hi, uint16_t* lo) {
                const float xs[4] = {x.x, x.y, x.z, x.w};
                uint16_t h[4], l[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const __nv_bfloat16 hb = __float2bfloat16_rn(xs[q]);
                    h[q] = __bfloat16_as_ushort(hb);
                    l[q] = __bfloat16_as_ushort(__float2bfloat16_rn(xs[q] - __bfloat162float(hb)));
                }
                *reinterpret_cast<uint2*>(hi) = make_uint2((uint32_t)h[0] | ((uint32_t)h[1] << 16), (uint32_t)h[2] | ((uint32_t)h[3] << 16));
                *reinterpret_cast<uint2*>(lo) = make_uint2((uint32_t)l[0] | ((uint32_t)l[1] << 16), (uint32_t)l[2] | ((uint32_t)l[3] << 16));
            };
            split4(av, a_hi + i * d + col, a_lo + i * d + col);
            split4(bv, b_hi + i * d + col, b_lo + i * d + col);
        }
    }
    if (lane == 0) { na[i] = n1; nb[i] = n2; }
}

constexpr int NT = 64;          // tile edge
constexpr int NS = NT + 4;      // smem row stride: float4-aligned rows, conflict-free 128-bit column access
// 256 threads = 16 (ty) x 16 (tx).  Shared-memory traffic is what bounds these tiles, so every operand
// is read with 128-bit loads along its contiguous axis (4 reduction steps per load).

// RAGGED: d is not a multiple of NT (d = 32, 96, 192), so the last chunk of the d axis sticks out past d and is zero-filled;
// off, the chunks tile d exactly and the instance compiles to the code it had before the flag existed.
template <bool RAGGED>
__device__ __forceinline__ void load_tile(float* sm, const float* __restrict__ src, int64_t row0, int64_t n, int d,
                                          int c0) {
    // sm[r][k] = src[(row0+r)*d + c0 + k], r,k < 64 (zero beyond n, and beyond d when RAGGED)
    for (int e = threadIdx.x; e < NT * (NT / 4); e += 256) {
        const int r = e / (NT / 4), k4 = (e % (NT / 4)) * 4;
        float4 v = f4zero();
        if (row0 + r < n && (!RAGGED || c0 + k4 < d)) v = ld4(src + (row0 + r) * (int64_t)d + c0 + k4);
        *reinterpret_cast<float4*>(sm + r * NS + k4) = v;
    }
}

// acc[ii][jj] += sum_k X[ty*4+ii][k] * Y[tx+16*jj][k]      (rows ty*4+ii, columns tx+16*jj)
__device__ __forceinline__ void tile_nt(float (&acc)[4][4], const float* X, const float* Y, int ty, int tx) {
#pragma unroll 4
    for (int k = 0; k < NT; k += 4) {
        float4 xv[4], yv[4];
#pragma unroll
        for (int ii = 0; ii < 4; ++ii) xv[ii] = *reinterpret_cast<const float4*>(X + (ty * 4 + ii) * NS + k);
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) yv[jj] = *reinterpret_cast<const float4*>(Y + (tx + 16 * jj) * NS + k);
#pragma unroll
        for (int ii = 0; ii < 4; ++ii)
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) acc[ii][jj] += dot4(xv[ii], yv[jj]);
    }
}
// acc[ii][jj] += sum_j P[ty*4+ii][j] * V[j][tx*4+jj]       (rows ty*4+ii, columns tx*4+jj)
__device__ __forceinline__ void tile_nn(float (&acc)[4][4], const float* P, const float* V, int ty, int tx) {
#pragma unroll 2
    for (int j = 0; j < NT; j += 4) {
        float4 pv[4];
#pragma unroll
        for (int ii = 0; ii < 4; ++ii) pv[ii] = *reinterpret_cast<const float4*>(P + (ty * 4 + ii) * NS + j);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float4 v = *reinterpret_cast<const float4*>(V + (j + q) * NS + tx * 4);
#pragma unroll
            for (int ii = 0; ii < 4; ++ii) {
                const float pq = q == 0 ? pv[ii].x : (q == 1 ? pv[ii].y : (q == 2 ? pv[ii].z : pv[ii].w));
                acc[ii][0] = fmaf(pq, v.x, acc[ii][0]); acc[ii][1] = fmaf(pq, v.y, acc[ii][1]);
                acc[ii][2] = fmaf(pq, v.z, acc[ii][2]); acc[ii][3] = fmaf(pq, v.w, acc[ii][3]);
            }
        }
    }
}
// acc[ii][jj] += sum_i Q[i][ty*4+ii] * V[i][tx*4+jj]       (rows ty*4+ii, columns tx*4+jj)
__device__ __forceinline__ void tile_tn(float (&acc)[4][4], const float* Q, const float* V, int ty, int tx) {
#pragma unroll 4
    for (int i = 0; i < NT; ++i) {
        const float4 q = *reinterpret_cast<const float4*>(Q + i * NS + ty * 4);
        const float4 v = *reinterpret_cast<const float4*>(V + i * NS + tx * 4);
        const float qv[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int ii = 0; ii < 4; ++ii) {
            acc[ii][0] = fmaf(qv[ii], v.x, acc[ii][0]); acc[ii][1] = fmaf(qv[ii], v.y, acc[ii][1]);
            acc[ii][2] = fmaf(qv[ii], v.z, acc[ii][2]); acc[ii][3] = fmaf(qv[ii], v.w, acc[ii][3]);
        }
    }
}

// stats layout: [diagR n][diagB n][loss n][unused n][partR ntj*n][partB ntj*n]
template <bool RAGGED>
__global__ void __launch_bounds__(256) nce_stats_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                        int64_t n, int d, float inv_tau, float* __restrict__ stats) {
    pdl_wait();
    extern __shared__ float sm[];
    float* Ai = sm; float* Aj = sm + NT * NS; float* Bj = sm + 2 * NT * NS;
    const int ty = threadIdx.x / 16, tx = threadIdx.x % 16;
    const int64_t i0 = blockIdx.x * (int64_t)NT, j0 = blockIdx.y * (int64_t)NT;
    float sr[4][4] = {}, sb[4][4] = {};
    for (int c0 = 0; c0 < d; c0 += NT) {
        load_tile<RAGGED>(Ai, a, i0, n, d, c0);
        load_tile<RAGGED>(Aj, a, j0, n, d, c0);
        load_tile<RAGGED>(Bj, b, j0, n, d, c0);
        __syncthreads();
        tile_nt(sr, Ai, Aj, ty, tx);
        tile_nt(sb, Ai, Bj, ty, tx);
        __syncthreads();
    }
    const int64_t ntj = gridDim.y;
    float* diag_r = stats; float* diag_b = stats + n;
    float* part_r = stats + 4 * n + blockIdx.y * n;
    float* part_b = stats + 4 * n + ntj * n + blockIdx.y * n;
#pragma unroll
    for (int ii = 0; ii < 4; ++ii) {
        const int64_t i = i0 + ty * 4 + ii;
        float rr = 0.f, rb = 0.f;
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
            const int64_t j = j0 + tx + 16 * jj;
            if (i < n && j < n) {
                const float er = expf(sr[ii][jj] * inv_tau), eb = expf(sb[ii][jj] * inv_tau);
                rr += er; rb += eb;
                if (i == j) { diag_r[i] = er; diag_b[i] = eb; }
            }
        }
        // the 16 threads sharing `ty` are 16 consecutive lanes
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) {
            rr += __shfl_xor_sync(0xffffffffu, rr, o, 16);
            rb += __shfl_xor_sync(0xffffffffu, rb, o, 16);
        }
        if (tx == 0 && i < n) { part_r[i] = rr; part_b[i] = rb; }
    }
}

__global__ void __launch_bounds__(256) nce_finalize_kernel(int64_t n, int64_t ntj, float* __restrict__ stats,
                                                           float* __restrict__ coef, const float* __restrict__ g_loss,
                                                           float* __restrict__ loss_part) {
    pdl_wait();
    __shared__ float red[32];
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    float li = 0.f;
    if (i < n) {
        float sr = 0.f, sb = 0.f;
        int64_t t = 0;
        for (; t + 4 <= ntj; t += 4) {      // independent loads first, fixed summation order
            float r_[4], b_[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) { r_[q] = stats[4 * n + (t + q) * n + i]; b_[q] = stats[4 * n + ntj * n + (t + q) * n + i]; }
#pragma unroll
            for (int q = 0; q < 4; ++q) { sr += r_[q]; sb += b_[q]; }
        }
        for (; t < ntj; ++t) {
            sr += stats[4 * n + t * n + i];
            sb += stats[4 * n + ntj * n + t * n + i];
        }
        const float dr = stats[i], db = stats[n + i];
        const float den = sr + sb - dr;
        const float r = db / den;
        li = -logf(r + 1e-8f);
        stats[2 * n + i] = li;
        const float g = (g_loss ? *g_loss : 1.f) / (float)n;
        const float w = -g / (r + 1e-8f);     // d total / d r_i
        coef[i] = w * r / den;                // u_i : -dL/dR_ij (j != i) and -dL/dB_ij
        coef[n + i] = w / den;                // v_i : extra dL/dB_ii
    }
    const float tot = block_sum(li, red);
    if (threadIdx.x == 0) loss_part[blockIdx.x] = tot;
}

template <bool RAGGED>
__global__ void __launch_bounds__(256) nce_grad_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                       int64_t n, int d, float inv_tau, const float* __restrict__ coef,
                                                       float* __restrict__ ga, float* __restrict__ gb) {
    pdl_wait();
    extern __shared__ float sm[];
    float* Ai = sm; float* Aj = sm + NT * NS; float* Bj = sm + 2 * NT * NS;
    float* P = sm + 3 * NT * NS; float* Q = sm + 4 * NT * NS;
    const int ty = threadIdx.x / 16, tx = threadIdx.x % 16;
    const int64_t i0 = blockIdx.x * (int64_t)NT, j0 = blockIdx.y * (int64_t)NT;
    float sr[4][4] = {}, sb[4][4] = {};
    for (int c0 = 0; c0 < d; c0 += NT) {
        load_tile<RAGGED>(Ai, a, i0, n, d, c0);
        load_tile<RAGGED>(Aj, a, j0, n, d, c0);
        load_tile<RAGGED>(Bj, b, j0, n, d, c0);
        __syncthreads();
        tile_nt(sr, Ai, Aj, ty, tx);
        tile_nt(sb, Ai, Bj, ty, tx);
        __syncthreads();
    }
    // coefficient tiles:  P_ij = -(u_i+u_j) R_ij / tau (i != j),   Q_ij = B_ij (-u_i + [i==j] v_i) / tau
#pragma unroll
    for (int ii = 0; ii < 4; ++ii) {
        const int64_t i = i0 + ty * 4 + ii;
        const float ui = (i < n) ? coef[i] : 0.f;
        const float vi = (i < n) ? coef[n + i] : 0.f;
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
            const int64_t j = j0 + tx + 16 * jj;
            float pv = 0.f, qv = 0.f;
            if (i < n && j < n) {
                const float uj = coef[j];
                const float er = expf(sr[ii][jj] * inv_tau), eb = expf(sb[ii][jj] * inv_tau);
                pv = (i == j) ? 0.f : -(ui + uj) * er * inv_tau;
                qv = eb * (-ui + ((i == j) ? vi : 0.f)) * inv_tau;
            }
            P[(ty * 4 + ii) * NS + tx + 16 * jj] = pv;
            Q[(ty * 4 + ii) * NS + tx + 16 * jj] = qv;
        }
    }
    __syncthreads();
    for (int c0 = 0; c0 < d; c0 += NT) {
        if (d > NT) {   // tiles of the first chunk pass are gone when d has several chunks
            load_tile<RAGGED>(Ai, a, i0, n, d, c0);
            load_tile<RAGGED>(Aj, a, j0, n, d, c0);
            load_tile<RAGGED>(Bj, b, j0, n, d, c0);
            __syncthreads();
        }
        float g1[4][4] = {}, g2[4][4] = {};
        tile_nn(g1, P, Aj, ty, tx);     // dL/da_i  += sum_j P_ij a_j
        tile_nn(g1, Q, Bj, ty, tx);     //           + sum_j Q_ij b_j
        tile_tn(g2, Q, Ai, ty, tx);     // dL/db_j  += sum_i Q_ij a_i
#pragma unroll
        for (int ii = 0; ii < 4; ++ii) {
            const int64_t i = i0 + ty * 4 + ii, j = j0 + ty * 4 + ii;
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
                const int c = c0 + tx * 4 + jj;
                if (RAGGED && c >= d) continue;
                if (i < n) atomicAdd(ga + i * d + c, g1[ii][jj]);
                if (j < n) atomicAdd(gb + j * d + c, g2[ii][jj]);
            }
        }
        __syncthreads();
    }
}

template <int G, int C>
__global__ void __launch_bounds__(256) nce_scatter_kernel(const float* __restrict__ ga, const float* __restrict__ gb,
                                                          const float* __restrict__ a, const float* __restrict__ b,
                                                          const float* __restrict__ na, const float* __restrict__ nb,
                                                          const int64_t* __restrict__ idx, int64_t n,
                                                          float* __restrict__ g_z1, int64_t ldg1,
                                                          float* __restrict__ g_z2, int64_t ldg2) {
    pdl_wait();
    const unsigned mask = group_mask<G>();
    const int lane = threadIdx.x & (G - 1);
    const int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / G;
    if (i >= n) return;
    const int64_t dst = idx ? idx[i] : i;
    const int d = 4 * G * C;
#pragma unroll
    for (int which = 0; which < 2; ++which) {
        const float* gsrc = which ? gb : ga;
        const float* xn = which ? b : a;
        const float nr = which ? nb[i] : na[i];
        float* out = which ? g_z2 : g_z1;
        const int64_t ldo = which ? ldg2 : ldg1;
        if (out == nullptr) continue;
        float4 g[C], x[C];
        float dot = 0.f;
#pragma unroll
        for (int c = 0; c < C; ++c) {
            const int col = lane * 4 + c * 4 * G;
            g[c] = ld4(gsrc + i * d + col);
            x[c] = ld4(xn + i * d + col);
            dot += dot4(g[c], x[c]);
        }
        dot = group_sum<G>(dot, mask);
#pragma unroll
        for (int c = 0; c < C; ++c) {
            const int col = lane * 4 + c * 4 * G;
            float4 o;
            if (nr > kNormEps) {
                const float k = 1.f / nr;
                o.x = k * (g[c].x - x[c].x * dot); o.y = k * (g[c].y - x[c].y * dot);
                o.z = k * (g[c].z - x[c].z * dot); o.w = k * (g[c].w - x[c].w * dot);
            } else {
                o = scale4(g[c], 1.f / kNormEps);
            }
            if (idx) atomic_add4(out + dst * ldo + col, o);
            else st4(out + dst * ldo + col, add4(ld4(out + dst * ldo + col), o));
        }
    }
}

// --------------------------------------------------------------------------- loss assembly
__device__ float ordered_sum(const float* p, int64_t n, float* red) {
    // fixed association: thread t sums p[t], p[t+1024], ... then a block tree -> deterministic
    float s = 0.f;
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) s += p[i];
    s = block_sum(s, red);
    __shared__ float bc;
    if (threadIdx.x == 0) bc = s;
    __syncthreads();
    const float r = bc;
    __syncthreads();
    return r;
}
__global__ void __launch_bounds__(1024) loss_assemble_kernel(const float* bpr_part, int64_t n_bpr, int64_t batch,
                                                             float reg_coef, const float* fr_u, int64_t n_fr_u,
                                                             const float* fr_i, int64_t n_fr_i, float feat_coef,
                                                             const float* nce1, int64_t n_nce1, const float* nce2,
                                                             int64_t n_nce2, int64_t n_nce_rows, float cl_rate,
                                                             float* out5) {
    pdl_wait();
    __shared__ float red[32];
    float mf = 0.f, emb = 0.f;
    {
        float a = 0.f, b = 0.f;
        for (int64_t i = threadIdx.x; i < n_bpr; i += blockDim.x) { a += bpr_part[2 * i]; b += bpr_part[2 * i + 1]; }
        a = block_sum(a, red);
        __shared__ float s0, s1;
        if (threadIdx.x == 0) s0 = a;
        __syncthreads();
        b = block_sum(b, red);
        if (threadIdx.x == 0) s1 = b;
        __syncthreads();
        mf = (batch > 0) ? s0 / (float)batch : 0.f;
        emb = reg_coef * s1;
        __syncthreads();
    }
    const float fu = fr_u ? ordered_sum(fr_u, n_fr_u, red) : 0.f;
    const float fi = fr_i ? ordered_sum(fr_i, n_fr_i, red) : 0.f;
    const float c1 = nce1 ? ordered_sum(nce1, n_nce1, red) : 0.f;
    const float c2 = nce2 ? ordered_sum(nce2, n_nce2, red) : 0.f;
    if (threadIdx.x == 0) {
        const float feat = feat_coef * (fu + fi);
        const float cl = (n_nce_rows > 0) ? (c1 + c2) / (float)n_nce_rows : 0.f;
        out5[0] = mf + emb + feat + cl_rate * cl;
        out5[1] = mf; out5[2] = emb; out5[3] = feat; out5[4] = cl;
    }
}

}  // namespace mmssl

using namespace mmssl;
#define GV(x) decltype(x)::value

extern "C" int64_t mmssl_bpr_blocks(int64_t batch, int d) { return (batch * width_shape(d).g + 255) / 256; }

extern "C" int mmssl_bpr(const float* uf, int64_t ldu, const float* itf, int64_t ldi, const float* itf_neg, int64_t ldin,
                         const int64_t* users, const int64_t* pos, const int64_t* neg, int64_t batch, int d, int mode,
                         float reg_coef, const float* g_mf, const float* g_emb, float* part, float* g_uf, int64_t ldgu,
                         float* g_pos, int64_t ldgp, float* g_neg, int64_t ldgn, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE(uf && itf && itf_neg, "null table");
    MMSSL_REQUIRE(aligned16(uf) && aligned16(itf) && aligned16(itf_neg) && ldu % 4 == 0 && ldi % 4 == 0 && ldin % 4 == 0, "alignment");
    MMSSL_REQUIRE(!(mode & 1) || part, "mode bit 0 needs the partials buffer");
    MMSSL_REQUIRE(!(mode & 2) || (g_uf && g_pos && g_neg && aligned16(g_uf) && aligned16(g_pos) && aligned16(g_neg) &&
                                  ldgu % 4 == 0 && ldgp % 4 == 0 && ldgn % 4 == 0), "mode bit 1 needs gradient buffers");
    if (batch == 0) return 0;
    return dispatch_width(d, [&](auto G, auto C) {
        const unsigned blocks = (unsigned)mmssl_bpr_blocks(batch, d);
        MMSSL_CUDA_LAUNCH((bpr_kernel<GV(G), GV(C)>), dim3(blocks), dim3(256), 0, st, uf, ldu, itf, ldi, itf_neg, ldin, users, pos, neg, batch, mode,
                                                         reg_coef, g_mf, g_emb, part, g_uf, ldgu, g_pos, ldgp, g_neg, ldgn);
        MMSSL_LAUNCH_OK();
        return 0;
    }, __func__);
}

extern "C" int mmssl_infonce_prepare(const float* z1, int64_t ldz1, const float* z2, int64_t ldz2, const int64_t* idx,
                                     int64_t n, int d, float* a, float* b, float* na, float* nb, float* ga, float* gb,
                                     void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE(aligned16(z1) && aligned16(z2) && ldz1 % 4 == 0 && ldz2 % 4 == 0 && aligned16(a) && aligned16(b), "alignment");
    if (n == 0) return 0;
    return dispatch_width(d, [&](auto G, auto C) {
        const unsigned blocks = (unsigned)((n * GV(G) + 255) / 256);
        MMSSL_CUDA_LAUNCH((nce_prepare_kernel<GV(G), GV(C)>), dim3(blocks), dim3(256), 0, st, z1, ldz1, z2, ldz2, idx, n, a, b, na, nb, ga, gb,
                          (uint16_t*)nullptr, (uint16_t*)nullptr, (uint16_t*)nullptr, (uint16_t*)nullptr);
        MMSSL_LAUNCH_OK();
        return 0;
    }, __func__);
}

// [diagR n][diagB n][loss n][unused n][partR ntj*n][partB ntj*n]; ntj <= ceil(n / 64) + 1 (the tensor-core path uses 2 per 128-tile)
extern "C" int64_t mmssl_infonce_stats_floats(int64_t n) { return 4 * n + 2 * n * ((n + NT - 1) / NT + 1); }
extern "C" int64_t mmssl_infonce_loss_blocks(int64_t n) { return (n + 255) / 256; }

template <bool RAGGED>
static int nce_smem_attr() {
    static bool done = false;
    if (done) return 0;
    MMSSL_CUDA(cudaFuncSetAttribute(nce_stats_kernel<RAGGED>, cudaFuncAttributeMaxDynamicSharedMemorySize, 3 * NT * NS * 4));
    MMSSL_CUDA(cudaFuncSetAttribute(nce_grad_kernel<RAGGED>, cudaFuncAttributeMaxDynamicSharedMemorySize, 5 * NT * NS * 4));
    done = true;
    return 0;
}

extern "C" int mmssl_infonce_stats(const float* a, const float* b, int64_t n, int d, float inv_tau, float* stats,
                                   float* coef, const float* g_loss, float* loss_part, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE(d > 0 && d % 4 == 0, "d must be a positive multiple of 4");
    if (n == 0) return 0;
    const bool ragged = d % NT != 0;
    if (int rc = ragged ? nce_smem_attr<true>() : nce_smem_attr<false>()) return rc;
    const unsigned nt = (unsigned)((n + NT - 1) / NT);
    MMSSL_REQUIRE(nt <= 65535, "batch too large for one InfoNCE call");
    if (ragged) MMSSL_CUDA_LAUNCH((nce_stats_kernel<true>), dim3(dim3(nt, nt)), dim3(256), 3 * NT * NS * 4, st, a, b, n, d, inv_tau, stats);
    else MMSSL_CUDA_LAUNCH((nce_stats_kernel<false>), dim3(dim3(nt, nt)), dim3(256), 3 * NT * NS * 4, st, a, b, n, d, inv_tau, stats);
    MMSSL_LAUNCH_OK();
    MMSSL_CUDA_LAUNCH((nce_finalize_kernel), dim3((unsigned)mmssl_infonce_loss_blocks(n)), dim3(256), 0, st, n, nt, stats, coef, g_loss, loss_part);
    MMSSL_LAUNCH_OK();
    return 0;
}

namespace mmssl {
// nce_prepare + bf16 hi / lo split of the normalised rows in one launch (tensor-core path, loss_tc.cu); ga / gb are not zeroed
// there (the tensor-core backward writes them)
int nce_prepare_split_launch(const float* z1, int64_t ldz1, const float* z2, int64_t ldz2, const int64_t* idx, int64_t n, int d, float* a,
                             float* b, float* na, float* nb, uint16_t* a_hi, uint16_t* a_lo, uint16_t* b_hi, uint16_t* b_lo, cudaStream_t st) {
    MMSSL_REQUIRE(aligned16(z1) && aligned16(z2) && ldz1 % 4 == 0 && ldz2 % 4 == 0 && aligned16(a) && aligned16(b), "alignment");
    if (n == 0) return 0;
    return dispatch_width(d, [&](auto G, auto C) {
        const unsigned blocks = (unsigned)((n * GV(G) + 255) / 256);
        MMSSL_CUDA_LAUNCH((nce_prepare_kernel<GV(G), GV(C)>), dim3(blocks), dim3(256), 0, st, z1, ldz1, z2, ldz2, idx, n, a, b, na, nb,
                          (float*)nullptr, (float*)nullptr, a_hi, a_lo, b_hi, b_lo);
        MMSSL_LAUNCH_OK();
        return 0;
    }, __func__);
}

// loss rows + backward coefficients from the row sums of `ntj` column tiles (used by the tensor-core path, loss_tc.cu)
int nce_finalize_launch(int64_t n, int64_t ntj, float* stats, float* coef, const float* g_loss, float* loss_part, cudaStream_t st) {
    MMSSL_CUDA_LAUNCH((nce_finalize_kernel), dim3((unsigned)mmssl_infonce_loss_blocks(n)), dim3(256), 0, st, n, ntj, stats, coef, g_loss, loss_part);
    MMSSL_LAUNCH_OK();
    return 0;
}
}  // namespace mmssl

extern "C" int mmssl_infonce_grad(const float* a, const float* b, int64_t n, int d, float inv_tau, const float* coef,
                                  float* ga, float* gb, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE(d > 0 && d % 4 == 0, "d must be a positive multiple of 4");
    if (n == 0) return 0;
    const bool ragged = d % NT != 0;
    if (int rc = ragged ? nce_smem_attr<true>() : nce_smem_attr<false>()) return rc;
    const unsigned nt = (unsigned)((n + NT - 1) / NT);
    MMSSL_REQUIRE(nt <= 65535, "batch too large for one InfoNCE call");
    if (ragged) MMSSL_CUDA_LAUNCH((nce_grad_kernel<true>), dim3(dim3(nt, nt)), dim3(256), 5 * NT * NS * 4, st, a, b, n, d, inv_tau, coef, ga, gb);
    else MMSSL_CUDA_LAUNCH((nce_grad_kernel<false>), dim3(dim3(nt, nt)), dim3(256), 5 * NT * NS * 4, st, a, b, n, d, inv_tau, coef, ga, gb);
    MMSSL_LAUNCH_OK();
    return 0;
}

extern "C" int mmssl_infonce_scatter(const float* ga, const float* gb, const float* a, const float* b, const float* na,
                                     const float* nb, const int64_t* idx, int64_t n, int d, float* g_z1, int64_t ldg1,
                                     float* g_z2, int64_t ldg2, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE((g_z1 == nullptr || (aligned16(g_z1) && ldg1 % 4 == 0)) && (g_z2 == nullptr || (aligned16(g_z2) && ldg2 % 4 == 0)), "alignment");
    if (n == 0) return 0;
    return dispatch_width(d, [&](auto G, auto C) {
        const unsigned blocks = (unsigned)((n * GV(G) + 255) / 256);
        MMSSL_CUDA_LAUNCH((nce_scatter_kernel<GV(G), GV(C)>), dim3(blocks), dim3(256), 0, st, ga, gb, a, b, na, nb, idx, n, g_z1, ldg1, g_z2, ldg2);
        MMSSL_LAUNCH_OK();
        return 0;
    }, __func__);
}

extern "C" int mmssl_loss_assemble(const float* bpr_part, int64_t n_bpr_blocks, int64_t batch, float reg_coef,
                                   const float* fr_u, int64_t n_fr_u, const float* fr_i, int64_t n_fr_i, float feat_coef,
                                   const float* nce1, int64_t n_nce1, const float* nce2, int64_t n_nce2,
                                   int64_t n_nce_rows, float cl_rate, float* out5, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE(out5 != nullptr, "null output");
    MMSSL_CUDA_LAUNCH((loss_assemble_kernel), dim3(1), dim3(1024), 0, st, bpr_part ? bpr_part : out5, bpr_part ? n_bpr_blocks : 0, batch, reg_coef,
                                             fr_u, n_fr_u, fr_i, n_fr_i, feat_coef, nce1, n_nce1, nce2, n_nce2,
                                             n_nce_rows, cl_rate, out5);
    MMSSL_LAUNCH_OK();
    return 0;
}
