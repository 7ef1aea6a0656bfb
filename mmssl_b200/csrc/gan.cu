// GAN side of the reference's training step -- SURVEY section 8f "next" row 2.  The device ops that
// mmssl_b200/gan.py sequences (one entry point == one op of tests/gan_ops_cpu.py, which is their specification):
//   Discriminator (Models.py:224-245): training-mode BatchNorm1d + dropout forward / backward, the sigmoid head,
//   the second-order sweep of gradient_penalty (main.py:140-160) through the batch statistics,
//   u_sim_calculation (main.py:283-298) masking + row normalisation and its backward,
//   the Gumbel-perturbed "real" rows (main.py:348-351), the interpolation of the penalty.
// The GEMMs between them go through the library's GEMM entry points.  All of this is HBM-bound reduction work on
// [2B, I/4], [2B, I/8] and [B, I] fp32 tiles (I/4 is not a multiple of 4 in general, so loads are scalar and coalesced
// along the row).  Two kernel shapes:
//   * column ops  -- CTA = 8 columns x 32 row lanes (h = I/4 = 1762 at Baby gives 221 CTAs: the 132 SMs are covered, which a
//                    32-column CTA would not do); a column's statistics are reduced in a fixed order (deterministic);
//                    multi-pass kernels re-read their 8-column stripe from L2.
//   * row ops     -- one CTA (256 threads) or one warp per row, block reductions in a fixed order.
#include "common.cuh"
#include "../../include/mmssl_b200.h"

namespace mmssl {

constexpr int kCT = 8;    // columns per CTA: 8 consecutive floats = one 32-byte sector per row
constexpr int kRL = 32;   // row lanes per CTA (a warp covers 4 rows x 8 columns: 4 full sectors per load instruction)
constexpr float kBnEps = 1e-5f, kBnMomentum = 0.1f;

// Sum over the kRL row lanes of every column; every thread of the column gets the result.
__device__ __forceinline__ float col_reduce(float v, float (*sh)[kCT]) {
    sh[threadIdx.y][threadIdx.x] = v;
    __syncthreads();
    float s = 0.f;
#pragma unroll
    for (int y = 0; y < kRL; ++y) s += sh[y][threadIdx.x];
    __syncthreads();
    return s;
}

// Block-wide (256 threads, 1-D) reductions whose result every thread receives.
__device__ __forceinline__ float block_sum_all(float v, float* sh33) {
    v = warp_sum(v);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();                       // sh33 may still be read from a previous call
    if (l == 0) sh33[w] = v;
    __syncthreads();
    if (w == 0) {
        float t = l < (int)(blockDim.x >> 5) ? sh33[l] : 0.f;
        t = warp_sum(t);
        if (l == 0) sh33[32] = t;
    }
    __syncthreads();
    return sh33[32];
}
__device__ __forceinline__ float block_max_all(float v, float* sh33) {
    v = group_max<32>(v, 0xffffffffu);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) sh33[w] = v;
    __syncthreads();
    if (w == 0) {
        float t = l < (int)(blockDim.x >> 5) ? sh33[l] : -INFINITY;
        t = group_max<32>(t, 0xffffffffu);
        if (l == 0) sh33[32] = t;
    }
    __syncthreads();
    return sh33[32];
}

// ------------------------------------------------------------------------------------------ column ops
__global__ void __launch_bounds__(kCT* kRL) bn_fwd_kernel(const float* __restrict__ a, const float* __restrict__ bias,
                                                          const float* __restrict__ gamma, const float* __restrict__ beta,
                                                          const float* __restrict__ mask, float* __restrict__ rmean,
                                                          float* __restrict__ rvar, int64_t n, int64_t h, float* __restrict__ hout,
                                                          float* __restrict__ ah, float* __restrict__ rout) {
    __shared__ float sh[kRL][kCT];
    const int64_t col = (int64_t)blockIdx.x * kCT + threadIdx.x;
    const bool ok = col < h;
    // The column is summed shifted by its row-0 value k0: a column whose mean is far above its spread loses no digits to the
    // running sum (fp32 sums of 1e3-sized values are off by far more than the spread's last bits), and a constant column
    // gives exactly zero deviations, var = 0.
    const float k0 = ok ? a[col] : 0.f;
    float s = 0.f;
    if (ok) for (int64_t r = threadIdx.y; r < n; r += kRL) s += a[r * h + col] - k0;
    const float ms = col_reduce(s, sh) / (float)n;                   // mean - k0
    s = 0.f;
    if (ok) for (int64_t r = threadIdx.y; r < n; r += kRL) { const float d = (a[r * h + col] - k0) - ms; s = fmaf(d, d, s); }
    const float var = col_reduce(s, sh) / (float)n;
    const float rs = 1.0f / sqrtf(var + kBnEps);
    if (!ok) return;
    const float g = gamma[col], b = beta[col];
    for (int64_t r = threadIdx.y; r < n; r += kRL) {
        const float x = ((a[r * h + col] - k0) - ms) * rs;
        ah[r * h + col] = x;
        hout[r * h + col] = fmaf(x, g, b) * mask[r * h + col];
    }
    if (threadIdx.y == 0) {
        rout[col] = rs;
        rmean[col] = (1.f - kBnMomentum) * rmean[col] + kBnMomentum * ((k0 + ms) + bias[col]);
        rvar[col] = (1.f - kBnMomentum) * rvar[col] + kBnMomentum * var * ((float)n / (float)(n - 1));
    }
}

__global__ void __launch_bounds__(kCT* kRL) bn_bwd_kernel(const float* __restrict__ dh, const float* __restrict__ mask,
                                                          const float* __restrict__ gamma, const float* __restrict__ ah,
                                                          const float* __restrict__ rstd, int64_t n, int64_t h, float* __restrict__ da,
                                                          float* __restrict__ dy, float* __restrict__ dgamma, float* __restrict__ dbeta) {
    __shared__ float sh[kRL][kCT];
    const int64_t col = (int64_t)blockIdx.x * kCT + threadIdx.x;
    const bool ok = col < h;
    float s1 = 0.f, s2 = 0.f;
    if (ok) for (int64_t r = threadIdx.y; r < n; r += kRL) {
        const float v = dh[r * h + col] * mask[r * h + col];
        dy[r * h + col] = v;
        s1 += v;
        s2 = fmaf(v, ah[r * h + col], s2);
    }
    const float S1 = col_reduce(s1, sh), S2 = col_reduce(s2, sh);
    if (!ok) return;
    const float g = gamma[col], rs = rstd[col];
    const float m = g * S1 / (float)n, cm = g * S2 / (float)n;
    for (int64_t r = threadIdx.y; r < n; r += kRL) da[r * h + col] = rs * (dy[r * h + col] * g - m - ah[r * h + col] * cm);
    if (threadIdx.y == 0) { dgamma[col] = S2; dbeta[col] = S1; }
}

// Adjoint of bn_bwd (see tests/gan_ops_cpu.py:gp_rev_bn, oracle/gan_oracle.py:rev_bn_bwd).
__global__ void __launch_bounds__(kCT* kRL) gp_rev_bn_kernel(const float* __restrict__ q, const float* __restrict__ dy,
                                                             const float* __restrict__ ah, const float* __restrict__ rstd,
                                                             const float* __restrict__ gamma, const float* __restrict__ mask,
                                                             int64_t n, int64_t h, float* __restrict__ dh_bar, float* __restrict__ ah_bar,
                                                             float* __restrict__ r_bar, float* __restrict__ g_gamma) {
    __shared__ float sh[kRL][kCT];
    const int64_t col = (int64_t)blockIdx.x * kCT + threadIdx.x;
    const bool ok = col < h;
    const float g = ok ? gamma[col] : 0.f, rs = ok ? rstd[col] : 0.f;
    float s1 = 0.f, s2 = 0.f;
    if (ok) for (int64_t r = threadIdx.y; r < n; r += kRL) {
        const float dah = dy[r * h + col] * g;
        s1 += dah;
        s2 = fmaf(dah, ah[r * h + col], s2);
    }
    const float m = col_reduce(s1, sh) / (float)n, cm = col_reduce(s2, sh) / (float)n;
    float t1 = 0.f, t2 = 0.f, t3 = 0.f;
    if (ok) for (int64_t r = threadIdx.y; r < n; r += kRL) {
        const float x = ah[r * h + col], dah = dy[r * h + col] * g, qq = q[r * h + col];
        const float u = dah - m - x * cm;
        const float ub = qq * rs;
        t1 = fmaf(qq, u, t1);
        t2 += ub;
        t3 = fmaf(ub, x, t3);
    }
    const float RB = col_reduce(t1, sh), ubm = col_reduce(t2, sh) / (float)n, c_bar = -col_reduce(t3, sh) / (float)n;
    float t4 = 0.f;
    if (ok) for (int64_t r = threadIdx.y; r < n; r += kRL) {
        const float x = ah[r * h + col], v = dy[r * h + col], dah = v * g, ub = q[r * h + col] * rs;
        const float dah_bar = ub - ubm + c_bar * x;
        ah_bar[r * h + col] = c_bar * dah - ub * cm;
        dh_bar[r * h + col] = dah_bar * g * mask[r * h + col];
        t4 = fmaf(dah_bar, v, t4);
    }
    const float GG = col_reduce(t4, sh);
    if (ok && threadIdx.y == 0) { r_bar[col] = RB; g_gamma[col] = GG; }
}

// Adjoint of bn_fwd with the extra adjoints of ah and r (tests/gan_ops_cpu.py:bn_fwd_rev).
__global__ void __launch_bounds__(kCT* kRL) bn_fwd_rev_kernel(const float* __restrict__ h_bar, const float* __restrict__ mask,
                                                              const float* __restrict__ gamma, const float* __restrict__ ah,
                                                              const float* __restrict__ rstd, const float* __restrict__ ah_bar,
                                                              const float* __restrict__ r_bar, int64_t n, int64_t h,
                                                              float* __restrict__ a_bar, float* __restrict__ g_gamma,
                                                              float* __restrict__ g_beta) {
    __shared__ float sh[kRL][kCT];
    const int64_t col = (int64_t)blockIdx.x * kCT + threadIdx.x;
    const bool ok = col < h;
    const float g = ok ? gamma[col] : 0.f;
    float s1 = 0.f, s2 = 0.f, s3 = 0.f, s4 = 0.f;
    if (ok) for (int64_t r = threadIdx.y; r < n; r += kRL) {
        const float x = ah[r * h + col], yb = h_bar[r * h + col] * mask[r * h + col];
        const float tot = ah_bar[r * h + col] + yb * g;
        s1 = fmaf(yb, x, s1);
        s2 += yb;
        s3 += tot;
        s4 = fmaf(tot, x, s4);
    }
    const float GG = col_reduce(s1, sh), GB = col_reduce(s2, sh);
    const float mt = col_reduce(s3, sh) / (float)n, mta = col_reduce(s4, sh) / (float)n;
    if (!ok) return;
    const float rs = rstd[col];
    const float extra = r_bar[col] * rs * rs / (float)n;
    for (int64_t r = threadIdx.y; r < n; r += kRL) {
        const float x = ah[r * h + col], yb = h_bar[r * h + col] * mask[r * h + col];
        const float tot = ah_bar[r * h + col] + yb * g;
        a_bar[r * h + col] = rs * (tot - mt - x * mta) - extra * x;
    }
    if (threadIdx.y == 0) { g_gamma[col] = GG; g_beta[col] = GB; }
}

__global__ void __launch_bounds__(kCT* kRL) colsum_any_kernel(const float* __restrict__ x, int64_t n, int64_t h, float* __restrict__ out) {
    __shared__ float sh[kRL][kCT];
    const int64_t col = (int64_t)blockIdx.x * kCT + threadIdx.x;
    float s = 0.f;
    if (col < h) for (int64_t r = threadIdx.y; r < n; r += kRL) s += x[r * h + col];
    s = col_reduce(s, sh);
    if (col < h && threadIdx.y == 0) out[col] = s;
}

// Head backward: dz = 100 s (1-s) coef ; dh2 = dz (x) w3 ; dw3 = sum_rows dz * h2 ; db3 = sum dz.
__global__ void __launch_bounds__(kCT* kRL) head_bwd_kernel(const float* __restrict__ s, float coef, const float* __restrict__ w3,
                                                            const float* __restrict__ h2, int64_t n, int64_t h, float* __restrict__ dh2,
                                                            float* __restrict__ dz_out, float* __restrict__ dw3, float* __restrict__ db3) {
    __shared__ float sh[kRL][kCT];
    const int64_t col = (int64_t)blockIdx.x * kCT + threadIdx.x;
    const bool ok = col < h;
    const float w = ok ? w3[col] : 0.f;
    float acc = 0.f;
    if (ok) for (int64_t r = threadIdx.y; r < n; r += kRL) {
        const float sv = s[r], dz = 100.f * sv * (1.f - sv) * coef;
        dh2[r * h + col] = dz * w;
        acc = fmaf(dz, h2[r * h + col], acc);
    }
    acc = col_reduce(acc, sh);
    if (ok && threadIdx.y == 0) dw3[col] = acc;
    if (blockIdx.x == 0) {                                  // the per-row vector and its sum, once
        const int tid = threadIdx.y * kCT + threadIdx.x;
        float t = 0.f;
        for (int64_t r = tid; r < n; r += kCT * kRL) {
            const float sv = s[r], dz = 100.f * sv * (1.f - sv) * coef;
            dz_out[r] = dz;
            t += dz;
        }
        t = col_reduce(t, sh);                              // per threadIdx.x partial over the row lanes ...
        if (threadIdx.y == 0) sh[0][threadIdx.x] = t;       // ... then over the kCT column slots, fixed order
        __syncthreads();
        if (tid == 0) {
            float tot = 0.f;
#pragma unroll
            for (int x = 0; x < kCT; ++x) tot += sh[0][x];
            db3[0] = tot;
        }
    }
}

// gp_head_rev, column part: h_bar = z_bar (x) w3 ; g_w3 = sum_rows dz * dh2_bar + z_bar * h2 ; g_b3 = sum z_bar.
__global__ void __launch_bounds__(kCT* kRL) gp_head_rev_cols_kernel(const float* __restrict__ dh2_bar, const float* __restrict__ dz,
                                                                    const float* __restrict__ z_bar, const float* __restrict__ w3,
                                                                    const float* __restrict__ h2, int64_t n, int64_t h,
                                                                    float* __restrict__ h_bar, float* __restrict__ g_w3,
                                                                    float* __restrict__ g_b3) {
    __shared__ float sh[kRL][kCT];
    const int64_t col = (int64_t)blockIdx.x * kCT + threadIdx.x;
    const bool ok = col < h;
    const float w = ok ? w3[col] : 0.f;
    float acc = 0.f;
    if (ok) for (int64_t r = threadIdx.y; r < n; r += kRL) {
        const float zb = z_bar[r];
        h_bar[r * h + col] = zb * w;
        acc = fmaf(dz[r], dh2_bar[r * h + col], acc);
        acc = fmaf(zb, h2[r * h + col], acc);
    }
    acc = col_reduce(acc, sh);
    if (ok && threadIdx.y == 0) g_w3[col] = acc;
    if (blockIdx.x == 0) {
        const int tid = threadIdx.y * kCT + threadIdx.x;
        float t = 0.f;
        for (int64_t r = tid; r < n; r += kCT * kRL) t += z_bar[r];
        t = col_reduce(t, sh);
        if (threadIdx.y == 0) sh[0][threadIdx.x] = t;
        __syncthreads();
        if (tid == 0) {
            float tot = 0.f;
#pragma unroll
            for (int x = 0; x < kCT; ++x) tot += sh[0][x];
            g_b3[0] = tot;
        }
    }
}

// ------------------------------------------------------------------------------------------ warp-per-row ops
// s = sigmoid(h2 . w3 + b3)
__global__ void __launch_bounds__(256) head_fwd_kernel(const float* __restrict__ h2, const float* __restrict__ w3,
                                                       const float* __restrict__ b3, int64_t n, int64_t h, float* __restrict__ s) {
    const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= n) return;                                   // warp-uniform
    float acc = 0.f;
    for (int64_t c = lane; c < h; c += 32) acc = fmaf(h2[row * h + c], w3[c], acc);
    acc = warp_sum(acc);
    if (lane == 0) s[row] = 1.f / (1.f + expf(-(acc + b3[0])));
}
// z_bar = (dh2_bar . w3) * 100 (1 - 2s) * s (1 - s)
__global__ void __launch_bounds__(256) gp_head_rev_rows_kernel(const float* __restrict__ dh2_bar, const float* __restrict__ w3,
                                                               const float* __restrict__ s, int64_t n, int64_t h, float* __restrict__ z_bar) {
    const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= n) return;
    float acc = 0.f;
    for (int64_t c = lane; c < h; c += 32) acc = fmaf(dh2_bar[row * h + c], w3[c], acc);
    acc = warp_sum(acc);
    if (lane == 0) { const float sv = s[row]; z_bar[row] = acc * 100.f * (1.f - 2.f * sv) * sv * (1.f - sv); }
}
// out[0] = scale * sum(x[0..n))   (one CTA, fixed order)
__global__ void __launch_bounds__(256) vec_sum_kernel(const float* __restrict__ x, int64_t n, float scale, float* __restrict__ out) {
    __shared__ float sh[33];
    float t = 0.f;
    for (int64_t i = threadIdx.x; i < n; i += 256) t += x[i];
    t = block_sum_all(t, sh);
    if (threadIdx.x == 0) out[0] = t * scale;
}

// ------------------------------------------------------------------------------------------ CTA-per-row ops
// gbar = (2 lam / n) (norm - 1) / norm * gx ; sq[row] = (norm - 1)^2.  A row with norm 0 (every head of the batch saturated
// in fp32, so d out / d x is exactly 0) gets torch's norm backward: a zero gradient, not (-inf) * 0 = NaN; it still adds 1 to sq.
__global__ void __launch_bounds__(256) gp_rows_kernel(const float* __restrict__ gx, int64_t n, int64_t w, float lam,
                                                      float* __restrict__ gbar, float* __restrict__ sq) {
    __shared__ float sh[33];
    const int64_t row = blockIdx.x;
    float t = 0.f;
    for (int64_t c = threadIdx.x; c < w; c += 256) { const float v = gx[row * w + c]; t = fmaf(v, v, t); }
    const float norm = sqrtf(block_sum_all(t, sh));
    const float f = norm > 0.f ? (2.f * lam / (float)n) * (norm - 1.f) / norm : 0.f;
    for (int64_t c = threadIdx.x; c < w; c += 256) gbar[row * w + c] = f * gx[row * w + c];
    if (threadIdx.x == 0) sq[row] = (norm - 1.f) * (norm - 1.f);
}

// y = normalize(scores with the user's training items zeroed), nrm = the row norm (clamped at 1e-12)
__global__ void __launch_bounds__(256) usim_finish_kernel(const float* __restrict__ scores, const int64_t* __restrict__ users,
                                                          const int64_t* __restrict__ indptr, const int64_t* __restrict__ indices,
                                                          int64_t w, float* __restrict__ y, float* __restrict__ nrm) {
    __shared__ float sh[33];
    const int64_t row = blockIdx.x, u = users[row];
    for (int64_t c = threadIdx.x; c < w; c += 256) y[row * w + c] = scores[row * w + c];
    __syncthreads();
    for (int64_t p = indptr[u] + threadIdx.x; p < indptr[u + 1]; p += 256) y[row * w + indices[p]] = 0.f;
    __syncthreads();
    float t = 0.f;
    for (int64_t c = threadIdx.x; c < w; c += 256) { const float v = y[row * w + c]; t = fmaf(v, v, t); }
    const float norm = fmaxf(sqrtf(block_sum_all(t, sh)), 1e-12f);
    for (int64_t c = threadIdx.x; c < w; c += 256) y[row * w + c] = y[row * w + c] / norm;
    if (threadIdx.x == 0) nrm[row] = norm;
}

// d_raw = (g - y <g, y>) / nrm, zero at the user's training items
__global__ void __launch_bounds__(256) usim_bwd_pre_kernel(const float* __restrict__ g, const float* __restrict__ y,
                                                           const float* __restrict__ nrm, const int64_t* __restrict__ users,
                                                           const int64_t* __restrict__ indptr, const int64_t* __restrict__ indices,
                                                           int64_t w, float* __restrict__ d_raw) {
    __shared__ float sh[33];
    const int64_t row = blockIdx.x, u = users[row];
    float t = 0.f;
    for (int64_t c = threadIdx.x; c < w; c += 256) t = fmaf(g[row * w + c], y[row * w + c], t);
    const float dot = block_sum_all(t, sh), inv = 1.f / nrm[row];
    for (int64_t c = threadIdx.x; c < w; c += 256) d_raw[row * w + c] = (g[row * w + c] - y[row * w + c] * dot) * inv;
    __syncthreads();
    for (int64_t p = indptr[u] + threadIdx.x; p < indptr[u + 1]; p += 256) d_raw[row * w + indices[p]] = 0.f;
}

// rr = normalize(softmax(R_row - c * log(-log(u + 1e-8) + 1e-8)) + pre_scale * ui_sim),  c = log_log_scale / tau
__global__ void __launch_bounds__(256) real_rows_kernel(const int64_t* __restrict__ users, const int64_t* __restrict__ indptr,
                                                        const int64_t* __restrict__ indices, const float* __restrict__ uniform,
                                                        const float* __restrict__ ui_sim, int64_t w, float c, float pre_scale,
                                                        float* __restrict__ out) {
    __shared__ float sh[33];
    const int64_t row = blockIdx.x, u = users[row];
    float* o = out + row * w;
    for (int64_t j = threadIdx.x; j < w; j += 256) o[j] = -c * logf(-logf(uniform[row * w + j] + 1e-8f) + 1e-8f);
    __syncthreads();
    for (int64_t p = indptr[u] + threadIdx.x; p < indptr[u + 1]; p += 256) o[indices[p]] += 1.f;
    __syncthreads();
    float mx = -INFINITY;
    for (int64_t j = threadIdx.x; j < w; j += 256) mx = fmaxf(mx, o[j]);
    mx = block_max_all(mx, sh);
    float t = 0.f;
    for (int64_t j = threadIdx.x; j < w; j += 256) { const float e = expf(o[j] - mx); o[j] = e; t += e; }
    const float inv = 1.f / block_sum_all(t, sh);
    t = 0.f;
    for (int64_t j = threadIdx.x; j < w; j += 256) {
        const float v = fmaf(ui_sim[row * w + j], pre_scale, o[j] * inv);
        o[j] = v;
        t = fmaf(v, v, t);
    }
    const float norm = fmaxf(sqrtf(block_sum_all(t, sh)), 1e-12f);
    for (int64_t j = threadIdx.x; j < w; j += 256) o[j] = o[j] / norm;
}

// ------------------------------------------------------------------------------------------ elementwise
__global__ void __launch_bounds__(256) interpolate_kernel(const float* __restrict__ alpha, const float* __restrict__ xr,
                                                          const float* __restrict__ xf, int64_t total, int64_t w, float* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= total) return;
    const float a = alpha[i / w];
    out[i] = a * xr[i] + (1.f - a) * xf[i];
}
__global__ void __launch_bounds__(256) add_scaled_kernel(float* __restrict__ acc, const float* __restrict__ x, float alpha, int64_t total) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i < total) acc[i] = fmaf(alpha, x[i], acc[i]);
}
__global__ void __launch_bounds__(256) gather_rows_kernel(const float* __restrict__ table, int64_t ld, const int64_t* __restrict__ rows,
                                                          int64_t total, int d, float* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= total) return;
    const int64_t r = i / d, c = i - r * d;
    out[i] = table[rows[r] * ld + c];
}
__global__ void __launch_bounds__(256) scatter_add_rows_kernel(float* __restrict__ table, int64_t ld, const int64_t* __restrict__ rows,
                                                               int64_t total, int d, const float* __restrict__ src) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= total) return;
    const int64_t r = i / d, c = i - r * d;
    atomicAdd(table + rows[r] * ld + c, src[i]);           // duplicates only when the batch exceeds the user count
}

static inline dim3 col_grid(int64_t h) { return dim3((unsigned)((h + kCT - 1) / kCT)); }
static inline unsigned flat_grid(int64_t total) { return (unsigned)((total + 255) / 256); }

}  // namespace mmssl

using namespace mmssl;
#define ST ((cudaStream_t)stream_)
#define COLS dim3(kCT, kRL)

extern "C" int mmssl_gan_bn_fwd(const float* a, const float* bias, const float* gamma, const float* beta, const float* mask,
                                float* running_mean, float* running_var, int64_t n, int64_t h, float* h_out, float* ah, float* rstd,
                                void* stream_) {
    MMSSL_REQUIRE(n >= 2 && h >= 1, "BatchNorm in training mode needs at least 2 rows");
    bn_fwd_kernel<<<col_grid(h), COLS, 0, ST>>>(a, bias, gamma, beta, mask, running_mean, running_var, n, h, h_out, ah, rstd);
    MMSSL_LAUNCH_OK();
    return 0;
}
extern "C" int mmssl_gan_bn_bwd(const float* dh, const float* mask, const float* gamma, const float* ah, const float* rstd, int64_t n,
                                int64_t h, float* da, float* dy, float* dgamma, float* dbeta, void* stream_) {
    MMSSL_REQUIRE(n >= 1 && h >= 1, "bad sizes");
    bn_bwd_kernel<<<col_grid(h), COLS, 0, ST>>>(dh, mask, gamma, ah, rstd, n, h, da, dy, dgamma, dbeta);
    MMSSL_LAUNCH_OK();
    return 0;
}
extern "C" int mmssl_gan_gp_rev_bn(const float* q, const float* dy, const float* ah, const float* rstd, const float* gamma,
                                   const float* mask, int64_t n, int64_t h, float* dh_bar, float* ah_bar, float* r_bar, float* g_gamma,
                                   void* stream_) {
    MMSSL_REQUIRE(n >= 1 && h >= 1, "bad sizes");
    gp_rev_bn_kernel<<<col_grid(h), COLS, 0, ST>>>(q, dy, ah, rstd, gamma, mask, n, h, dh_bar, ah_bar, r_bar, g_gamma);
    MMSSL_LAUNCH_OK();
    return 0;
}
extern "C" int mmssl_gan_bn_fwd_rev(const float* h_bar, const float* mask, const float* gamma, const float* ah, const float* rstd,
                                    const float* ah_bar, const float* r_bar, int64_t n, int64_t h, float* a_bar, float* g_gamma,
                                    float* g_beta, void* stream_) {
    MMSSL_REQUIRE(n >= 1 && h >= 1, "bad sizes");
    bn_fwd_rev_kernel<<<col_grid(h), COLS, 0, ST>>>(h_bar, mask, gamma, ah, rstd, ah_bar, r_bar, n, h, a_bar, g_gamma, g_beta);
    MMSSL_LAUNCH_OK();
    return 0;
}
extern "C" int mmssl_gan_colsum(const float* x, int64_t n, int64_t h, float* out, void* stream_) {
    MMSSL_REQUIRE(n >= 0 && h >= 1, "bad sizes");
    colsum_any_kernel<<<col_grid(h), COLS, 0, ST>>>(x, n, h, out);
    MMSSL_LAUNCH_OK();
    return 0;
}
extern "C" int mmssl_gan_head_fwd(const float* h2, const float* w3, const float* b3, int64_t n, int64_t h, float* s, float* s_sum,
                                  void* stream_) {
    MMSSL_REQUIRE(n >= 1 && h >= 1, "bad sizes");
    head_fwd_kernel<<<(unsigned)((n + 7) / 8), 256, 0, ST>>>(h2, w3, b3, n, h, s);
    MMSSL_LAUNCH_OK();
    vec_sum_kernel<<<1, 256, 0, ST>>>(s, n, 1.f, s_sum);
    MMSSL_LAUNCH_OK();
    return 0;
}
extern "C" int mmssl_gan_head_bwd(const float* s, float coef, const float* w3, const float* h2, int64_t n, int64_t h, float* dh2,
                                  float* dz, float* dw3, float* db3, void* stream_) {
    MMSSL_REQUIRE(n >= 1 && h >= 1, "bad sizes");
    head_bwd_kernel<<<col_grid(h), COLS, 0, ST>>>(s, coef, w3, h2, n, h, dh2, dz, dw3, db3);
    MMSSL_LAUNCH_OK();
    return 0;
}
extern "C" int mmssl_gan_gp_rows(const float* gx, int64_t n, int64_t w, float lam, float* gbar, float* sq_scratch, float* gp,
                                 void* stream_) {
    MMSSL_REQUIRE(n >= 1 && w >= 1, "bad sizes");
    gp_rows_kernel<<<(unsigned)n, 256, 0, ST>>>(gx, n, w, lam, gbar, sq_scratch);
    MMSSL_LAUNCH_OK();
    vec_sum_kernel<<<1, 256, 0, ST>>>(sq_scratch, n, lam / (float)n, gp);
    MMSSL_LAUNCH_OK();
    return 0;
}
extern "C" int mmssl_gan_gp_head_rev(const float* dh2_bar, const float* dz, const float* s, const float* w3, const float* h2,
                                     int64_t n, int64_t h, float* z_bar_scratch, float* h_bar, float* g_w3, float* g_b3,
                                     void* stream_) {
    MMSSL_REQUIRE(n >= 1 && h >= 1, "bad sizes");
    gp_head_rev_rows_kernel<<<(unsigned)((n + 7) / 8), 256, 0, ST>>>(dh2_bar, w3, s, n, h, z_bar_scratch);
    MMSSL_LAUNCH_OK();
    gp_head_rev_cols_kernel<<<col_grid(h), COLS, 0, ST>>>(dh2_bar, dz, z_bar_scratch, w3, h2, n, h, h_bar, g_w3, g_b3);
    MMSSL_LAUNCH_OK();
    return 0;
}
extern "C" int mmssl_gan_usim_finish(const float* scores, const int64_t* users, const int64_t* indptr, const int64_t* indices,
                                     int64_t rows, int64_t w, float* y, float* nrm, void* stream_) {
    MMSSL_REQUIRE(rows >= 0 && w >= 1, "bad sizes");
    if (rows == 0) return 0;
    usim_finish_kernel<<<(unsigned)rows, 256, 0, ST>>>(scores, users, indptr, indices, w, y, nrm);
    MMSSL_LAUNCH_OK();
    return 0;
}
extern "C" int mmssl_gan_usim_bwd_pre(const float* g, const float* y, const float* nrm, const int64_t* users, const int64_t* indptr,
                                      const int64_t* indices, int64_t rows, int64_t w, float* d_raw, void* stream_) {
    MMSSL_REQUIRE(rows >= 0 && w >= 1, "bad sizes");
    if (rows == 0) return 0;
    usim_bwd_pre_kernel<<<(unsigned)rows, 256, 0, ST>>>(g, y, nrm, users, indptr, indices, w, d_raw);
    MMSSL_LAUNCH_OK();
    return 0;
}
extern "C" int mmssl_gan_real_rows(const int64_t* users, const int64_t* indptr, const int64_t* indices, const float* uniform,
                                   const float* ui_sim, int64_t rows, int64_t w, float log_log_scale, float tau, float pre_scale,
                                   float* out, void* stream_) {
    MMSSL_REQUIRE(rows >= 0 && w >= 1 && tau > 0.f, "bad sizes");
    if (rows == 0) return 0;
    real_rows_kernel<<<(unsigned)rows, 256, 0, ST>>>(users, indptr, indices, uniform, ui_sim, w, log_log_scale / tau, pre_scale, out);
    MMSSL_LAUNCH_OK();
    return 0;
}
extern "C" int mmssl_gan_interpolate(const float* alpha, const float* xr, const float* xf, int64_t rows, int64_t w, float* out,
                                     void* stream_) {
    if (rows * w == 0) return 0;
    interpolate_kernel<<<flat_grid(rows * w), 256, 0, ST>>>(alpha, xr, xf, rows * w, w, out);
    MMSSL_LAUNCH_OK();
    return 0;
}
extern "C" int mmssl_gan_add_scaled(float* acc, const float* x, float alpha, int64_t total, void* stream_) {
    if (total == 0) return 0;
    add_scaled_kernel<<<flat_grid(total), 256, 0, ST>>>(acc, x, alpha, total);
    MMSSL_LAUNCH_OK();
    return 0;
}
extern "C" int mmssl_gan_gather_rows(const float* table, int64_t ld, const int64_t* rows, int64_t n_rows, int d, float* out,
                                     void* stream_) {
    if (n_rows * d == 0) return 0;
    gather_rows_kernel<<<flat_grid(n_rows * d), 256, 0, ST>>>(table, ld, rows, n_rows * d, d, out);
    MMSSL_LAUNCH_OK();
    return 0;
}
extern "C" int mmssl_gan_scatter_add_rows(float* table, int64_t ld, const int64_t* rows, int64_t n_rows, int d, const float* src,
                                          void* stream_) {
    if (n_rows * d == 0) return 0;
    scatter_add_rows_kernel<<<flat_grid(n_rows * d), 256, 0, ST>>>(table, ld, rows, n_rows * d, d, src);
    MMSSL_LAUNCH_OK();
    return 0;
}
