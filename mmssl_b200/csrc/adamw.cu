// Multi-tensor AdamW with torch.optim.AdamW semantics (reference: main.py:76-80 builds
// optim.AdamW(model.parameters(), lr=args.lr) -> betas (0.9, 0.999), eps 1e-8, weight_decay 1e-2;
// stepped at main.py:427-429).  One launch covers all live parameters; the step counter lives on
// the device so the kernel can be replayed inside a CUDA graph.
#include "common.cuh"
#include "../../include/mmssl_b200.h"

namespace mmssl {

struct AdamPack {
    float* p[MMSSL_ADAMW_MAX_TENSORS];
    const float* g[MMSSL_ADAMW_MAX_TENSORS];
    float* m[MMSSL_ADAMW_MAX_TENSORS];
    float* v[MMSSL_ADAMW_MAX_TENSORS];
    int64_t start4[MMSSL_ADAMW_MAX_TENSORS + 1];   // prefix of ceil(numel/4)
    int64_t numel[MMSSL_ADAMW_MAX_TENSORS];
    int n;
};

// 1 - beta^step.  Formed as 1.f - powf(beta, step) it cancels: beta^step near 1 is rounded to 2^-24 of 1, which is 3e-5 of
// 1 - 0.999^2.  beta - 1 is exact in fp32 (beta in [0.5, 1)) and log1pf / expm1f keep the relative accuracy of a small argument.
__device__ __forceinline__ float bias_correction(float beta, int step) {
    return -expm1f((float)step * log1pf(beta - 1.f)); }

__global__ void step_tick_kernel(int32_t* step) {
    pdl_wait(); *step += 1; }

__global__ void __launch_bounds__(256) adamw_kernel(const AdamPack pk, const int32_t* __restrict__ step_dev, float lr,
                                                    float b1, float b2, float eps, float wd) {
    pdl_wait();
    const int step = *step_dev;
    const float bc1 = bias_correction(b1, step);
    const float bc2 = bias_correction(b2, step);
    const float step_size = lr / bc1;
    const float inv_sqrt_bc2 = rsqrtf(bc2);
    const float decay = 1.f - lr * wd;
    const int64_t total4 = pk.start4[pk.n];
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total4; i += (int64_t)gridDim.x * blockDim.x) {
        int t = 0;
        while (t + 1 < pk.n && i >= pk.start4[t + 1]) ++t;
        const int64_t e = (i - pk.start4[t]) * 4;
        const int64_t left = pk.numel[t] - e;
        float* p = pk.p[t] + e; const float* g = pk.g[t] + e; float* m = pk.m[t] + e; float* v = pk.v[t] + e;
        if (left >= 4) {
            float4 pv = ld4(p), gv = ld4(g), mv = ld4(m), vv = ld4(v);
            float* pp = &pv.x; float* gg = &gv.x; float* mm = &mv.x; float* vq = &vv.x;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float gk = gg[k];
                mm[k] = b1 * mm[k] + (1.f - b1) * gk;
                vq[k] = b2 * vq[k] + (1.f - b2) * gk * gk;
                const float den = sqrtf(vq[k]) * inv_sqrt_bc2 + eps;
                pp[k] = pp[k] * decay - step_size * (mm[k] / den);
            }
            st4(p, pv); st4(m, mv); st4(v, vv);
        } else {
            for (int k = 0; k < left; ++k) {
                const float gk = g[k];
                const float mk = b1 * m[k] + (1.f - b1) * gk;
                const float vk = b2 * v[k] + (1.f - b2) * gk * gk;
                m[k] = mk; v[k] = vk;
                p[k] = p[k] * decay - step_size * (mk / (sqrtf(vk) * inv_sqrt_bc2 + eps));
            }
        }
    }
}

// Data-parallel optimiser step in ONE kernel over NVSwitch multicast (SURVEY 8f next #4, sharded AdamW):
//   g   = multimem.ld_reduce(add) over every rank's gradient bucket      (reduce-scatter, summed in the switch)
//   AdamW on this rank's slice only (m, v exist only for the slice)
//   multimem.st of the new parameters into every rank's parameter buffer  (all-gather)
// Buckets are symmetric-memory buffers with the same layout on every rank; callers barrier before (all
// gradients written) and after (all slices published).
__global__ void __launch_bounds__(256) dp_fused_adamw_kernel(const float* __restrict__ p_local, float* p_mc,
                                                             const float* g_mc, float* __restrict__ m,
                                                             float* __restrict__ v, int64_t begin, int64_t count4,
                                                             float inv_world, int step_host, const int32_t* __restrict__ step_dev,
                                                             float lr, float b1, float b2, float eps, float wd) {
    // step_dev != NULL: the 1-based step number lives on the device (mmssl_step_tick), so the launch can sit in a CUDA graph
    const int step = step_dev != nullptr ? *step_dev : step_host;
    const float bc1 = bias_correction(b1, step);
    const float bc2 = bias_correction(b2, step);
    const float step_size = lr / bc1;
    const float inv_sqrt_bc2 = rsqrtf(bc2);
    const float decay = 1.f - lr * wd;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < count4; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t e = begin + i * 4;
        float4 g;
        asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
                     : "=f"(g.x), "=f"(g.y), "=f"(g.z), "=f"(g.w) : "l"(g_mc + e) : "memory");
        float4 pv = ld4(p_local + e), mv = ld4(m + i * 4), vv = ld4(v + i * 4);
        float* pp = &pv.x; float* gg = &g.x; float* mm = &mv.x; float* vq = &vv.x;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float gk = gg[k] * inv_world;
            mm[k] = b1 * mm[k] + (1.f - b1) * gk;
            vq[k] = b2 * vq[k] + (1.f - b2) * gk * gk;
            pp[k] = pp[k] * decay - step_size * (mm[k] / (sqrtf(vq[k]) * inv_sqrt_bc2 + eps));
        }
        st4(m + i * 4, mv); st4(v + i * 4, vv);
        asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p_mc + e), "f"(pv.x), "f"(pv.y),
                     "f"(pv.z), "f"(pv.w) : "memory");
    }
}

}  // namespace mmssl

using namespace mmssl;

static int dp_fused_launch(const float* p_local, float* p_mc, const float* g_mc, float* m, float* v, int64_t begin, int64_t count,
                           float inv_world, int step, const int32_t* step_dev, float lr, float beta1, float beta2, float eps,
                           float weight_decay, cudaStream_t st) {
    MMSSL_REQUIRE(begin % 4 == 0 && count % 4 == 0, "slice must be a multiple of 4 floats");
    MMSSL_REQUIRE(aligned16(p_local) && aligned16(p_mc) && aligned16(g_mc) && aligned16(m) && aligned16(v), "alignment");
    MMSSL_REQUIRE(step_dev != nullptr || step >= 1, "step is 1-based");
    if (count == 0) return 0;
    int64_t blocks = (count / 4 + 255) / 256;
    if (blocks > kNumSMs * 8) blocks = kNumSMs * 8;
    dp_fused_adamw_kernel<<<(unsigned)blocks, 256, 0, st>>>(p_local, p_mc, g_mc, m, v, begin, count / 4, inv_world, step, step_dev, lr,
                                                           beta1, beta2, eps, weight_decay);
    MMSSL_LAUNCH_OK();
    return 0;
}

extern "C" int mmssl_dp_fused_adamw(const float* p_local, float* p_mc, const float* g_mc, float* m, float* v, int64_t begin,
                                    int64_t count, float inv_world, int step, float lr, float beta1, float beta2, float eps,
                                    float weight_decay, void* stream_) {
    return dp_fused_launch(p_local, p_mc, g_mc, m, v, begin, count, inv_world, step, nullptr, lr, beta1, beta2, eps, weight_decay,
                           (cudaStream_t)stream_);
}

extern "C" int mmssl_dp_fused_adamw_dev(const float* p_local, float* p_mc, const float* g_mc, float* m, float* v, int64_t begin,
                                        int64_t count, float inv_world, const int32_t* step_dev, float lr, float beta1, float beta2,
                                        float eps, float weight_decay, void* stream_) {
    MMSSL_REQUIRE(step_dev != nullptr, "device step counter missing");
    return dp_fused_launch(p_local, p_mc, g_mc, m, v, begin, count, inv_world, 0, step_dev, lr, beta1, beta2, eps, weight_decay,
                           (cudaStream_t)stream_);
}

extern "C" int mmssl_step_tick(int32_t* step_dev, void* stream_) {
    MMSSL_CUDA_LAUNCH((step_tick_kernel), dim3(1), dim3(1), 0, (cudaStream_t)stream_, step_dev);
    MMSSL_LAUNCH_OK();
    return 0;
}

extern "C" int mmssl_adamw(int n_tensors, float* const* p, const float* const* g, float* const* m, float* const* v,
                           const int64_t* numel, const int32_t* step_dev, float lr, float beta1, float beta2, float eps,
                           float weight_decay, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    MMSSL_REQUIRE(n_tensors >= 1 && n_tensors <= MMSSL_ADAMW_MAX_TENSORS, "1..16 tensors per call");
    AdamPack pk;
    memset(&pk, 0, sizeof(pk));
    pk.n = n_tensors;
    int64_t acc = 0;
    for (int t = 0; t < n_tensors; ++t) {
        MMSSL_REQUIRE(p[t] && g[t] && m[t] && v[t], "null tensor");
        MMSSL_REQUIRE(aligned16(p[t]) && aligned16(g[t]) && aligned16(m[t]) && aligned16(v[t]), "tensors must be 16-byte aligned");
        pk.p[t] = p[t]; pk.g[t] = g[t]; pk.m[t] = m[t]; pk.v[t] = v[t];
        pk.numel[t] = numel[t];
        pk.start4[t] = acc;
        acc += (numel[t] + 3) / 4;
    }
    pk.start4[n_tensors] = acc;
    if (acc == 0) return 0;
    int64_t blocks = (acc + 255) / 256;
    if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
    MMSSL_CUDA_LAUNCH((adamw_kernel), dim3((unsigned)blocks), dim3(256), 0, st, pk, step_dev, lr, beta1, beta2, eps, weight_decay);
    MMSSL_LAUNCH_OK();
    return 0;
}
