// Shared helpers for the mmssl_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <type_traits>
namespace mmssl {

// ---- error reporting (thread-local message, C-ABI functions return non-zero on failure) ----
char* last_error_buffer();
int fail(const char* where, const char* what);
int fail_cuda(const char* where, cudaError_t e);

#define MMSSL_REQUIRE(cond, msg)                                   \
    do {                                                           \
        if (!(cond)) return ::mmssl::fail(__func__, msg);          \
    } while (0)

#define MMSSL_CUDA(call)                                           \
    do {                                                           \
        cudaError_t e__ = (call);                                  \
        if (e__ != cudaSuccess) return ::mmssl::fail_cuda(__func__, e__); \
    } while (0)

// Launch check that is legal during stream capture (no sync).
#define MMSSL_LAUNCH_OK()                                          \
    do {                                                           \
        cudaError_t e__ = cudaPeekAtLastError();                   \
        if (e__ != cudaSuccess) { cudaGetLastError(); return ::mmssl::fail_cuda(__func__, e__); } \
    } while (0)

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

constexpr int kNumSMs = 132;   // H100 SXM

// ---- programmatic dependent launch (PDL) ----
// Kernels on the critical path of the captured step are launched with
// cudaLaunchAttributeProgrammaticStreamSerialization: the next kernel's launch and prologue overlap the
// tail of its predecessor, and `pdl_wait()` (griddepcontrol.wait, first statement of every such kernel)
// blocks until the predecessor has fully completed and flushed.  MMSSL_PDL=0 disables it.
bool pdl_enabled();
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr.val.programmaticStreamSerializationAllowed = 1;
    if (pdl_enabled()) { cfg.attrs = &attr; cfg.numAttrs = 1; }
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
#define MMSSL_CUDA_LAUNCH(kernel, grid, block, smem, stream, ...)                                          \
    do {                                                                                                   \
        cudaError_t e__ = ::mmssl::launch_k(kernel, grid, block, smem, stream, __VA_ARGS__);               \
        if (e__ != cudaSuccess) return ::mmssl::fail_cuda(__func__, e__);                                   \
    } while (0)

// ---- device helpers ----
__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 ldcg4(const float* p) { return __ldcg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ float4 f4zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }

// ---- L2 / L1 residency hints (large graphs: what streams must not evict what is gathered) ----
// 64-bit L2 cache-policy words (createpolicy encodings, the ones the TMA kernels already use on hardware)
constexpr uint64_t kL2EvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kL2EvictLast = 0x14F0000000000000ull;
__device__ __forceinline__ int ldg_i32_stream(const int* p) {
    int v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.b32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(kL2EvictFirst));
    return v;
}
__device__ __forceinline__ float ldg_f32_stream(const float* p) {
    float v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(v) : "l"(p), "l"(kL2EvictFirst));
    return v;
}
__device__ __forceinline__ float4 ldg4_stream(const float* p) {
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p), "l"(kL2EvictFirst));
    return v;
}
__device__ __forceinline__ float4 ld4_stream(const float* p) {      // coherent (the buffer may be written by this kernel elsewhere)
    float4 v;
    asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p), "l"(kL2EvictFirst) : "memory");
    return v;
}
__device__ __forceinline__ void st4_stream(float* p, const float4& v) {
    asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(kL2EvictFirst) : "memory");
}
// gathered row: keep it in L2 (policy word chosen by the caller: evict-last when the gathered table fits L2, else normal)
__device__ __forceinline__ float4 ldg4_l2(const float* p, uint64_t policy) {
    float4 v;
    asm volatile("ld.global.nc.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p), "l"(policy));
    return v;
}
// gathered row with an L1 priority: hot columns (the head of the degree distribution) are pinned (evict_last), the cold ones
// do not allocate -- two predicated loads into the same registers, no branch
__device__ __forceinline__ float4 ldg4_l1_hot_cold(const float* p, int hot, uint64_t policy) {
    float4 v;
    asm volatile(
        "{\n\t.reg .pred q;\n\t"
        "setp.ne.b32 q, %5, 0;\n\t"
        "@q ld.global.nc.L1::evict_last.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %6;\n\t"
        "@!q ld.global.nc.L1::no_allocate.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %6;\n\t}"
        : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p), "r"(hot), "l"(policy));
    return v;
}
__device__ __forceinline__ void fma4(float4& a, float s, const float4& x) {
    a.x = fmaf(s, x.x, a.x); a.y = fmaf(s, x.y, a.y); a.z = fmaf(s, x.z, a.z); a.w = fmaf(s, x.w, a.w);
}
__device__ __forceinline__ float dot4(const float4& a, const float4& b) {
    return fmaf(a.x, b.x, fmaf(a.y, b.y, fmaf(a.z, b.z, a.w * b.w)));
}
__device__ __forceinline__ float4 add4(const float4& a, const float4& b) {
    return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
}
__device__ __forceinline__ float4 scale4(const float4& a, float s) {
    return make_float4(a.x * s, a.y * s, a.z * s, a.w * s);
}
__device__ __forceinline__ float max4(const float4& a) { return fmaxf(fmaxf(a.x, a.y), fmaxf(a.z, a.w)); }

// Reduction over a group of G consecutive lanes (G = 8, 16 or 32) using a group-local mask.
template <int G>
__device__ __forceinline__ unsigned group_mask() {
    if (G == 32) return 0xffffffffu;
    const unsigned lane = threadIdx.x & 31u;
    return ((1u << G) - 1u) << (lane & ~(unsigned)(G - 1));
}
template <int G>
__device__ __forceinline__ float group_sum(float v, unsigned mask) {
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(mask, v, o, G);
    return v;
}
template <int G>
__device__ __forceinline__ float group_max(float v, unsigned mask) {
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(mask, v, o, G));
    return v;
}
__device__ __forceinline__ float warp_sum(float v) { return group_sum<32>(v, 0xffffffffu); }

// ---- embedding widths ----
// The row kernels (SpMM, row ops, losses) lay a row of d floats over a group of G consecutive lanes, G a power of two from 8
// to 32 (group_sum), each lane holding C float4 per right-hand side at columns 4 lane + 4 G c: d = 4 G C.  These six widths
// are the ones the library is built for; kernel dispatch and host-side sizes derived from G both come from this rule.
struct WidthShape { int g, c; };
constexpr WidthShape width_shape(int d) {
    return d == 32 ? WidthShape{8, 1} : d == 64 ? WidthShape{16, 1} : d == 96 ? WidthShape{8, 3}
         : d == 128 ? WidthShape{32, 1} : d == 192 ? WidthShape{16, 3} : d == 256 ? WidthShape{32, 2} : WidthShape{0, 0};
}
constexpr bool width_supported(int d) { return width_shape(d).g != 0; }
int fail_width(const char* where, int d);   // "<where>: embedding width <d> is not supported (...)"

// The SpMM work plan's current row cuts (graph.cu, mmssl_spmm_plan_set_cuts): {split threshold, segment length, heavy threshold,
// heavy segment length}.  The fold-in kernel (rowops.cu) cuts a query row where the plan would cut a training row.
int4 spmm_plan_cuts();

// f(integral_constant G, integral_constant C) for one of the six widths, an error naming the width otherwise.
template <typename F>
static inline int dispatch_width(int d, F&& f, const char* where = "embedding width") {
#define MMSSL_WIDTH_CASE(D) \
    case D: return f(std::integral_constant<int, width_shape(D).g>(), std::integral_constant<int, width_shape(D).c>());
    switch (d) {
        MMSSL_WIDTH_CASE(32) MMSSL_WIDTH_CASE(64) MMSSL_WIDTH_CASE(96) MMSSL_WIDTH_CASE(128) MMSSL_WIDTH_CASE(192) MMSSL_WIDTH_CASE(256)
    }
#undef MMSSL_WIDTH_CASE
    return fail_width(where, d);
}

// Block-wide sum for blockDim.x <= 1024 (result valid in thread 0).
__device__ __forceinline__ float block_sum(float v, float* smem32) {
    v = warp_sum(v);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) smem32[w] = v;
    __syncthreads();
    const int nw = (blockDim.x + 31) >> 5;
    v = (threadIdx.x < nw) ? smem32[threadIdx.x] : 0.f;
    if (w == 0) v = warp_sum(v);
    return v;
}

// The ranking key of the top-k lists (eval.cu: the sweep and the merge of partial lists).  Larger key == better: higher score
// first, then lower id.  fp32 -> order-preserving u32 of its bits, so -0.0 orders below +0.0 exactly as the sweep orders them.
__device__ __forceinline__ uint64_t eval_key(float s, uint32_t item) {
    uint32_t b = __float_as_uint(s);
    b = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
    return ((uint64_t)b << 32) | (uint64_t)(0xFFFFFFFFu - item);
}
__device__ __forceinline__ float eval_key_score(uint64_t key) {
    uint32_t b = (uint32_t)(key >> 32);
    b = (b & 0x80000000u) ? (b & 0x7FFFFFFFu) : ~b;
    return __uint_as_float(b);
}

}  // namespace mmssl
