// cuemu -- a host-side executor for plain CUDA C++ kernels.  TEST INFRASTRUCTURE ONLY.
//
// Purpose: the build container has nvcc but no GPU.  This header lets g++ compile the *unmodified kernel bodies* of
// mmssl_b200/csrc/*.cu (after tests/cuemu/build.py rewrites the three pieces of syntax g++ cannot parse: `<<<...>>>`
// launches, `extern __shared__` declarations and inline asm statements) and run them on the CPU with CUDA's execution model:
//   * one fiber per CUDA thread, all fibers of a block alive at the same time, blocks executed one after the other;
//   * __syncthreads / __syncthreads_or|and|count are block barriers, __shfl_*_sync / __ballot_sync / __syncwarp are
//     barriers over the lanes named by the mask, with the value exchange in between (exited lanes are ignored, like
//     the hardware does);
//   * atomics are plain read-modify-writes (single OS thread, fibers switch only at barriers);
//   * static __shared__ variables are function-local statics (one block at a time), dynamic shared memory is a
//     per-launch buffer re-poisoned with NaN bytes for every block;
//   * the fiber order inside a block is selectable (CUEMU_ORDER=fwd|rev|shuffle:<seed>) so that a missing barrier
//     shows up as a result that depends on the order; CUEMU_BLOCK_ORDER=rev runs the blocks of a grid last to first;
//   * a block in which every live fiber waits at a barrier that cannot complete is reported as a deadlock
//     (divergent __syncthreads, a shuffle mask naming a lane that went elsewhere).
//   * inline PTX is routed to cuemu_ptx.cpp: a functional model of the subset the tensor-core kernels use (mbarrier, 2-D
//     TMA tensor copies with the 128-byte swizzle, wgmma with register accumulators); anything else fails the launch;
//   * CUB's two device primitives are host shims.
// It proves indexing, reduction order, barrier / pipeline protocol and the host-side argument marshalling; it says nothing
// about performance, memory coalescing, true asynchrony or device math rounding.  Nothing under mmssl_b200/ includes this.
#pragma once
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <tuple>
#include <type_traits>
#include <utility>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline __attribute__((always_inline))
#define __noinline__ __attribute__((noinline))
#define __launch_bounds__(...)
#define __shared__ static
#define __constant__ static
#define __align__(n) __attribute__((aligned(n)))
#define __grid_constant__
#define CUEMU 1

// ------------------------------------------------------------------------------------------ vector types
struct uint3 { unsigned x, y, z; };
struct dim3 {
    unsigned x, y, z;
    constexpr dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct __attribute__((aligned(8))) float2 { float x, y; };
struct __attribute__((aligned(16))) float4 { float x, y, z, w; };
struct __attribute__((aligned(8))) int2 { int x, y; };
struct __attribute__((aligned(16))) int4 { int x, y, z, w; };
struct __attribute__((aligned(8))) uint2 { unsigned x, y; };
struct __attribute__((aligned(16))) uint4 { unsigned x, y, z, w; };
struct __attribute__((aligned(16))) double2 { double x, y; };
struct __attribute__((aligned(16))) longlong2 { long long x, y; };
static inline float2 make_float2(float x, float y) { return float2{x, y}; }
static inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
static inline int2 make_int2(int x, int y) { return int2{x, y}; }
static inline int4 make_int4(int x, int y, int z, int w) { return int4{x, y, z, w}; }
static inline uint2 make_uint2(unsigned x, unsigned y) { return uint2{x, y}; }
static inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { return uint4{x, y, z, w}; }
static inline double2 make_double2(double x, double y) { return double2{x, y}; }

// ------------------------------------------------------------------------------------------ runtime API subset
typedef void* cudaStream_t;
typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorLaunchFailure = 719 };
enum cudaMemcpyKind { cudaMemcpyHostToHost, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice, cudaMemcpyDefault };
enum cudaDeviceAttr { cudaDevAttrComputeCapabilityMajor = 75, cudaDevAttrMultiProcessorCount = 16 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8, cudaFuncAttributePreferredSharedMemoryCarveout = 9 };
enum cudaSharedCarveout { cudaSharedmemCarveoutDefault = -1, cudaSharedmemCarveoutMaxShared = 100, cudaSharedmemCarveoutMaxL1 = 0 };
enum cudaLaunchAttributeID { cudaLaunchAttributeProgrammaticStreamSerialization = 4 };
struct cudaLaunchAttributeValue { int programmaticStreamSerializationAllowed; };
struct cudaLaunchAttribute { cudaLaunchAttributeID id; cudaLaunchAttributeValue val; };
struct cudaLaunchConfig_t {
    dim3 gridDim, blockDim;
    size_t dynamicSmemBytes;
    cudaStream_t stream;
    cudaLaunchAttribute* attrs;
    unsigned numAttrs;
};

namespace cuemu {
struct Fiber {
    void* sp;
    uint3 tid;
    int lin, warp, lane;
    bool done;
};
extern Fiber* cur;
extern int g_error;                                  // sticky per launch; read by cudaPeekAtLastError

void run_grid(dim3 grid, dim3 block, size_t smem, void (*thunk)(void*), void* arg, const char* name);
void* dyn_smem();
void syncthreads();
int syncthreads_red(int pred, int op);               // op 0 = or, 1 = and, 2 = count
void syncwarp(unsigned mask);
void exchange_begin(unsigned mask, uint64_t bits);   // deposit + barrier
uint64_t exchange_peek(int lane, bool* valid);
void exchange_end(unsigned mask);
// Inline PTX, as rewritten by build.py: template text, pointers to / sizes of the outputs, the inputs as 64-bit values.
// cuemu_ptx.cpp models the subset the library uses (mbarrier, TMA copies with the 128-byte swizzle, wgmma m64nNk16 bf16,
// multimem over registered replica groups, griddepcontrol) and fails the launch on anything else.
void ptx_op(const char* text, void** outs, const int* out_sizes, int n_out, const uint64_t* ins, int n_in);
void ptx_block_reset();
void yield_blocked();                                 // give the CPU to the other fibers of the block (a failed try_wait)
void note_progress();
size_t dyn_smem_bytes();
const char* error_text();
void fail(const char* what);

static inline uint64_t as_u64(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static inline uint64_t as_u64(double d) { uint64_t u; memcpy(&u, &d, 8); return u; }
template <typename T> static inline uint64_t as_u64(T* p) { return (uint64_t)(uintptr_t)p; }
template <typename T> static inline typename std::enable_if<std::is_integral<T>::value || std::is_enum<T>::value, uint64_t>::type as_u64(T v) { return (uint64_t)v; }

template <typename T> struct ident { typedef T type; };

struct Cfg {
    dim3 grid, block;
    size_t smem;
    Cfg(dim3 g, dim3 b, size_t s = 0, cudaStream_t = nullptr) : grid(g), block(b), smem(s) {}
};
static inline Cfg cfg(dim3 g, dim3 b, size_t s = 0, cudaStream_t st = nullptr) { return Cfg(g, b, s, st); }

template <typename... KArgs>
struct Launcher {
    void (*kernel)(KArgs...);
    Cfg c;
    const char* name;
    template <typename... Args>
    void operator()(Args&&... args) const {
        typedef std::tuple<typename std::decay<KArgs>::type...> Tup;
        struct Pack { void (*k)(KArgs...); Tup t; } pack{kernel, Tup(static_cast<KArgs>(args)...)};
        run_grid(c.grid, c.block, c.smem, [](void* p) {
            Pack* q = static_cast<Pack*>(p);
            std::apply(q->k, q->t);
        }, &pack, name);
    }
};
template <typename... KArgs>
static inline Launcher<KArgs...> launch(void (*kernel)(KArgs...), Cfg c, const char* name = "kernel") {
    return Launcher<KArgs...>{kernel, c, name};
}
}  // namespace cuemu

// The scheduler copies the running fiber's coordinates into these before every switch (single OS thread).
extern uint3 threadIdx, blockIdx;
extern dim3 blockDim, gridDim;
#define warpSize 32

static inline const char* cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : cuemu::error_text(); }
static inline cudaError_t cudaPeekAtLastError() { return cuemu::g_error; }
static inline cudaError_t cudaGetLastError() { int e = cuemu::g_error; cuemu::g_error = 0; return e; }
static inline cudaError_t cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t = nullptr) { memset(p, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemset(void* p, int v, size_t n) { memset(p, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
static inline cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr a, int) { *v = a == cudaDevAttrMultiProcessorCount ? 132 : 9; return cudaSuccess; }
template <typename F> static inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int* n, F, int, size_t) { *n = 8; return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
template <typename F> static inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int) { return cudaSuccess; }
template <typename... KArgs, typename... Args>
static inline cudaError_t cudaLaunchKernelEx(const cudaLaunchConfig_t* c, void (*kernel)(KArgs...), Args&&... args) {
    cuemu::launch(kernel, cuemu::Cfg(c->gridDim, c->blockDim, c->dynamicSmemBytes))(static_cast<Args&&>(args)...);
    return cuemu::g_error;
}

// ------------------------------------------------------------------------------------------ barriers and warp primitives
// shared-memory "addresses" are byte offsets into the block's dynamic shared memory (1024-byte aligned base)
static inline size_t __cvta_generic_to_shared(const void* p) { return (size_t)((const char*)p - (const char*)cuemu::dyn_smem()); }
static inline void __trap() { cuemu::fail("__trap()"); }
static inline void __syncthreads() { cuemu::syncthreads(); }
static inline int __syncthreads_or(int p) { return cuemu::syncthreads_red(p, 0); }
static inline int __syncthreads_and(int p) { return cuemu::syncthreads_red(p, 1); }
static inline int __syncthreads_count(int p) { return cuemu::syncthreads_red(p, 2); }
static inline void __syncwarp(unsigned mask = 0xffffffffu) { cuemu::syncwarp(mask); }
static inline void __threadfence() { __asm__ volatile("" ::: "memory"); }
static inline void __threadfence_block() { __asm__ volatile("" ::: "memory"); }
static inline void __threadfence_system() { __asm__ volatile("" ::: "memory"); }
static inline unsigned __activemask() { cuemu::fail("__activemask is not emulated"); return 0; }

namespace cuemu {
template <typename T>
static inline T shfl_from(unsigned mask, T v, int src) {
    static_assert(sizeof(T) <= 8, "shuffle of a type wider than 64 bits");
    uint64_t bits = 0;
    memcpy(&bits, &v, sizeof(T));
    exchange_begin(mask, bits);
    bool valid = false;
    const uint64_t got = exchange_peek(src, &valid);
    exchange_end(mask);
    if (!valid) return v;                            // reading an inactive lane is undefined; keep the own value
    T r;
    memcpy(&r, &got, sizeof(T));
    return r;
}
}  // namespace cuemu
template <typename T> static inline T __shfl_sync(unsigned mask, T v, int src, int width = 32) {
    const int lane = cuemu::cur->lane;
    return cuemu::shfl_from(mask, v, (lane & ~(width - 1)) | (src & (width - 1)));
}
template <typename T> static inline T __shfl_xor_sync(unsigned mask, T v, int lanemask, int width = 32) {
    const int lane = cuemu::cur->lane, src = lane ^ lanemask;
    return cuemu::shfl_from(mask, v, ((src & ~(width - 1)) == (lane & ~(width - 1))) ? src : lane);
}
template <typename T> static inline T __shfl_down_sync(unsigned mask, T v, unsigned delta, int width = 32) {
    const int lane = cuemu::cur->lane, src = lane + (int)delta;
    return cuemu::shfl_from(mask, v, ((src & ~(width - 1)) == (lane & ~(width - 1))) ? src : lane);
}
template <typename T> static inline T __shfl_up_sync(unsigned mask, T v, unsigned delta, int width = 32) {
    const int lane = cuemu::cur->lane, src = lane - (int)delta;
    return cuemu::shfl_from(mask, v, (src >= (lane & ~(width - 1))) ? src : lane);
}
static inline unsigned __ballot_sync(unsigned mask, int pred) {
    cuemu::exchange_begin(mask, pred ? 1u : 0u);
    unsigned r = 0;
    for (int l = 0; l < 32; ++l) {
        bool valid = false;
        const uint64_t b = cuemu::exchange_peek(l, &valid);
        if (valid && ((mask >> l) & 1u) && b) r |= 1u << l;
    }
    cuemu::exchange_end(mask);
    return r;
}
static inline int __any_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) != 0; }
static inline int __all_sync(unsigned mask, int pred) {
    // all lanes named by the mask that are still alive
    cuemu::exchange_begin(mask, pred ? 1u : 0u);
    int r = 1;
    for (int l = 0; l < 32; ++l) {
        bool valid = false;
        const uint64_t b = cuemu::exchange_peek(l, &valid);
        if (valid && ((mask >> l) & 1u) && !b) r = 0;
    }
    cuemu::exchange_end(mask);
    return r;
}

// ------------------------------------------------------------------------------------------ atomics (plain RMW: one OS thread)
template <typename T> static inline T atomicAdd(T* p, typename cuemu::ident<T>::type v) { T o = *p; *p = o + v; return o; }
template <typename T> static inline T atomicSub(T* p, typename cuemu::ident<T>::type v) { T o = *p; *p = o - v; return o; }
template <typename T> static inline T atomicExch(T* p, typename cuemu::ident<T>::type v) { T o = *p; *p = v; return o; }
template <typename T> static inline T atomicMax(T* p, typename cuemu::ident<T>::type v) { T o = *p; if (v > o) *p = v; return o; }
template <typename T> static inline T atomicMin(T* p, typename cuemu::ident<T>::type v) { T o = *p; if (v < o) *p = v; return o; }
template <typename T> static inline T atomicOr(T* p, typename cuemu::ident<T>::type v) { T o = *p; *p = o | v; return o; }
template <typename T> static inline T atomicAnd(T* p, typename cuemu::ident<T>::type v) { T o = *p; *p = o & v; return o; }
template <typename T> static inline T atomicCAS(T* p, typename cuemu::ident<T>::type cmp, typename cuemu::ident<T>::type v) {
    T o = *p;
    if (o == cmp) *p = v;
    return o;
}
// sm_90+ vector float atomics (element-wise, returns the old vector)
static inline float4 atomicAdd(float4* p, float4 v) { float4 o = *p; p->x += v.x; p->y += v.y; p->z += v.z; p->w += v.w; return o; }
static inline float2 atomicAdd(float2* p, float2 v) { float2 o = *p; p->x += v.x; p->y += v.y; return o; }
static inline unsigned atomicInc(unsigned* p, unsigned v) { unsigned o = *p; *p = (o >= v) ? 0 : o + 1; return o; }

// ------------------------------------------------------------------------------------------ loads / stores with cache hints
template <typename T> static inline T __ldg(const T* p) { return *p; }
template <typename T> static inline T __ldcg(const T* p) { return *p; }
template <typename T> static inline T __ldcs(const T* p) { return *p; }
template <typename T> static inline T __ldca(const T* p) { return *p; }
template <typename T> static inline T __ldlu(const T* p) { return *p; }
template <typename T> static inline void __stcg(T* p, T v) { *p = v; }
template <typename T> static inline void __stcs(T* p, T v) { *p = v; }
template <typename T> static inline void __stwt(T* p, T v) { *p = v; }

// ------------------------------------------------------------------------------------------ math / bit intrinsics
static inline float rsqrtf(float x) { return 1.0f / sqrtf(x); }
static inline double rsqrt(double x) { return 1.0 / sqrt(x); }
#define __expf(x) expf(x)        /* glibc declares these names itself */
#define __logf(x) logf(x)
#define __log2f(x) log2f(x)
#define __exp2f(x) exp2f(x)
static inline float __fdividef(float a, float b) { return a / b; }
static inline float __frcp_rn(float a) { return 1.0f / a; }
static inline float __fsqrt_rn(float a) { return sqrtf(a); }
static inline float __fmaf_rn(float a, float b, float c) { return fmaf(a, b, c); }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __saturatef(float x) { return x < 0.f ? 0.f : (x > 1.f ? 1.f : x); }
static inline unsigned __float_as_uint(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
static inline int __float_as_int(float f) { int u; memcpy(&u, &f, 4); return u; }
static inline float __uint_as_float(unsigned u) { float f; memcpy(&f, &u, 4); return f; }
static inline float __int_as_float(int u) { float f; memcpy(&f, &u, 4); return f; }
static inline long long __double_as_longlong(double d) { long long u; memcpy(&u, &d, 8); return u; }
static inline double __longlong_as_double(long long u) { double d; memcpy(&d, &u, 8); return d; }
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline int __popcll(unsigned long long x) { return __builtin_popcountll(x); }
static inline int __clz(int x) { return x == 0 ? 32 : __builtin_clz((unsigned)x); }
static inline int __clzll(long long x) { return x == 0 ? 64 : __builtin_clzll((unsigned long long)x); }
static inline int __ffs(int x) { return __builtin_ffs(x); }
static inline int __ffsll(long long x) { return __builtin_ffsll(x); }
static inline unsigned __brev(unsigned x) {
    unsigned r = 0;
    for (int i = 0; i < 32; ++i) r |= ((x >> i) & 1u) << (31 - i);
    return r;
}
static inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((uint64_t)a * b) >> 32); }
static inline unsigned long long __umul64hi(unsigned long long a, unsigned long long b) { return (unsigned long long)(((unsigned __int128)a * b) >> 64); }
static inline long long clock64() { return 0; }

template <typename A, typename B> static inline typename std::common_type<A, B>::type min(A a, B b) {
    typedef typename std::common_type<A, B>::type C;
    return (C)b < (C)a ? (C)b : (C)a;
}
template <typename A, typename B> static inline typename std::common_type<A, B>::type max(A a, B b) {
    typedef typename std::common_type<A, B>::type C;
    return (C)a < (C)b ? (C)b : (C)a;
}
