// Kernels that exercise the emulator itself (tests/test_emu_selftest.py): correct ones with known answers and
// deliberately broken ones that the emulator must catch.  CUDA syntax, compiled through the same rewrite as csrc/*.cu.
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
using namespace mmssl;

__global__ void st_shuffles(int* out) {          // out[5][blockDim.x]
    const int t = threadIdx.x, lane = t & 31, n = blockDim.x;
    int v = t * 3 + 1;
    out[0 * n + t] = __shfl_xor_sync(0xffffffffu, v, 5);
    out[1 * n + t] = __shfl_down_sync(0xffffffffu, v, 3, 16);
    out[2 * n + t] = __shfl_up_sync(0xffffffffu, v, 2, 8);
    out[3 * n + t] = __shfl_sync(0xffffffffu, v, 7, 16);
    out[4 * n + t] = (int)__ballot_sync(0xffffffffu, (lane % 3) == 0);
}

// half-warp groups with group-local masks, both halves active at the same time
__global__ void st_group_masks(float* out) {
    const int t = threadIdx.x, lane = t & 31;
    const unsigned mask = (lane < 16) ? 0x0000ffffu : 0xffff0000u;
    float v = (float)(t + 1);
    for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(mask, v, o, 16);
    out[t] = v;
}

__global__ void st_block_reduce(const float* x, int n, float* out, int* flags) {
    __shared__ float sh[256];
    extern __shared__ float dyn[];
    const int t = threadIdx.x;
    float s = 0.f;
    for (int i = blockIdx.x * blockDim.x + t; i < n; i += gridDim.x * blockDim.x) s += x[i];
    sh[t] = s;
    dyn[t] = s;
    __syncthreads();
    for (int o = blockDim.x / 2; o > 0; o >>= 1) {
        if (t < o) sh[t] += sh[t + o];
        __syncthreads();
    }
    const int any = __syncthreads_or(t == 3), all = __syncthreads_and(t < 1000), cnt = __syncthreads_count(t % 2);
    if (t == 0) {
        atomicAdd(out, sh[0]);
        flags[0] = any; flags[1] = all; flags[2] = cnt;
        flags[3] = (dyn[blockDim.x - 1] == dyn[blockDim.x - 1]);   // written by another thread before the barrier
    }
}

// early exit of whole warps and of single lanes before barriers / shuffles: legal, the hardware ignores exited threads
__global__ void st_early_exit(int* out, int limit) {
    const int t = threadIdx.x;
    if (t >= limit) return;
    int v = 1;
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    out[t] = v;
}

// BROKEN: neighbour read without a barrier -> the result depends on the thread order
__global__ void st_missing_barrier(int* out) {
    __shared__ int sh[64];
    const int t = threadIdx.x;
    sh[t] = t + 100;
    out[t] = sh[(t + 1) % 64];
}

// BROKEN: full mask while half of the warp is in another branch and never arrives
__global__ void st_bad_mask(int* out) {
    const int t = threadIdx.x;
    if ((t & 31) < 16) out[t] = __shfl_xor_sync(0xffffffffu, t, 1);
    else { __syncthreads(); out[t] = t; }
    __syncthreads();
}

__global__ void st_ptx(int* out) {
    asm volatile("griddepcontrol.wait;" ::: "memory");
    out[0] = 1;
    if (out[1] == 7) asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %1, %1, %1};" ::"l"(out), "f"(1.f) : "memory");
}

// the cache-hinted accesses of common.cuh: out[0..3] <- stream loads, out[4..7] <- L2-policy / L1 hot / cold loads of a
// (hot and cold alike), out[8] <- b32 stream load, out[9] <- f32 stream load; out[12..15] <- st4_stream of out[0..3] + 1
__global__ void st_cache_hints(const float* a, float* out) {
    const float4 v = ldg4_stream(a), w = ld4_stream(a + 4);
    const float4 l2 = ldg4_l2(a + 8, kL2EvictLast), hot = ldg4_l1_hot_cold(a + 12, 1, kL2EvictLast), cold = ldg4_l1_hot_cold(a + 16, 0, 0);
    out[0] = v.x; out[1] = v.y; out[2] = w.z; out[3] = w.w;
    out[4] = l2.x; out[5] = hot.y; out[6] = cold.z; out[7] = cold.w;
    out[8] = (float)ldg_i32_stream(reinterpret_cast<const int*>(a + 20));
    out[9] = ldg_f32_stream(a + 21);
    st4_stream(out + 12, make_float4(out[0] + 1.f, out[1] + 1.f, out[2] + 1.f, out[3] + 1.f));
}

extern "C" int cuemu_st_run(int which, void* a, void* b, void* c, int n, int block, int grid) {
    cudaGetLastError();
    switch (which) {
        case 0: st_shuffles<<<1, block>>>((int*)a); break;
        case 1: st_group_masks<<<1, block>>>((float*)a); break;
        case 2: st_block_reduce<<<grid, block, block * sizeof(float)>>>((const float*)a, n, (float*)b, (int*)c); break;
        case 3: st_early_exit<<<1, block>>>((int*)a, n); break;
        case 4: st_missing_barrier<<<1, 64>>>((int*)a); break;
        case 6: st_bad_mask<<<1, 64>>>((int*)a); break;
        case 7: st_ptx<<<1, 1>>>((int*)a); break;
        case 8: st_shuffles<<<1, 2048>>>((int*)a); break;       // invalid configuration
        case 9: st_cache_hints<<<1, 1>>>((const float*)a, (float*)b); break;
        default: return -1;
    }
    return (int)cudaPeekAtLastError();
}
extern "C" const char* cuemu_st_error(void) { return cudaGetErrorString(cudaPeekAtLastError()); }
