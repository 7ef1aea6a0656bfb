// SpMM variant for large power-law graphs: the rows of X that belong to the highest-degree columns
// ("hot" neighbours) are staged ONCE per CTA into shared memory by TMA bulk copies
// (cp.async.bulk, mbarrier complete_tx) and every gather of a hot neighbour is served from shared
// memory; only cold neighbours go through the L2 gather path.
//
// Why: at 1M x 200k / 20M edges the LDG kernel (spmm.cu) is bound by the L2 -> SM gather stream
// (each of the nnz neighbour rows crosses L2 once: 4*d*nnz bytes), not by HBM.  With
// Zipf-like item popularity a few hundred columns carry about half of the edges, and ~200 KB of
// shared memory holds 400 (d=128) .. 800 (d=64) rows, so about half of that stream disappears.
//
// Same operator contract, work plan, split-row protocol and epilogues as spmm_csr_kernel; the grid is
// persistent (one CTA of 1024 threads per SM) so the staging cost is paid once per SM per launch.
// `colidx_hot` is the operand's column index array with hot columns encoded as -(slot+1)
// (slots ordered by decreasing degree; slots beyond the staged count fall back to hot_ids[slot]).
#include "spmm_common.cuh"

namespace mmssl {

constexpr int kHotThreads = 1024;
constexpr int kHotSmemBytes = 200 * 1024;

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void hot_mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_addr(bar);
    uint32_t done = 0, spins = 0;
    while (true) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done) : "r"(addr), "r"(parity) : "memory");
        if (done) break;
        if (++spins > (1u << 24)) __trap();
    }
}

template <int G, int C, int R>
__global__ void __launch_bounds__(kHotThreads, 1)
spmm_hot_kernel(const SpmmParams p, const int32_t* __restrict__ colidx_hot, const int32_t* __restrict__ hot_ids,
                int n_staged) {
    constexpr int D = 4 * G * C;
    constexpr int RC = R * C;
    constexpr int UNR = (8 / RC) >= 2 ? (8 / RC) : 2;
    constexpr int W = R * D;
    extern __shared__ __align__(128) uint8_t smem_raw[];
    float* hot = reinterpret_cast<float*>(smem_raw);                       // [n_staged][R][D]
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw + (size_t)n_staged * W * 4);

    // ---- stage the hot rows with TMA bulk copies (one mbarrier, byte-count completion) ----
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_addr(bar)));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x < 32) {
        if (threadIdx.x == 0)
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"((uint32_t)(n_staged * W * 4)) : "memory");
        __syncwarp();
        for (int s = threadIdx.x; s < n_staged; s += 32) {
            const int64_t col = __ldg(hot_ids + s);
#pragma unroll
            for (int r = 0; r < R; ++r) {
                const float* src = p.x[r] + col * p.ldx[r];
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             ::"r"(smem_addr(hot + ((size_t)s * R + r) * D)), "l"(src), "r"((uint32_t)(D * 4)), "r"(smem_addr(bar)) : "memory");
            }
        }
    }
    hot_mbar_wait(bar, 0);

    const unsigned gmask = group_mask<G>();
    const int lane = threadIdx.x & (G - 1);
    const int64_t gstride = (int64_t)gridDim.x * (blockDim.x / G);
    int64_t it = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / G;
    int4 item = make_int4(-1, 0, 0, -1);
    if (it < p.n_items) item = __ldg(&p.items[it]);
    int c_nxt = 0;
    float v_nxt = 0.f;
    if (item.x >= 0 && item.y + lane < item.z) { c_nxt = __ldg(colidx_hot + item.y + lane); v_nxt = __ldg(p.vals + item.y + lane); }

    for (; it < p.n_items; it += gstride) {
        const int row = item.x, begin = item.y, end = item.z, splitw = item.w;
        int4 item2 = make_int4(-1, 0, 0, -1);
        if (it + gstride < p.n_items) item2 = __ldg(&p.items[it + gstride]);
        int c_first2 = 0;
        float v_first2 = 0.f;
        bool first2_done = false;
        if (row >= 0) {
            float4 acc[R][C];
#pragma unroll
            for (int r = 0; r < R; ++r)
#pragma unroll
                for (int c = 0; c < C; ++c) acc[r][c] = f4zero();

            for (int base = begin; base < end; base += G) {
                const int c_l = c_nxt;
                const float v_l = v_nxt;
                c_nxt = 0; v_nxt = 0.f;
                if (base + G < end) {
                    const int e2 = base + G + lane;
                    if (e2 < end) { c_nxt = __ldg(colidx_hot + e2); v_nxt = __ldg(p.vals + e2); }
                } else if (item2.x >= 0) {
                    if (item2.y + lane < item2.z) { c_first2 = __ldg(colidx_hot + item2.y + lane); v_first2 = __ldg(p.vals + item2.y + lane); }
                    first2_done = true;
                }
                const int cnt = min(G, end - base);
                for (int j = 0; j < cnt; j += UNR) {
                    int cc[UNR];
                    float vv[UNR];
#pragma unroll
                    for (int k = 0; k < UNR; ++k) {
                        cc[k] = __shfl_sync(gmask, c_l, j + k, G);
                        vv[k] = __shfl_sync(gmask, v_l, j + k, G);
                    }
                    float4 xv[UNR][R][C];
#pragma unroll
                    for (int k = 0; k < UNR; ++k) {
                        const bool on = (j + k) < cnt;
                        int col = cc[k];
                        int slot = -1;
                        if (col < 0) {                                  // hot column
                            slot = -col - 1;
                            if (slot >= n_staged) { col = __ldg(hot_ids + slot); slot = -1; }
                        }
#pragma unroll
                        for (int r = 0; r < R; ++r) {
#pragma unroll
                            for (int c = 0; c < C; ++c) {
                                float4 v = f4zero();
                                if (on) {
                                    if (slot >= 0) v = *reinterpret_cast<const float4*>(hot + ((size_t)slot * R + r) * D + lane * 4 + c * (4 * G));
                                    else v = ldg4(p.x[r] + (int64_t)col * p.ldx[r] + lane * 4 + c * (4 * G));
                                }
                                xv[k][r][c] = v;
                            }
                        }
                    }
#pragma unroll
                    for (int k = 0; k < UNR; ++k)
#pragma unroll
                        for (int r = 0; r < R; ++r)
#pragma unroll
                            for (int c = 0; c < C; ++c) fma4(acc[r][c], vv[k], xv[k][r][c]);
                }
            }

            // ---- split rows (same protocol as spmm_csr_kernel) ----
            bool finish = true;
            if (splitw >= 0) {
                const int4 st = __ldg(&p.split_table[splitw]);
                if (st.w != 0) {
                    float* slotp = p.partials + (int64_t)st.x * W;
#pragma unroll
                    for (int r = 0; r < R; ++r)
#pragma unroll
                        for (int c = 0; c < C; ++c)
                            atomicAdd(reinterpret_cast<float4*>(slotp + (r * C + c) * (4 * G) + lane * 4), acc[r][c]);
                } else {
                    const int k = (begin - __ldg(p.rowptr + row)) / st.z;
                    float* part = p.partials + ((int64_t)st.x + k) * W;
#pragma unroll
                    for (int r = 0; r < R; ++r)
#pragma unroll
                        for (int c = 0; c < C; ++c) st4(part + (r * C + c) * (4 * G) + lane * 4, acc[r][c]);
                }
                __threadfence();
                __syncwarp(gmask);
                int old = 0;
                if (lane == 0) old = atomicAdd(p.counters + splitw, 1);
                old = __shfl_sync(gmask, old, 0, G);
                finish = (old == st.y - 1);
                if (finish) {
                    __threadfence();
                    if (lane == 0) p.counters[splitw] = 0;
                    if (st.w != 0) {
                        float* slotp = p.partials + (int64_t)st.x * W;
#pragma unroll
                        for (int r = 0; r < R; ++r)
#pragma unroll
                            for (int c = 0; c < C; ++c) {
                                float* q = slotp + (r * C + c) * (4 * G) + lane * 4;
                                acc[r][c] = ldcg4(q);
                                __stcg(reinterpret_cast<float4*>(q), f4zero());
                            }
                    } else {
#pragma unroll
                        for (int r = 0; r < R; ++r)
#pragma unroll
                            for (int c = 0; c < C; ++c) acc[r][c] = f4zero();
                        constexpr int PB = (8 / RC) >= 1 ? (8 / RC) : 1;
                        for (int s0 = 0; s0 < st.y; s0 += PB) {
                            float4 pv[PB][R][C];
#pragma unroll
                            for (int q = 0; q < PB; ++q) {
                                const bool on = (s0 + q) < st.y;
                                const float* ps = p.partials + ((int64_t)st.x + s0 + q) * W;
#pragma unroll
                                for (int r = 0; r < R; ++r)
#pragma unroll
                                    for (int c = 0; c < C; ++c)
                                        pv[q][r][c] = on ? ldcg4(ps + (r * C + c) * (4 * G) + lane * 4) : f4zero();
                            }
#pragma unroll
                            for (int q = 0; q < PB; ++q)
#pragma unroll
                                for (int r = 0; r < R; ++r)
#pragma unroll
                                    for (int c = 0; c < C; ++c) acc[r][c] = add4(acc[r][c], pv[q][r][c]);
                        }
                    }
                }
            }
            if (finish) spmm_epilogue<G, C, R>(p, acc, row, lane, gmask);
        }
        if (!first2_done && item2.x >= 0 && item2.y + lane < item2.z) {
            c_first2 = __ldg(colidx_hot + item2.y + lane); v_first2 = __ldg(p.vals + item2.y + lane);
        }
        item = item2; c_nxt = c_first2; v_nxt = v_first2;
    }
}

template <int G, int C, int R>
static int launch_hot(const SpmmParams& p, const int32_t* colidx_hot, const int32_t* hot_ids, int n_hot, cudaStream_t stream) {
    constexpr int D = 4 * G * C;
    const int cap = (kHotSmemBytes - 64) / (R * D * 4);
    const int n_staged = n_hot < cap ? n_hot : cap;
    const int smem = n_staged * R * D * 4 + 64;
    static bool attr = false;
    if (!attr) {
        MMSSL_CUDA(cudaFuncSetAttribute(spmm_hot_kernel<G, C, R>, cudaFuncAttributeMaxDynamicSharedMemorySize, kHotSmemBytes));
        attr = true;
    }
    int64_t blocks = (p.n_items + (kHotThreads / G) - 1) / (kHotThreads / G);
    if (blocks > kNumSMs) blocks = kNumSMs;
    if (blocks == 0) return 0;
    spmm_hot_kernel<G, C, R><<<(unsigned)blocks, kHotThreads, smem, stream>>>(p, colidx_hot, hot_ids, n_staged);
    MMSSL_LAUNCH_OK();
    return 0;
}

int launch_spmm_hot(const SpmmParams& p, int d, int nrhs, const int32_t* colidx_hot, const int32_t* hot_ids, int n_hot,
                    cudaStream_t stream) {
#define MMSSL_HOT_CASE(G, C)                                                            \
    switch (nrhs) {                                                                     \
        case 1: return launch_hot<G, C, 1>(p, colidx_hot, hot_ids, n_hot, stream);      \
        case 2: return launch_hot<G, C, 2>(p, colidx_hot, hot_ids, n_hot, stream);      \
        default: return launch_hot<G, C, 3>(p, colidx_hot, hot_ids, n_hot, stream);     \
    }
    if (d == 64) { MMSSL_HOT_CASE(16, 1) }
    if (d == 128) { MMSSL_HOT_CASE(32, 1) }
    MMSSL_HOT_CASE(32, 2)
#undef MMSSL_HOT_CASE
}

}  // namespace mmssl

using namespace mmssl;

extern "C" int mmssl_spmm_hot_f32(const mmssl_csr_t* a, const int32_t* colidx_hot, const int32_t* hot_ids, int n_hot, int d,
                                  int nrhs, const mmssl_spmm_rhs_t* rhs, int epilogue, float alpha, int s_mode,
                                  float* partials, int64_t partials_floats, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    MMSSL_REQUIRE(colidx_hot != nullptr && hot_ids != nullptr && n_hot >= 0, "missing hot-column plan");
    SpmmParams p;
    if (int rc = fill_spmm_params(p, a, d, nrhs, rhs, epilogue, alpha, s_mode, partials, partials_floats)) return rc;
    for (int r = 0; r < nrhs; ++r) MMSSL_REQUIRE(p.ldx[r] % 4 == 0, "TMA staging needs 16-byte aligned rows");
    return launch_spmm_hot(p, d, nrhs, colidx_hot, hot_ids, n_hot, stream);
}
