// Row-sharded hot step (SURVEY section 8e, mmssl_b200/rowshard_step.py): the two kernels that connect the batch -- global
// user / item ids (main.py:368-370, :411-412 index the full tables with them) -- to a rank's row block [lo, hi).
//   gather_owned      out[j] = table[idx[j] - lo] if lo <= idx[j] < hi else 0     -> summed over ranks by one all-reduce
//                     this gives every rank the batch rows of the full table
//   scatter_add_owned table[idx[j] - lo] += src[j] for the owned j only           -> the loss kernels' gradient rows
//                     return to the rank that owns the row; duplicates (the same item drawn twice) accumulate atomically
// One thread per float4 of a row (d % 4 == 0, rows 16-byte aligned like every table of the library).
#include "spmm_common.cuh"

namespace mmssl {

__global__ void __launch_bounds__(256) gather_owned_kernel(const float* __restrict__ table, int64_t ld, const int64_t* __restrict__ idx,
                                                           int64_t lo, int64_t hi, int64_t n, int d4, float* __restrict__ out, int64_t ldo) {
    const int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (t >= n * d4) return;
    const int64_t j = t / d4;
    const int c = (int)(t - j * d4) * 4;
    const int64_t r = idx[j];
    float4 v = f4zero();
    if (r >= lo && r < hi) v = ld4(table + (r - lo) * ld + c);
    st4(out + j * ldo + c, v);
}

__global__ void __launch_bounds__(256) scatter_add_owned_kernel(float* __restrict__ table, int64_t ld, const int64_t* __restrict__ idx,
                                                                int64_t lo, int64_t hi, int64_t n, int d4, const float* __restrict__ src,
                                                                int64_t lds) {
    const int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (t >= n * d4) return;
    const int64_t j = t / d4;
    const int c = (int)(t - j * d4) * 4;
    const int64_t r = idx[j];
    if (r < lo || r >= hi) return;
    atomicAdd(reinterpret_cast<float4*>(table + (r - lo) * ld + c), ld4(src + j * lds + c));     // 128-bit reduction (sm_90+)
}

}  // namespace mmssl

using namespace mmssl;

extern "C" int mmssl_gather_owned(const float* table, int64_t ld, const int64_t* idx, int64_t lo, int64_t hi, int64_t n, int d, float* out,
                                  int64_t ldo, void* stream_) {
    MMSSL_REQUIRE(d % 4 == 0 && ld % 4 == 0 && ldo % 4 == 0 && aligned16(table) && aligned16(out), "alignment");
    MMSSL_REQUIRE(lo >= 0 && hi >= lo && n >= 0, "bad range");
    if (n == 0) return 0;
    gather_owned_kernel<<<(unsigned)((n * (d / 4) + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(table, ld, idx, lo, hi, n, d / 4, out, ldo);
    MMSSL_LAUNCH_OK();
    return 0;
}

extern "C" int mmssl_scatter_add_owned(float* table, int64_t ld, const int64_t* idx, int64_t lo, int64_t hi, int64_t n, int d,
                                       const float* src, int64_t lds, void* stream_) {
    MMSSL_REQUIRE(d % 4 == 0 && ld % 4 == 0 && lds % 4 == 0 && aligned16(table) && aligned16(src), "alignment");
    MMSSL_REQUIRE(lo >= 0 && hi >= lo && n >= 0, "bad range");
    if (n == 0) return 0;
    scatter_add_owned_kernel<<<(unsigned)((n * (d / 4) + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(table, ld, idx, lo, hi, n, d / 4, src, lds);
    MMSSL_LAUNCH_OK();
    return 0;
}

// ---- all-gather of a rank's row block without NCCL: every rank PUBLISHES its rows into every rank's copy of the full table
// (CUDA symmetric memory) -- one multimem.st per 16 bytes through the NVSwitch multicast address (y_mode 1; the switch replicates
// the store, the local copy included), or a local store plus one NVLink store per peer-mapped table (y_mode 2).  The same store
// paths as the SpMM epilogue (spmm.cu), for operands that are not SpMM outputs (projection, id fusion, parameter blocks,
// gradients).  The caller orders producers and consumers with the symmetric memory's signal-pad barrier.
namespace mmssl {
struct PublishPeers { float* p[8]; };

__global__ void __launch_bounds__(256) publish_rows_kernel(const float* __restrict__ src, int64_t lds, int64_t rows, int d4,
                                                           float* dst, int64_t ldd, int y_mode, int n_peers, PublishPeers peers) {
    const int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (t >= rows * d4) return;
    const int64_t r = t / d4;
    const int c = (int)(t - r * d4) * 4;
    const float4 v = ld4(src + r * lds + c);
    const int64_t off = r * ldd + c;
    if (y_mode == 1) {
        asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst + off), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
                     : "memory");
    } else {
        st4(dst + off, v);
        for (int q = 0; q < n_peers; ++q) st4(peers.p[q] + off, v);
    }
}
}  // namespace mmssl

extern "C" int mmssl_publish_rows(const float* src, int64_t lds, int64_t rows, int d, float* dst, int64_t ldd, int y_mode, int n_peers,
                                  float* const* peers, void* stream_) {
    MMSSL_REQUIRE(d % 4 == 0 && lds % 4 == 0 && ldd % 4 == 0 && aligned16(src) && aligned16(dst), "alignment");
    MMSSL_REQUIRE((y_mode == 1 && n_peers == 0) || (y_mode == 2 && n_peers >= 0 && n_peers <= 8) || (y_mode == 0 && n_peers == 0),
                  "y_mode 0 (local), 1 (multicast address) or 2 (local + up to 8 peers)");
    if (rows == 0) return 0;
    PublishPeers pp{};
    for (int q = 0; q < n_peers; ++q) { MMSSL_REQUIRE(aligned16(peers[q]), "peer table alignment"); pp.p[q] = peers[q]; }
    publish_rows_kernel<<<(unsigned)((rows * (d / 4) + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(src, lds, rows, d / 4, dst, ldd, y_mode,
                                                                                                     n_peers, pp);
    MMSSL_LAUNCH_OK();
    return 0;
}

// ---- all-reduce(sum) without NCCL: every rank wrote its contribution into its copy of a symmetric buffer; after a barrier each
// rank reads the SUM over all copies through the buffer's multicast address (multimem.ld_reduce: the switch adds the replicas)
// into a private result.  A second barrier lets the buffer be rewritten.  Used for the [5, B, d] batch rows and the small
// replicated gradients of the row-sharded step.
namespace mmssl {
__global__ void __launch_bounds__(256) mc_allreduce_kernel(const float* src_mc, float* __restrict__ dst, int64_t n4) {
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n4; i += (int64_t)gridDim.x * 256) {
        float4 v;
        asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
                     : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(src_mc + i * 4) : "memory");
        st4(dst + i * 4, v);
    }
}
}  // namespace mmssl

extern "C" int mmssl_mc_allreduce_sum(const float* src_mc, float* dst, int64_t n, void* stream_) {
    MMSSL_REQUIRE(n >= 0 && n % 4 == 0 && aligned16(src_mc) && aligned16(dst), "count must be a multiple of 4 floats, 16-byte aligned buffers");
    if (n == 0) return 0;
    int64_t blocks = (n / 4 + 255) / 256;
    if (blocks > kNumSMs * 8) blocks = kNumSMs * 8;
    mc_allreduce_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream_>>>(src_mc, dst, n / 4);
    MMSSL_LAUNCH_OK();
    return 0;
}

// ---- exact all-reduce(sum) of 64-bit integers (the row-sharded sampler's batch ids) through the same fp32 multicast reduction:
// an fp32 sum of the ids themselves would round them above 2^24, so each id travels as four 16-bit limbs held as floats
// (ids_to_limbs_kernel writes a rank's contribution into its copy of the symmetric buffer, one float4 per id).
// multimem.ld_reduce.add.v4.f32 then adds each limb over the ranks; a limb sum is an integer below 256 * 2^16 < 2^24 for up to
// 256 ranks, so fp32 holds it exactly, and the reassembled value is the exact integer sum mod 2^64.  The row-sharded sampler has
// one writer per entry (zeros elsewhere): the sum is that writer's id.
namespace mmssl {
__global__ void __launch_bounds__(256) ids_to_limbs_kernel(const uint64_t* __restrict__ src, float* __restrict__ dst, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) {
        const uint64_t v = src[i];
        st4(dst + i * 4, make_float4((float)(v & 0xFFFFu), (float)((v >> 16) & 0xFFFFu), (float)((v >> 32) & 0xFFFFu), (float)(v >> 48)));
    }
}

__global__ void __launch_bounds__(256) mc_allreduce_ids_kernel(const float* src_mc, uint64_t* __restrict__ dst, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) {
        float4 v;
        asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
                     : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(src_mc + i * 4) : "memory");
        dst[i] = (uint64_t)v.x + ((uint64_t)v.y << 16) + ((uint64_t)v.z << 32) + ((uint64_t)v.w << 48);
    }
}

static unsigned id_blocks(int64_t n) {
    const int64_t b = (n + 255) / 256;
    return (unsigned)(b > kNumSMs * 8 ? kNumSMs * 8 : b);
}
}  // namespace mmssl

extern "C" int mmssl_ids_to_limbs(const int64_t* src, float* dst, int64_t n, void* stream_) {
    MMSSL_REQUIRE(n >= 0 && ((uintptr_t)src % 8) == 0 && aligned16(dst), "8-byte aligned ids, 16-byte aligned limb buffer");
    if (n == 0) return 0;
    ids_to_limbs_kernel<<<id_blocks(n), 256, 0, (cudaStream_t)stream_>>>(reinterpret_cast<const uint64_t*>(src), dst, n);
    MMSSL_LAUNCH_OK();
    return 0;
}

extern "C" int mmssl_mc_allreduce_ids(const float* src_mc, int64_t* dst, int64_t n, void* stream_) {
    MMSSL_REQUIRE(n >= 0 && aligned16(src_mc) && ((uintptr_t)dst % 8) == 0, "16-byte aligned limb buffer, 8-byte aligned ids");
    if (n == 0) return 0;
    mc_allreduce_ids_kernel<<<id_blocks(n), 256, 0, (cudaStream_t)stream_>>>(src_mc, reinterpret_cast<uint64_t*>(dst), n);
    MMSSL_LAUNCH_OK();
    return 0;
}

// ---- reduce-scatter + SpMM epilogue of the row-sharded step's "partial product" schedule (rowshard_step.py): for a product
// whose dense operand lives in the LARGE (user) row space, every rank multiplies the column block of A it owns,
// A[:, U_r] * X[U_r], into its copy of a full-height partial table (symmetric memory).  After a barrier this kernel gives a rank
// the rows it owns of the SUM over the ranks' copies -- one multimem.ld_reduce per 16 bytes through the table's multicast
// address (the switch adds the replicas), or a plain load when `reduced` rows are handed in (NCCL / gloo reduce-scatter) -- and
// applies what the SpMM would have applied to a finished row: + alpha*C, row softmax / softmax backward, the store, the running
// layer sum.  Only the item-sized table crosses NVLink; the user-sized operand never moves (SURVEY 8e; VERDICT r1 #2).
namespace mmssl {
template <int G, int C, int R>
__global__ void __launch_bounds__(256) reduce_rows_epilogue_kernel(const SpmmParams p, int64_t n_rows, int multicast) {
    const unsigned gmask = group_mask<G>();
    const int lane = threadIdx.x & (G - 1);
    const int64_t row = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / G;
    if (row >= n_rows) return;            // whole group exits together
    float4 acc[R][C];
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
        for (int c = 0; c < C; ++c) {
            const float* src = p.x[r] + row * p.ldx[r] + lane * 4 + c * (4 * G);
            if (multicast) {
                asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
                             : "=f"(acc[r][c].x), "=f"(acc[r][c].y), "=f"(acc[r][c].z), "=f"(acc[r][c].w) : "l"(src) : "memory");
            } else {
                acc[r][c] = ld4(src);
            }
        }
    spmm_epilogue<G, C, R>(p, acc, (int)row, lane, gmask);
}

template <int G, int C>
static int launch_reduce_rows(const SpmmParams& p, int nrhs, int64_t n_rows, int multicast, cudaStream_t st) {
    const int T = 256;
    const int64_t blocks = (n_rows * G + T - 1) / T;
    if (blocks == 0) return 0;
    if (nrhs == 1) reduce_rows_epilogue_kernel<G, C, 1><<<(unsigned)blocks, T, 0, st>>>(p, n_rows, multicast);
    else if (nrhs == 2) reduce_rows_epilogue_kernel<G, C, 2><<<(unsigned)blocks, T, 0, st>>>(p, n_rows, multicast);
    else reduce_rows_epilogue_kernel<G, C, 3><<<(unsigned)blocks, T, 0, st>>>(p, n_rows, multicast);
    MMSSL_LAUNCH_OK();
    return 0;
}
}  // namespace mmssl

// rhs[r].x = the rank's row block inside the partial table: the MULTICAST address of its first row (multicast != 0) or a local
// pointer to already reduced rows (multicast == 0); every other field as for mmssl_spmm_csr_f32 (y, c, ysaved, s, sbase: local rows).
extern "C" int mmssl_reduce_rows_epilogue(int64_t n_rows, int d, int nrhs, const mmssl_spmm_rhs_t* rhs, int epilogue, float alpha,
                                          int s_mode, int multicast, void* stream_) {
    MMSSL_REQUIRE(n_rows >= 0 && n_rows < (1ll << 31), "row count");
    mmssl_csr_t a;
    memset(&a, 0, sizeof(a));
    a.items = reinterpret_cast<const int32_t*>(rhs);      // unused by the epilogue; fill_spmm_params only checks presence
    SpmmParams p;
    if (int rc = fill_spmm_params(p, &a, d, nrhs, rhs, epilogue, alpha, s_mode, nullptr, 0)) return rc;
    cudaStream_t st = (cudaStream_t)stream_;
    return dispatch_width(d, [&](auto G, auto C) {
        return launch_reduce_rows<decltype(G)::value, decltype(C)::value>(p, nrhs, n_rows, multicast, st);
    }, __func__);
}
