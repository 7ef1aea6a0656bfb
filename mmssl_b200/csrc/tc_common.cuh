// wgmma / TMA / mbarrier building blocks shared by the tensor-core GEMM kernels (proj_tc.cu, gemm_wide.cu, loss_tc.cu), sm_90a.
//
// CTA layout of every such kernel: warps 0-7 = two consumer warpgroups (wgmma issue, accumulators in registers, epilogue),
// warp 8 = TMA producer.  A 128-row tile is split between the warpgroups: warpgroup g owns rows 64 g .. 64 g + 63 and issues
// m64nNk16 MMAs on them against the whole N-row B tile.
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace mmssl {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;                       // bf16 elements = 128 bytes = one swizzle span
constexpr int kTileABytes = kBlockM * kBlockK * 2;   // 16 KB
constexpr int kWgRowBytes = 64 * kBlockK * 2;     // the 64 rows of one warpgroup inside an A tile: 8 KB
constexpr int kConsumerWarps = 8;
constexpr int kProducerWarp = kConsumerWarps;
constexpr int kThreads = 32 * (kConsumerWarps + 1);   // 288
constexpr int kMaxSplit = 1024;
constexpr int kMaxChainKb = 48;                  // k-blocks (64 of K each) accumulated into one register accumulator by one CTA of the split-K GEMM: 576 chained MMAs

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    uint32_t done = 0;
    uint32_t spins = 0;
    while (true) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done) : "r"(addr), "r"(parity) : "memory");
        if (done) break;
        if (++spins > (1u << 24)) __trap();   // never hang the GPU on a protocol bug
    }
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* dst, int x, int y, uint64_t hint) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
        " [%0], [%1, {%3, %4}], [%2], %5;"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(x), "r"(y), "l"(hint) : "memory");
}
__device__ __forceinline__ uint64_t make_sw128_kmajor_desc(uint32_t saddr) {
    // sm_90 GMMA shared-memory descriptor: start>>4 [0,14) | LBO>>4 [16,30) (unused for swizzled K-major, 1) |
    // SBO>>4 [32,46) = 8 rows * 128 B | base offset [49,52) = 0 (1024-byte aligned tiles) | layout SWIZZLE_128B = 1 [62,64)
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024u >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x N] += A[64 x 16] * B[N x 16]^T, bf16 operands K-major in shared memory, fp32 accumulator fragment in registers:
// d[j] holds row 16 (warp % 4) + lane / 4 + 8 ((j / 2) % 2), column 8 (j / 4) + 2 (lane % 4) + j % 2 (frag_row / frag_col).
template <int N>
__device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], uint64_t da, uint64_t db);
template <> __device__ __forceinline__ void wgmma_bf16<64>(float (&d)[32], uint64_t da, uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31"
        "}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_bf16<128>(float (&d)[64], uint64_t da, uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
        "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
        "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63"
        "}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_bf16<256>(float (&d)[128], uint64_t da, uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
        "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
        "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,"
        "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,"
        "%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,"
        "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,"
        "%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127"
        "}, %128, %129, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
          "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
          "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
          "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
          "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
          "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(da), "l"(db), "r"(1));
}


__device__ __forceinline__ int frag_row(int warp, int lane, int j) { return 16 * (warp & 3) + (lane >> 2) + 8 * ((j >> 1) & 1); }
__device__ __forceinline__ int frag_col(int lane, int j) { return 8 * (j >> 2) + 2 * (lane & 3) + (j & 1); }

// A stage's MMAs are complete: one arrival per consumer warp (empty barriers count kConsumerWarps), after every lane of the warp
// has passed its wgmma wait.
__device__ __forceinline__ void release_stage(uint64_t* bar) {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(bar);
}

// acc (+)= the k-blocks [i0, i1) of the TMA pipeline: stage s holds A_hi, A_lo (kBlockM rows each), B_hi, B_lo (N rows each);
// three MMAs per 16 of K (hi hi + hi lo + lo hi, lo lo dropped).  With two or more stages a stage is released while the next
// one's MMAs run; with one stage it must be released before the producer can refill it.
template <int N, int kStages, int kStageBytes>
__device__ __forceinline__ void mma_kblocks(float (&acc)[N / 2], uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar, int i0, int i1) {
    const int wg = (threadIdx.x >> 7);
    for (int i = i0; i < i1; ++i) {
        const int s = i % kStages;
        mbar_wait(&full_bar[s], (uint32_t)(i / kStages) & 1u);
        const uint32_t a_hi = smem_u32(smem + s * kStageBytes) + wg * kWgRowBytes;
        const uint32_t a_lo = a_hi + kTileABytes;
        const uint32_t b_hi = smem_u32(smem + s * kStageBytes) + 2 * kTileABytes;
        const uint32_t b_lo = b_hi + N * kBlockK * 2;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / 16; ++k) {
            const uint32_t off = k * 32;   // 16 bf16 = 32 bytes inside the 128-byte swizzle span
            const uint64_t dah = make_sw128_kmajor_desc(a_hi + off), dal = make_sw128_kmajor_desc(a_lo + off);
            const uint64_t dbh = make_sw128_kmajor_desc(b_hi + off), dbl = make_sw128_kmajor_desc(b_lo + off);
            wgmma_bf16<N>(acc, dah, dbh);
            wgmma_bf16<N>(acc, dah, dbl);
            wgmma_bf16<N>(acc, dal, dbh);
        }
        wgmma_commit();
        if (kStages == 1) {
            wgmma_wait<0>();
            release_stage(&empty_bar[s]);
        } else if (i > i0) {
            wgmma_wait<1>();
            release_stage(&empty_bar[(i - 1) % kStages]);
        }
    }
    if (kStages > 1) {
        wgmma_wait<0>();
        if (i1 > i0) release_stage(&empty_bar[(i1 - 1) % kStages]);
    }
}

constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;   // streamed operand (features)
constexpr uint64_t kEvictLast = 0x14F0000000000000ull;    // operand shared by every CTA (weights)

// ---- host side: tensor maps through the driver entry point (no link-time libcuda dependency) ----
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (fn == nullptr) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

static int make_map(CUtensorMap* map, const uint16_t* base, int64_t rows, int64_t ld, int box_rows) {
    EncodeTiledFn fn = get_encode_fn();
    MMSSL_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled is not available from the driver");
    cuuint64_t dims[2] = {(cuuint64_t)ld, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
    cuuint32_t box[2] = {(cuuint32_t)kBlockK, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (void*)base, dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        snprintf(last_error_buffer(), 512, "cuTensorMapEncodeTiled failed with CUresult %d (rows=%lld ld=%lld box=%d)", (int)r,
                 (long long)rows, (long long)ld, box_rows);
        return 3;
    }
    return 0;
}

}  // namespace mmssl
