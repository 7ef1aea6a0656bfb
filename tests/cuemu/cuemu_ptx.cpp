// cuemu: functional model of the inline PTX the library uses.  TEST INFRASTRUCTURE ONLY (see include/cuemu.h).
//
// Scope = exactly what csrc/tc_common.cuh and the kernels built on it issue:
//   mbarrier.init / arrive / arrive.expect_tx / try_wait.parity         phase + pending-arrival + transaction-byte counters
//   cp.async.bulk (1-D) ... mbarrier::complete_tx::bytes       contiguous copy global -> shared (spmm_hot.cu)
//   cp.async.bulk.tensor.2d ... mbarrier::complete_tx::bytes    box copy global -> shared through the tensor map: out-of-bounds
//                                                               elements read as zero, SWIZZLE_128B (address bits [4:6] ^= [7:9])
//   wgmma.mma_async.sync.aligned.m64nNk16.f32.bf16.bf16         D[64 x N] += A[64 x 16] * B[N x 16]^T, bf16 operands read from
//                                                               shared memory through K-major SWIZZLE_128B descriptors; each
//                                                               thread updates its own accumulator fragment when it issues the
//                                                               instruction (the model executes an MMA at once)
//   wgmma.fence / commit_group / wait_group                     no-ops (the MMA has already executed)
//   multimem.ld_reduce.add.v4.f32 / multimem.st.v4.f32         over multicast groups registered by the test (cuemu_mc_register):
//                                                               several ranks' replicas in one process
//   fences, prefetch.tensormap, griddepcontrol.wait             no-ops
//   ld.global[.nc] / st.global with L1:: / L2::cache_hint       plain loads and stores (.b32, .f32, .v4.f32, incl. the predicated
//                                                               @q / @!q pair of common.cuh:ldg4_l1_hot_cold); hints are not modelled
// What the model asserts on the way: 1024-byte aligned swizzled tiles, transaction bytes that add up, barrier phases, the
// descriptor fields the kernels are supposed to encode, the accumulator fragment size of the instruction shape.  A kernel that
// passes here and shares tc_common.cuh's descriptor / swizzle code with proj_tc.cu (tests/test_emu_tensor_core.py) differs
// from the kernel the GPU tests check only in its own logic.
// It says nothing about timing, asynchrony bugs that need real concurrency, or PTX outside this list (fails the launch).
#include <map>
#include <string>
#include <vector>

#include "cuda.h"

namespace cuemu {

namespace {
struct TensorMap {
    uint32_t magic;
    int elem_bytes, swizzle;
    const uint8_t* base;
    uint64_t dims[2];          // elements: [0] = contiguous dimension
    uint64_t stride1;          // bytes between rows
    uint32_t box[2];
};
static_assert(sizeof(TensorMap) <= sizeof(CUtensorMap), "tensor map record does not fit");
constexpr uint32_t kMagic = 0x7E45AB01u;

struct MBar {
    bool init = false;
    int expected = 0, pending = 0;
    int64_t tx = 0;
    unsigned phase = 0;
};
std::map<uint32_t, MBar> g_bars;

// NVSwitch multicast objects, for tests that play several ranks in one process: a fake "multicast address range" stands for n
// replicas (one buffer per rank).  multimem.st writes every replica, multimem.ld_reduce.add sums them in rank order.
struct McGroup { uint64_t base, bytes; std::vector<uint8_t*> replicas; };
std::vector<McGroup> g_mc;
const McGroup& mc_find(uint64_t addr, size_t bytes, uint64_t* off) {
    for (const McGroup& g : g_mc)
        if (addr >= g.base && addr + bytes <= g.base + g.bytes) { *off = addr - g.base; return g; }
    fail("multimem: the address is not inside a registered multicast group");
    static McGroup none{};
    *off = 0;
    return none;
}
uint8_t* smem_at(uint64_t addr, size_t bytes) {
    if (addr + bytes > dyn_smem_bytes()) fail("shared-memory address outside the block's dynamic shared memory");
    return static_cast<uint8_t*>(dyn_smem()) + addr;
}
inline uint64_t swz128(uint64_t a) { return a ^ (((a >> 7) & 7u) << 4); }
inline float bf16(uint16_t b) {
    const uint32_t u = (uint32_t)b << 16;
    float f;
    memcpy(&f, &u, 4);
    return f;
}
MBar& bar_at(uint64_t addr, bool must_exist = true) {
    if (addr % 8) fail("mbarrier address is not 8-byte aligned");
    MBar& b = g_bars[(uint32_t)addr];
    if (must_exist && !b.init) fail("mbarrier used before mbarrier.init");
    return b;
}
void bar_check(MBar& b) {
    if (b.tx < 0) fail("mbarrier: more bytes completed than expected (complete_tx without a matching expect_tx)");
    if (b.pending == 0 && b.tx == 0) {
        b.phase ^= 1u;
        b.pending = b.expected;
        note_progress();
    }
}
void bar_arrive(MBar& b) {
    if (b.pending <= 0) fail("mbarrier: more arrivals than the count it was initialised with");
    --b.pending;
    note_progress();
    bar_check(b);
}
void out32(void** outs, const int* sizes, int i, uint32_t v) {
    if (sizes[i] != 4) fail("ptx model: a 32-bit result is written to an operand of another size");
    memcpy(outs[i], &v, 4);
}
}  // namespace

CUresult encode_tiled(CUtensorMap* map, CUtensorMapDataType dt, cuuint32_t rank, void* base, const cuuint64_t* dims, const cuuint64_t* strides,
                      const cuuint32_t* box, const cuuint32_t* estr, CUtensorMapInterleave il, CUtensorMapSwizzle sw, CUtensorMapL2promotion,
                      CUtensorMapFloatOOBfill) {
    // the driver's documented requirements for the case the library uses
    if (rank != 2 || dt != CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 || il != CU_TENSOR_MAP_INTERLEAVE_NONE) return CUDA_ERROR_INVALID_VALUE;
    if (((uintptr_t)base & 15u) || (strides[0] & 15u) || strides[0] < dims[0] * 2) return CUDA_ERROR_INVALID_VALUE;
    if (box[0] == 0 || box[1] == 0 || box[0] > 256 || box[1] > 256 || estr[0] != 1 || estr[1] != 1) return CUDA_ERROR_INVALID_VALUE;
    if (sw == CU_TENSOR_MAP_SWIZZLE_128B && box[0] * 2 > 128) return CUDA_ERROR_INVALID_VALUE;      // inner box <= swizzle span
    if (sw != CU_TENSOR_MAP_SWIZZLE_128B && sw != CU_TENSOR_MAP_SWIZZLE_NONE) return CUDA_ERROR_INVALID_VALUE;
    if (dims[0] == 0 || dims[1] == 0) return CUDA_ERROR_INVALID_VALUE;
    TensorMap t{};
    t.magic = kMagic; t.elem_bytes = 2; t.swizzle = (int)sw; t.base = static_cast<const uint8_t*>(base);
    t.dims[0] = dims[0]; t.dims[1] = dims[1]; t.stride1 = strides[0]; t.box[0] = box[0]; t.box[1] = box[1];
    memset(map, 0, sizeof(*map));
    memcpy(map, &t, sizeof(t));
    return CUDA_SUCCESS;
}

void ptx_block_reset() {
    g_bars.clear();
}

void ptx_op(const char* text, void** outs, const int* out_sizes, int n_out, const uint64_t* in, int n_in) {
    auto has = [&](const char* s) { return strstr(text, s) != nullptr; };
    if (has("griddepcontrol") || has("fence.mbarrier_init") || has("prefetch.tensormap") || has("wgmma.fence") ||
        has("wgmma.commit_group") || has("wgmma.wait_group"))
        return;
    if (has("ex2.approx")) {                                  // MUFU.EX2: the model returns the correctly rounded value
        float x;
        const uint32_t xb = (uint32_t)in[0];
        memcpy(&x, &xb, 4);
        const float y = exp2f(x);
        uint32_t yb;
        memcpy(&yb, &y, 4);
        out32(outs, out_sizes, 0, yb);
        return;
    }
    if (has("mbarrier.init")) {
        MBar& b = bar_at(in[0], false);
        b = MBar();
        b.init = true;
        int count = 0;
        if (n_in >= 2) count = (int)in[1];
        else if (const char* c = strrchr(text, ',')) count = atoi(c + 1);          // immediate count in the template
        b.expected = b.pending = count;
        if (b.expected <= 0) fail("mbarrier.init with a non-positive count");
        return;
    }
    if (has("mbarrier.arrive.expect_tx")) {
        MBar& b = bar_at(in[0]);
        b.tx += (int64_t)in[1];
        bar_arrive(b);
        return;
    }
    if (has("mbarrier.arrive.shared::cta.b64 _")) {       // plain arrival (consumer release)
        bar_arrive(bar_at(in[0]));
        return;
    }
    if (has("mbarrier.try_wait.parity")) {
        MBar& b = bar_at(in[0]);
        const unsigned parity = (unsigned)in[1] & 1u;
        const bool done = b.phase != parity;     // the phase with this parity has completed
        out32(outs, out_sizes, 0, done ? 1u : 0u);
        if (!done) yield_blocked();
        return;
    }
    if (has("cp.async.cg.shared.global")) {                 // Ampere-style 16-byte asynchronous copy: executed at once in this model
        if ((in[0] % 16) || (in[1] % 16)) fail("cp.async.cg 16: addresses must be multiples of 16 bytes");
        memcpy(smem_at(in[0], 16), reinterpret_cast<const void*>((uintptr_t)in[1]), 16);
        return;
    }
    if (has("cp.async.commit_group") || has("cp.async.wait_group")) return;      // copies execute at once in this model
    if (has("cp.async.mbarrier.arrive.noinc")) {            // the lane's earlier copies have landed (model: they always have)
        bar_arrive(bar_at(in[0]));
        return;
    }
    if (has("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes")) {      // 1-D bulk copy: dst, src, bytes, barrier
        const uint64_t dst = in[0], bytes = in[2];
        if ((dst % 16) || (in[1] % 16) || (bytes % 16)) fail("cp.async.bulk: addresses and size must be multiples of 16 bytes");
        memcpy(smem_at(dst, bytes), reinterpret_cast<const void*>((uintptr_t)in[1]), bytes);
        MBar& b = bar_at(in[3]);
        b.tx -= (int64_t)bytes;
        note_progress();
        bar_check(b);
        return;
    }
    if (has("cp.async.bulk.tensor.2d")) {
        TensorMap t;
        memcpy(&t, reinterpret_cast<const void*>((uintptr_t)in[1]), sizeof(t));
        if (t.magic != kMagic) fail("cp.async.bulk.tensor: the tensor map was not made by cuTensorMapEncodeTiled");
        const uint64_t dst = in[0];
        const int64_t x = (int32_t)in[3], y = (int32_t)in[4];
        const uint32_t row_bytes = t.box[0] * t.elem_bytes;
        if (t.swizzle == CU_TENSOR_MAP_SWIZZLE_128B && (dst % 1024)) fail("TMA destination of a SWIZZLE_128B tile is not 1024-byte aligned");
        if (dst % 128) fail("TMA destination is not 128-byte aligned");
        const size_t total = (size_t)t.box[1] * row_bytes;
        uint8_t* sm = smem_at(dst, total);
        (void)sm;
        for (uint32_t r = 0; r < t.box[1]; ++r)
            for (uint32_t c = 0; c < t.box[0]; ++c) {
                const int64_t gx = x + c, gy = y + r;
                uint16_t v = 0;                                    // out of bounds reads as zero
                if (gx >= 0 && gy >= 0 && (uint64_t)gx < t.dims[0] && (uint64_t)gy < t.dims[1])
                    memcpy(&v, t.base + (uint64_t)gy * t.stride1 + (uint64_t)gx * 2, 2);
                uint64_t a = dst + (uint64_t)r * row_bytes + (uint64_t)c * 2;
                if (t.swizzle == CU_TENSOR_MAP_SWIZZLE_128B) a = swz128(a);
                memcpy(smem_at(a, 2), &v, 2);
            }
        MBar& b = bar_at(in[2]);
        b.tx -= (int64_t)total;
        note_progress();
        bar_check(b);
        return;
    }
    if (has("wgmma.mma_async")) {
        if (!has(".f32.bf16.bf16") || !has("m64n") || !has("p, 1, 1, 0, 0")) fail("wgmma: only m64nNk16.f32.bf16.bf16, unscaled, K-major operands are modelled");
        const int N = atoi(strstr(text, "m64n") + 4);
        if (N < 8 || N > 256 || (N % 8)) fail("wgmma: N must be a multiple of 8 up to 256");
        if (n_out != N / 2 || n_in != 3) fail("wgmma: an m64nNk16 fp32 accumulator fragment is N / 2 registers per thread");
        const uint64_t da = in[0], db = in[1];
        const bool acc = in[2] != 0;
        auto dec = [&](uint64_t d, uint64_t& start) {
            start = (d & 0x3FFFu) << 4;
            const uint64_t sbo = ((d >> 32) & 0x3FFFu) << 4;
            if ((d >> 62) != 1u) fail("wgmma: shared-memory descriptor is not SWIZZLE_128B (layout type 1)");
            if ((d >> 49) & 7u) fail("wgmma: base offset set (the kernels use 1024-byte aligned tiles)");
            if (sbo != 1024) fail("wgmma: stride-byte-offset of a K-major SWIZZLE_128B tile must be 1024 (8 rows x 128 B)");
            if ((start & ~(uint64_t)127) % 1024) fail("wgmma: swizzled operand tile is not 1024-byte aligned");
        };
        uint64_t sa, sb;
        dec(da, sa);
        dec(db, sb);
        auto elem = [&](uint64_t start, int row, int k) {
            const uint64_t a = swz128(start + (uint64_t)(row / 8) * 1024 + (uint64_t)(row % 8) * 128 + (uint64_t)k * 2);
            uint16_t v;
            memcpy(&v, smem_at(a, 2), 2);
            return bf16(v);
        };
        const int w = cur->warp % 4, l = cur->lane;
        for (int j = 0; j < N / 2; ++j) {          // the thread's fragment (tc_common.cuh: frag_row / frag_col)
            const int row = 16 * w + l / 4 + 8 * ((j / 2) % 2), col = 8 * (j / 4) + 2 * (l % 4) + j % 2;
            if (out_sizes[j] != 4) fail("wgmma: accumulator registers are 32-bit");
            float d;
            memcpy(&d, outs[j], 4);
            if (!acc) d = 0.f;
            for (int k = 0; k < 16; ++k) d += elem(sa, row, k) * elem(sb, col, k);
            memcpy(outs[j], &d, 4);
        }
        note_progress();
        return;
    }
    if (has("multimem.ld_reduce") && has("add.v4.f32")) {
        uint64_t off;
        const McGroup& g = mc_find(in[0], 16, &off);
        if (in[0] % 16) fail("multimem.ld_reduce.v4: misaligned address");
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        for (uint8_t* r : g.replicas) {
            float v[4];
            memcpy(v, r + off, 16);
            for (int k = 0; k < 4; ++k) acc[k] += v[k];
        }
        for (int k = 0; k < 4; ++k) {
            uint32_t u;
            memcpy(&u, &acc[k], 4);
            out32(outs, out_sizes, k, u);
        }
        return;
    }
    if (has("multimem.st") && has("v4.f32")) {
        uint64_t off;
        const McGroup& g = mc_find(in[0], 16, &off);
        if (in[0] % 16) fail("multimem.st.v4: misaligned address");
        uint32_t v[4] = {(uint32_t)in[1], (uint32_t)in[2], (uint32_t)in[3], (uint32_t)in[4]};
        for (uint8_t* r : g.replicas) memcpy(r + off, v, 16);
        return;
    }
    if ((has("ld.global") || has("st.global")) && (has("L2::cache_hint") || has("L1::"))) {
        // cache-hinted loads / stores (common.cuh): plain memory accesses here, the hints only steer residency.  A load
        // writes n_out consecutive 32-bit values from in[0]; the predicated @q / @!q pair of ldg4_l1_hot_cold loads the same
        // address into the same registers on both branches, so it is one load.  A store takes the address and its values,
        // then the policy word.
        const bool st = has("st.global");
        const int nv = st ? n_in - 2 : n_out;
        if (nv != 1 && nv != 4) fail("cache-hinted access: only .b32 / .f32 and .v4.f32 are modelled");
        if (in[0] % (4u * (unsigned)nv)) fail("cache-hinted access: misaligned address");
        if (st) {
            uint32_t v[4];
            for (int k = 0; k < nv; ++k) v[k] = (uint32_t)in[1 + k];
            memcpy(reinterpret_cast<void*>((uintptr_t)in[0]), v, 4 * nv);
        } else {
            uint32_t v[4];
            memcpy(v, reinterpret_cast<const void*>((uintptr_t)in[0]), 4 * nv);
            for (int k = 0; k < nv; ++k) out32(outs, out_sizes, k, v[k]);
        }
        return;
    }
    std::string m = std::string("inline PTX is not emulated: ") + text;
    fail(m.c_str());
}

}  // namespace cuemu

extern "C" void cuemu_mc_register(uint64_t base, uint64_t bytes, int n, void** replicas) {
    cuemu::McGroup g;
    g.base = base; g.bytes = bytes;
    for (int i = 0; i < n; ++i) g.replicas.push_back(static_cast<uint8_t*>(replicas[i]));
    cuemu::g_mc.push_back(g);
}
extern "C" void cuemu_mc_clear() { cuemu::g_mc.clear(); }
