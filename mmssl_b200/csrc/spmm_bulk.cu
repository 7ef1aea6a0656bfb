// SpMM, staged-gather pipeline:  Y_r = epilogue( A * X_r ),  r < nrhs  -- same operator contract as spmm.cu
// (reference: MMSSL.mm / torch.sparse.mm, Models.py:69-73, and torch.mm(sparse, dense), Models.py:203-208).
//
// Why a second kernel.  The LDG kernel (spmm.cu) keeps the neighbour rows it has in flight in REGISTERS: 8 float4 per lane, so a
// row walk of n non-zeros costs n/8 dependent memory round trips (up to 8 for its longest work item).  Here the neighbour rows are
// staged through shared memory by asynchronous copies: no register holds a row in flight, and ALL rows of a work unit (up to 32)
// are requested before the first one is consumed.
//
// Work decomposition (plan: graph.cu, mmssl_spmm_bulk_plan): BUCKETS of at most 32 consecutive non-zeros -- one position per
// lane -- that never cut a row of <= 32 non-zeros: a bucket is up to 8 consecutive whole rows, or one 32-chunk of a longer row.
// One warp owns one bucket:
//   round trip 1   the bucket descriptor {first row, #rows, first position, #positions}, {split-row slot, chunk index}
//   round trip 2   (col, val) of its positions and the row pointers of its rows, coalesced, parked in shared memory
//   round trip 3   every neighbour row of the bucket and the row-indexed epilogue operands of its rows (alpha*C[row], saved
//                  softmax output, running-sum base): asynchronous copies into the warp's shared-memory slots
//   then           accumulate from shared memory (every lane owns d/32 columns of every right-hand side), epilogue, store.
// Chunks of long rows publish partial sums; the last chunk to arrive adds them in chunk order (deterministic), as in spmm.cu;
// rows of more than 32 chunks accumulate with vector reductions into a zeroed slot instead.
//
// Two copy engines, same pipeline (template parameter TMA):
//   LDGSTS the whole warp issues 16-byte cp.async copies (512 B per instruction: one d=128 row, two d=64 rows), completion by
//          cp.async.wait_group.
//   TMA    one cp.async.bulk per neighbour row, issued by the lane that owns the position, completion counted in bytes on an
//          mbarrier (the arrangement north_star sketches).
// Shared memory per warp: 32 slots x (nrhs * d * 4) bytes + 8 rows per staged epilogue operand + 0.5 KB of indices.
// No tensor cores: the contraction is a sparse gather.
#include "spmm_common.cuh"

namespace mmssl {

constexpr int kBk = 32;        // positions per bucket (one per lane)
constexpr int kBkRows = 8;     // rows per bucket (= rows of epilogue operands staged per bucket)

struct BulkParams {
    SpmmParams p;
    const int4* buckets;       // [n_buckets][2]: {row0, n_rows, nz0, count}, {split (-1: whole rows), chunk index, 0, 0}
    int64_t n_buckets;
    int tasks_per_warp;
    int n_ops;                 // staged epilogue operands: 0, 1 or 2   (A = alpha*C, B = ysaved | S | SB)
    int warp_bytes;            // shared memory per warp
};

__device__ __forceinline__ uint32_t bsm(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void bk_mbar_init(uint64_t* bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bsm(bar)), "r"(count)); }
__device__ __forceinline__ void bk_cp16(void* dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(bsm(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void bk_cp_commit_wait() {
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 0;" ::: "memory");
}
__device__ __forceinline__ void bk_expect(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bsm(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bk_copy(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(bsm(dst)), "l"(src), "r"(bytes), "r"(bsm(bar)) : "memory");
}
__device__ __forceinline__ void bk_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = bsm(bar);
    uint32_t done = 0, spins = 0;
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

// Lane layout of a d-wide row: V = d/32 floats per lane in chunks of CW (vector width) floats.
template <int V>
struct Lay {
    static constexpr int CW = V >= 4 ? 4 : 2;
    static constexpr int NCH = V / CW;
    __device__ static __forceinline__ int off(int lane, int ch) { return ch * (32 * CW) + lane * CW; }
};
template <int CW> __device__ __forceinline__ void ldv(float (&dst)[CW], const float* src);
template <> __device__ __forceinline__ void ldv<2>(float (&dst)[2], const float* src) {
    const float2 v = *reinterpret_cast<const float2*>(src); dst[0] = v.x; dst[1] = v.y;
}
template <> __device__ __forceinline__ void ldv<4>(float (&dst)[4], const float* src) {
    const float4 v = *reinterpret_cast<const float4*>(src); dst[0] = v.x; dst[1] = v.y; dst[2] = v.z; dst[3] = v.w;
}
template <int CW> __device__ __forceinline__ void ldv_cg(float (&dst)[CW], const float* src);
template <> __device__ __forceinline__ void ldv_cg<2>(float (&dst)[2], const float* src) {
    const float2 v = __ldcg(reinterpret_cast<const float2*>(src)); dst[0] = v.x; dst[1] = v.y;
}
template <> __device__ __forceinline__ void ldv_cg<4>(float (&dst)[4], const float* src) {
    const float4 v = __ldcg(reinterpret_cast<const float4*>(src)); dst[0] = v.x; dst[1] = v.y; dst[2] = v.z; dst[3] = v.w;
}
template <int CW> __device__ __forceinline__ void stv(float* dst, const float (&v)[CW]);
template <> __device__ __forceinline__ void stv<2>(float* dst, const float (&v)[2]) { *reinterpret_cast<float2*>(dst) = make_float2(v[0], v[1]); }
template <> __device__ __forceinline__ void stv<4>(float* dst, const float (&v)[4]) { *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]); }
template <int CW> __device__ __forceinline__ void stv_cg(float* dst, const float (&v)[CW]);
template <> __device__ __forceinline__ void stv_cg<2>(float* dst, const float (&v)[2]) { __stcg(reinterpret_cast<float2*>(dst), make_float2(v[0], v[1])); }
template <> __device__ __forceinline__ void stv_cg<4>(float* dst, const float (&v)[4]) { __stcg(reinterpret_cast<float4*>(dst), make_float4(v[0], v[1], v[2], v[3])); }
template <int CW> __device__ __forceinline__ void redv(float* dst, const float (&v)[CW]);
template <> __device__ __forceinline__ void redv<2>(float* dst, const float (&v)[2]) { atomicAdd(reinterpret_cast<float2*>(dst), make_float2(v[0], v[1])); }
template <> __device__ __forceinline__ void redv<4>(float* dst, const float (&v)[4]) { atomicAdd(reinterpret_cast<float4*>(dst), make_float4(v[0], v[1], v[2], v[3])); }
template <int CW> __device__ __forceinline__ void mcstv(float* dst, const float (&v)[CW]);
template <> __device__ __forceinline__ void mcstv<2>(float* dst, const float (&v)[2]) {
    asm volatile("multimem.st.relaxed.sys.global.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(v[0]), "f"(v[1]) : "memory");
}
template <> __device__ __forceinline__ void mcstv<4>(float* dst, const float (&v)[4]) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(v[0]), "f"(v[1]), "f"(v[2]), "f"(v[3]) : "memory");
}

// Warp-cooperative copy of one D-float row (16 bytes per lane per instruction): rows of 64 floats take a half warp, so two rows
// travel per instruction; 128 floats one instruction; 256 floats two.
template <int D>
__device__ __forceinline__ void bk_row_ldgsts(float* dst, const float* src, int lane, bool on) {
    if (D == 64) {
        if (on) bk_cp16(dst + (lane & 15) * 4, src + (lane & 15) * 4);
    } else {
#pragma unroll
        for (int o = 0; o < D; o += 128)
            if (on) bk_cp16(dst + o + lane * 4, src + o + lane * 4);
    }
}

// V floats per lane (d = 32 V), R right-hand sides, TMA: copy engine (see the file header).
template <int V, int R, bool TMA>
__global__ void __launch_bounds__(256) spmm_bulk_kernel(const BulkParams bp) {
    using L = Lay<V>;
    constexpr int CW = L::CW, NCH = L::NCH;
    constexpr int D = 32 * V;
    constexpr int RD = R * D;                       // floats per slot / staged operand row
    constexpr uint32_t ROWB = RD * 4;
    constexpr int RPI = (D == 64) ? 2 : 1;          // rows per LDGSTS instruction
    const SpmmParams& p = bp.p;
    extern __shared__ __align__(128) uint8_t smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint8_t* wbase = smem_raw + (size_t)warp * bp.warp_bytes;
    float* ring = reinterpret_cast<float*>(wbase);                                   // [32][RD]
    float* stg = ring + kBk * RD;                                                    // [n_ops][kBkRows][RD]
    int* cols_s = reinterpret_cast<int*>(stg + (size_t)bp.n_ops * kBkRows * RD);     // [32]
    float* vals_s = reinterpret_cast<float*>(cols_s + kBk);                          // [32]
    int* bnd_s = reinterpret_cast<int*>(vals_s + kBk);                               // [kBkRows + 1] (+ padding to 16)
    uint64_t* bar = reinterpret_cast<uint64_t*>(bnd_s + 16);
    uint32_t phase = 0;
    if (TMA) {
        if (lane == 0) {
            bk_mbar_init(bar, 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncwarp();
    }
    pdl_wait();

    const int64_t gwarp = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
    const int64_t t_begin = gwarp * bp.tasks_per_warp;
    const int64_t t_end = min(bp.n_buckets, t_begin + bp.tasks_per_warp);
    const bool has_a = p.has_c != 0;
    const bool has_b = bp.n_ops > (has_a ? 1 : 0);

    for (int64_t t = t_begin; t < t_end; ++t) {
        // ---- round trip 1: descriptor
        const int4 d0 = __ldg(&bp.buckets[2 * t]), d1 = __ldg(&bp.buckets[2 * t + 1]);
        const int row0 = d0.x, n_rows = d0.y, nz0 = d0.z, cnt = d0.w;
        const int sp = d1.x, seg = d1.y;
        if (n_rows <= 0) continue;
        // ---- round trip 2: indices, values, row bounds (relative to nz0), split-row entry
        int c = 0;
        float v = 0.f;
        if (lane < cnt) { c = __ldg(p.colidx + nz0 + lane); v = __ldg(p.vals + nz0 + lane); }
        int bnd = 0;
        if (sp >= 0) bnd = (lane == 0) ? 0 : cnt;
        else if (lane <= n_rows) bnd = __ldg(p.rowptr + row0 + lane) - nz0;
        int4 st = make_int4(0, 0, 0, 0);
        if (sp >= 0) st = __ldg(&p.split_table[sp]);                 // {first partial slot, #chunks, -, heavy}: same address in every lane
        __syncwarp();                                                 // every lane has finished reading the previous bucket's slots
        cols_s[lane] = c;
        vals_s[lane] = v;
        if (lane <= kBkRows) bnd_s[lane] = bnd;
        __syncwarp();

        // ---- round trip 3: neighbour rows -> slots, epilogue operands of the bucket's rows -> staging
        if (TMA) {
            if (lane == 0) bk_expect(bar, (uint32_t)(cnt + n_rows * bp.n_ops) * ROWB);
            __syncwarp();
            if (lane < cnt) {
#pragma unroll
                for (int r = 0; r < R; ++r) bk_copy(ring + (size_t)lane * RD + r * D, p.x[r] + (int64_t)c * p.ldx[r], D * 4, bar);
            }
            if (lane < n_rows) {
                const int64_t row = row0 + lane;
                int o = 0;
                if (has_a) {
#pragma unroll
                    for (int r = 0; r < R; ++r) bk_copy(stg + (size_t)lane * RD + r * D, p.c[r] + row * p.ldc[r], D * 4, bar);
                    o = 1;
                }
                if (has_b) {
#pragma unroll
                    for (int r = 0; r < R; ++r) {
                        const float* src = (p.epilogue == MMSSL_EPI_SOFTMAX_BWD) ? p.ys[r] + row * p.ldys[r]
                                           : (p.s_mode == 2)                     ? p.sb[r] + row * p.ldsb[r]
                                                                                 : p.s[r] + row * p.lds[r];
                        bk_copy(stg + (size_t)(o * kBkRows + lane) * RD + r * D, src, D * 4, bar);
                    }
                }
            }
            bk_wait(bar, phase);
            phase ^= 1u;
        } else {
            for (int j = 0; j < cnt; j += RPI) {
                const int mj = j + (RPI == 2 ? (lane >> 4) : 0);
                const int col = cols_s[mj & (kBk - 1)];
                float* dst = ring + (size_t)mj * RD;
#pragma unroll
                for (int r = 0; r < R; ++r) bk_row_ldgsts<D>(dst + r * D, p.x[r] + (int64_t)col * p.ldx[r], lane, mj < cnt);
            }
            if (bp.n_ops > 0) {
                for (int i = 0; i < n_rows; i += RPI) {
                    const int mi = i + (RPI == 2 ? (lane >> 4) : 0);
                    const int64_t row = row0 + min(mi, n_rows - 1);
                    int o = 0;
                    if (has_a) {
#pragma unroll
                        for (int r = 0; r < R; ++r) bk_row_ldgsts<D>(stg + (size_t)mi * RD + r * D, p.c[r] + row * p.ldc[r], lane, mi < n_rows);
                        o = 1;
                    }
                    if (has_b) {
#pragma unroll
                        for (int r = 0; r < R; ++r) {
                            const float* src = (p.epilogue == MMSSL_EPI_SOFTMAX_BWD) ? p.ys[r] + row * p.ldys[r]
                                               : (p.s_mode == 2)                     ? p.sb[r] + row * p.ldsb[r]
                                                                                     : p.s[r] + row * p.lds[r];
                            bk_row_ldgsts<D>(stg + (size_t)(o * kBkRows + mi) * RD + r * D, src, lane, mi < n_rows);
                        }
                    }
                }
            }
            bk_cp_commit_wait();
            __syncwarp();
        }

        // ---- consume: rows of the bucket one after the other, all lanes on each
        for (int i = 0; i < n_rows; ++i) {
            const int jb = bnd_s[i], je = bnd_s[i + 1];
            const int row = row0 + i;
            float acc[R][V];
#pragma unroll
            for (int r = 0; r < R; ++r)
#pragma unroll
                for (int e = 0; e < V; ++e) acc[r][e] = 0.f;
#pragma unroll 4
            for (int j = jb; j < je; ++j) {
                const float w = vals_s[j];
                const float* slot = ring + (size_t)j * RD;
#pragma unroll
                for (int r = 0; r < R; ++r)
#pragma unroll
                    for (int ch = 0; ch < NCH; ++ch) {
                        float x[CW];
                        ldv<CW>(x, slot + r * D + L::off(lane, ch));
#pragma unroll
                        for (int e = 0; e < CW; ++e) acc[r][ch * CW + e] = fmaf(w, x[e], acc[r][ch * CW + e]);
                    }
            }

            // ---- chunk of a long row: publish the partial sum, the last chunk to arrive reduces in chunk order
            if (sp >= 0) {
                if (st.w != 0) {
                    float* slot = p.partials + (int64_t)st.x * RD;
#pragma unroll
                    for (int r = 0; r < R; ++r)
#pragma unroll
                        for (int ch = 0; ch < NCH; ++ch) {
                            float x[CW];
#pragma unroll
                            for (int e = 0; e < CW; ++e) x[e] = acc[r][ch * CW + e];
                            redv<CW>(slot + r * D + L::off(lane, ch), x);
                        }
                } else {
                    float* part = p.partials + ((int64_t)st.x + seg) * RD;
#pragma unroll
                    for (int r = 0; r < R; ++r)
#pragma unroll
                        for (int ch = 0; ch < NCH; ++ch) {
                            float x[CW];
#pragma unroll
                            for (int e = 0; e < CW; ++e) x[e] = acc[r][ch * CW + e];
                            stv<CW>(part + r * D + L::off(lane, ch), x);
                        }
                }
                __threadfence();
                __syncwarp();
                int old = 0;
                if (lane == 0) old = atomicAdd(p.counters + sp, 1);
                old = __shfl_sync(0xffffffffu, old, 0);
                if (old != st.y - 1) continue;
                __threadfence();
                if (lane == 0) p.counters[sp] = 0;    // self-cleaning for the next launch
                if (st.w != 0) {
                    float* slot = p.partials + (int64_t)st.x * RD;
#pragma unroll
                    for (int r = 0; r < R; ++r)
#pragma unroll
                        for (int ch = 0; ch < NCH; ++ch) {
                            float x[CW], z[CW];
                            ldv_cg<CW>(x, slot + r * D + L::off(lane, ch));
#pragma unroll
                            for (int e = 0; e < CW; ++e) { acc[r][ch * CW + e] = x[e]; z[e] = 0.f; }
                            stv_cg<CW>(slot + r * D + L::off(lane, ch), z);      // leave the slot clean for the next launch
                        }
                } else {
#pragma unroll
                    for (int r = 0; r < R; ++r)
#pragma unroll
                        for (int e = 0; e < V; ++e) acc[r][e] = 0.f;
                    constexpr int PB = (8 / (R * NCH)) >= 1 ? (8 / (R * NCH)) : 1;   // partial rows fetched per round trip
                    for (int s0 = 0; s0 < st.y; s0 += PB) {
                        float pv[PB][R][V];
#pragma unroll
                        for (int qq = 0; qq < PB; ++qq) {
                            const bool on = (s0 + qq) < st.y;
                            const float* ps = p.partials + ((int64_t)st.x + s0 + qq) * RD;
#pragma unroll
                            for (int r = 0; r < R; ++r)
#pragma unroll
                                for (int ch = 0; ch < NCH; ++ch) {
                                    float x[CW];
                                    if (on) ldv_cg<CW>(x, ps + r * D + L::off(lane, ch));
#pragma unroll
                                    for (int e = 0; e < CW; ++e) pv[qq][r][ch * CW + e] = on ? x[e] : 0.f;
                                }
                        }
#pragma unroll
                        for (int qq = 0; qq < PB; ++qq)      // fixed (chunk) order -> deterministic sum
#pragma unroll
                            for (int r = 0; r < R; ++r)
#pragma unroll
                                for (int e = 0; e < V; ++e) acc[r][e] += pv[qq][r][e];
                    }
                }
            }

            // ---- epilogue
            const float* sa = stg + (size_t)i * RD;                                      // operand A row (alpha * C)
            const float* sb_ = stg + (size_t)((has_a ? kBkRows : 0) + i) * RD;           // operand B row
#pragma unroll
            for (int r = 0; r < R; ++r) {
                if (has_a && p.c[r] != nullptr) {
#pragma unroll
                    for (int ch = 0; ch < NCH; ++ch) {
                        float x[CW];
                        ldv<CW>(x, sa + r * D + L::off(lane, ch));
#pragma unroll
                        for (int e = 0; e < CW; ++e) acc[r][ch * CW + e] = fmaf(p.alpha, x[e], acc[r][ch * CW + e]);
                    }
                }
                if (p.epilogue == MMSSL_EPI_SOFTMAX) {
                    float m = -INFINITY;
#pragma unroll
                    for (int e = 0; e < V; ++e) m = fmaxf(m, acc[r][e]);
                    m = group_max<32>(m, 0xffffffffu);
                    float sum = 0.f;
#pragma unroll
                    for (int e = 0; e < V; ++e) { acc[r][e] = __expf(acc[r][e] - m); sum += acc[r][e]; }
                    sum = group_sum<32>(sum, 0xffffffffu);
                    const float inv = 1.f / sum;
#pragma unroll
                    for (int e = 0; e < V; ++e) acc[r][e] *= inv;
                } else if (p.epilogue == MMSSL_EPI_SOFTMAX_BWD) {
                    float yv[V];
                    float dotp = 0.f;
#pragma unroll
                    for (int ch = 0; ch < NCH; ++ch) {
                        float x[CW];
                        ldv<CW>(x, sb_ + r * D + L::off(lane, ch));
#pragma unroll
                        for (int e = 0; e < CW; ++e) { yv[ch * CW + e] = x[e]; dotp = fmaf(acc[r][ch * CW + e], x[e], dotp); }
                    }
                    dotp = group_sum<32>(dotp, 0xffffffffu);
#pragma unroll
                    for (int e = 0; e < V; ++e) acc[r][e] = yv[e] * (acc[r][e] - dotp);
                }
#pragma unroll
                for (int ch = 0; ch < NCH; ++ch) {
                    float x[CW];
#pragma unroll
                    for (int e = 0; e < CW; ++e) x[e] = acc[r][ch * CW + e];
                    const int64_t off = (int64_t)row * p.ldy[r] + L::off(lane, ch);
                    if (p.y_mode[r] == 1) {       // NVSwitch multicast: the store is replicated into every GPU's table
                        mcstv<CW>(p.y[r] + off, x);
                    } else {
                        stv<CW>(p.y[r] + off, x);
                        if (p.y_mode[r] == 2)     // peer-mapped tables over NVLink
                            for (int qq = 0; qq < p.n_peers[r]; ++qq) stv<CW>(p.y_peers[r][qq] + off, x);
                    }
                }
                if (p.s_mode != 0 && p.s[r] != nullptr) {
#pragma unroll
                    for (int ch = 0; ch < NCH; ++ch) {
                        float x[CW], o[CW];
                        ldv<CW>(x, sb_ + r * D + L::off(lane, ch));
#pragma unroll
                        for (int e = 0; e < CW; ++e) o[e] = x[e] + acc[r][ch * CW + e];
                        stv<CW>(p.s[r] + (int64_t)row * p.lds[r] + L::off(lane, ch), o);
                    }
                }
            }
        }
    }
}

template <int V, int R, bool TMA>
static int launch_bulk(const BulkParams& bp_in, cudaStream_t stream, int wpb, int tpw) {
    constexpr int D = 32 * V, RD = R * D;
    BulkParams bp = bp_in;
    const int warp_bytes = ((kBk + bp.n_ops * kBkRows) * RD * 4 + (2 * kBk + 16) * 4 + 16 + 127) & ~127;
    bp.warp_bytes = warp_bytes;
    bp.tasks_per_warp = tpw;
    while (wpb > 1 && warp_bytes * wpb > 227 * 1024) --wpb;       // wide slots: fewer warps per block
    const int smem = warp_bytes * wpb;
    static int attr_smem = 0;
    if (smem > attr_smem) {
        MMSSL_CUDA(cudaFuncSetAttribute(spmm_bulk_kernel<V, R, TMA>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        attr_smem = smem;
    }
    const int64_t warps = (bp.n_buckets + tpw - 1) / tpw;
    const int64_t blocks = (warps + wpb - 1) / wpb;
    if (blocks == 0) return 0;
    if (blocks > 0x7fffffffll) return fail("mmssl_spmm_bulk_f32", "grid too large");
    MMSSL_CUDA_LAUNCH((spmm_bulk_kernel<V, R, TMA>), dim3((unsigned)blocks), dim3(32 * wpb), (size_t)smem, stream, bp);
    MMSSL_LAUNCH_OK();
    return 0;
}

}  // namespace mmssl

using namespace mmssl;

// variant: bits 4-7 warps per block (0 = 4), bits 8-15 buckets per warp (0 = automatic: 1 under 2M edges, 4 above),
// bit 16: TMA bulk copies instead of LDGSTS.
extern "C" int mmssl_spmm_bulk_f32(const mmssl_csr_t* a, const int32_t* buckets8, int64_t n_buckets, int d, int nrhs,
                                   const mmssl_spmm_rhs_t* rhs, int epilogue, float alpha, int s_mode, float* partials,
                                   int64_t partials_floats, int variant, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    MMSSL_REQUIRE(a != nullptr && (buckets8 != nullptr || n_buckets == 0) && n_buckets >= 0, "missing bucket table (mmssl_spmm_bulk_plan)");
    MMSSL_REQUIRE(nrhs >= 1 && nrhs <= 2, "the staged-gather SpMM takes 1 or 2 right-hand sides");
    if (d != 64 && d != 128 && d != 256) return fail_width("mmssl_spmm_bulk_f32 (64, 128 or 256 only)", d);
    BulkParams bp;
    mmssl_csr_t a2 = *a;            // the classic plan's item list is not used here: only the split table / counters of the bucket plan
    a2.n_items = 0;
    a2.items = a->rowptr;           // any non-null pointer (fill_spmm_params checks presence)
    if (int rc = fill_spmm_params(bp.p, &a2, d, nrhs, rhs, epilogue, alpha, s_mode, partials, partials_floats)) return rc;
    bp.buckets = reinterpret_cast<const int4*>(buckets8);
    bp.n_buckets = n_buckets;
    const bool has_b = (epilogue == MMSSL_EPI_SOFTMAX_BWD) || (s_mode != 0 && bp.p.s[0] != nullptr);
    MMSSL_REQUIRE(!(epilogue == MMSSL_EPI_SOFTMAX_BWD && s_mode != 0), "softmax-backward epilogue and running sum together: use mmssl_spmm_csr_f32");
    for (int r = 0; r < nrhs; ++r) {
        MMSSL_REQUIRE((bp.p.c[r] != nullptr) == (bp.p.c[0] != nullptr), "C must be given for all right-hand sides or none");
        MMSSL_REQUIRE((bp.p.s[r] != nullptr) == (bp.p.s[0] != nullptr), "S must be given for all right-hand sides or none");
    }
    bp.n_ops = (bp.p.has_c ? 1 : 0) + (has_b ? 1 : 0);
    int wpb = (variant >> 4) & 15, tpw = (variant >> 8) & 255;
    const bool tma = (variant >> 16) & 1;
    if (wpb == 0) wpb = 4;
    if (tpw == 0) tpw = a->nnz >= (1ll << 21) ? 4 : 1;
    MMSSL_REQUIRE(wpb >= 1 && wpb <= 8, "warps per block must be 1..8");
#define MMSSL_BULK_CASE(V)                                                                                              \
    if (nrhs == 1) return tma ? launch_bulk<V, 1, true>(bp, stream, wpb, tpw) : launch_bulk<V, 1, false>(bp, stream, wpb, tpw); \
    return tma ? launch_bulk<V, 2, true>(bp, stream, wpb, tpw) : launch_bulk<V, 2, false>(bp, stream, wpb, tpw);
    if (d == 64) { MMSSL_BULK_CASE(2) }
    if (d == 128) { MMSSL_BULK_CASE(4) }
    if (d == 256) { MMSSL_BULK_CASE(8) }
#undef MMSSL_BULK_CASE
    return fail_width(__func__, d);
}
