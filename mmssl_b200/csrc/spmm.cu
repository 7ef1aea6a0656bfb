// CSR SpMM  Y_r = epilogue( A * X_r ),  r < nrhs  -- the propagation operator of the MMSSL hot
// path (reference: MMSSL.mm / torch.sparse.mm, Models.py:69-73, and torch.mm(sparse, dense),
// Models.py:203-208; the transposed products autograd derives from them use the CSR of A^T).
//
// Design (sparse gather: latency bound on small graphs, L2-gather / resident-row-walk bound on
// large ones -- DESIGN.md section 6; no tensor cores):
//  * one lane *group* (16 lanes for d=64, 32 lanes for d>=128) owns one work item = one row or one
//    fixed-length segment of a long row (plan built by mmssl_spmm_plan); every lane owns one
//    float4 column slice per right-hand side, so a neighbour row is fetched with one coalesced
//    128-bit load per lane (256 B .. 1 KB contiguous per neighbour).
//  * column indices / values of the row are loaded coalesced (one per lane) and broadcast with
//    warp shuffles; the next chunk is prefetched and 8 neighbour gathers (float4 each) are in flight per
//    lane before the first FMA consumes one.
//  * up to 3 right-hand sides share one pass over the sparsity pattern (e.g. image|text features),
//    which divides the index traffic and the launch count.
//  * long rows (power-law item degrees) are cut into segments handled by different groups; the
//    last group to arrive sums the partials in segment order -> deterministic.  Rows over 1024
//    non-zeros (the head of a power-law degree distribution) instead accumulate 64-nnz segments with
//    128-bit float reductions into a zeroed slot: a serial reduction over hundreds of partials would be
//    the critical path of a small (latency-bound) graph.
//  * output rows can be stored to the NVSwitch multicast address of a symmetric table (multimem.st) or to
//    peer-mapped tables: the all-gather of the row-sharded scheme is part of the epilogue.
//  * fused epilogues: + alpha*C[row], row softmax over d (last GCN layer, Models.py:203-204),
//    softmax backward y*(g - <g,y>), running layer sum S (+)= out (Models.py:213-214).
#include <cstdlib>

#include "spmm_common.cuh"

namespace mmssl {

// G lanes per group, C float4 chunks per lane per rhs (d = 4*G*C), R right-hand sides.
// UNR neighbour gathers are issued back to back before the first FMA consumes one, and the next
// chunk of (col, val) pairs is prefetched while the current one is processed, so a row walk costs
// about one memory round trip per UNR non-zeros instead of one per load.
// PRE (impl bit 6, candidate awaiting measurement): the row-indexed epilogue operands -- alpha*C[row], the saved softmax
// output, the running-sum base -- are requested as soon as the work item is known, so that they travel while the
// index -> gather chain runs instead of adding one more dependent round trip after it.  Only for R*C <= 2 (register cost).
// HINT (large graphs, impl bits 7 / 8): 1 = the streams (col, val, outputs, row-indexed operands) are marked L2 evict-first and
// bypass L1 so that they do not push the gathered table out of L2 (at 1M x 200k a 102 MB table shares the L2 with 670 MB of
// streams, so the gathered rows are re-fetched from DRAM); 2 = additionally the column indices carry a
// "hot" flag in the sign bit (the head of the column-degree distribution, graph.py:hot_flag_plan) and hot rows are loaded
// with L1::evict_last, cold ones with L1::no_allocate, so that the ~200 KB of L1 serve the popular rows.
// One work item, from its descriptor and the first chunk of (col, val) pairs (one per lane, 0 beyond the item's end) to the
// stored output row.  `return` = this group is done with the item.
template <int G, int C, int R, int UMUL, bool PRE, int HINT, bool EARLY>
__device__ __forceinline__ void spmm_item(const SpmmParams& p, const int4 item, int c_nxt, float v_nxt, const int lane,
                                          const unsigned gmask) {
    constexpr int RC = R * C;
    constexpr bool PRE_ON = PRE && RC <= 2;
    constexpr int UNR0 = ((8 / RC) >= 2 ? (8 / RC) : 2) * UMUL;
    constexpr int UNR = UNR0 > G ? G : UNR0;
    const int row = item.x;
    const int begin = item.y, end = item.z;
    // split rows: the table entry and the row start are requested now, not after the gathers (one dependent trip less) -- EARLY:
    // not in the register-capped variants of the large graphs, where the five extra live registers become spills
    int4 st = make_int4(0, 0, 0, 0);
    int row_begin = 0;
    if (EARLY && item.w >= 0) {
        st = __ldg(&p.split_table[item.w]);   // {first partial slot, #segments, segment length, heavy}
        row_begin = __ldg(p.rowptr + row);
    }

    float4 pre_c[PRE_ON ? R : 1][PRE_ON ? C : 1], pre_e[PRE_ON ? R : 1][PRE_ON ? C : 1];
    if (PRE_ON) {
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
            for (int c = 0; c < C; ++c) {
                const int64_t cofs = lane * 4 + c * (4 * G);
                pre_c[r][c] = (p.has_c && p.c[r] != nullptr) ? ld4(p.c[r] + (int64_t)row * p.ldc[r] + cofs) : f4zero();
                if (p.epilogue == MMSSL_EPI_SOFTMAX_BWD) pre_e[r][c] = ldg4(p.ys[r] + (int64_t)row * p.ldys[r] + cofs);
                else if (p.s_mode == 1 && p.s[r] != nullptr) pre_e[r][c] = ld4(p.s[r] + (int64_t)row * p.lds[r] + cofs);
                else if (p.s_mode == 2 && p.s[r] != nullptr) pre_e[r][c] = ldg4(p.sb[r] + (int64_t)row * p.ldsb[r] + cofs);
                else pre_e[r][c] = f4zero();
            }
    }

    float4 acc[R][C];
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
        for (int c = 0; c < C; ++c) acc[r][c] = f4zero();

    for (int base = begin; base < end; base += G) {
        const int c_l = c_nxt;
        const float v_l = v_nxt;
        const int e2 = base + G + lane;
        c_nxt = 0; v_nxt = 0.f;
        if (e2 < end) {                                                                // prefetch the next chunk
            c_nxt = HINT ? ldg_i32_stream(p.colidx + e2) : __ldg(p.colidx + e2);
            v_nxt = HINT ? ldg_f32_stream(p.vals + e2) : __ldg(p.vals + e2);
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
#pragma unroll
                for (int r = 0; r < R; ++r) {
                    const int col = (HINT == 2) ? (cc[k] & 0x7fffffff) : cc[k];
                    const float* xr = p.x[r] + (int64_t)col * p.ldx[r] + lane * 4;
#pragma unroll
                    for (int c = 0; c < C; ++c) {
                        if (HINT == 0) xv[k][r][c] = on ? ldg4(xr + c * (4 * G)) : f4zero();
                        else if (HINT == 1) xv[k][r][c] = on ? ldg4_l2(xr + c * (4 * G), p.x_policy) : f4zero();
                        else xv[k][r][c] = on ? ldg4_l1_hot_cold(xr + c * (4 * G), cc[k] < 0, p.x_policy) : f4zero();
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

    // ---- split rows: publish the partial, the last arriver reduces in segment order ----
    if (item.w >= 0) {
        if (!EARLY) {
            st = __ldg(&p.split_table[item.w]);
            row_begin = __ldg(p.rowptr + row);
        }
        const int W = R * C * G * 4;
        if (st.w != 0) {
            // heavy row: accumulate into the row's own zeroed slot with 128-bit reductions
            float* slot = p.partials + (int64_t)st.x * W;
#pragma unroll
            for (int r = 0; r < R; ++r)
#pragma unroll
                for (int c = 0; c < C; ++c)
                    atomicAdd(reinterpret_cast<float4*>(slot + (r * C + c) * (4 * G) + lane * 4), acc[r][c]);
            __threadfence();
            __syncwarp(gmask);
            int old = 0;
            if (lane == 0) old = atomicAdd(p.counters + item.w, 1);
            old = __shfl_sync(gmask, old, 0, G);
            if (old != st.y - 1) return;
            __threadfence();
            if (lane == 0) p.counters[item.w] = 0;
#pragma unroll
            for (int r = 0; r < R; ++r)
#pragma unroll
                for (int c = 0; c < C; ++c) {
                    float* q = slot + (r * C + c) * (4 * G) + lane * 4;
                    acc[r][c] = ldcg4(q);
                    __stcg(reinterpret_cast<float4*>(q), f4zero());   // leave the slot clean for the next launch
                }
        } else {
        const int k = (begin - row_begin) / st.z;
        float* part = p.partials + ((int64_t)st.x + k) * W;
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
            for (int c = 0; c < C; ++c) st4(part + (r * C + c) * (4 * G) + lane * 4, acc[r][c]);
        __threadfence();
        __syncwarp(gmask);
        int old = 0;
        if (lane == 0) old = atomicAdd(p.counters + item.w, 1);
        old = __shfl_sync(gmask, old, 0, G);
        if (old != st.y - 1) return;
        __threadfence();
        if (lane == 0) p.counters[item.w] = 0;   // self-cleaning for the next launch
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
            for (int c = 0; c < C; ++c) acc[r][c] = f4zero();
        constexpr int PB = (8 / RC) >= 1 ? (8 / RC) : 1;   // partial rows fetched per round trip
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
            for (int q = 0; q < PB; ++q)      // fixed (segment) order -> deterministic sum
#pragma unroll
                for (int r = 0; r < R; ++r)
#pragma unroll
                    for (int c = 0; c < C; ++c) acc[r][c] = add4(acc[r][c], pv[q][r][c]);
        }
        }
    }

    // ---- epilogue ----
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const int64_t col0 = lane * 4;
        if (p.has_c && p.c[r] != nullptr) {
#pragma unroll
            for (int c = 0; c < C; ++c) {
                const float* cp_ = p.c[r] + (int64_t)row * p.ldc[r] + col0 + c * (4 * G);
                const float4 cv = PRE_ON ? pre_c[r][c] : HINT ? ld4_stream(cp_) : ld4(cp_);   // may alias Y (read before the row is written, by the same lanes)
                fma4(acc[r][c], p.alpha, cv);
            }
        }
        if (p.epilogue == MMSSL_EPI_SOFTMAX) {
            float m = -INFINITY;
#pragma unroll
            for (int c = 0; c < C; ++c) m = fmaxf(m, max4(acc[r][c]));
            m = group_max<G>(m, gmask);
            float sum = 0.f;
#pragma unroll
            for (int c = 0; c < C; ++c) {
                acc[r][c].x = __expf(acc[r][c].x - m); acc[r][c].y = __expf(acc[r][c].y - m);
                acc[r][c].z = __expf(acc[r][c].z - m); acc[r][c].w = __expf(acc[r][c].w - m);
                sum += (acc[r][c].x + acc[r][c].y) + (acc[r][c].z + acc[r][c].w);
            }
            sum = group_sum<G>(sum, gmask);
            const float inv = 1.f / sum;
#pragma unroll
            for (int c = 0; c < C; ++c) acc[r][c] = scale4(acc[r][c], inv);
        } else if (p.epilogue == MMSSL_EPI_SOFTMAX_BWD) {
            float4 yv[C];
            float dotp = 0.f;
#pragma unroll
            for (int c = 0; c < C; ++c) {
                yv[c] = PRE_ON ? pre_e[r][c] : ldg4(p.ys[r] + (int64_t)row * p.ldys[r] + col0 + c * (4 * G));
                dotp += dot4(acc[r][c], yv[c]);
            }
            dotp = group_sum<G>(dotp, gmask);
#pragma unroll
            for (int c = 0; c < C; ++c) {
                acc[r][c].x = yv[c].x * (acc[r][c].x - dotp); acc[r][c].y = yv[c].y * (acc[r][c].y - dotp);
                acc[r][c].z = yv[c].z * (acc[r][c].z - dotp); acc[r][c].w = yv[c].w * (acc[r][c].w - dotp);
            }
        }
#pragma unroll
        for (int c = 0; c < C; ++c) {
            const int64_t off = (int64_t)row * p.ldy[r] + col0 + c * (4 * G);
            if (p.y_mode[r] == 1) {           // NVSwitch multicast: the store is replicated into every GPU's table
                asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p.y[r] + off), "f"(acc[r][c].x),
                             "f"(acc[r][c].y), "f"(acc[r][c].z), "f"(acc[r][c].w) : "memory");
            } else {
                if (HINT) st4_stream(p.y[r] + off, acc[r][c]); else st4(p.y[r] + off, acc[r][c]);
                if (p.y_mode[r] == 2)         // peer-mapped tables over NVLink
                    for (int q = 0; q < p.n_peers[r]; ++q) st4(p.y_peers[r][q] + off, acc[r][c]);
            }
        }
        if (p.s_mode != 0 && p.s[r] != nullptr) {
#pragma unroll
            for (int c = 0; c < C; ++c) {
                float* sp = p.s[r] + (int64_t)row * p.lds[r] + col0 + c * (4 * G);
                const float4 prev = PRE_ON ? pre_e[r][c]
                                           : (p.s_mode == 1) ? ld4(sp) : ldg4(p.sb[r] + (int64_t)row * p.ldsb[r] + col0 + c * (4 * G));
                st4(sp, add4(prev, acc[r][c]));
            }
        }
    }
}

// first chunk of an item's (col, val) pairs: one per lane
template <int HINT>
__device__ __forceinline__ void spmm_first_chunk(const SpmmParams& p, const int4 item, const int lane, int& c, float& v) {
    c = 0; v = 0.f;
    if (item.x >= 0 && item.y + lane < item.z) {
        c = HINT ? ldg_i32_stream(p.colidx + item.y + lane) : __ldg(p.colidx + item.y + lane);
        v = HINT ? ldg_f32_stream(p.vals + item.y + lane) : __ldg(p.vals + item.y + lane);
    }
}

// one item per lane group (the grid covers the plan)
template <int G, int C, int R, int UMUL, int MINB, bool PRE = false, int HINT = 0>
__global__ void __launch_bounds__(256, MINB) spmm_csr_kernel(const SpmmParams p) {
    pdl_wait();
    const unsigned gmask = group_mask<G>();
    const int lane = threadIdx.x & (G - 1);
    const int64_t gid = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / G;
    int4 item = make_int4(-1, 0, 0, -1);
    if (gid < p.n_items) item = __ldg(&p.items[gid]);
    if (item.x < 0) return;   // whole group exits together (items are per group)
    int c0; float v0;
    spmm_first_chunk<HINT>(p, item, lane, c0, v0);
    spmm_item<G, C, R, UMUL, PRE, HINT, MINB == 1>(p, item, c0, v0, lane, gmask);
}

// Software-pipelined walk for small (latency-bound) graphs: the grid is one resident wave of lane groups and every group walks
// items gid, gid + stride, ... .  While item k is gathered, the (col, val) chunk of item k+1 and the descriptor of item k+2 are
// already in flight (and, PRE, the row-indexed epilogue operands of item k are requested before its gathers), so that an item
// costs about one memory round trip (its gathers) instead of the four of the one-item kernel (descriptor -> indices ->
// gathers -> epilogue operands), and a plan of several waves no longer pays them per wave.  Per-item arithmetic is spmm_item's: results are identical.
template <int G, int C, int R, bool PRE>
__global__ void __launch_bounds__(128) spmm_csr_pipe_kernel(const SpmmParams p) {
    pdl_wait();
    const unsigned gmask = group_mask<G>();
    const int lane = threadIdx.x & (G - 1);
    const int64_t stride = (int64_t)gridDim.x * (blockDim.x / G);
    int64_t gid = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / G;
    const int4 none = make_int4(-1, 0, 0, -1);
    int4 it0 = gid < p.n_items ? __ldg(&p.items[gid]) : none;
    int4 it1 = gid + stride < p.n_items ? __ldg(&p.items[gid + stride]) : none;
    int c0; float v0;
    spmm_first_chunk<0>(p, it0, lane, c0, v0);
    while (it0.x >= 0) {
        int c1; float v1;
        spmm_first_chunk<0>(p, it1, lane, c1, v1);
        const int4 it2 = gid + 2 * stride < p.n_items ? __ldg(&p.items[gid + 2 * stride]) : none;
        spmm_item<G, C, R, 1, PRE, 0, true>(p, it0, c0, v0, lane, gmask);
        it0 = it1; c0 = c1; v0 = v1; it1 = it2; gid += stride;
    }
}

static int g_pipe_blocks = 0;        // mmssl_spmm_pipe_set_blocks: 0 = one resident wave

template <int G, int C, int R, bool PRE>
static int launch_spmm_pipe(const SpmmParams& p, cudaStream_t stream) {
    constexpr int T = 128;
    static int resident = 0;                         // blocks of this instantiation one device holds at once
    if (resident == 0) {
        int per_sm = 0, dev = 0, sms = 0;
        MMSSL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, spmm_csr_pipe_kernel<G, C, R, PRE>, T, 0));
        MMSSL_CUDA(cudaGetDevice(&dev));
        MMSSL_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        resident = per_sm * sms;
        if (resident <= 0) return fail("mmssl_spmm_csr_f32", "pipelined kernel does not fit an SM");
    }
    const int64_t groups_per_block = T / G;
    int64_t blocks = (p.n_items + groups_per_block - 1) / groups_per_block;
    if (blocks == 0) return 0;
    const int64_t cap = g_pipe_blocks > 0 ? g_pipe_blocks : resident;
    if (blocks > cap) blocks = cap;
    MMSSL_CUDA_LAUNCH((spmm_csr_pipe_kernel<G, C, R, PRE>), dim3((unsigned)blocks), dim3(T), 0, stream, p);
    MMSSL_LAUNCH_OK();
    return 0;
}

template <int G, int C, int R, int UMUL, int MINB, bool PRE = false, int HINT = 0>
static int launch_spmm_v(const SpmmParams& p, cudaStream_t stream, int T) {
    const int64_t groups_per_block = T / G;
    const int64_t blocks = (p.n_items + groups_per_block - 1) / groups_per_block;
    if (blocks == 0) return 0;
    if (blocks > 0x7fffffffll) return fail("mmssl_spmm_csr_f32", "grid too large");
    static bool attr = false;
    if (!attr) {                     // MMSSL_SPMM_CARVEOUT (percent): experiment knob, the SM's shared-memory configuration this kernel asks for
        if (const char* e = getenv("MMSSL_SPMM_CARVEOUT"))
            MMSSL_CUDA(cudaFuncSetAttribute(spmm_csr_kernel<G, C, R, UMUL, MINB, PRE, HINT>, cudaFuncAttributePreferredSharedMemoryCarveout, atoi(e)));
        attr = true;
    }
    MMSSL_CUDA_LAUNCH((spmm_csr_kernel<G, C, R, UMUL, MINB, PRE, HINT>), dim3((unsigned)blocks), dim3(T), 0, stream, p);
    MMSSL_LAUNCH_OK();
    return 0;
}

// impl bit 3 (8): twice as many gathers in flight per lane; bit 4 (16): cap registers for 6 blocks/SM;
// bit 6 (64): early epilogue-operand prefetch (only with the two policy defaults, i.e. bit 3 clear)
template <int G, int C, int R>
static int launch_spmm(const SpmmParams& p, cudaStream_t stream, int T, int impl) {
    if (impl & 512) return (impl & 64) ? launch_spmm_pipe<G, C, R, true>(p, stream) : launch_spmm_pipe<G, C, R, false>(p, stream);
    if (impl & 256) return launch_spmm_v<G, C, R, 1, 6, false, 2>(p, stream, T);       // L2 streams + L1 hot / cold rows
    if (impl & 128) return launch_spmm_v<G, C, R, 1, 6, false, 1>(p, stream, T);       // L2 streams
    if ((impl & 64) && R * C <= 2 && !(impl & 8))
        return (impl & 16) ? launch_spmm_v<G, C, R, 1, 6, true>(p, stream, T) : launch_spmm_v<G, C, R, 1, 1, true>(p, stream, T);
    switch ((impl >> 3) & 3) {
        case 1: return launch_spmm_v<G, C, R, 2, 1>(p, stream, T);
        case 2: return launch_spmm_v<G, C, R, 1, 6>(p, stream, T);
        case 3: return launch_spmm_v<G, C, R, 2, 4>(p, stream, T);
        default: return launch_spmm_v<G, C, R, 1, 1>(p, stream, T);
    }
}

int fill_spmm_params(SpmmParams& p, const mmssl_csr_t* a, int d, int nrhs, const mmssl_spmm_rhs_t* rhs, int epilogue,
                     float alpha, int s_mode, float* partials, int64_t partials_floats) {
    MMSSL_REQUIRE(a != nullptr && rhs != nullptr, "null argument");
    MMSSL_REQUIRE(nrhs >= 1 && nrhs <= kMaxRhs, "nrhs must be 1..3");
    MMSSL_REQUIRE(d == 64 || d == 128 || d == 256, "embedding width must be 64, 128 or 256");
    MMSSL_REQUIRE(epilogue >= MMSSL_EPI_NONE && epilogue <= MMSSL_EPI_SOFTMAX_BWD, "bad epilogue");
    MMSSL_REQUIRE(s_mode >= 0 && s_mode <= 2, "bad s_mode");
    MMSSL_REQUIRE(a->n_items >= 0 && a->items != nullptr, "missing work plan");
    MMSSL_REQUIRE(a->segs_cap * (int64_t)nrhs * d <= partials_floats || a->segs_cap == 0,
                  "partials buffer too small for the split rows");
    memset(&p, 0, sizeof(p));
    p.rowptr = a->rowptr; p.colidx = a->colidx; p.vals = a->vals;
    p.items = (const int4*)a->items; p.n_items = a->n_items;
    p.split_table = (const int4*)a->split_table; p.counters = a->counters; p.partials = partials;
    p.alpha = alpha; p.epilogue = epilogue; p.s_mode = s_mode;
    for (int r = 0; r < nrhs; ++r) {
        const mmssl_spmm_rhs_t& q = rhs[r];
        MMSSL_REQUIRE(q.x && q.y, "null X or Y");
        MMSSL_REQUIRE(aligned16(q.x) && aligned16(q.y) && q.ldx % 4 == 0 && q.ldy % 4 == 0, "X/Y must be 16-byte aligned with ld % 4 == 0");
        p.x[r] = q.x; p.ldx[r] = q.ldx; p.y[r] = q.y; p.ldy[r] = q.ldy;
        MMSSL_REQUIRE(q.y_mode >= 0 && q.y_mode <= 2 && q.n_peers >= 0 && q.n_peers <= 8, "bad y_mode / n_peers");
        p.y_mode[r] = q.y_mode; p.n_peers[r] = q.n_peers;
        for (int k = 0; k < q.n_peers; ++k) { MMSSL_REQUIRE(aligned16(q.y_peers[k]), "peer table alignment"); p.y_peers[r][k] = q.y_peers[k]; }
        if (q.c) {
            MMSSL_REQUIRE(aligned16(q.c) && q.ldc % 4 == 0, "C alignment");
            p.c[r] = q.c; p.ldc[r] = q.ldc; p.has_c = 1;
        }
        if (epilogue == MMSSL_EPI_SOFTMAX_BWD) {
            MMSSL_REQUIRE(q.ysaved && aligned16(q.ysaved) && q.ldysaved % 4 == 0, "softmax-backward epilogue needs ysaved");
            p.ys[r] = q.ysaved; p.ldys[r] = q.ldysaved;
        }
        if (s_mode != 0 && q.s) {
            MMSSL_REQUIRE(aligned16(q.s) && q.lds % 4 == 0, "S alignment");
            p.s[r] = q.s; p.lds[r] = q.lds;
            if (s_mode == 2) {
                MMSSL_REQUIRE(q.sbase && aligned16(q.sbase) && q.ldsbase % 4 == 0, "s_mode 2 needs sbase");
                p.sb[r] = q.sbase; p.ldsb[r] = q.ldsbase;
            }
        }
    }
    return 0;
}

}  // namespace mmssl

using namespace mmssl;

extern "C" int mmssl_spmm_pipe_set_blocks(int blocks) {
    MMSSL_REQUIRE(blocks >= 0, "blocks must be >= 0 (0 = one resident wave)");
    g_pipe_blocks = blocks;
    return 0;
}

extern "C" int mmssl_spmm_csr_f32(const mmssl_csr_t* a, int d, int nrhs, const mmssl_spmm_rhs_t* rhs, int epilogue,
                                  float alpha, int s_mode, float* partials, int64_t partials_floats, int impl,
                                  void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    SpmmParams p;
    if (int rc = fill_spmm_params(p, a, d, nrhs, rhs, epilogue, alpha, s_mode, partials, partials_floats)) return rc;
    // gathered rows: evict-last in L2 when every right-hand side table fits it with room to spare, else no preference
    p.x_policy = ((int64_t)a->n_cols * d * nrhs * 4 <= (96ll << 20)) ? kL2EvictLast : 0x1000000000000000ull;
    // impl 0 = automatic policy from measurements (tools/probe.py): small graphs are launch/latency
    // bound and prefer 128-thread blocks; large graphs are bound by the number of resident row walks
    // and prefer the register-capped variant (6 blocks/SM).
    if (impl == 0) impl = (a->nnz >= (1ll << 21)) ? 16 : 4;
    // impl: bit 1 -> 8-lane groups for d = 64 (each lane owns two float4 slices; twice as many rows
    // resident per SM, so a small graph fits one wave); bit 2 -> 128-thread blocks.
    const int T = (impl & 4) ? 128 : 256;
#define MMSSL_SPMM_CASE(G, C)                                           \
    switch (nrhs) {                                                     \
        case 1: return launch_spmm<G, C, 1>(p, stream, T, impl);        \
        case 2: return launch_spmm<G, C, 2>(p, stream, T, impl);        \
        default: return launch_spmm<G, C, 3>(p, stream, T, impl);       \
    }
    if (d == 64 && (impl & 2)) { MMSSL_SPMM_CASE(8, 2) }
    if (d == 64) { MMSSL_SPMM_CASE(16, 1) }
    if (d == 128) { MMSSL_SPMM_CASE(32, 1) }
    MMSSL_SPMM_CASE(32, 2)
#undef MMSSL_SPMM_CASE
}
